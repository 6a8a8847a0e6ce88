"""Every pair-force kernel instantiation against the f64 oracle, and known answers at the cutoff edges.

The non-bonded force is compiled as separate instantiations per dtype T (engine.cu launch_pairs):
  allpairs_force_kernel<T, COUL, CUTM, EN>       no-list path (no neighbour list, or a box under 2.5 r_list)
  brick_force_kernel<T, COUL, UNI, CUTM, EN>     cell-list path
COUL: none / plain Coulomb / reaction field / Ewald real space; CUTM: plain / shifted / two-point cutoff family;
UNI: uniform-LJ fast path (only without Coulomb); EN: energy and virial computed. That is 24 + 30 = 54 kernels per
dtype, 108 in all, each with its own inlined copy of pair_eval / pair_eval_rt (pair.cuh): a mistake in one of them
leaves the others correct.

Each row of VARIANTS runs in f64 and f32 through mbhelpers.check (forces, energy and virial against the oracle at the
tolerances stated in test_gpu_parity.py). The evaluations run under torch.profiler with CUDA activities; the row
asserts that the demangled kernel names recorded on the device carry its expected (COUL, CUTM, UNI), with both EN
values (mb.forces launches EN = false, mb.potential_energy and mb.forces_virial EN = true), and adds what ran to
OBSERVED. The last test of the file asserts that all 108 instantiations were observed.

The known-answer tests put a pair exactly at the cutoff (rc = 1.0, coordinates exact in f32 and f64) and one ulp
beyond it, inside the box and across the periodic boundary, on both paths, and pin geometric sigma mixing by the
reference's literal.
"""
import re
from collections import namedtuple

import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import mbhelpers as H
import mollyb200 as mb
from oracle import oracle as o

pytestmark = pytest.mark.gpu

C_NONE, C_PLAIN, C_CRF, C_EWALD = 0, 1, 2, 3          # COUL template argument (pair.cuh)
M_PLAIN, M_SHIFTED, M_TWO = 0, 1, 2                   # CUTM template argument
DTYPES = {np.float64: "double", np.float32: "float"}


# ---------------------------------------------------------------------------------------------------
# interaction pairs (mollyb200 descriptor, oracle descriptor)
# ---------------------------------------------------------------------------------------------------
_MB_CUT = {"distance": mb.DistanceCutoff, "sp": mb.ShiftedPotentialCutoff, "sf": mb.ShiftedForceCutoff,
           "cubic": mb.CubicSplineCutoff, "poly": mb.PolynomialCutoff}
_O_CUT = {"none": o.CUT_NONE, "distance": o.CUT_DISTANCE, "sp": o.CUT_SHIFTED_POTENTIAL, "sf": o.CUT_SHIFTED_FORCE,
          "cubic": o.CUT_CUBIC_SPLINE, "poly": o.CUT_POLYNOMIAL}


def _cut(kind, rc, ra):
    if kind == "none":
        return mb.NoCutoff()
    return _MB_CUT[kind](ra, rc) if kind in ("cubic", "poly") else _MB_CUT[kind](rc)


def LJ(kind="none", rc=0.0, ra=0.0, w=1.0, nl=True, geo=False):
    return (mb.LennardJones(cutoff=_cut(kind, rc, ra), use_neighbors=nl, weight_special=w,
                            sigma_mixing="geometric" if geo else "lorentz"),
            o.Inter(o.LJ, _O_CUT[kind], rc, r_act=ra, weight_special=w, use_neighbors=nl,
                    sigma_mix=o.MIX_GEOMETRIC if geo else o.MIX_LORENTZ))


def COUL(kind, rc, ra=0.0, w=1.0, nl=True):
    return (mb.Coulomb(cutoff=_cut(kind, rc, ra), use_neighbors=nl, weight_special=w),
            o.Inter(o.COULOMB, _O_CUT[kind], rc, r_act=ra, weight_special=w, use_neighbors=nl))


def CRF(rc, w=1.0, nl=True, solvent=78.3):
    return (mb.CoulombReactionField(dist_cutoff=rc, solvent_dielectric=solvent, use_neighbors=nl, weight_special=w),
            o.Inter(o.CRF, o.CUT_DISTANCE, rc, weight_special=w, use_neighbors=nl, solvent_dielectric=solvent))


def EWALD(rc, w=1.0, nl=True, approx=True):
    alpha = float(np.sqrt(-np.log(2 * 5e-4)) / rc)
    return (mb.CoulombEwald(dist_cutoff=rc, use_neighbors=nl, weight_special=w, approximate_erfc=approx),
            o.Inter(o.EWALD_REAL, o.CUT_DISTANCE, rc, weight_special=w, ewald_alpha=alpha, use_neighbors=nl,
                    approx_erfc=approx))


# ---------------------------------------------------------------------------------------------------
# systems
# ---------------------------------------------------------------------------------------------------
def readme():
    return H.readme_system(100, 2.0, seed=1)


def readme_mixed_sigma():
    """The README system with per-atom sigma in [0.2, 0.4]: with equal sigmas geometric and Lorentz mixing agree."""
    sd = readme()
    return dict(sd, sigma=np.random.default_rng(2).uniform(0.2, 0.4, sd["n"]))


def mol_small(seed=11):
    return H.molecular_system(150, [3.0, 3.2, 3.4], seed=seed)  # 3.0 nm < 2.5 r_list: the no-list kernel


def mol_mixed():
    sd = mol_small(13)
    return dict(sd, charge=sd["charge"] * 0.1)


def mol_mixed_lj_all_pairs():
    """LJ over all pairs meets the excluded 1-2 pairs at 0.11 nm; half sigma keeps those forces moderate, so that the
    f32 tolerance (relative to max|F|) still resolves the rest."""
    sd = mol_small(13)
    return dict(sd, sigma=sd["sigma"] * 0.5)


def mol_large():
    return H.molecular_system(1000, [5.1, 5.4, 5.8], seed=5)  # 4000 atoms: the cell-list path


def mol_uncharged():
    sd = mol_large()
    return dict(sd, charge=np.zeros(sd["n"]))


def _lam_zero(sd, every):
    lam = np.ones(sd["n"])
    lam[::every] = 0.0
    return dict(sd, lam=lam)


def mol_uncharged_lam0():
    return _lam_zero(mol_uncharged(), 7)


def fluid(cells):
    return H.lj_fluid(cells, seed=42, dtype=np.float64)


def fluid_lam0():
    return _lam_zero(fluid(6), 11)


def fluid_exceptions():
    """864-atom LJ fluid with disjoint nearest-neighbour pairs, alternately excluded and special (1-4)."""
    sd = fluid(6)
    used, excl, spec = set(), [], []
    for k, hub in enumerate(range(0, sd["n"], 8)):
        if hub in used:
            continue
        j = int(H.nearest_partners(sd, hub, 1, skip=used)[0])
        used |= {hub, j}
        (excl if k % 2 == 0 else spec).append((hub, j))
    return dict(sd, excluded=np.array(excl, np.int32), special=np.array(spec, np.int32))


Row = namedtuple("Row", "id system inters r_list path coul cutm uni nl_radius", defaults=(None,))
B = 1  # path: brick (cell-list); 0: all-pairs

VARIANTS = [
    # ---- all-pairs, no Coulomb
    Row("ap-readme-lj", readme, [LJ(nl=False)], 0.0, 0, C_NONE, M_PLAIN, None),
    Row("ap-readme-lj-geometric", readme_mixed_sigma, [LJ(nl=False, geo=True)], 0.0, 0, C_NONE, M_PLAIN, None),
    Row("ap-readme-lj-shifted-potential", readme, [LJ("sp", 0.9, nl=False)], 0.0, 0, C_NONE, M_SHIFTED, None),
    Row("ap-readme-lj-polynomial", readme, [LJ("poly", 0.9, 0.7, nl=False)], 0.0, 0, C_NONE, M_TWO, None),
    # ---- all-pairs, plain Coulomb
    *[Row(f"ap-mol-lj-coulomb-{c}", mol_small, [LJ(c, 1.2, w=0.5), COUL(c, 1.2, w=0.8333)], 1.3, 0, C_PLAIN,
          M_PLAIN if c == "distance" else M_SHIFTED, None) for c in ("distance", "sp", "sf")],
    *[Row(f"ap-mol-lj-coulomb-{c}", mol_small, [LJ(c, 1.0, 0.8, w=0.5), COUL(c, 1.0, 0.8, w=0.8333)], 1.25,
          0, C_PLAIN, M_TWO, None) for c in ("cubic", "poly")],
    Row("ap-mol-lj-nl-coulomb-all-pairs", mol_mixed, [LJ("distance", 1.2, w=0.5), COUL("distance", 1.2, w=0.8333, nl=False)],
        1.3, 0, C_PLAIN, M_PLAIN, None),
    Row("ap-mol-lj-all-pairs-coulomb-nl", mol_mixed_lj_all_pairs,
        [LJ("distance", 1.2, w=0.5, nl=False), COUL("distance", 1.2, w=0.8333)], 1.3, 0, C_PLAIN, M_PLAIN, None),
    # ---- all-pairs, reaction field / Ewald
    Row("ap-mol-lj-distance-crf", mol_small, [LJ("distance", 1.0, w=0.5), CRF(1.2, w=0.8333)], 1.3, 0, C_CRF, M_PLAIN, None),
    Row("ap-mol-lj-sf-crf-inf", mol_small, [LJ("sf", 1.2, w=0.5), CRF(1.2, w=0.8333, solvent=float("inf"))], 1.3, 0,
        C_CRF, M_SHIFTED, None),
    Row("ap-mol-lj-cubic-crf", mol_small, [LJ("cubic", 1.2, 1.0, w=0.5), CRF(1.2, w=0.8333)], 1.3, 0, C_CRF, M_TWO, None),
    Row("ap-mol-lj-distance-ewald-approx", mol_small, [LJ("distance", 1.2, w=0.5), EWALD(1.2, w=0.8333)], 1.3, 0,
        C_EWALD, M_PLAIN, None),
    Row("ap-mol-lj-sf-ewald-exact", mol_small, [LJ("sf", 1.2, w=0.5), EWALD(1.2, w=0.8333, approx=False)], 1.3, 0,
        C_EWALD, M_SHIFTED, None),
    Row("ap-mol-lj-poly-ewald", mol_small, [LJ("poly", 1.2, 1.0, w=0.5), EWALD(1.2, w=0.8333)], 1.3, 0, C_EWALD, M_TWO,
        None),
    # ---- brick, no Coulomb, uniform LJ
    Row("br-fluid6-lj-distance", lambda: fluid(6), [LJ("distance", 0.9)], 1.0, B, C_NONE, M_PLAIN, True),
    Row("br-fluid9-lj-distance", lambda: fluid(9), [LJ("distance", 1.2)], 1.3, B, C_NONE, M_PLAIN, True),
    Row("br-fluid6-lj-shifted-potential", lambda: fluid(6), [LJ("sp", 0.9)], 1.0, B, C_NONE, M_SHIFTED, True),
    Row("br-fluid6-lj-sp-exclusions-special", fluid_exceptions, [LJ("sp", 0.9, w=0.5)], 1.0, B, C_NONE, M_SHIFTED, True),
    *[Row(f"br-fluid9-lj-{c}", lambda: fluid(9), [LJ(c, 1.0, 0.8)], 1.1, B, C_NONE, M_TWO, True) for c in ("cubic", "poly")],
    # ---- brick, no Coulomb, per-atom LJ
    Row("br-fluid6-lj-sp-lambda0", fluid_lam0, [LJ("sp", 0.9)], 1.0, B, C_NONE, M_SHIFTED, False),
    Row("br-mol0-lj-distance-geometric", mol_uncharged, [LJ("distance", 1.0, w=0.5, geo=True)], 1.1, B, C_NONE, M_PLAIN,
        False),
    Row("br-mol0-lj-sp-lambda0", mol_uncharged_lam0, [LJ("sp", 1.0, w=0.5)], 1.1, B, C_NONE, M_SHIFTED, False),
    Row("br-mol0-lj-cubic", mol_uncharged, [LJ("cubic", 1.0, 0.8, w=0.5)], 1.1, B, C_NONE, M_TWO, False),
    # ---- brick, plain Coulomb
    Row("br-mol-lj-coulomb-distance", mol_large, [LJ("distance", 1.0, w=0.5), COUL("distance", 1.0, w=0.8333)], 1.1, B,
        C_PLAIN, M_PLAIN, False),
    Row("br-mol-lj-coulomb-sf", mol_large, [LJ("distance", 1.0, w=0.5), COUL("sf", 1.0, w=0.8333)], 1.1, B, C_PLAIN,
        M_SHIFTED, False),
    *[Row(f"br-mol-lj-coulomb-{c}", mol_large, [LJ(c, 1.0, 0.8, w=0.5), COUL(c, 1.0, 0.8, w=0.8333)], 1.1, B, C_PLAIN,
          M_TWO, False) for c in ("cubic", "poly")],
    # ---- brick, reaction field
    Row("br-mol-lj-crf", mol_large, [LJ("distance", 1.0, w=0.5), CRF(1.0, w=0.8333)], 1.1, B, C_CRF, M_PLAIN, False),
    Row("br-mol-lj-nocutoff-nl-crf", mol_large, [LJ("none", w=0.5), CRF(1.0, w=0.8333)], 1.2, B, C_CRF, M_PLAIN, False,
        1.2),
    Row("br-mol-lj-sf0.9-geometric-crf1.1", mol_large, [LJ("sf", 0.9, w=0.5, geo=True), CRF(1.1, w=0.8333)], 1.2, B,
        C_CRF, M_SHIFTED, False),
    Row("br-mol-lj-poly-crf", mol_large, [LJ("poly", 1.0, 0.8, w=0.5), CRF(1.0, w=0.8333)], 1.1, B, C_CRF, M_TWO, False),
    # ---- brick, Ewald
    *[Row(f"br-mol-lj-ewald-{'approx' if a else 'exact'}", mol_large, [LJ("distance", 1.0, w=0.5),
          EWALD(1.0, w=0.8333, approx=a)], 1.1, B, C_EWALD, M_PLAIN, False) for a in (False, True)],
    Row("br-mol-lj-sf1.1-ewald0.9", mol_large, [LJ("sf", 1.1, w=0.5), EWALD(0.9, w=0.8333)], 1.2, B, C_EWALD, M_SHIFTED,
        False),
    Row("br-mol-lj-cubic-ewald-exact", mol_large, [LJ("cubic", 1.0, 0.8, w=0.5), EWALD(1.0, w=0.8333, approx=False)], 1.1,
        B, C_EWALD, M_TWO, False),
]


# ---------------------------------------------------------------------------------------------------
# which kernel ran: demangled names of the device activity recorded by torch.profiler (Kineto / CUPTI)
# ---------------------------------------------------------------------------------------------------
_KERNEL = re.compile(r"\b(allpairs|brick)_force_kernel<([^<>]*)>")


def _targ(s):
    s = re.sub(r"^\(\w+\)", "", s.strip())  # a cast prefix such as "(int)2"
    if s.isdigit():
        return int(s)
    return {"true": True, "false": False}.get(s, s)


def force_kernels(prof):
    """{(path, T, COUL, UNI, CUTM, EN)} of the pair-force kernels the profile recorded; UNI is None for all-pairs."""
    out = set()
    for ev in prof.events():
        m = _KERNEL.search(ev.name)
        if not m:
            continue
        a = [_targ(x) for x in m.group(2).split(",")]
        if m.group(1) == "allpairs":
            out.add(("allpairs", a[0], a[1], None, a[2], a[3]))
        else:
            out.add(("brick", a[0], a[1], a[2], a[3], a[4]))
    return out


def all_instantiations():
    s = set()
    for t in DTYPES.values():
        for en in (False, True):
            for cutm in (M_PLAIN, M_SHIFTED, M_TWO):
                for coul in (C_NONE, C_PLAIN, C_CRF, C_EWALD):
                    s.add(("allpairs", t, coul, None, cutm, en))
                    s.add(("brick", t, coul, False, cutm, en))
                s.add(("brick", t, C_NONE, True, cutm, en))
    return s


OBSERVED = set()
RAN = set()


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("row", VARIANTS, ids=[r.id for r in VARIANTS])
def test_variant_matches_oracle(row, dtype):
    sd = row.system()
    mbi, oi = [i[0] for i in row.inters], [i[1] for i in row.inters]
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        H.check(sd, tuple(mbi), oi, dtype, r_list=row.r_list, expect_path=row.path, label=row.id,
                nl_radius=row.nl_radius)
    ran = force_kernels(prof)
    print(f"    kernels: {sorted(ran, key=str)}")
    t = DTYPES[dtype]
    expect = {("brick" if row.path else "allpairs", t, row.coul, row.uni if row.path else None, row.cutm, en)
              for en in (False, True)}
    assert ran == expect, (ran, expect)
    OBSERVED.update(ran)
    RAN.add((row.id, t))
    if "lam" in sd and dtype == np.float64:
        # lambda = 0 is the LJ zero shortcut: bit-identical to the same atoms given eps = 0
        zeroed = {k: v for k, v in sd.items() if k != "lam"}
        zeroed["eps"] = np.where(sd["lam"] == 0, 0.0, sd["eps"])
        lam = H.make_system(sd, tuple(mbi), dtype, r_list=row.r_list)
        ref = H.make_system(zeroed, tuple(mbi), dtype, r_list=row.r_list)
        assert np.array_equal(mb.forces(lam), mb.forces(ref))
        assert mb.potential_energy(lam) == mb.potential_energy(ref)
        assert lam.stats()["path"] == ref.stats()["path"] == row.path
        lam.close(); ref.close()


# ---------------------------------------------------------------------------------------------------
# known answers at the edges
# ---------------------------------------------------------------------------------------------------
L_BOX, R_LIST = 8.0, 1.25
KE = o.COULOMB_CONST


def _lj_closed(r, sig=0.3, eps=0.2):
    s6 = (sig / r) ** 6
    return 24 * eps / r * (2 * s6 * s6 - s6), 4 * eps * (s6 * s6 - s6)  # F (along r, repulsive > 0), E


def _crf_consts(rc, solvent=78.3):
    return (1 / rc ** 3) * (solvent - 1) / (2 * solvent + 1), (1 / rc) * 3 * solvent / (2 * solvent + 1)


def _spectators(pair_x):
    """Atoms on a 1.6 nm grid, more than 2 nm (> r_list) from both pair atoms: they put the system on the cell-list path
    (n >= 64) without interacting with anything."""
    g = 0.8 + 1.6 * np.arange(5)
    pts = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    keep = np.ones(len(pts), bool)
    for p in pair_x:
        d = pts - p
        d -= L_BOX * np.round(d / L_BOX)
        keep &= np.einsum("ij,ij->i", d, d) > 4.0
    return pts[keep]


def _pair_run(inter, xi, xj, dtype, brick, charges=(0.0, 0.0), sigmas=(0.3, 0.3), epss=(0.2, 0.2)):
    """Force on atom j along x and total energy of a pair at xi, xj (x coordinates; y = z = 4), on the all-pairs path
    (2 atoms) or on the cell-list path (spectators added)."""
    x = np.array([[xi, 4.0, 4.0], [xj, 4.0, 4.0]], np.float64)
    q, sig, eps = list(charges), list(sigmas), list(epss)
    if brick:
        sp = _spectators(x.astype(dtype).astype(np.float64))
        x = np.vstack([x, sp])
        q += [0.0] * len(sp); sig += [0.3] * len(sp); eps += [0.2] * len(sp)
    n = len(x)
    atoms = mb.atoms_from_arrays(np.full(n, 10.0), q, sig, eps, dtype)
    xs = x.astype(dtype)
    xs[1, 0] = xj  # xj is given in dtype (an ulp-exact value)
    s = mb.System(atoms=atoms, coords=xs, boundary=mb.CubicBoundary(L_BOX), pairwise_inters=(inter,), dtype=dtype,
                  neighbor_finder=mb.GPUNeighborFinder(dist_cutoff=R_LIST) if brick else None)
    f = mb.forces(s)
    e = mb.potential_energy(s)
    st = s.stats()
    s.close()
    assert st["path"] == (1 if brick else 0), st
    if brick:
        assert n >= 64 and not f[2:].any()
    return float(f[1, 0]), float(e), f


# cutoff kind -> (interaction builder(use_neighbors), charges, closed-form (F, E) at r = rc = 1, (F, E) at r_act or None)
_F1, _E1 = _lj_closed(1.0)
_KRF, _CRF = _crf_consts(1.0)
_EDGE_CASES = {
    "lj-distance": (lambda nl: mb.LennardJones(cutoff=mb.DistanceCutoff(1.0), use_neighbors=nl), (0.0, 0.0), (_F1, _E1), abs(_E1), None),
    "coulomb-distance": (lambda nl: mb.Coulomb(cutoff=mb.DistanceCutoff(1.0), use_neighbors=nl), (1.0, -1.0), (-KE, -KE), KE, None),
    "lj-shifted-potential": (lambda nl: mb.LennardJones(cutoff=mb.ShiftedPotentialCutoff(1.0), use_neighbors=nl), (0.0, 0.0), (_F1, 0.0), abs(_E1), None),
    "lj-shifted-force": (lambda nl: mb.LennardJones(cutoff=mb.ShiftedForceCutoff(1.0), use_neighbors=nl), (0.0, 0.0), (0.0, 0.0), abs(_E1) + abs(_F1), None),
    "crf": (lambda nl: mb.CoulombReactionField(dist_cutoff=1.0, use_neighbors=nl), (1.0, -1.0), (-KE * (1 - 2 * _KRF), 0.0), KE * _CRF, None),
    "lj-cubic-spline": (lambda nl: mb.LennardJones(cutoff=mb.CubicSplineCutoff(0.5, 1.0), use_neighbors=nl), (0.0, 0.0), (0.0, 0.0), 1.0, _lj_closed(0.5)),
    "lj-polynomial": (lambda nl: mb.LennardJones(cutoff=mb.PolynomialCutoff(0.5, 1.0), use_neighbors=nl), (0.0, 0.0), (0.0, 0.0), 1.0, _lj_closed(0.5)),
}


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("path", ["allpairs", "brick"])
@pytest.mark.parametrize("where", ["inside", "periodic"])
@pytest.mark.parametrize("case", list(_EDGE_CASES))
def test_pair_exactly_at_cutoff(case, where, path, dtype):
    """The reference keeps a pair with r <= dist_cutoff (src/cutoffs.jl:20, :36). rc = 1.0 and the coordinates below are
    exact in f32 and f64, and so is their difference on both paths (the all-pairs minimum image, the cell-list path's
    ghost copies at x -/+ L), hence r^2 = 1 = rc^2 exactly: the pair counts; one ulp further it gives exactly zero.
    Values against closed-form float64 within 64 ulp of the dtype times the size of the terms involved."""
    build, q, (f_rc, e_rc), scale, act = _EDGE_CASES[case]
    brick = path == "brick"
    inter = build(brick)
    T = np.dtype(dtype).type
    tol = 64 * np.finfo(dtype).eps
    # (x_i, x_j) at distance r, and the sign of F(r) in the force on j along x
    place = {"inside": lambda r: (3.0, T(3.0 + r), 1.0), "periodic": lambda r: (r / 2, T(L_BOX - r / 2), -1.0)}[where]
    xi, xj, sgn = place(1.0)
    fj, e, _ = _pair_run(inter, xi, xj, dtype, brick, charges=q)
    fs = max(abs(f_rc), scale)
    print(f"[{case} {where} {path} {np.dtype(dtype).name}] r = rc: F = {fj:.9e} (closed form {sgn * f_rc:.9e}), "
          f"E = {e:.9e} (closed form {e_rc:.9e})")
    assert abs(fj - sgn * f_rc) <= tol * fs
    assert abs(e - e_rc) <= tol * max(abs(e_rc), scale)
    if f_rc != 0.0 or e_rc != 0.0:
        assert fj != 0.0 or e != 0.0  # the pair counted
    # one ulp beyond the cutoff
    xj_out = np.nextafter(xj, T(np.inf) if where == "inside" else T(-np.inf))
    fj, e, f = _pair_run(inter, xi, xj_out, dtype, brick, charges=q)
    assert not f.any() and e == 0.0, (f[:2], e)
    if act is not None:  # two-point cutoffs leave the interaction unchanged up to dist_activation
        xi, xj, sgn = place(0.5)
        fj, e, _ = _pair_run(inter, xi, xj, dtype, brick, charges=q)
        assert abs(fj - sgn * act[0]) <= tol * abs(act[0]) and abs(e - act[1]) <= tol * abs(act[1])


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("path", ["allpairs", "brick"])
def test_geometric_sigma_literal(path, dtype):
    """test/interactions.jl:15-18: sigma (0.3, 0.2), eps (0.2, 0.1); geometric sigma sqrt(0.06) = 0.2449489742783178,
    eps sqrt(0.02). E(sigma) = 0 and E(2^(1/6) sigma) = -eps with F = 0. The second atom's coordinate is rounded to the
    dtype, so the bound adds |dE/dr| or |dF/dr| times the rounding of r."""
    sig, eps = 0.2449489742783178, 0.14142135623730953
    brick = path == "brick"
    inter = mb.LennardJones(cutoff=mb.DistanceCutoff(1.0), use_neighbors=brick, sigma_mixing="geometric")
    tol = 64 * np.finfo(dtype).eps
    dx = 2 * np.finfo(dtype).eps * 4.0  # rounding of x_j near 4
    T = np.dtype(dtype).type
    fj, e, _ = _pair_run(inter, 3.0, T(3.0 + sig), dtype, brick, sigmas=(0.3, 0.2), epss=(0.2, 0.1))
    print(f"[geometric {path} {np.dtype(dtype).name}] E(sigma) = {e:.3e}, F = {fj:.6e}")
    assert abs(e) <= 24 * eps / sig * dx + tol * 4 * eps
    assert abs(fj - 24 * eps / sig) <= (456 * eps / sig ** 2) * dx + tol * 48 * eps / sig
    rmin = sig * 2 ** (1 / 6)
    fj, e, _ = _pair_run(inter, 3.0, T(3.0 + rmin), dtype, brick, sigmas=(0.3, 0.2), epss=(0.2, 0.1))
    print(f"[geometric {path} {np.dtype(dtype).name}] E(2^(1/6) sigma) = {e:.12f}, F = {fj:.3e}")
    assert abs(e + eps) <= tol * 4 * eps + 36 * eps / rmin ** 2 * dx ** 2
    assert abs(fj) <= 72 * eps / rmin ** 2 * dx + tol * 48 * eps / rmin


# ---------------------------------------------------------------------------------------------------
def test_zz_every_instantiation_ran():
    """All 108 pair-force instantiations were observed on the device by the rows above."""
    want_rows = {(r.id, t) for r in VARIANTS for t in DTYPES.values()}
    if RAN != want_rows:
        pytest.skip(f"{len(want_rows - RAN)} of {len(want_rows)} rows did not run in this session")
    want = all_instantiations()
    assert len(want) == 108
    print(f"observed {len(OBSERVED & want)} of {len(want)} pair-force instantiations (profiler kernel names)")
    assert OBSERVED == want, sorted(want - OBSERVED, key=str)
