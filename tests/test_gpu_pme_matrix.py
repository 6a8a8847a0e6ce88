"""The device PME (csrc/pme.cuh, launch_pme / pme_prepare in csrc/engine.cu) against the f64 checker oracle/pme.py across
meshes, precisions, both force paths and the charge and coordinate edges, plus the live-context setters.

A PME-only System (no pairwise interaction, PME as the only general interaction) runs on the all-pairs path (path 0): its
forces are the reciprocal-space part plus the Ewald exclusion forces, its energy those two plus the self and
neutralising-background terms, i.e. oracle.pme.pme_reciprocal + oracle.pme.ewald_exclusion. The brick path (path 1) needs
a pairwise interaction on the neighbour list, so the path tests add CoulombEwald (exact erfc) and subtract the C oracle's
real-space term. tests/test_pme_direct_ewald.py pins oracle/pme.py itself against a direct Ewald sum on these shapes.

Bars. f64: max|dF| <= 1e-9 max|F_ref| and |dE| <= 1e-9 |E_ref| (tests/test_pme_host.py's bars). f32 against the same f64
oracle: F32_BAR_F / F32_BAR_E below, set from runs on an H100 with about 5x headroom."""
import ctypes as C

import numpy as np
import pytest

import mbhelpers as H
import mollyb200 as mb
from oracle import oracle as o
from oracle import pme
from test_pme_direct_ewald import charged_system

pytestmark = pytest.mark.gpu

F64, F32 = np.float64, np.float32
# f32 bars. Measured on one H100 80GB HBM3 at a 700 W power limit over this file's systems: worst max|dF|/max|F| 2.2e-5
# (the 154^3 mesh with uncharged atoms, whose max|F| is the smallest), at most 4.0e-6 on every other mesh and 2.0e-6 on
# 6mrr (2.2e-6 in another run); worst |dE|/|E| 1.5e-6. Bars: about 5x those.
F32_BAR_F, F32_BAR_E = 1e-4, 7e-6

# name -> box, r_cut, error_tol. "aniso" and "cubic" also fit the brick path (box >= 2.5 r_list with r_list = r_cut + 0.1).
MESHES = {
    "cubic": (np.array([3.0, 3.0, 3.0]), 1.0, 5e-4),
    "cubic-tol1e-3": (np.array([3.0, 3.0, 3.0]), 1.0, 1e-3),
    "aniso": (np.array([2.0, 3.3, 5.1]), 0.7, 5e-4),
    "k6": (np.array([0.8, 1.0, 3.1]), 1.0, 1e-3),  # K = (6, 7, 21)
    "fine": (np.array([7.0, 7.0, 7.0]), 1.0, 1e-5),  # 154^3 mesh: 28 500 convolution blocks
}
CHARGES = ["neutral", "plus3", "minus3", "zeros"]
N_ATOMS = 200


def plan(box, r_cut, tol):
    """Mesh dimensions from the library's own plan (mb_pme_plan), the K that pme_prepare uses."""
    L = mb.capi.load()
    alpha, mesh = C.c_double(), (C.c_int32 * 3)()
    mb.capi.check(L.mb_pme_plan((C.c_double * 3)(*box), r_cut, tol, 5, C.byref(alpha), mesh, None, 0))
    return tuple(mesh)


def test_matrix_meshes():
    """The matrix contains what it claims: K = 6 in one dimension, odd and even K (the Nyquist fold k < (K+1)/2 both
    ways), a strongly anisotropic mesh and a mesh with tens of thousands of convolution blocks; and the library's plan
    is the oracle's."""
    ks = {name: plan(*m) for name, m in MESHES.items()}
    for name, (box, rc, tol) in MESHES.items():
        assert ks[name] == pme.pme_mesh_dims(box, pme.pme_alpha(rc, tol), tol), name
    flat = [k for kk in ks.values() for k in kk]
    assert ks["k6"][0] == 6
    # a coarse odd dimension: there the Gaussian weight at the fold is not negligible (exp(-pi^2 m^2 / alpha^2) ~ 6e-7)
    assert ks["k6"][1] == 7
    assert any(k % 2 for k in flat) and any(k % 2 == 0 for k in flat)
    assert max(ks["aniso"]) >= 2 * min(ks["aniso"])
    assert np.prod(ks["fine"]) / 128 > 20000


def system_with_edges(mesh, charges, coords, seed=3, n=N_ATOMS):
    """n charged atoms at least 0.15 nm apart (except the pairs below) and the exclusion pairs, 0-based (m, 2), PME's list:
      0-1  straddles the x faces (raw |dx| > L/2);  2-3 the y faces;  4-5 the z faces
      6-7  listed twice: once as excluded, once as special
      8-9  at r = 1e-4 nm;  10-11 coincident (the erf(alpha r) <= 1e-6 branch)
      12.. bonded-like pairs 0.1-0.25 nm apart
    coords: 'wrapped' (in [0, L)), 'shifted' (every atom moved by a random +-1 box length per dimension) or 'planes'
    (atoms exactly on the 0 and L planes and 1e-7 nm outside them)."""
    box, rc, tol = MESHES[mesh]
    rng = np.random.default_rng(seed)
    _, q = charged_system(box, n, charges, seed)
    x = np.zeros((n, 3))
    k = 0
    while k < n:
        c = rng.random(3) * box
        d = x[:k] - c
        d -= box * np.round(d / box)
        if k == 0 or (d * d).sum(1).min() > 0.15 ** 2:
            x[k] = c
            k += 1
    for a, dim in ((0, 0), (2, 1), (4, 2)):  # straddling pairs
        x[a + 1] = x[a]
        x[a, dim], x[a + 1, dim] = 0.04, box[dim] - 0.07
    x[7] = x[6] + np.array([0.06, -0.08, 0.05])
    x[9] = x[8] + np.array([1e-4, 0.0, 0.0])
    x[11] = x[10]
    pairs = [(0, 1), (2, 3), (4, 5), (6, 7), (6, 7), (8, 9), (10, 11)]
    for a in range(12, 40, 2):
        v = rng.normal(size=3)
        x[a + 1] = (x[a] + v / np.linalg.norm(v) * rng.uniform(0.1, 0.25)) % box
        pairs.append((a, a + 1))
    x %= box
    if coords == "shifted":
        x = x + box * rng.choice([-1.0, 1.0], size=(n, 3))
    elif coords == "planes":
        x[40, 0], x[41, 0], x[42, 1], x[43, 2] = 0.0, box[0], 0.0, box[2]
        x[44, 0], x[45, 1], x[46, 2], x[47, 0] = -1e-7, box[1] + 1e-7, -1e-7, box[0] + 1e-7
        pairs.append((40, 41))  # a pair across the x planes, both atoms exactly on one of them
    pairs = np.array(pairs, np.int32)
    excluded = np.delete(pairs, 4, axis=0)  # the second (6, 7) goes to the special list
    special = np.array([[6, 7]], np.int32)
    return dict(n=n, box=box, coords=x, velocities=np.zeros((n, 3)), mass=np.full(n, 12.0), charge=q,
                sigma=np.full(n, 0.3), eps=np.zeros(n), excluded=excluded, special=special, pairs=pairs), rc, tol


def pme_system(sd, rc, tol, dtype, eps_r=1.0, pairwise=(), r_list=0.0):
    atoms = mb.atoms_from_arrays(sd["mass"], sd["charge"], sd["sigma"], sd["eps"], dtype)
    nf = None
    if pairwise:
        nf = mb.GPUNeighborFinder(dist_cutoff=r_list, excluded_pairs=sd["excluded"] + 1, special_pairs=sd["special"] + 1)
    return mb.System(atoms=atoms, coords=sd["coords"].astype(dtype), boundary=mb.CubicBoundary(*sd["box"]),
                     pairwise_inters=pairwise, neighbor_finder=nf, dtype=dtype,
                     general_inters=(mb.PME(dist_cutoff=rc, error_tol=tol, eps_r=eps_r, excluded_pairs=sd["pairs"] + 1),))


def pme_reference(sd, rc, tol, dtype, eps_r=1.0):
    """oracle/pme.py at the coordinates the device sees (rounded to dtype), in f64."""
    x = sd["coords"].astype(dtype).astype(F64)
    q = sd["charge"].astype(dtype).astype(F64)
    fr, er, _ = pme.pme_reciprocal(x, q, sd["box"], r_cut=rc, error_tol=tol, eps_r=eps_r)
    with np.errstate(divide="ignore", invalid="ignore"):  # (the coincident pair: np.where evaluates both branches)
        fx, ex = pme.ewald_exclusion(x, q, sd["box"], sd["pairs"], r_cut=rc, error_tol=tol, eps_r=eps_r)
    return fr + fx, er + ex


def evaluate(s):
    """forces_energy, forces and potential_energy: they must agree with one another."""
    f, e = mb.forces_energy(s)
    f2, e2 = mb.forces(s), mb.potential_energy(s)
    tol_f = (1e-12 if s.dtype == F64 else 1e-6) * np.abs(f).max()
    assert np.abs(f2 - f).max() <= tol_f and abs(e2 - e) <= (1e-12 if s.dtype == F64 else 1e-6) * abs(e), (e, e2)
    return f.astype(F64), e


def check(f, e, f_ref, e_ref, dtype, label):
    df = np.abs(f - f_ref).max() / np.abs(f_ref).max()
    de = abs(e - e_ref) / abs(e_ref)
    bf, be = (1e-9, 1e-9) if dtype == F64 else (F32_BAR_F, F32_BAR_E)
    print(f"[{label} {np.dtype(dtype).name}] max|dF|/max|F| = {df:.2e} (bar {bf:g})  |dE|/|E| = {de:.2e} (bar {be:g})  "
          f"E = {e_ref:.6f}")
    assert df <= bf and de <= be


CASES = ([(m, c, 1.0, "wrapped") for m in MESHES for c in CHARGES]
         + [(m, "plus3", 4.0, "wrapped") for m in MESHES]
         + [(m, "zeros", 1.0, co) for m in MESHES for co in ("shifted", "planes")])


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("mesh,charges,eps_r,coords", CASES, ids=[f"{m}-{c}-eps{e:g}-{co}" for m, c, e, co in CASES])
def test_pme_only_vs_oracle(mesh, charges, eps_r, coords, dtype):
    sd, rc, tol = system_with_edges(mesh, charges, coords)
    if charges == "zeros":
        assert (sd["charge"] == 0).sum() >= 0.2 * sd["n"]
    s = pme_system(sd, rc, tol, dtype, eps_r=eps_r)
    f, e = evaluate(s)
    assert s.stats()["path"] == 0
    f_ref, e_ref = pme_reference(sd, rc, tol, dtype, eps_r)
    check(f, e, f_ref, e_ref, dtype, f"PME-only {mesh} {charges} eps_r {eps_r:g} {coords} K={plan(*MESHES[mesh])}")
    s.close()


def real_space_reference(sd, rc, tol, dtype, wrap):
    """CoulombEwald(rc, tol, use_neighbors=true, approximate_erfc=false) from the C oracle, f64. The pair kernels see the
    coordinates as the reference's forces() does: the all-pairs kernel applies vector_1D (one image shift, src/spatial.jl)
    to them as given, the brick path wraps them into the box when it bins them (wrap=True)."""
    inter = o.Inter(o.EWALD_REAL, o.CUT_DISTANCE, rc, ewald_alpha=pme.pme_alpha(rc, tol), use_neighbors=True)
    x = sd["coords"].astype(dtype).astype(F64)
    if wrap:
        x = x - np.floor(x / sd["box"]) * sd["box"]
    orc = H.make_oracle(dict(sd, charge=sd["charge"].astype(dtype).astype(F64)), [inter])
    f, e, _ = orc.forces_allpairs(x)
    return f, e


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("coords", ["wrapped", "shifted", "planes"])
@pytest.mark.parametrize("mesh", ["cubic", "aniso"])
def test_pme_paths_agree_and_match_oracle(mesh, coords, dtype):
    """The same system on the all-pairs path and on the brick path (where slot_of() remaps the exclusion pairs): each
    against real space (C oracle) + PME (oracle/pme.py), and the two paths against each other to 1e-12 in f64. With
    coordinates a box length outside the box the two paths' real-space terms differ as the reference's would (see
    real_space_reference), so there the paths are compared through their PME parts only."""
    sd, rc, tol = system_with_edges(mesh, "plus3", coords)
    ce = (mb.CoulombEwald(dist_cutoff=rc, error_tol=tol, use_neighbors=True, approximate_erfc=False),)
    fp, ep = pme_reference(sd, rc, tol, dtype)
    out = {}
    for path, r_list in ((0, 0.0), (1, rc + 0.1)):
        fr, er = real_space_reference(sd, rc, tol, dtype, wrap=path == 1)
        s = pme_system(sd, rc, tol, dtype, pairwise=ce, r_list=r_list)
        f, e = evaluate(s)
        assert s.stats()["path"] == path
        out[path] = (f - fr, e - er) if coords == "shifted" else (f, e)
        # the PME part: what the device computed beyond the real-space term, against oracle/pme.py
        check(f - fr, e - er, fp, ep, dtype, f"path {path} {mesh} {coords} (CoulombEwald subtracted)")
        check(f, e, fr + fp, er + ep, dtype, f"path {path} {mesh} {coords} (total)")
        s.close()
    if dtype == F64:
        (f0, e0), (f1, e1) = out[0], out[1]
        assert np.abs(f1 - f0).max() <= 1e-12 * np.abs(f0).max() and abs(e1 - e0) <= 1e-12 * abs(e0)


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_6mrr_pme_only_vs_oracle(golden_6mrr, dtype):
    """PME-only on 6mrr: 15 954 atoms, mesh 46 x 46 x 51, 18k excluded + special pairs (the f32 PME path on a real
    system)."""
    g = golden_6mrr
    sd = H.sixmrr_description(g)
    sd["pairs"] = np.concatenate([g["excluded"], g["special"]]).astype(np.int32)
    assert len(sd["pairs"]) > 18000
    s = pme_system(sd, 1.0, 5e-4, dtype)
    f, e = evaluate(s)
    assert s.stats()["path"] == 0
    f_ref, e_ref = pme_reference(sd, 1.0, 5e-4, dtype)
    check(f, e, f_ref, e_ref, dtype, "6mrr PME-only")
    s.close()


def test_pme_forces_are_the_energy_gradient_f64():
    """Independent of the oracle: SPME forces are the exact gradient of the SPME energy (order-5 B-splines are C^3), so a
    central difference of the device energy (h = 1e-5 nm) matches the device force to 1e-6 of max|F|. Ten atoms x three
    directions on the anisotropic mesh with net charge, including atoms of ordinary exclusion pairs."""
    sd, rc, tol = system_with_edges("aniso", "plus3", "wrapped")
    s = pme_system(sd, rc, tol, F64)
    f, _ = evaluate(s)
    fmax = np.abs(f).max()
    h = 1e-5
    worst = 0.0
    for i in [12, 13, 20, 21, 50, 77, 101, 140, 170, 199]:
        for d in range(3):
            x0 = s.coords[i, d]
            s.coords[i, d] = x0 + h
            ep = mb.potential_energy(s)
            s.coords[i, d] = x0 - h
            em = mb.potential_energy(s)
            s.coords[i, d] = x0
            fd = -(ep - em) / (2 * h)
            worst = max(worst, abs(fd - f[i, d]) / fmax)
    print(f"[PME finite difference f64] max |F_fd - F| / max|F| = {worst:.2e} (bar 1e-6)")
    assert worst <= 1e-6
    s.close()


# ---- live contexts: a setter between evaluations gives what a fresh context gives -----------------------------------
def _same(a, b, tol=1e-12):
    (fa, ea), (fb, eb) = a, b
    assert np.abs(fa - fb).max() <= tol * np.abs(fb).max() and abs(ea - eb) <= tol * abs(eb), (ea, eb)


def _set_atoms(s, sd, dtype):
    atoms = mb.atoms_from_arrays(sd["mass"], sd["charge"], sd["sigma"], sd["eps"], dtype)
    mb.capi.check(s._L.mb_set_atoms(s.engine(), len(atoms), atoms.ctypes.data))


def test_live_set_box_replans_pme():
    """mb_set_box to a larger box and then to a smaller one on a live PME context: each gives another mesh (a new grid,
    cuFFT plan, moduli and partial buffer), and the same forces and energy as a fresh context in that box."""
    sd, rc, tol = system_with_edges("cubic", "plus3", "wrapped")
    s = pme_system(sd, rc, tol, F64)
    evaluate(s)
    meshes = {plan(sd["box"], rc, tol)}
    for scale in (1.3, 0.9):
        box = MESHES["cubic"][0] * scale
        meshes.add(plan(box, rc, tol))
        mb.capi.check(s._L.mb_set_box(s.engine(), (C.c_double * 3)(*box)))
        sd2 = dict(sd, box=box)
        ref = pme_system(sd2, rc, tol, F64)
        _same(evaluate(s), evaluate(ref))
        check(*evaluate(s), *pme_reference(sd2, rc, tol, F64), F64, f"live set_box x{scale}")
        ref.close()
    assert len(meshes) == 3
    s.close()


def test_live_set_atoms_new_charges_pme():
    """mb_set_atoms with every charge scaled by 0.7 (same n) on a live PME context: the self and background energy must
    follow the new charges, as the forces do."""
    sd, rc, tol = system_with_edges("aniso", "plus3", "wrapped")
    s = pme_system(sd, rc, tol, F64)
    evaluate(s)
    sd2 = dict(sd, charge=sd["charge"] * 0.7)
    _set_atoms(s, sd2, F64)
    ref = pme_system(sd2, rc, tol, F64)
    _same(evaluate(s), evaluate(ref))
    check(*evaluate(s), *pme_reference(sd2, rc, tol, F64), F64, "live set_atoms q x 0.7")
    s.close()
    ref.close()


def test_live_set_atoms_new_lj_dispersion_correction():
    """The same for LJDispersionCorrection: its factors follow the sigma / epsilon of mb_set_atoms."""
    sd = H.readme_system(100, 2.0, seed=1)
    inters = (mb.LennardJones(cutoff=mb.DistanceCutoff(0.9)),)

    def make(d):
        atoms = mb.atoms_from_arrays(d["mass"], d["charge"], d["sigma"], d["eps"], F64)
        return mb.System(atoms=atoms, coords=d["coords"], boundary=mb.CubicBoundary(*d["box"]), pairwise_inters=inters,
                         dtype=F64, general_inters=(mb.LJDispersionCorrection(0.9),))

    s = make(sd)
    e0 = mb.potential_energy(s)
    rng = np.random.default_rng(4)
    sd2 = dict(sd, sigma=sd["sigma"] * rng.uniform(0.8, 1.2, sd["n"]), eps=sd["eps"] * rng.uniform(0.5, 2.0, sd["n"]))
    _set_atoms(s, sd2, F64)
    ref = make(sd2)
    e_live, e_ref = mb.potential_energy(s), mb.potential_energy(ref)
    assert abs(e_ref - e0) > 1e-3 * abs(e0)
    assert abs(e_live - e_ref) <= 1e-12 * abs(e_ref), (e_live, e_ref)
    s.close()
    ref.close()


def test_live_set_atoms_fewer_atoms_refused_until_set_pme():
    """mb_set_atoms with fewer atoms while PME exclusion pairs index past the new n: the next evaluation is refused on the
    host with MB_ERR_STATE, before anything launches; after mb_set_pme with pairs inside the new n it gives what a fresh
    context gives."""
    sd, rc, tol = system_with_edges("cubic", "neutral", "wrapped")
    s = pme_system(sd, rc, tol, F64)
    evaluate(s)
    m = 150
    assert sd["pairs"].max() < m  # every pair is inside the first m atoms except the one added below
    sd2 = {k: (v[:m] if k in ("coords", "velocities", "mass", "charge", "sigma", "eps") else v) for k, v in sd.items()}
    sd2["n"] = m
    pairs_old = np.concatenate([sd["pairs"], [[3, 170]]]).astype(np.int32)
    pi, pj = np.ascontiguousarray(pairs_old[:, 0] + 1), np.ascontiguousarray(pairs_old[:, 1] + 1)
    L, ctx = s._L, s.engine()
    mb.capi.check(L.mb_set_pme(ctx, rc, tol, 5, 1.0, len(pi), pi.ctypes.data, pj.ctypes.data))
    _set_atoms(s, sd2, F64)
    x = np.ascontiguousarray(sd2["coords"], F64)
    f, pe = np.zeros((m, 3)), np.zeros(1)
    rc_call = L.mb_forces_energy_all(ctx, x.ctypes.data, f.ctypes.data, pe.ctypes.data, 0)
    assert rc_call == mb.capi.MB_ERR_STATE, rc_call
    assert b"mb_set_pme" in L.mb_last_error()
    assert not f.any() and pe[0] == 0
    pi, pj = np.ascontiguousarray(sd["pairs"][:, 0] + 1), np.ascontiguousarray(sd["pairs"][:, 1] + 1)
    mb.capi.check(L.mb_set_pme(ctx, rc, tol, 5, 1.0, len(pi), pi.ctypes.data, pj.ctypes.data))
    mb.capi.check(L.mb_forces_energy_all(ctx, x.ctypes.data, f.ctypes.data, pe.ctypes.data, 0))
    ref = pme_system(sd2, rc, tol, F64)
    _same((f, float(pe[0])), evaluate(ref))
    ref.close()
    s.close()
