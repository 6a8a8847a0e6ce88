"""Deterministic synthetic systems shared by the tests, bench.py and smoke().

Generators follow the reference's benchmark scripts (SURVEY.md §8d):
  * argon LJ fluid, rho = 1400 kg/m^3, sigma 0.34 nm, eps 0.997 kJ/mol, m 39.948
    (benchmark/benchmark_gpu_tiles.jl:13-56), FCC lattice + N(0, 0.01 nm) jitter for dynamics;
  * README example: 100 atoms, box 2.0 nm, sigma 0.3, eps 0.2, m 10 (README.md:72-95).
"""
from __future__ import annotations

import numpy as np

ARGON = dict(mass=39.948, sigma=0.34, eps=0.997)
ARGON_DENSITY = 1400.0 * 6.02214076e23 / (39.948e-3) / 1e27  # atoms / nm^3 = 21.105
K_B = 8.31446261815324e-3


def fcc_lattice(cells: int, a: float):
    base = np.array([[0, 0, 0], [0.5, 0.5, 0], [0.5, 0, 0.5], [0, 0.5, 0.5]])
    g = np.stack(np.meshgrid(np.arange(cells), np.arange(cells), np.arange(cells), indexing="ij"), -1).reshape(-1, 3)
    x = (g[:, None, :] + base[None, :, :]).reshape(-1, 3) * a
    return x, cells * a


def lj_fluid(cells: int, seed: int = 42, jitter: float = 0.01, temp: float = 90.0, dtype=np.float32):
    """4*cells^3 argon atoms on an FCC lattice at the reference density, jittered; MB velocities, CM removed."""
    a = (4.0 / ARGON_DENSITY) ** (1.0 / 3.0)
    x, L = fcc_lattice(cells, a)
    rng = np.random.default_rng(seed)
    x = x + rng.normal(0.0, jitter, x.shape) + 0.25 * a
    x = x - np.floor(x / L) * L
    n = len(x)
    v = rng.normal(0.0, np.sqrt(K_B * temp / ARGON["mass"]), (n, 3))
    v -= v.mean(0)
    return dict(n=n, box=np.array([L, L, L]), coords=x.astype(dtype), velocities=v.astype(dtype),
                mass=np.full(n, ARGON["mass"]), charge=np.zeros(n), sigma=np.full(n, ARGON["sigma"]),
                eps=np.full(n, ARGON["eps"]))


def _argon(x, box, seed, temp, dtype):
    rng = np.random.default_rng(seed + 1)
    n = len(x)
    v = rng.normal(0.0, np.sqrt(K_B * temp / ARGON["mass"]), (n, 3))
    v -= v.mean(0)
    box = np.asarray(box, float)
    x = x - np.floor(x / box) * box
    return dict(n=n, box=box, coords=x.astype(dtype), velocities=v.astype(dtype), mass=np.full(n, ARGON["mass"]),
                charge=np.zeros(n), sigma=np.full(n, ARGON["sigma"]), eps=np.full(n, ARGON["eps"]))


def fluid_in_box(box, seed: int = 3, jitter: float = 0.01, temp: float = 90.0, dtype=np.float64):
    """Argon filling a rectangular box: an FCC lattice of about the reference density, stretched per axis to tile the box."""
    box = np.asarray(box, float)
    a = (4.0 / ARGON_DENSITY) ** (1.0 / 3.0)
    m = np.maximum(1, np.round(box / a)).astype(int)
    base = np.array([[0, 0, 0], [0.5, 0.5, 0], [0.5, 0, 0.5], [0, 0.5, 0.5]])
    g = np.stack(np.meshgrid(*[np.arange(k) for k in m], indexing="ij"), -1).reshape(-1, 3)
    x = (g[:, None, :] + base[None, :, :] + 0.25).reshape(-1, 3) * (box / m)
    x = x + np.random.default_rng(seed).normal(0.0, jitter, x.shape)
    return _argon(x, box, seed, temp, dtype)


def argon_droplet(radius: float, box, center, seed: int = 5, jitter: float = 0.01, temp: float = 90.0, dtype=np.float64):
    """A sphere carved out of an FCC argon crystal at the reference density (vacuum around it), wrapped into the box."""
    box = np.asarray(box, float)
    a = (4.0 / ARGON_DENSITY) ** (1.0 / 3.0)
    k = int(np.ceil(radius / a)) + 1
    x, _ = fcc_lattice(2 * k, a)
    x = x - k * a + 0.25 * a
    x = x[np.einsum("ij,ij->i", x, x) <= radius * radius]
    x = x + np.random.default_rng(seed).normal(0.0, jitter, x.shape) + np.asarray(center, float)
    return _argon(x, box, seed, temp, dtype)


def argon_slab(thickness: float, box, seed: int = 9, dtype=np.float64):
    """A liquid argon film filling x and y, `thickness` nm thick in z and centred in the box, with vacuum above and below."""
    box = np.asarray(box, float)
    f = fluid_in_box([box[0], box[1], thickness], seed=seed, dtype=np.float64)
    x = f["coords"] + np.array([0.0, 0.0, 0.5 * (box[2] - thickness)])
    return _argon(x, box, seed, 90.0, dtype)


def nearest_partners(sysd, hub: int, count: int, skip=()):
    """The `count` atoms nearest to atom `hub` (minimum image) that are not `hub` and not in `skip`."""
    d = sysd["coords"].astype(np.float64) - sysd["coords"][hub].astype(np.float64)
    d -= sysd["box"] * np.round(d / sysd["box"])
    order = np.argsort(np.einsum("ij,ij->i", d, d), kind="stable")
    skip = set(skip) | {hub}
    return np.array([j for j in order if j not in skip][:count], np.int32)


def readme_system(n: int = 100, box: float = 2.0, seed: int = 1, min_dist: float = 0.3, dtype=np.float64):
    """README.md:72-95: place_atoms-style rejection sampling (setup.jl:23-60), T = 298 K."""
    rng = np.random.default_rng(seed)
    pts = []
    while len(pts) < n:
        c = rng.random(3) * box
        ok = True
        for p in pts:
            d = c - p
            d -= box * np.round(d / box)
            if d @ d < min_dist * min_dist:
                ok = False
                break
        if ok:
            pts.append(c)
    x = np.array(pts)
    v = rng.normal(0.0, np.sqrt(K_B * 298.0 / 10.0), (n, 3))
    return dict(n=n, box=np.array([box] * 3), coords=x.astype(dtype), velocities=v.astype(dtype),
                mass=np.full(n, 10.0), charge=np.zeros(n), sigma=np.full(n, 0.3), eps=np.full(n, 0.2))


def molecular_system(n_mol: int, box, seed: int = 7, dtype=np.float64, stable: bool = False):
    """Small charged 4-site chain molecules A-B-C-D on a jittered grid: 1-2 and 1-3 pairs excluded,
    1-4 pairs special; three LJ types including a zero-epsilon one (TIP3P-hydrogen-like)."""
    rng = np.random.default_rng(seed)
    box = np.asarray(box, float)
    per_dim = int(np.ceil(n_mol ** (1 / 3)))
    grid = np.stack(np.meshgrid(*[np.arange(per_dim)] * 3, indexing="ij"), -1).reshape(-1, 3)[:n_mol]
    centers = (grid + 0.5) / per_dim * box
    coords, q, sig, eps, mass = [], [], [], [], []
    excl, spec = [], []
    tq = [0.4, -0.4, 0.3, -0.3]
    ts = [0.32, 0.30, 0.25, 0.10]
    te = [0.6, 0.4, 0.2, 0.0]
    tm = [12.0, 14.0, 16.0, 1.008]
    if stable:  # for dynamics without bonded terms: every site keeps a repulsive core, charges are mild
        te = [0.6, 0.4, 0.2, 0.15]
        ts = [0.32, 0.30, 0.25, 0.22]
        tq = [0.2, -0.2, 0.15, -0.15]
        tm = [12.0, 14.0, 16.0, 4.0]
    for m, c in enumerate(centers):
        d = rng.normal(size=3)
        d /= np.linalg.norm(d)
        e = np.cross(d, rng.normal(size=3))
        e /= np.linalg.norm(e)
        pos = [c, c + 0.11 * d, c + 0.11 * d + 0.11 * e, c + 0.11 * e + 0.18 * d]
        base = 4 * m
        for k in range(4):
            coords.append(pos[k] + rng.normal(0, 0.005, 3))
            q.append(tq[k]); sig.append(ts[k]); eps.append(te[k]); mass.append(tm[k])
        excl += [(base, base + 1), (base + 1, base + 2), (base + 2, base + 3), (base, base + 2), (base + 1, base + 3)]
        spec += [(base, base + 3)]
    x = np.array(coords)
    x = x - np.floor(x / box) * box
    n = len(x)
    v = rng.normal(0.0, 0.3, (n, 3))
    return dict(n=n, box=box, coords=x.astype(dtype), velocities=v.astype(dtype), mass=np.array(mass),
                charge=np.array(q), sigma=np.array(sig), eps=np.array(eps),
                excluded=np.array(excl, np.int32), special=np.array(spec, np.int32))


def make_oracle(sysd, inters, dtype=np.float64):
    """The oracle has no lambda: an atom with lam == 0 (optional key "lam") gets eps = 0, which is what the reference's
    zero shortcut does to its LJ pairs (src/mixing.jl:7-11)."""
    from oracle import oracle as o
    eps = sysd["eps"] if "lam" not in sysd else np.where(np.asarray(sysd["lam"]) == 0, 0.0, sysd["eps"])
    return o.OracleSystem(box=sysd["box"], mass=sysd["mass"], charge=sysd["charge"], sigma=sysd["sigma"],
                          eps=eps, inters=inters, excluded_pairs=sysd.get("excluded", np.zeros((0, 2), np.int32)),
                          special_pairs=sysd.get("special", np.zeros((0, 2), np.int32)), dtype=dtype)


def make_system(sysd, inters, dtype, r_list=0.0, n_steps=0):
    """mollyb200.System for the same description (exception pairs become 1-based; optional per-atom "lam")."""
    import mollyb200 as mb
    atoms = mb.atoms_from_arrays(sysd["mass"], sysd["charge"], sysd["sigma"], sysd["eps"], dtype)
    if "lam" in sysd:
        atoms["lam"] = sysd["lam"]
    nf = None
    if r_list > 0 or "excluded" in sysd:
        nf = mb.GPUNeighborFinder(dist_cutoff=r_list,
                                  excluded_pairs=sysd.get("excluded", np.zeros((0, 2), np.int32)) + 1,
                                  special_pairs=sysd.get("special", np.zeros((0, 2), np.int32)) + 1, n_steps=n_steps)
    return mb.System(atoms=atoms, coords=sysd["coords"].astype(dtype), boundary=mb.CubicBoundary(*sysd["box"]),
                     velocities=sysd["velocities"].astype(dtype), pairwise_inters=inters, neighbor_finder=nf, dtype=dtype)


# ---------------------------------------------------------------------------------------------------
# CUDA path vs the oracle
# ---------------------------------------------------------------------------------------------------
def tol(dtype, fmax):
    return (1e-9 * fmax + 1e-9) if np.dtype(dtype) == np.float64 else (5e-5 * fmax + 2e-3)


def etol(dtype, e):
    return (1e-11 if np.dtype(dtype) == np.float64 else 2e-6) * max(abs(e), 1.0)


def boundary_atoms(orc, x64, o_inters, delta=3e-6):
    """Atoms that own a pair sitting on a cutoff within f32 rounding of r^2, where a DistanceCutoff /
    reaction-field force is discontinuous (it jumps by F(rc) ~ 1-2 kJ/mol/nm for CRF with water charges), and
    a bound on that jump. The reference has the same sensitivity between its f32 and f64 paths."""
    n = len(x64)
    count = np.zeros(n)
    for rc in sorted({it.r_cut for it in o_inters if it.r_cut > 0}):
        hi = orc.neighbor_list(x64, rc * (1 + delta))
        lo = orc.neighbor_list(x64, rc * (1 - delta))
        key = lambda a: set(map(tuple, a[:, :2].tolist()))
        for i, j in key(hi) - key(lo):
            count[i] += 1
            count[j] += 1
    return count


def cutoff_force_bound(sysd, o_inters):
    """max |F(rc)| of a single pair over the interaction tuple."""
    from oracle import oracle as o
    b = 0.0
    qmax = np.abs(sysd["charge"]).max()
    for it in o_inters:
        rc = it.r_cut
        if rc <= 0:
            continue
        if it.kind == o.LJ and it.cutoff_kind == o.CUT_DISTANCE:
            sig, eps = sysd["sigma"].max(), sysd["eps"].max()
            s6 = (sig / rc) ** 6
            b += abs(24 * eps / rc * (2 * s6 * s6 - s6))
        elif it.kind == o.CRF:
            e = it.solvent_dielectric
            krf = (1 / rc ** 3) * (e - 1) / (2 * e + 1)
            b += it.coulomb_const * qmax * qmax * abs(1 / rc ** 2 - 2 * krf * rc)
        elif it.kind in (o.COULOMB, o.EWALD_REAL) and it.cutoff_kind == o.CUT_DISTANCE:
            b += it.coulomb_const * qmax * qmax / rc ** 2
    return b


def check(sysd, mb_inters, o_inters, dtype, r_list=0.0, expect_path=None, label="", nl_radius=None):
    """Forces, energy and virial of the CUDA path against the f64 oracle on the same dtype-rounded inputs, at the
    tolerances stated in test_gpu_parity.py. The reference is the oracle's all-pairs sum, or its neighbour-list sum
    at `nl_radius` where an interaction's effective cutoff is the list radius (NoCutoff with use_neighbors=true)."""
    import mollyb200 as mb
    xin = sysd["coords"].astype(dtype)
    sd = dict(sysd, coords=xin)
    s = make_system(sd, mb_inters, dtype, r_list=r_list)
    orc = make_oracle(sd, o_inters, dtype=np.float64)
    x64 = xin.astype(np.float64)
    if nl_radius is None:
        f_ref, e_ref, vir_ref = orc.forces_allpairs(x64, virial=True)
    else:
        f_ref, e_ref, vir_ref = orc.forces_nl(x64, orc.neighbor_list(x64, nl_radius), virial=True)
    f = mb.forces(s)
    e = mb.potential_energy(s)
    f2, vir = mb.forces_virial(s)
    st = s.stats()
    if expect_path is not None:
        assert st["path"] == expect_path, st
    fmax = np.abs(f_ref).max()
    err = np.abs(f.astype(np.float64) - f_ref).max()
    print(f"[{label}] n={sysd['n']} dtype={np.dtype(dtype).name} path={st['path']} bricks={st['n_bricks']} "
          f"brick={st['brick_dims']} stride={st['list_stride']} maxnb={st['max_neighbors']} halo={st['max_halo']} "
          f"max|dF|={err:.3e} (max|F|={fmax:.3e}) dE={e - e_ref:.3e} (E={e_ref:.6e})")
    vtol = (1e-9 if np.dtype(dtype) == np.float64 else 1e-4) * max(np.abs(vir_ref).max(), 1.0)
    verr = np.abs(vir.astype(np.float64) - vir_ref).max()
    ferr2 = np.abs(f2.astype(np.float64) - f.astype(np.float64)).max()
    print(f"    virial err={verr:.3e} (tol {vtol:.3e}) |f(force-only) - f(force+virial)|={ferr2:.3e} repeat-equal={np.array_equal(f, mb.forces(s))}")
    if np.dtype(dtype) == np.float32 and err > tol(dtype, fmax):
        # pairs sitting on the cutoff within f32 rounding may land on either side: allow one F(rc) jump each
        nb_pairs = boundary_atoms(orc, xin.astype(np.float64), o_inters)
        fc = cutoff_force_bound(sysd, o_inters)
        per_atom = np.abs(f.astype(np.float64) - f_ref).max(axis=1)
        allowed = tol(dtype, fmax) + nb_pairs * fc
        print(f"    cutoff-boundary atoms: {int((nb_pairs > 0).sum())}; atoms over the plain tolerance: "
              f"{int((per_atom > tol(dtype, fmax)).sum())}; F(rc) bound {fc:.3f}; "
              f"max err off-boundary={per_atom[nb_pairs == 0].max():.3e}")
        assert (per_atom <= allowed).all()
    else:
        assert err <= tol(dtype, fmax)
    assert abs(e - e_ref) <= etol(dtype, e_ref)
    assert np.array_equal(f, mb.forces(s))  # deterministic: same kernel, no atomics
    assert ferr2 <= tol(dtype, fmax)       # the energy/virial variant may contract FMAs differently
    assert verr <= vtol
    s.close()
    return f, e


# ---------------------------------------------------------------------------------------------------
# 6mrr (BASELINE config 3): full system from the golden fixture
# ---------------------------------------------------------------------------------------------------
def sixmrr_description(g):
    box = g["box"]
    x = g["coords"] - np.floor(g["coords"] / box) * box
    return dict(n=len(x), box=box, coords=x, velocities=g["velocities_300K"], mass=g["mass"], charge=g["charge"],
                sigma=g["sigma"], eps=g["eps"], excluded=g["excluded"], special=g["special"])


def sixmrr_specific_lists(g):
    import mollyb200 as mb
    b, a = g["bond_idx"] + 1, g["angle_idx"] + 1
    t = np.concatenate([g["proper_idx"], g["improper_idx"]]) + 1
    tp = np.concatenate([g["proper_par"], g["improper_par"]])
    return (mb.InteractionList2Atoms(b[:, 0], b[:, 1], g["bond_par"][:, 0], g["bond_par"][:, 1]),
            mb.InteractionList3Atoms(a[:, 0], a[:, 1], a[:, 2], g["angle_par"][:, 0], g["angle_par"][:, 1]),
            mb.InteractionList4Atoms(t[:, 0], t[:, 1], t[:, 2], t[:, 3], tp[:, 0], tp[:, 1], tp[:, 2]))


def sixmrr_system(g, dtype, r_list=1.2, n_steps=0, bonded=True, coords=None, velocities=None, device=0, dispersion=False):
    """System(6mrr_equil.pdb, ff99SBildn + tip3p; nonbonded_method=:cutoff) as benchmark/protein.jl:24-37 builds it:
    LJ(rc 1.0, w14 0.5) + CoulombReactionField(rc 1.0, eps 78.3, w14 0.8333) + bonds/angles/torsions."""
    import mollyb200 as mb
    sd = sixmrr_description(g)
    atoms = mb.atoms_from_arrays(sd["mass"], sd["charge"], sd["sigma"], sd["eps"], dtype)
    inters = (mb.LennardJones(cutoff=mb.DistanceCutoff(1.0), use_neighbors=True, weight_special=float(g["lj14scale"])),
              mb.CoulombReactionField(dist_cutoff=1.0, use_neighbors=True, weight_special=float(g["coulomb14scale"])))
    nf = mb.GPUNeighborFinder(dist_cutoff=r_list, excluded_pairs=g["excluded"] + 1, special_pairs=g["special"] + 1, n_steps=n_steps)
    x = sd["coords"] if coords is None else coords
    v = sd["velocities"] if velocities is None else velocities
    return mb.System(atoms=atoms, coords=np.asarray(x).astype(dtype), boundary=mb.CubicBoundary(*sd["box"]),
                     velocities=np.asarray(v).astype(dtype), pairwise_inters=inters, neighbor_finder=nf, dtype=dtype,
                     specific_inter_lists=sixmrr_specific_lists(g) if bonded else (), device=device,
                     general_inters=(mb.LJDispersionCorrection(1.0),) if dispersion else ())  # setup.jl:2000-2004


def sixmrr_oracle(g, dtype=np.float64):
    from oracle import oracle as o
    sd = sixmrr_description(g)
    inters = [o.Inter(o.LJ, o.CUT_DISTANCE, 1.0, weight_special=float(g["lj14scale"]), use_neighbors=True),
              o.Inter(o.CRF, o.CUT_DISTANCE, 1.0, weight_special=float(g["coulomb14scale"]), use_neighbors=True)]
    return make_oracle(sd, inters, dtype=dtype), sd


def bonded_forces_oracle(g, x):
    from oracle import bonded as bd
    box = g["box"]
    f = np.zeros_like(x, dtype=np.float64)
    e = 0.0
    for fn, idx, par in ((bd.bond_forces, "bond_idx", "bond_par"), (bd.angle_forces, "angle_idx", "angle_par"),
                         (bd.torsion_forces, "proper_idx", "proper_par"), (bd.torsion_forces, "improper_idx", "improper_par")):
        ff, ee = fn(np.asarray(x, np.float64), box, g[idx], g[par])
        f += ff
        e += ee
    return f, e


def oracle_vv_with_bonded(g, x, v, dt, n_steps, r_list=1.2, nl_every=10):
    """VelocityVerlet simulate! (src/simulators.jl:547-668) with pairwise (C oracle, neighbour list) + bonded (numpy)
    forces, f64, remove_CM_motion = 1."""
    orc, sd = sixmrr_oracle(g)
    box, m = sd["box"], sd["mass"]
    x = x - np.floor(x / box) * box
    v = orc.remove_cm(v)

    def forces(xx, nl):
        f, _, _ = orc.forces_nl(xx, nl, energy=False)
        return f + bonded_forces_oracle(g, xx)[0]
    nl = orc.neighbor_list(x, r_list)
    f = forces(x, nl)
    for step in range(1, n_steps + 1):
        v = v + f / m[:, None] * (dt / 2)
        x = x + v * dt
        x = x - np.floor(x / box) * box
        f = forces(x, nl)
        v = v + f / m[:, None] * (dt / 2)
        v = orc.remove_cm(v)
        if step % nl_every == 0:
            nl = orc.neighbor_list(x, r_list)
    return x, v


def oracle_vv_pme(g, x, v, dt, n_steps, r_list=1.2, nl_every=10):
    """simulate!(sys_pme_exact, VelocityVerlet(dt), n) of test/protein.jl:277-299 restated with the oracle's pieces (f64):
    LJ + CoulombEwald real space (C oracle over the neighbour list) + bonded + EwaldExclusion + PME reciprocal space
    (oracle/pme.py, numpy), remove_CM_motion = 1."""
    from oracle import oracle as o, pme
    sd = sixmrr_description(g)
    box, m = sd["box"], sd["mass"]
    alpha = pme.pme_alpha(1.0)
    inters = [o.Inter(o.LJ, o.CUT_DISTANCE, 1.0, weight_special=float(g["lj14scale"]), use_neighbors=True),
              o.Inter(o.EWALD_REAL, o.CUT_DISTANCE, 1.0, weight_special=float(g["coulomb14scale"]), ewald_alpha=alpha,
                      use_neighbors=True)]
    orc = make_oracle(sd, inters)
    excl = np.concatenate([g["excluded"], g["special"]])
    x = x - np.floor(x / box) * box
    v = orc.remove_cm(v)

    def forces(xx, nl):
        f, _, _ = orc.forces_nl(xx, nl, energy=False)
        fr, _, _ = pme.pme_reciprocal(xx, g["charge"], box, r_cut=1.0, error_tol=0.0005, order=5)
        fx, _ = pme.ewald_exclusion(xx, g["charge"], box, excl)
        return f + fr + fx + bonded_forces_oracle(g, xx)[0]
    nl = orc.neighbor_list(x, r_list)
    f = forces(x, nl)
    for step in range(1, n_steps + 1):
        v = v + f / m[:, None] * (dt / 2)
        x = x + v * dt
        x = x - np.floor(x / box) * box
        f = forces(x, nl)
        v = v + f / m[:, None] * (dt / 2)
        v = orc.remove_cm(v)
        if step % nl_every == 0:
            nl = orc.neighbor_list(x, r_list)
    return x, v


def sixmrr_pme_system(g, dtype, r_list=1.2, exact=True, velocities=None):
    """System(6mrr; nonbonded_method=:pme, approximate_pme=!exact) of test/protein.jl:76-85 / setup.jl:1894-1927: LJ +
    CoulombEwald + bonded lists + PME + EwaldExclusion(excluded or special) + LJDispersionCorrection."""
    import mollyb200 as mb
    sd = sixmrr_description(g)
    atoms = mb.atoms_from_arrays(sd["mass"], sd["charge"], sd["sigma"], sd["eps"], dtype)
    inters = (mb.LennardJones(cutoff=mb.DistanceCutoff(1.0), use_neighbors=True, weight_special=float(g["lj14scale"])),
              mb.CoulombEwald(dist_cutoff=1.0, error_tol=0.0005, use_neighbors=True, weight_special=float(g["coulomb14scale"]),
                              approximate_erfc=not exact))
    nf = mb.GPUNeighborFinder(dist_cutoff=r_list, excluded_pairs=g["excluded"] + 1, special_pairs=g["special"] + 1)
    pme = mb.PME(dist_cutoff=1.0, error_tol=0.0005, excluded_pairs=np.concatenate([g["excluded"], g["special"]]) + 1)
    v = sd["velocities"] if velocities is None else velocities
    return mb.System(atoms=atoms, coords=sd["coords"].astype(dtype), boundary=mb.CubicBoundary(*sd["box"]),
                     velocities=np.asarray(v).astype(dtype), pairwise_inters=inters, neighbor_finder=nf, dtype=dtype,
                     specific_inter_lists=sixmrr_specific_lists(g), general_inters=(pme, mb.LJDispersionCorrection(1.0)))
