"""The specific interaction kinds 3-9 on the device (HarmonicPositionRestraint, MorseBond, FENEBond, CosineAngle,
UreyBradley, HarmonicTorsion, RBTorsion): each kind alone on the reference's literal geometry, a molecular system holding
every kind at once on the all-pairs, cell-list and triclinic paths, f64 trajectories of VelocityVerlet, NoseHoover and
MTSIntegrator against numpy loops over the oracle's forces, energy conservation, steepest descent with restraints, the
reference's "Position restraints" protocol and the C-ABI refusals. The CPU counterpart is
tests/test_specific_kinds_host.py."""
import numpy as np
import pytest

import bonded_kinds_oracle as bk
import mbhelpers as H
import mollyb200 as mb
import mts_oracle as mo
import nosehoover_oracle as nho
import sd_oracle as sdo
from oracle import oracle as o
from test_gpu_parity import _pos_err
from test_specific_kinds_host import (DRIFT_BAR, DRIFT_DT, DRIFT_SAMPLES, DRIFT_STEPS, LITERALS, RB_ENERGY, RB_NORMS, RB_PARAMS,
                                      RB_X, drift_system)

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64


def _coords(s):
    c = s.coords
    return c.detach().cpu().numpy() if hasattr(c, "data_ptr") else np.array(c)


def _lone_system(kind, x, side, par, dtype):
    """The atoms of one term and nothing else: zero-epsilon, uncharged atoms, so only the term acts."""
    x = np.asarray(x, np.float64)
    n = len(x)
    idx = [np.arange(1, n + 1)] if kind == bk.POSITION_RESTRAINT else [[a + 1] for a in range(n)]
    par = np.asarray(par, np.float64)
    make = {bk.POSITION_RESTRAINT: lambda: mb.InteractionList1Atoms(idx[0], [par[0]], [par[1:4]]),
            bk.MORSE_BOND: lambda: mb.MorseBonds(*idx, *[[p] for p in par]),
            bk.FENE_BOND: lambda: mb.FENEBonds(*idx, *[[p] for p in par]),
            bk.COSINE_ANGLE: lambda: mb.CosineAngles(*idx, *[[p] for p in par]),
            bk.UREY_BRADLEY: lambda: mb.UreyBradleys(*idx, *[[p] for p in par]),
            bk.HARMONIC_TORSION: lambda: mb.HarmonicTorsions(*idx, *[[p] for p in par]),
            bk.RB_TORSION: lambda: mb.RBTorsions(*idx, *[[p] for p in par])}
    atoms = mb.atoms_from_arrays(np.full(n, 12.0), np.zeros(n), np.full(n, 0.3), np.zeros(n), dtype)
    return mb.System(atoms=atoms, coords=x.astype(dtype), boundary=mb.CubicBoundary(side, side, side), dtype=dtype,
                     pairwise_inters=(mb.LennardJones(),), specific_inter_lists=(make[kind](),))


def _literal_case(name):
    kind, x, side, par, f_exp, e_exp, fatol, eatol = LITERALS[name]
    if kind == bk.HARMONIC_TORSION:  # moved next to the origin (the term is translation invariant): f32 keeps the digits
        x = np.asarray(x) - np.asarray(x)[0] + 1.0
    return kind, x, side, par, f_exp, e_exp, fatol, eatol


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", sorted(LITERALS) + ["rb_torsion"])
def test_each_kind_alone_on_the_literal_geometry(name, dtype):
    if name == "rb_torsion":
        kind, x, side, par, f_exp, e_exp, fatol, eatol = bk.RB_TORSION, RB_X, 5.0, RB_PARAMS, None, RB_ENERGY, 1e-9, 1e-9
    else:
        kind, x, side, par, f_exp, e_exp, fatol, eatol = _literal_case(name)
    s = _lone_system(kind, x, side, par, dtype)
    try:
        f, e = mb.forces_energy(s)
    finally:
        s.close()
    f = f.astype(F64)
    x_in = np.asarray(x, dtype).astype(F64)
    idx = np.arange(bk.ATOMS[kind])[None, :]
    f_ref, e_ref = bk.FORCES[kind](x_in, np.full(3, side), idx, np.asarray(par, F64)[None, :])
    print(f"[{name} {np.dtype(dtype).name}] f={f.tolist()} e={e!r} (oracle e={e_ref!r})")
    if dtype == F64:
        if kind == bk.RB_TORSION:
            np.testing.assert_allclose(np.linalg.norm(f, axis=1), RB_NORMS, rtol=0, atol=fatol)
        elif f_exp is not None and fatol is not None:
            np.testing.assert_allclose(f, np.asarray(f_exp, F64), rtol=0, atol=fatol)
        elif f_exp is not None:
            for a, b in zip(f, np.asarray(f_exp, F64)):
                assert np.linalg.norm(a - b) <= np.sqrt(np.finfo(float).eps) * np.linalg.norm(b)
        assert abs(e - e_exp) <= (eatol if eatol is not None else np.sqrt(np.finfo(float).eps) * abs(e_exp))
        assert np.abs(f - f_ref).max() <= 1e-9 * max(np.abs(f_ref).max(), 1.0)
    else:  # energies on the scale |F| x 0.1 nm, the size of the geometry: a small sum of stiff terms keeps f32 digits of those
        assert np.abs(f - f_ref).max() <= H.tol(F32, np.abs(f_ref).max())
        assert abs(e - e_ref) <= H.etol(F32, max(abs(e_ref), 0.1 * np.abs(f_ref).max()))
    if name in ("restraint_at_x0", "fene_2", "cosine_collinear", "cosine_right"):
        assert np.all(f == 0)  # exactly zero, not NaN


# ---- a molecular system holding every kind at once ----------------------------------------------------------------------
def _all_kinds_lists(sd, n_mol, rng):
    """Per 4-site molecule A-B-C-D of H.molecular_system (1-based): every kind, PeriodicTorsion and RBTorsion in two lists."""
    a = np.arange(0, 4 * n_mol, 4) + 1
    b, c, d = a + 1, a + 2, a + 3
    one = np.ones(n_mol)
    x = sd["coords"].astype(F64)
    th = bk._torsion(x, sd["box"], np.stack([a, b, c, d], 1) - 1)[-1]
    half = n_mol // 2
    return (mb.InteractionList2Atoms(np.r_[a, b, c], np.r_[b, c, d], np.full(3 * n_mol, 2e5), np.full(3 * n_mol, 0.11)),
            mb.InteractionList3Atoms(np.r_[a, b], np.r_[b, c], np.r_[c, d], np.full(2 * n_mol, 400.0), np.full(2 * n_mol, 1.9)),
            mb.InteractionList4Atoms(a, b, c, d, 3 * one, 0.3 * one, 5 * one),
            mb.InteractionList1Atoms(a, np.full(n_mol, 800.0), x[a - 1] + rng.normal(0, 0.02, (n_mol, 3))),
            mb.MorseBonds(a, b, 300 * one, 15 * one, 0.11 * one),
            mb.FENEBonds(a, c, 30 * one, 0.3 * one, 0.15 * one, one),
            mb.CosineAngles(b, c, d, 20 * one, 1.2 * one),
            mb.UreyBradleys(a, b, c, 300 * one, 1.9 * one, 5000 * one, 0.18 * one),
            mb.HarmonicTorsions(a, b, c, d, 40 * one, th + 0.1),
            mb.RBTorsions(d[:half], c[:half], b[:half], a[:half], 2 * one[:half], -1 * one[:half], 1.5 * one[:half], 0.5 * one[:half]),
            mb.InteractionList4Atoms(a, b, c, d, 2 * one, 0.0 * one, 1.5 * one),
            mb.RBTorsions(a[half:], b[half:], c[half:], d[half:], 3 * one[half:], 1 * one[half:], -2 * one[half:], 0 * one[half:]))


PAIR_MB = lambda: (mb.LennardJones(cutoff=mb.DistanceCutoff(1.0), use_neighbors=True, weight_special=0.5),
                   mb.CoulombReactionField(dist_cutoff=1.0, use_neighbors=True, weight_special=0.8333))
PAIR_O = [o.Inter(o.LJ, o.CUT_DISTANCE, 1.0, weight_special=0.5, use_neighbors=True),
          o.Inter(o.CRF, o.CUT_DISTANCE, 1.0, weight_special=0.8333, use_neighbors=True)]


def _molecules(n_mol, box, dtype, seed=3, triclinic=False, r_list=1.2, pick=slice(None)):
    sd = H.molecular_system(n_mol, box, seed=seed, stable=True)
    sd["box"] = np.asarray(sd["box"], F64)
    lists = _all_kinds_lists(sd, n_mol, np.random.default_rng(seed))[pick]
    L = sd["box"]
    bnd = mb.TriclinicBoundary([L[0], 0, 0], [L[0], L[1], 0], [-L[0], 0, L[2]]) if triclinic else mb.CubicBoundary(*L)
    atoms = mb.atoms_from_arrays(sd["mass"], sd["charge"], sd["sigma"], sd["eps"], dtype)
    nf = mb.GPUNeighborFinder(dist_cutoff=r_list, excluded_pairs=sd["excluded"] + 1, special_pairs=sd["special"] + 1)
    s = mb.System(atoms=atoms, coords=sd["coords"].astype(dtype), velocities=sd["velocities"].astype(dtype), boundary=bnd,
                  pairwise_inters=PAIR_MB(), neighbor_finder=nf, dtype=dtype, specific_inter_lists=lists)
    return sd, s, lists


def _oracle_fe(sd, lists, dtype=F64):
    orc = H.make_oracle(dict(sd, coords=sd["coords"].astype(dtype)), PAIR_O)
    ol = bk.oracle_lists(lists)

    def fe(x):
        fp, ep, _ = orc.forces_allpairs(x)
        fb, eb = bk.specific_forces(x, sd["box"], ol)
        return fp + fb, ep + eb
    return fe, orc


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("where", ["allpairs", "celllist", "triclinic"])
def test_every_kind_at_once(where, dtype):
    if where == "celllist":
        n_mol, box, path = 729, [5.1, 5.4, 5.8], 1
    else:
        n_mol, box, path = 100, [2.4, 2.4, 2.4], 0
    sd, s, lists = _molecules(n_mol, box, dtype, triclinic=where == "triclinic")
    x = sd["coords"].astype(dtype).astype(F64)
    if where == "triclinic":  # every atom moved by lattice vectors: bonded partners sit in different images
        L = sd["box"][0]
        bv = np.array([[L, 0, 0], [L, L, 0], [-L, 0, L]])
        s.coords[:] = (x + np.random.default_rng(4).integers(-1, 2, (len(x), 3)) @ bv).astype(dtype)
    fe, orc = _oracle_fe(sd, lists, dtype)
    try:
        f, e = mb.forces_energy(s)
        st = s.stats()
    finally:
        s.close()
    f_ref, e_ref = fe(x)
    fmax = np.abs(f_ref).max()
    err = np.abs(f.astype(F64) - f_ref).max()
    print(f"[every kind {where} {np.dtype(dtype).name}] path={st['path']} max|dF|={err:.3e} (max|F| {fmax:.3e}) "
          f"dE={e - e_ref:.3e} (E {e_ref:.6e})")
    assert st["path"] == path
    scale = 10 if where == "triclinic" else 1  # the wrapped f32 inputs of the moved atoms carry rounding of their own
    if dtype == F32 and err > scale * H.tol(dtype, fmax):
        # pairs sitting on the cutoff within f32 rounding may land on either side: one F(rc) jump each (as H.check)
        nb_pairs = H.boundary_atoms(orc, x, PAIR_O)
        per_atom = np.abs(f.astype(F64) - f_ref).max(axis=1)
        assert (per_atom <= scale * H.tol(dtype, fmax) + nb_pairs * H.cutoff_force_bound(sd, PAIR_O)).all()
    else:
        assert err <= scale * H.tol(dtype, fmax)
    assert abs(e - e_ref) <= scale * H.etol(dtype, e_ref)


# ---- f64 trajectories against numpy loops over the oracle's forces -----------------------------------------------------
def _wrap(box):
    return lambda x: x - np.floor(x / box) * box


def _vv_oracle(fe, x, v, mass, dt, n, box):
    m = mass[:, None]
    rcm = lambda v: v - (m * v).sum(0) / m.sum()
    x, v = _wrap(box)(x), rcm(v)
    f = fe(x)[0]
    for _ in range(n):
        v = v + f / m * (dt / 2)
        x = _wrap(box)(x + v * dt)
        f = fe(x)[0]
        v = rcm(v + f / m * (dt / 2))
    return x, v


def test_vv_trajectory_f64():
    sd, s, lists = _molecules(100, [2.4, 2.4, 2.4], F64)
    fe, _ = _oracle_fe(sd, lists)
    dt, n = 0.0005, 40
    x_ref, v_ref = _vv_oracle(fe, sd["coords"], sd["velocities"], sd["mass"], dt, n, sd["box"])
    mb.simulate(s, mb.VelocityVerlet(dt=dt), n)
    ex, ev = _pos_err(s.coords, x_ref, sd["box"]), np.abs(s.velocities - v_ref).max()
    print(f"[VV every kind f64] dx={ex:.3e} dv={ev:.3e}")
    assert ex < 1e-9 and ev < 1e-8
    s.close()


def test_nose_hoover_trajectory_f64():
    sd, s, lists = _molecules(100, [2.4, 2.4, 2.4], F64)
    fe, _ = _oracle_fe(sd, lists)
    dt, n, T = 0.0005, 40, 150.0
    sim = mb.NoseHoover(dt=dt, temperature=T, damping=0.05)
    x_ref, v_ref, _ = nho.simulate_nose_hoover(lambda x: fe(x)[0], sd["coords"], sd["velocities"], sd["mass"], dt, n,
                                               mb.BOLTZMANN_K * T, 0.05, _wrap(sd["box"]))
    mb.simulate(s, sim, n)
    ex, ev = _pos_err(s.coords, x_ref, sd["box"]), np.abs(s.velocities - v_ref).max()
    print(f"[NoseHoover every kind f64] dx={ex:.3e} dv={ev:.3e}")
    assert ex < 1e-9 and ev < 1e-8
    s.close()


def test_mts_new_kinds_inner_level_f64():
    """Kinds 3-9 at fraction 2 (level 1), kinds 0-2 and the pairs at fraction 1 (level 0): the level ranges of every kind."""
    sd, s, lists = _molecules(100, [2.4, 2.4, 2.4], F64)
    _, orc = _oracle_fe(sd, lists)
    si = tuple(2 if li.kind >= 3 else 1 for li in lists)
    sim = mb.MTSIntegrator(0.001, pi_fractions=(1, 1), si_fractions=si)
    box = sd["box"]

    def level(lv):
        mine = bk.oracle_lists([li for li, f in zip(lists, si) if sim.ordered_fractions.index(f) == lv])
        return lambda x: (orc.forces_allpairs(x, energy=False)[0] if lv == 0 else 0) + bk.specific_forces(x, box, mine)[0]
    n = 20
    x_ref, v_ref = mo.simulate_mts([level(0), level(1)], sd["coords"], sd["velocities"], sd["mass"], sim.dt, n,
                                   sim.ordered_fractions, _wrap(box))
    mb.simulate(s, sim, n)
    ex, ev = _pos_err(s.coords, x_ref, box), np.abs(s.velocities - v_ref).max()
    print(f"[MTS {sim.ordered_fractions} every kind f64] dx={ex:.3e} dv={ev:.3e}")
    assert ex < 1e-9 and ev < 1e-8
    s.close()


# ---- energy conservation with restraints, RB torsions and Morse bonds ---------------------------------------------------
# VelocityVerlet, f64, 0.5 fs, 2000 steps: the largest |E(t) - E(0)| over 10 samples stays under DRIFT_BAR kJ/mol. With the
# reference's RBTorsion force sign the same run drifts far beyond it (test_specific_kinds_host checks that on the numpy
# oracle).


def test_energy_conservation_restraints_rb_morse():
    sd, lists = drift_system()
    atoms = mb.atoms_from_arrays(sd["mass"], sd["charge"], sd["sigma"], sd["eps"], F64)
    s = mb.System(atoms=atoms, coords=sd["coords"], velocities=sd["velocities"], boundary=mb.CubicBoundary(*sd["box"]), dtype=F64,
                  pairwise_inters=(mb.LennardJones(),), specific_inter_lists=lists)
    etot = lambda: mb.potential_energy(s) + mb.kinetic_energy(s)
    e0 = etot()
    es = []
    for _ in range(DRIFT_SAMPLES):
        mb.simulate(s, mb.VelocityVerlet(dt=DRIFT_DT, remove_CM_motion=0), DRIFT_STEPS // DRIFT_SAMPLES)
        es.append(etot())
    drift = np.abs(np.array(es) - e0).max()
    print(f"[energy drift] E0={e0:.6f} max|E-E0|={drift:.3e} (bar {DRIFT_BAR})")
    assert drift < DRIFT_BAR
    s.close()


# ---- steepest descent with restraints ------------------------------------------------------------------------------------
def test_steepest_descent_with_restraints_f64():
    sd, base, _ = _molecules(100, [2.4, 2.4, 2.4], F64, pick=slice(0, 3))
    x0 = sd["coords"] + np.random.default_rng(1).normal(0, 0.05, sd["coords"].shape)
    s = mb.add_position_restraints(base, 500.0, atom_selector=np.arange(1, sd["n"] + 1, 4), restrain_coords=x0)
    fe, _ = _oracle_fe(sd, s.specific_inter_lists)
    kw = dict(step_size=0.01, max_steps=60, tol=10.0)
    x_ref, _ = sdo.steepest_descent(sd["coords"], sd["box"], fe, **kw)
    mb.simulate(s, mb.SteepestDescentMinimizer(**kw))
    ex = _pos_err(_coords(s), x_ref, sd["box"])
    print(f"[SD restraints f64] dx={ex:.3e} steps={s.minimize_result}")
    assert ex < 1e-9
    s.close()


# ---- the reference's "Position restraints" testset (test/simulation.jl:737-768) ------------------------------------------
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_reference_position_restraints_protocol(dtype):
    n, n_res = 10, 5
    sd = H.readme_system(n, 2.0, seed=11, min_dist=0.3)
    atoms = mb.atoms_from_arrays(np.full(n, 10.0), np.zeros(n), np.full(n, 0.2), np.full(n, 0.2), dtype)
    start = sd["coords"].astype(F64)
    s = mb.System(atoms=atoms, coords=start.astype(dtype), boundary=mb.CubicBoundary(2.0), pairwise_inters=(mb.LennardJones(),),
                  dtype=dtype)
    sel = np.arange(n) < n_res
    sr = mb.add_position_restraints(s, 100_000.0, atom_selector=sel)
    mb.simulate(sr, mb.Langevin(dt=0.001, temperature=300.0, friction=1.0), 2000, rng=np.random.default_rng(5))
    d = _coords(sr).astype(F64) - start
    d -= 2.0 * np.round(d / 2.0)
    dists = np.linalg.norm(d, axis=1)
    print(f"[position restraints {np.dtype(dtype).name}] restrained max {dists[:n_res].max():.4f} nm, "
          f"free median {np.median(dists[n_res:]):.4f} nm")
    assert dists[:n_res].max() < 0.1
    assert np.median(dists[n_res:]) > 0.2
    sr.close()
    s.close()


# ---- refusals ------------------------------------------------------------------------------------------------------------
def test_refusals_leave_the_context_usable():
    kind, x, side, par, *_ = LITERALS["morse_1"]
    s = _lone_system(kind, x, side, par, F64)
    f0, e0 = mb.forces_energy(s)
    ctx, L = s.engine(), s._L
    one = np.array([1], np.int32)
    p4 = np.zeros(4)
    for k in (-1, 10):
        assert L.mb_set_specific(ctx, k, 1, one.ctypes.data, p4.ctypes.data) == mb.capi.MB_ERR_INVALID
    for bad in (0, 3):  # n = 2 atoms: 0 and n + 1 are outside 1 .. n
        i = np.array([bad], np.int32)
        assert L.mb_set_specific(ctx, mb.capi.MB_SPECIFIC_POSITION_RESTRAINT, 1, i.ctypes.data, p4.ctypes.data) == mb.capi.MB_ERR_INVALID
    lv = np.zeros(2, np.int32)
    assert L.mb_set_specific_levels(ctx, mb.capi.MB_SPECIFIC_MORSE_BOND, 2, lv.ctypes.data) == mb.capi.MB_ERR_INVALID
    assert L.mb_set_specific_levels(ctx, mb.capi.MB_SPECIFIC_RB_TORSION, 1, lv.ctypes.data) == mb.capi.MB_ERR_INVALID
    f1, e1 = mb.forces_energy(s)
    assert np.array_equal(f0, f1) and e0 == e1
    s.close()
