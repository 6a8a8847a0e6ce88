"""GPU tests of DPDInteraction and DPDVelocityVerlet (src/interactions/dpd.jl:57-142, src/simulators.jl:670-842): one
evaluation against the f64 restatement in tests/dpd_oracle.py on the all-pairs and cell-list paths, in a sheared box,
with exclusions and special pairs; f64 trajectories against the oracle's loop (bead-spring polymer, CM-removal schedules,
init_step, chunked calls); the engine's identities (graph = stream, loggers do not change the trajectory, DPDVelocityVerlet
without DPD is VelocityVerlet, momentum conservation); the reference's "DPD simulation" protocol and a production-size
temperature check; and the refusals."""
import ctypes as C
import math
import os
import socket

import numpy as np
import pytest

import dpd_oracle as do
import mbhelpers as H
import mollyb200 as mb

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
KEY = 0x0123456789ABCDEF
GW = dict(a=25.0, gamma=4.5, sigma=3.0, r_c=1.0)  # Groot-Warren: sigma^2 = 2 gamma kT with kT = 1


def _fluid(box, rho=3.0, seed=1, mass2=False):
    """Beads at uniform random positions (overlaps allowed: the potential is soft), Maxwell-Boltzmann velocities at kT = 1."""
    b = np.asarray(box, np.float64)
    vol = np.prod(b) if b.ndim == 1 else b[0, 0] * b[1, 1] * b[2, 2]
    n = int(round(rho * vol))
    r = np.random.default_rng(seed)
    frac = r.uniform(0, 1, (n, 3))
    x = frac * b if b.ndim == 1 else frac @ b
    m = np.where(r.uniform(size=n) < 0.3, 2.0, 1.0) if mass2 else np.ones(n)
    v = r.normal(0, 1, (n, 3)) / np.sqrt(m)[:, None]
    return x, v, m


def _inter(use_neighbors, dt=0.02, **kw):
    p = dict(GW, dt=dt, key=KEY)
    p.update(kw)
    return mb.DPDInteraction(a=p["a"], gamma=p["gamma"], sigma=p["sigma"], r_c=p["r_c"], dt=p["dt"],
                             use_neighbors=use_neighbors, key=p["key"]), p


def _system(x, v, m, box, inter, dtype, r_list=0.0, excluded=None, special=None, bonds=None, loggers=None, n_steps=0):
    b = np.asarray(box, np.float64)
    boundary = mb.CubicBoundary(*b) if b.ndim == 1 else mb.TriclinicBoundary(*b)
    atoms = mb.atoms_from_arrays(m, np.zeros(len(m)), np.zeros(len(m)), np.zeros(len(m)), dtype)
    nf = None
    if r_list > 0 or excluded is not None or special is not None:
        nf = mb.GPUNeighborFinder(dist_cutoff=r_list, excluded_pairs=excluded, special_pairs=special, n_steps=n_steps)
    sil = ()
    if bonds is not None:
        sil = (mb.InteractionList2Atoms(bonds[:, 0].astype(int) + 1, bonds[:, 1].astype(int) + 1, bonds[:, 2], bonds[:, 3]),)
    # (copies: a System with f64 host state updates its arrays in place, and the callers keep x and v for the oracle)
    return mb.System(atoms, np.array(x), boundary, velocities=np.array(v), pairwise_inters=(inter,), neighbor_finder=nf,
                     dtype=dtype, k=1.0, specific_inter_lists=sil, loggers=loggers)


def _polymer(n, chain=10, k=100.0, r0=0.7):
    """Harmonic-bond chains of `chain` consecutive beads: rows (i, j, k, r0), 0-based."""
    rows = [(i, i + 1, k, r0) for c in range(0, n - chain + 1, chain) for i in range(c, c + chain - 1)]
    return np.array(rows, np.float64)


def _chain_coords(x, box, chain=10, step=0.6, seed=3):
    """Random walks of `chain` beads with bond length `step` from the first bead of each chain."""
    r = np.random.default_rng(seed)
    x = x.copy()
    for c in range(0, len(x) - chain + 1, chain):
        for i in range(c + 1, c + chain):
            u = r.normal(size=3)
            x[i] = x[i - 1] + step * u / np.linalg.norm(u)
    return do.wrap(x, box)


def _pos_err(a, b, box):
    d = np.asarray(a, np.float64) - np.asarray(b, np.float64)
    bx = np.asarray(box, np.float64)
    return float(np.abs(d - bx * np.round(d / bx)).max())


def _near_pairs(x, box, count, lo=0.2, hi=0.9, seed=5):
    """`count` distinct 0-based pairs at distances in (lo, hi): exclusions / specials that matter."""
    i, j, dr = do.pairs_within(x, box, hi)
    r = np.sqrt((dr * dr).sum(-1))
    keep = np.nonzero(r > lo)[0]
    pick = np.random.default_rng(seed).choice(keep, count, replace=False)
    return np.stack([i[pick], j[pick]], 1)


SHEAR = np.array([[6.0, 0.0, 0.0], [1.5, 6.0, 0.0], [-1.0, 2.0, 6.0]])
FORCE_CASES = {
    # name: box, use_neighbors, r_list, exclusions, specials, expected path
    "allpairs": (np.full(3, 4.0), False, 0.0, 0, 0, 0),
    "brick-8": (np.full(3, 8.0), True, 1.5, 0, 0, 1),
    "brick-20": (np.full(3, 20.0), True, 1.5, 0, 0, 1),
    "triclinic": (SHEAR, False, 0.0, 0, 0, 0),
    "brick-exclusions": (np.full(3, 8.0), True, 1.5, 300, 0, 1),
    "brick-special": (np.full(3, 8.0), True, 1.5, 0, 300, 1),
    "allpairs-nl-exclusions": (np.full(3, 3.5), True, 1.5, 100, 0, 0),
}


@pytest.mark.parametrize("dtype", [F64, F32])
@pytest.mark.parametrize("case", list(FORCE_CASES))
def test_one_evaluation_matches_oracle(case, dtype):
    box, nl, r_list, n_ex, n_sp, path = FORCE_CASES[case]
    x, v, m = _fluid(box, seed=11)
    inter, p = _inter(nl)
    ex = _near_pairs(x, box, n_ex) if n_ex else None
    sp = _near_pairs(x, box, n_sp, seed=6) if n_sp else None
    s = _system(x, v, m, box, inter, dtype, r_list=r_list, excluded=None if ex is None else ex + 1,
                special=None if sp is None else sp + 1)
    step = 17
    f, pe = mb.forces_energy(s, step_n=step)
    assert s.stats()["path"] == path
    x64, v64 = s.coords.astype(F64), s.velocities.astype(F64)
    excluded = set() if ex is None or not nl else {(int(a), int(b)) for a, b in np.sort(ex, 1)}
    f_ref, e_ref = do.forces(x64, v64, box, p, step, excluded)
    fmax = np.abs(f_ref).max()
    rel = 1e-12 if dtype == F64 else 1e-5
    assert np.abs(f - f_ref).max() <= rel * fmax, (np.abs(f - f_ref).max(), fmax)
    assert abs(pe - e_ref) <= rel * abs(e_ref) * 10, (pe, e_ref)
    assert np.abs(mb.forces(s, step_n=step) - f_ref).max() <= rel * fmax  # the force-only kernel variant
    tot = np.abs(f.astype(F64).sum(0)).max()
    assert tot <= (1e-10 if dtype == F64 else 1e-5) * np.abs(f).sum(), tot
    if case == "allpairs":  # a different step draws different numbers; the energy does not depend on them
        f2, pe2 = mb.forces_energy(s, step_n=step + 1)
        assert not np.array_equal(f2, f) and pe2 == pe


def test_coincident_beads_give_finite_forces():
    box = np.full(3, 4.0)
    x, v, m = _fluid(box, seed=2)
    x[1] = x[0]
    inter, p = _inter(False)
    s = _system(x, v, m, box, inter, F64)
    f = mb.forces(s, step_n=3)
    assert np.all(np.isfinite(f))
    f_ref, _ = do.forces(x, v, box, p, 3)
    assert np.abs(f - f_ref).max() <= 1e-12 * np.abs(f_ref).max()


# ---- trajectories (f64) ---------------------------------------------------------------------------------------------------
TRAJ_PATHS = {"allpairs": (np.full(3, 4.0), False, 0.0), "brick": (np.full(3, 5.0), True, 1.5)}
TRAJ_CASES = {  # name: remove_CM_motion, init_step, chunks, bonds
    "rcm1": (1, 0, None, False),
    "rcm0-init9": (0, 9, None, False),
    "rcm5-init3": (5, 3, None, False),
    "polymer": (1, 0, None, True),
    "chunked": (1, 0, [40, 60], False),
}


@pytest.mark.parametrize("case", list(TRAJ_CASES))
@pytest.mark.parametrize("path", list(TRAJ_PATHS))
def test_trajectory_matches_oracle(path, case):
    box, nl, r_list = TRAJ_PATHS[path]
    rcm, init_step, chunks, poly = TRAJ_CASES[case]
    x, v, m = _fluid(box, seed=21, mass2=True)
    bonds = None
    if poly:
        x = _chain_coords(x, box)
        bonds = _polymer(len(x))
    inter, p = _inter(nl)
    dt, lam = 0.02, 0.65
    s = _system(x, v, m, box, inter, F64, r_list=r_list, bonds=bonds)
    x_ref, v_ref, step = x, v, init_step
    for k in (chunks or [100]):
        x_ref, v_ref = do.simulate_dpd_vv(x_ref, v_ref, m, box, p, dt, lam, k, remove_cm_every=rcm, init_step=step, bonds=bonds)
        mb.simulate(s, mb.DPDVelocityVerlet(dt=dt, lam=lam, remove_CM_motion=rcm), k, init_step=step)
        step += k
    assert s.stats()["path"] == (1 if nl else 0)
    assert _pos_err(s.coords, x_ref, box) < 1e-9, _pos_err(s.coords, x_ref, box)
    assert np.abs(s.velocities - v_ref).max() < 1e-8


def test_chunked_calls_differ_from_one_call():
    """Each call's F0 uses v(t), not the predicted velocity: two calls of 50 steps are not one call of 100 (as in the
    reference), and the oracle agrees on both."""
    box = np.full(3, 4.0)
    x, v, m = _fluid(box, seed=4)
    inter, p = _inter(False)
    one = _system(x, v, m, box, inter, F64)
    two = _system(x, v, m, box, inter, F64)
    mb.simulate(one, mb.DPDVelocityVerlet(dt=0.02), 100)
    mb.simulate(two, mb.DPDVelocityVerlet(dt=0.02), 50)
    mb.simulate(two, mb.DPDVelocityVerlet(dt=0.02), 50, init_step=50)
    assert _pos_err(one.coords, two.coords, box) > 1e-9


# ---- identities -------------------------------------------------------------------------------------------------------------
def _brick_fluid(dtype, seed=8, loggers=None, box=6.0):
    b = np.full(3, box)
    x, v, m = _fluid(b, seed=seed)
    inter, p = _inter(True)
    return _system(x, v, m, b, inter, dtype, r_list=1.5, loggers=loggers), (x, v, m, b, p)


@pytest.mark.parametrize("dtype", [F32, F64])
def test_graph_and_stream_runs_are_bitwise_equal(dtype, monkeypatch):
    s, _ = _brick_fluid(dtype)
    mb.simulate(s, mb.DPDVelocityVerlet(dt=0.04), 200)
    assert s.stats()["graph_mode"] == 1
    monkeypatch.setenv("MOLLYB200_NO_GRAPH", "1")
    t, _ = _brick_fluid(dtype)
    mb.simulate(t, mb.DPDVelocityVerlet(dt=0.04), 200)
    assert t.stats()["graph_mode"] == 0
    assert np.array_equal(s.coords, t.coords) and np.array_equal(s.velocities, t.velocities)


def test_loggers_do_not_change_the_trajectory_and_match_oracle():
    every = 5
    lg = {"pe": mb.PotentialEnergyLogger(every), "ke": mb.KineticEnergyLogger(every), "te": mb.TotalEnergyLogger(every),
          "t": mb.TemperatureLogger(every), "x": mb.CoordinatesLogger(every), "v": mb.VelocitiesLogger(every)}
    s, (x, v, m, b, p) = _brick_fluid(F64, loggers=lg)
    t, _ = _brick_fluid(F64)
    n = 60
    mb.simulate(s, mb.DPDVelocityVerlet(dt=0.02), n)
    mb.simulate(t, mb.DPDVelocityVerlet(dt=0.02), n)
    assert np.array_equal(s.coords, t.coords) and np.array_equal(s.velocities, t.velocities)
    rec = {}
    do.simulate_dpd_vv(x, v, m, b, p, 0.02, 0.65, n, record=lambda st, xx, vv, pe: rec.__setitem__(st, (vv, pe)))
    steps = [k for k in range(0, n + 1) if k % every == 0]
    df = 3 * len(m) - 3
    pe_ref = np.array([rec[k][1] for k in steps])
    ke_ref = np.array([0.5 * (m[:, None] * rec[k][0] ** 2).sum() for k in steps])
    assert np.allclose(np.array(mb.values(lg["pe"]), F64), pe_ref, rtol=1e-10)
    assert np.allclose(np.array(mb.values(lg["ke"]), F64), ke_ref, rtol=1e-10)
    assert np.allclose(np.array(mb.values(lg["te"]), F64), pe_ref + ke_ref, rtol=1e-10)
    assert np.allclose(np.array(mb.values(lg["t"]), F64), 2 * ke_ref / df, rtol=1e-10)
    assert len(mb.values(lg["x"])) == len(steps) and len(mb.values(lg["v"])) == len(steps)


@pytest.mark.parametrize("dtype", [F32, F64])
def test_without_dpd_it_is_velocity_verlet(dtype):
    """DPDVelocityVerlet on a system without a DPDInteraction runs mb_simulate_vv's step, bit for bit."""
    sd = H.lj_fluid(6, seed=3, dtype=dtype)
    inter = (mb.LennardJones(cutoff=mb.DistanceCutoff(1.0), use_neighbors=True),)
    a = H.make_system(sd, inter, dtype, r_list=1.2)
    b = H.make_system(sd, inter, dtype, r_list=1.2)
    mb.simulate(a, mb.VelocityVerlet(dt=0.002), 50)
    mb.simulate(b, mb.DPDVelocityVerlet(dt=0.002, lam=0.9), 50)
    assert np.array_equal(a.coords, b.coords) and np.array_equal(a.velocities, b.velocities)


def test_momentum_is_conserved_without_cm_removal():
    s, (x, v, m, b, p) = _brick_fluid(F64, seed=12)
    p0 = (m[:, None] * s.velocities).sum(0)
    scale = (m[:, None] * np.abs(s.velocities)).sum()
    mb.simulate(s, mb.DPDVelocityVerlet(dt=0.04, remove_CM_motion=0), 1000)
    p1 = (m[:, None] * s.velocities).sum(0)
    assert np.abs(p1 - p0).max() <= 1e-9 * scale, (p0, p1)


# ---- physics ------------------------------------------------------------------------------------------------------------------
def test_reference_dpd_simulation_protocol():
    """test/simulation.jl:1257-1304: 100 beads in a 5^3 box, 10 000 steps of dt = 0.01, kT = 1, use_neighbors with
    r_list = 1.5 r_c rebuilt every 10 steps; mean T of the second half in (0.5, 1.5), |P| < 1."""
    n, box, dt = 100, 5.0, 0.01
    r = np.random.default_rng(12345)
    x, v, m = r.uniform(0, box, (n, 3)), r.normal(size=(n, 3)), np.ones(n)
    inter = mb.DPDInteraction(a=25.0, gamma=4.5, sigma=math.sqrt(2 * 4.5 * 1.0), r_c=1.0, dt=dt, use_neighbors=True)
    lg = {"temp": mb.TemperatureLogger(100)}
    s = _system(x, v, m, np.full(3, box), inter, F64, r_list=1.5, loggers=lg, n_steps=10)
    mb.simulate(s, mb.DPDVelocityVerlet(dt=dt, lam=0.65), 10_000)
    temps = np.array(mb.values(lg["temp"]), F64)
    mean_t = temps[len(temps) // 2:].mean()
    assert 0.5 < mean_t < 1.5, mean_t
    assert np.all(np.abs((m[:, None] * s.velocities).sum(0)) < 1.0)
    assert s.stats()["path"] == 1


def test_production_size_temperature():
    """N = 24 000 at rho = 3 (box 20), dt = 0.02, 5000 steps, f32 on the cell-list path: the mean T of the second half is
    within 3 % of kT = 1."""
    b = np.full(3, 20.0)
    x, v, m = _fluid(b, seed=30)
    inter, _ = _inter(True, dt=0.02)
    lg = {"temp": mb.TemperatureLogger(50)}
    s = _system(x, v, m, b, inter, F32, r_list=1.5, loggers=lg)
    mb.simulate(s, mb.DPDVelocityVerlet(dt=0.02), 5000)
    temps = np.array(mb.values(lg["temp"]), F64)
    mean_t = temps[len(temps) // 2:].mean()
    print(f"DPD production run: N = {len(m)}, mean T (second half) = {mean_t:.4f}")
    assert abs(mean_t - 1.0) < 0.03, mean_t
    assert s.stats()["path"] == 1


# ---- refusals -----------------------------------------------------------------------------------------------------------------
def _raw_dpd(**kw):
    p = dict(GW, dt=0.02, key=KEY, use_neighbors=0)
    p.update(kw)
    return mb.capi.MBDpd(p["a"], p["gamma"], p["sigma"], p["r_c"], p["dt"], p["key"], p["use_neighbors"])


def _dpd_params(lam=0.65, n=5):
    q = mb.capi.MBDpdVVParams()
    q.dt, q.n_steps, q.init_step, q.remove_cm_every, q.lambda_ = 0.02, n, 0, 1, lam
    return q


def _refused(s, fn):
    x0, v0 = s.coords.copy(), s.velocities.copy()
    with pytest.raises(mb.MollyB200Error) as e:
        fn()
    assert e.value.code == mb.capi.MB_ERR_INVALID, str(e.value)
    assert np.array_equal(s.coords, x0) and np.array_equal(s.velocities, v0)
    return str(e.value)


def test_refusals():
    box = np.full(3, 4.0)
    x, v, m = _fluid(box, seed=9)
    inter, _ = _inter(False)
    s = _system(x, v, m, box, inter, F64)
    ctx, L = s.engine(), s._L
    X, V = s.coords.ctypes.data, s.velocities.ctypes.data
    # bad interaction parameters
    for bad in (dict(r_c=0.0), dict(r_c=math.inf), dict(dt=0.0), dict(dt=math.nan), dict(gamma=-1.0), dict(sigma=math.nan),
                dict(a=math.inf)):
        _refused(s, lambda: mb.capi.check(L.mb_set_dpd(ctx, C.byref(_raw_dpd(**bad)))))
    # lambda not finite
    _refused(s, lambda: mb.capi.check(L.mb_simulate_dpd_vv(ctx, X, V, C.byref(_dpd_params(lam=math.inf)), None)))
    # other integrators and the minimiser
    for sim in (mb.VelocityVerlet(dt=0.02), mb.Langevin(dt=0.02, temperature=1.0, friction=1.0), mb.Verlet(dt=0.02)):
        assert "mb_simulate_dpd_vv" in _refused(s, lambda: mb.simulate(s, sim, 5))
    _refused(s, lambda: mb.simulate(s, mb.SteepestDescentMinimizer(), run_loggers=False))
    # a velocity coupling on the context
    vc = mb.capi.MBVCoupling(mb.capi.MB_VC_BERENDSEN, 1, 1.0, 1.0)
    mb.capi.check(L.mb_set_velocity_coupling(ctx, C.byref(vc)))
    _refused(s, lambda: mb.capi.check(L.mb_simulate_dpd_vv(ctx, X, V, C.byref(_dpd_params()), None)))
    mb.capi.check(L.mb_set_velocity_coupling(ctx, None))
    with pytest.raises(TypeError):
        mb.simulate(s, mb.DPDVelocityVerlet(dt=0.02, coupling=mb.AndersenThermostat(1.0, 1.0)), 5)
    # forces without velocities; the energy needs none
    fs = np.zeros((s.n, 3))
    for call in (lambda: L.mb_forces(ctx, X, fs.ctypes.data, None, 0),
                 lambda: L.mb_forces_energy(ctx, X, fs.ctypes.data, None, None, 0),
                 lambda: L.mb_forces_energy_all(ctx, X, fs.ctypes.data, None, 0)):
        assert "mb_forces_energy_vel" in _refused(s, lambda: mb.capi.check(call()))
    # a DPDInteraction has no virial
    pe, vir = np.zeros(1), np.zeros(9)
    assert "virial" in _refused(s, lambda: mb.capi.check(L.mb_forces_energy(ctx, X, None, pe.ctypes.data, vir.ctypes.data, 0)))
    assert mb.potential_energy(s) > 0
    mb.simulate(s, mb.DPDVelocityVerlet(dt=0.02), 5)  # the context still runs

    # combinations refused at the next call
    n = len(m)
    for extra in (dict(pairwise_inters=(inter, mb.LennardJones(cutoff=mb.DistanceCutoff(1.0)))),
                  dict(general_inters=(mb.LJDispersionCorrection(1.0),)),
                  dict(general_inters=(mb.PME(1.0),)),
                  dict(general_inters=(mb.ImplicitSolventOBC(np.full(n, 0.15), np.full(n, 0.12)),))):
        atoms = mb.atoms_from_arrays(m, np.zeros(len(m)), np.full(len(m), 0.3), np.full(len(m), 0.5), F64)
        t = mb.System(atoms, x, mb.CubicBoundary(4.0), velocities=v, dtype=F64, k=1.0,
                      **dict(dict(pairwise_inters=(inter,)), **extra))
        assert "cannot be combined" in _refused(t, lambda: mb.simulate(t, mb.DPDVelocityVerlet(dt=0.02), 5))
        assert "cannot be combined" in _refused(t, lambda: mb.forces(t))
    # the neighbour list radius below r_c on the cell-list path
    b5 = np.full(3, 5.0)
    x5, v5, m5 = _fluid(b5, seed=2)
    u = _system(x5, v5, m5, b5, _inter(True)[0], F64, r_list=0.8)
    _refused(u, lambda: mb.simulate(u, mb.DPDVelocityVerlet(dt=0.02), 5))


def test_f32_index_limit():
    """An f32 context of more than 2^24 atoms is refused: the position records carry the atom index as a float."""
    n = (1 << 24) + 1
    L = mb.capi.load()
    ctx = C.c_void_p()
    mb.capi.check(L.mb_ctx_create(0, 32, None, C.byref(ctx)))
    try:
        z = np.zeros(n, F32)
        one = np.ones(n, F32)
        mb.capi.check(L.mb_set_atoms_soa(ctx, n, one.ctypes.data, z.ctypes.data, z.ctypes.data, z.ctypes.data))
        mb.capi.check(L.mb_set_box(ctx, (C.c_double * 3)(200.0, 200.0, 200.0)))
        mb.capi.check(L.mb_set_dpd(ctx, C.byref(_raw_dpd())))
        x = np.zeros((n, 3), F32)
        pe = np.zeros(1, F32)
        assert L.mb_energy(ctx, x.ctypes.data, pe.ctypes.data, 0) == mb.capi.MB_ERR_INVALID
        assert "2^24" in L.mb_last_error().decode()
    finally:
        L.mb_ctx_destroy(ctx)


@pytest.mark.parametrize("case", ["allpairs", "brick-8"])
def test_conservative_only_skips_gather_and_draw(case):
    """gamma = sigma = 0: the pair kernels neither gather v_j nor draw; the forces are the conservative ones (the oracle with
    the same parameters) whatever the velocities are."""
    box, nl, r_list = FORCE_CASES[case][:3]
    x, v, m = _fluid(box, seed=13)
    inter, p = _inter(nl, gamma=0.0, sigma=0.0)
    s = _system(x, v, m, box, inter, F64, r_list=r_list)
    f, pe = mb.forces_energy(s, step_n=5)
    f_ref, e_ref = do.forces(x, v, box, p, 5)
    assert np.abs(f - f_ref).max() <= 1e-12 * np.abs(f_ref).max()
    assert abs(pe - e_ref) <= 1e-11 * abs(e_ref)
    s.velocities[...] = np.nan  # never read
    assert np.array_equal(mb.forces(s, step_n=6), mb.forces(s, step_n=5))


def _free_port():
    sk = socket.socket()
    sk.bind(("127.0.0.1", 0))
    p = sk.getsockname()[1]
    sk.close()
    return p


def _decomposed_worker(rank, world, port, out_dir):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    box = np.full(3, 8.0)
    x, v, m = _fluid(box, seed=3)
    s = _system(x, v, m, box, _inter(True)[0], F64, r_list=1.5)
    s.device = rank
    s.engine()
    uid = [mb.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    x0, out = s.coords.copy(), []
    try:
        mb.comm_init(s, uid[0], rank, world)
        mb.simulate(s, mb.DPDVelocityVerlet(dt=0.02), 5)
        out.append("ok")
    except mb.MollyB200Error as e:
        out.append(str(e))
    assert np.array_equal(s.coords, x0)  # refused before any work
    s.close()
    np.save(os.path.join(out_dir, f"rank{rank}.npy"), np.array(out))
    dist.destroy_process_group()


def test_decomposed_context_refuses():
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_decomposed_worker, args=(2, _free_port(), d), nprocs=2, join=True)
        for rank in range(2):
            for r in np.load(os.path.join(d, f"rank{rank}.npy")):
                assert str(mb.capi.MB_ERR_INVALID) in r and "decomposed" in r, r
