"""GPU tests of the Nose-Hoover integrator (src/simulators.jl:1491-1614): trajectory parity with the numpy restatement of
the reference loop (tests/nosehoover_oracle.py) on the all-pairs, brick, triclinic and PME paths; zeta reset per call; the
reference's test/simulation.jl protocol; and the observer / determinism properties of the step graph. No draws are involved,
so every trajectory is pinned."""
import ctypes as C
import math

import numpy as np
import pytest

import mbhelpers as H
import mollyb200 as mb
import nosehoover_oracle as nho
from oracle import oracle as o
from test_gpu_parity import _pos_err

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
KB = mb.BOLTZMANN_K


def _box_wrap(box):
    return lambda x: x - np.floor(x / box) * box


def _readme():
    sd = H.readme_system(100, 2.0, seed=1)
    orc = H.make_oracle(sd, [o.Inter(o.LJ)])
    return sd, H.make_system(sd, (mb.LennardJones(),), F64), lambda x: orc.forces_allpairs(x, energy=False)[0], 0


def _lj_brick(dtype=F64):
    """864 argon atoms on the brick path with a 0.02 nm skin: the neighbour structure is rebuilt inside the run."""
    sd = H.lj_fluid(6, seed=3, dtype=F64)
    s = H.make_system(sd, (mb.LennardJones(cutoff=mb.ShiftedForceCutoff(0.9), use_neighbors=True),), dtype, r_list=0.92)
    orc = H.make_oracle(sd, [o.Inter(o.LJ, o.CUT_SHIFTED_FORCE, 0.9, use_neighbors=True)])
    return sd, s, lambda x: orc.forces_allpairs(x, energy=False)[0], 1


def _molecular():
    sd = H.molecular_system(729, [5.1, 5.4, 5.8], seed=5, stable=True)
    s = H.make_system(sd, (mb.LennardJones(cutoff=mb.ShiftedForceCutoff(1.0), use_neighbors=True, weight_special=0.5),
                           mb.CoulombReactionField(dist_cutoff=1.0, use_neighbors=True, weight_special=0.8333)), F64, r_list=1.15)
    orc = H.make_oracle(sd, [o.Inter(o.LJ, o.CUT_SHIFTED_FORCE, 1.0, weight_special=0.5, use_neighbors=True),
                             o.Inter(o.CRF, o.CUT_DISTANCE, 1.0, weight_special=0.8333, use_neighbors=True)])
    return sd, s, lambda x: orc.forces_allpairs(x, energy=False)[0], 1


def _sixmrr(g):
    s = H.sixmrr_system(g, F64, r_list=1.2)
    orc, sd = H.sixmrr_oracle(g)
    return sd, s, lambda x: orc.forces_nl(x, orc.neighbor_list(x, 1.2), energy=False)[0] + H.bonded_forces_oracle(g, x)[0], 1


def _sixmrr_pme(g):
    """LJ + CoulombEwald real space (C oracle) + PME reciprocal space + Ewald exclusions (oracle/pme.py) + bonded terms."""
    from oracle import pme
    s = H.sixmrr_pme_system(g, F64, exact=True)
    sd = H.sixmrr_description(g)
    alpha = pme.pme_alpha(1.0)
    orc = H.make_oracle(sd, [o.Inter(o.LJ, o.CUT_DISTANCE, 1.0, weight_special=float(g["lj14scale"]), use_neighbors=True),
                             o.Inter(o.EWALD_REAL, o.CUT_DISTANCE, 1.0, weight_special=float(g["coulomb14scale"]),
                                     ewald_alpha=alpha, use_neighbors=True)])
    excl = np.concatenate([g["excluded"], g["special"]])

    def fe(x):
        f = orc.forces_nl(x, orc.neighbor_list(x, 1.2), energy=False)[0]
        f += pme.pme_reciprocal(x, g["charge"], sd["box"], r_cut=1.0, error_tol=0.0005, order=5)[0]
        f += pme.ewald_exclusion(x, g["charge"], sd["box"], excl)[0]
        return f + H.bonded_forces_oracle(g, x)[0]
    return sd, s, fe, 1


SYSTEMS = {"readme-allpairs": _readme, "lj-brick-rebuilds": _lj_brick, "molecular-brick": _molecular}


def _parity(sd, s, fe, path, T=300.0, damping=None, rcm=1, init_step=0, n=50, dt=0.002, wrap=None, chunks=None, graph=None):
    """n steps in one call (chunks=None) or in calls of `chunks` steps, each restarting zeta at 0, against the oracle's
    restatement of the same calls."""
    sim = mb.NoseHoover(dt=dt, temperature=T, damping=damping, remove_CM_motion=rcm)
    x_ref, v_ref, step = sd["coords"], sd["velocities"], init_step
    rb0 = s.stats()["n_rebuilds"] if s._ctx is not None else 0
    for k in (chunks or [n]):
        x_ref, v_ref, _ = nho.simulate_nose_hoover(fe, x_ref, v_ref, sd["mass"], dt, k, KB * T, sim.damping,
                                                   wrap or _box_wrap(sd["box"]), remove_cm_every=rcm, init_step=step)
        mb.simulate(s, sim, k, init_step=step)
        step += k
    st = s.stats()
    ex = _pos_err(s.coords, x_ref, sd["box"]) if wrap is None else np.abs(s.coords - x_ref).max()
    ev = np.abs(s.velocities - v_ref).max()
    print(f"[NoseHoover rcm={rcm} init={init_step} chunks={chunks} path={st['path']} graph={st['graph_mode']} "
          f"rebuilds={st['n_rebuilds'] - rb0}] dx={ex:.3e} dv={ev:.3e}")
    assert st["path"] == path
    if graph is not None:
        assert st["graph_mode"] == graph
    assert ex < 1e-9 and ev < 1e-8
    return st["n_rebuilds"] - rb0, x_ref, v_ref


@pytest.mark.parametrize("name", list(SYSTEMS))
def test_parity_f64(name):
    sd, s, fe, path = SYSTEMS[name]()
    rebuilds, _, _ = _parity(sd, s, fe, path, T=120.0 if name != "readme-allpairs" else 300.0, graph=1)
    if name == "lj-brick-rebuilds":
        assert rebuilds > 1
    s.close()


def test_parity_6mrr_bonded(golden_6mrr):
    sd, s, fe, path = _sixmrr(golden_6mrr)
    _parity(sd, s, fe, path, n=20)
    s.close()


def test_parity_6mrr_pme_stream_path(golden_6mrr):
    """PME runs the stream path (cuFFT stays outside the captured step)."""
    sd, s, fe, path = _sixmrr_pme(golden_6mrr)
    _parity(sd, s, fe, path, n=10, dt=0.0005, graph=0)
    s.close()


@pytest.mark.parametrize("rcm", [0, 1, 3])
@pytest.mark.parametrize("init_step", [0, 13])
def test_parity_remove_cm_and_init_step(rcm, init_step):
    sd, s, fe, path = _readme()
    _parity(sd, s, fe, path, rcm=rcm, init_step=init_step, T=250.0)
    s.close()


def test_parity_triclinic_allpairs():
    from oracle import triclinic as tri
    bv = np.array([[3.0, 0.0, 0.0], [0.8, 3.1, 0.0], [0.5, -0.6, 3.2]])
    t = tri.Triclinic(bv)
    rng = np.random.default_rng(21)
    pts = []
    while len(pts) < 40:
        c = rng.random(3) @ bv
        if all(np.linalg.norm(t.vector(c, q)) > 0.3 for q in pts):
            pts.append(c)
    x = np.array(pts)
    n = len(x)
    sig, eps, mass = np.full(n, 0.3), np.full(n, 0.5), np.linspace(1.0, 20.0, n)
    v = rng.normal(0, 0.3, (n, 3))
    atoms = mb.atoms_from_arrays(mass, np.zeros(n), sig, eps, F64)
    s = mb.System(atoms=atoms, coords=x.copy(), velocities=v.copy(), boundary=mb.TriclinicBoundary(*bv),
                  pairwise_inters=(mb.LennardJones(cutoff=mb.DistanceCutoff(1.2)),), dtype=F64)
    sd = dict(coords=x, velocities=v, mass=mass, box=np.diag(bv))
    wrap = lambda y: np.array([t.wrap(r) for r in y])  # noqa: E731
    _parity(sd, s, lambda y: tri.forces_energy(t, y, sig, eps, r_cut=1.2)[0], 0, wrap=wrap)
    d = np.array([t.vector(a, b) for a, b in zip(s.coords, wrap(s.coords))])
    assert np.abs(d).max() < 1e-12
    s.close()


def test_chunked_calls_restart_zeta():
    """25 + 25 steps match the oracle's two calls, each starting from zeta = 0 (the reference keeps zeta as a local of
    simulate!), and differ from one 50-step call, which matches the oracle's single call. T0 = 150 K against a 90 K start,
    so that zeta is far from 0 after 25 steps."""
    sd, a, fe, path = _lj_brick()
    _, b, _, _ = _lj_brick()
    _, x1, v1 = _parity(sd, a, fe, path, T=150.0, n=50)
    _, x2, v2 = _parity(sd, b, fe, path, T=150.0, chunks=[25, 25])
    assert np.abs(v1 - v2).max() > 1e-4 and np.abs(a.velocities - b.velocities).max() > 1e-4
    a.close(); b.close()


@pytest.mark.parametrize("dtype", [F32, F64])
def test_reference_simulation_protocol(dtype):
    """test/simulation.jl:805-831: 256 argon atoms (m 39.98, sigma 0.34 nm, eps 0.2 kJ/mol, LennardJones without cutoff) in
    a 4 nm box placed at least 0.36 nm apart, velocities at 100 K; SteepestDescentMinimizer, then NoseHoover(dt 2 fs,
    100 K) for 50 000 steps with TemperatureLogger(1): the mean temperature lies within 1 K of 100 K and its standard
    deviation exceeds 2 K."""
    n, box, T0, m = 256, 4.0, 100.0, 39.98
    sd = H.readme_system(n, box, seed=12, min_dist=0.36)
    v = np.random.default_rng(13).normal(0.0, math.sqrt(KB * T0 / m), (n, 3))
    atoms = mb.atoms_from_arrays(np.full(n, m), np.zeros(n), np.full(n, 0.34), np.full(n, 0.2), dtype)
    s = mb.System(atoms=atoms, coords=sd["coords"].astype(dtype), velocities=v.astype(dtype), boundary=mb.CubicBoundary(box),
                  pairwise_inters=(mb.LennardJones(),), dtype=dtype, loggers={"temp": mb.TemperatureLogger(1)})
    mb.simulate(s, mb.SteepestDescentMinimizer())
    mb.simulate(s, mb.NoseHoover(dt=0.002, temperature=T0), 50_000)
    temps = np.array(mb.values(s.loggers["temp"]))
    assert len(temps) == 50_001
    print(f"[simulation.jl NoseHoover {np.dtype(dtype).name}] <T> = {temps.mean():.3f} K, std {temps.std():.3f} K, "
          f"graph={s.stats()['graph_mode']}")
    assert T0 - 1.0 < temps.mean() < T0 + 1.0
    assert temps.std() > 2.0
    s.close()


def _run(n=40, loggers=None, dtype=F64, device=False, T=120.0):
    sd, s, _, _ = _lj_brick(dtype)
    if loggers:
        s.loggers = loggers
    if device:
        import torch
        s.coords = torch.from_numpy(s.coords).cuda()
        s.velocities = torch.from_numpy(s.velocities).cuda()
    mb.simulate(s, mb.NoseHoover(dt=0.002, temperature=T), n)
    out = [a.cpu().numpy() if hasattr(a, "cpu") else a.copy() for a in (s.coords, s.velocities)] + [s.stats()["graph_mode"]]
    s.close()
    return out


def test_two_identical_runs_bit_identical():
    x0, v0, g = _run()
    x1, v1, _ = _run()
    assert g == 1
    assert np.array_equal(x0, x1) and np.array_equal(v0, v1)


def test_graph_and_stream_paths_bit_identical(monkeypatch):
    res = []
    for no_graph in ("0", "1"):
        monkeypatch.setenv("MOLLYB200_NO_GRAPH", no_graph)
        lg = {"ke": mb.KineticEnergyLogger(5)}
        x, v, g = _run(loggers=lg)
        res.append((x, v, list(lg["ke"].history), g))
    (xa, va, ka, ga), (xb, vb, kb, gb) = res
    assert (ga, gb) == (1, 0)
    assert np.array_equal(xa, xb) and np.array_equal(va, vb) and ka == kb


def test_host_and_device_buffers_identical():
    a, b = _run(), _run(device=True)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


@pytest.mark.parametrize("dtype", [F32, F64])
def test_loggers_are_observers(dtype):
    x0, v0, _ = _run(n=30, dtype=dtype)
    lg = {"v": mb.VelocitiesLogger(7), "e": mb.TotalEnergyLogger(7), "pe": mb.PotentialEnergyLogger(7),
          "ke": mb.KineticEnergyLogger(7), "t": mb.TemperatureLogger(7), "x": mb.CoordinatesLogger(10)}
    x1, v1, _ = _run(n=30, loggers=lg, dtype=dtype)
    assert np.array_equal(x0, x1) and np.array_equal(v0, v1)
    # a logged record equals an unlogged run stopped at that step
    for k, step in enumerate(mb.record_steps(7, 30)):
        if step == 0:
            continue
        xs, vs, _ = _run(n=step, dtype=dtype)
        assert np.array_equal(lg["v"].history[k], vs)
        sd, s, _, _ = _lj_brick()
        ref = H.make_system(dict(sd, coords=xs, velocities=vs), s.pairwise_inters, dtype, r_list=0.92)
        s.close()
        pe, ke = mb.potential_energy(ref), mb.kinetic_energy(ref)
        ref.close()
        tol = 1e-5 if dtype == F32 else 1e-10
        assert abs(lg["pe"].history[k] - pe) < tol * abs(pe)
        assert abs(lg["ke"].history[k] - ke) < 1e-12 * ke
        assert abs(lg["e"].history[k] - (pe + ke)) < tol * abs(pe)
        assert abs(lg["t"].history[k] - 2 * ke / ((3 * sd["n"] - 3) * KB)) < 1e-12 * lg["t"].history[k]


def test_refusals_leave_coordinates_untouched():
    sd, s, _, _ = _readme()
    ctx = s.engine()
    L = s._L
    x, v = s.coords.copy(), s.velocities.copy()
    P = mb.capi.MBNoseHooverParams
    bad = [P(0.0, 10, 0, 1, 2.0, 0.2), P(-0.002, 10, 0, 1, 2.0, 0.2), P(math.nan, 10, 0, 1, 2.0, 0.2),
           P(0.002, -1, 0, 1, 2.0, 0.2),
           P(0.002, 10, 0, 1, -2.0, 0.2), P(0.002, 10, 0, 1, 0.0, 0.2), P(0.002, 10, 0, 1, math.nan, 0.2),
           P(0.002, 10, 0, 1, math.inf, 0.2),
           P(0.002, 10, 0, 1, 2.0, 0.0), P(0.002, 10, 0, 1, 2.0, -0.2), P(0.002, 10, 0, 1, 2.0, math.nan),
           P(0.002, 10, 0, 1, 2.0, math.inf)]
    for p in bad:
        assert L.mb_simulate_nose_hoover(ctx, s.coords.ctypes.data, s.velocities.ctypes.data, C.byref(p), None) == mb.capi.MB_ERR_INVALID
        assert np.array_equal(x, s.coords) and np.array_equal(v, s.velocities)
    assert L.mb_simulate_nose_hoover(ctx, s.coords.ctypes.data, s.velocities.ctypes.data, None, None) == mb.capi.MB_ERR_INVALID
    # a logging request the call cannot honour: capacity below the records it writes
    rec = np.zeros((2, 3))
    lg = mb.capi.MBLog(energy_every=1, log_initial=1, energies=rec.ctypes.data, energy_capacity=2)
    p = P(0.002, 10, 0, 1, 2.0, 0.2)
    assert L.mb_simulate_nose_hoover(ctx, s.coords.ctypes.data, s.velocities.ctypes.data, C.byref(p), C.byref(lg)) == mb.capi.MB_ERR_INVALID
    assert np.array_equal(x, s.coords) and np.array_equal(v, s.velocities)
    # a velocity coupling set on the context
    assert L.mb_set_velocity_coupling(ctx, C.byref(mb.capi.MBVCoupling(mb.capi.MB_VC_IMMEDIATE, 0, 2.0, 0.0))) == 0
    assert L.mb_simulate_nose_hoover(ctx, s.coords.ctypes.data, s.velocities.ctypes.data, C.byref(p), None) == mb.capi.MB_ERR_INVALID
    assert b"velocity coupling" in L.mb_last_error()
    assert np.array_equal(x, s.coords) and np.array_equal(v, s.velocities)
    # simulate clears it: the run goes through
    mb.simulate(s, mb.NoseHoover(0.002, 300.0), 5)
    s.close()
    # one atom: Nf = 0
    one = mb.System(atoms=mb.atoms_from_arrays([10.0], [0.0], [0.3], [0.2], F64), coords=np.array([[0.5, 0.5, 0.5]]),
                    velocities=np.array([[0.1, 0.2, 0.3]]), boundary=mb.CubicBoundary(2.0), pairwise_inters=(mb.LennardJones(),),
                    dtype=F64)
    x1, v1 = one.coords.copy(), one.velocities.copy()
    p = P(0.002, 10, 0, 0, 2.0, 0.2)
    ctx1 = one.engine()
    assert one._L.mb_simulate_nose_hoover(ctx1, one.coords.ctypes.data, one.velocities.ctypes.data, C.byref(p), None) == mb.capi.MB_ERR_INVALID
    assert b"2 atoms" in one._L.mb_last_error()
    assert np.array_equal(x1, one.coords) and np.array_equal(v1, one.velocities)
    one.close()


def test_velocity_verlet_after_nose_hoover_equals_fresh_system():
    """No zeta or v_cm state of the Nose-Hoover call leaks into a later VelocityVerlet call on the same context."""
    sd, s, _, _ = _lj_brick()
    mb.simulate(s, mb.NoseHoover(dt=0.002, temperature=150.0), 20)
    ref = H.make_system(dict(sd, coords=s.coords.copy(), velocities=s.velocities.copy()), s.pairwise_inters, F64, r_list=0.92)
    mb.simulate(s, mb.VelocityVerlet(dt=0.002), 30, init_step=20)
    mb.simulate(ref, mb.VelocityVerlet(dt=0.002), 30, init_step=20)
    assert _pos_err(s.coords, ref.coords, sd["box"]) < 1e-12
    assert np.abs(s.velocities - ref.velocities).max() < 1e-12
    s.close(); ref.close()
