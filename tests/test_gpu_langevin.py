"""GPU tests of the Langevin integrator (src/simulators.jl:1065-1210): trajectory parity with the numpy restatement of the
reference loop (tests/langevin_oracle.py) on the all-pairs, brick and triclinic paths; the exact statistics of the O step on
free particles; the reference's test/simulation.jl protocol; canonical sampling of the kinetic energy; and the observer /
determinism properties of the step graph."""
import ctypes as C
import math

import numpy as np
import pytest

import langevin_oracle as lo
import mbhelpers as H
import mollyb200 as mb
import thermostat_oracle as tho
from oracle import oracle as o
from test_gpu_parity import _pos_err

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
KB = mb.BOLTZMANN_K


def _keys(seed):
    """The (rng_ctr1, rng_key) words simulate(..., rng=np.random.default_rng(seed)) passes to the engine."""
    r = np.random.default_rng(seed)
    return tho.rng_words(int(r.integers(0, 2 ** 63)), int(r.integers(0, 2 ** 63)))


def _box_wrap(box):
    return lambda x: x - np.floor(x / box) * box


def _readme():
    sd = H.readme_system(100, 2.0, seed=1)
    orc = H.make_oracle(sd, [o.Inter(o.LJ)])
    return sd, H.make_system(sd, (mb.LennardJones(),), F64), lambda x: orc.forces_allpairs(x, energy=False)[0], 0


def _lj_brick():
    """864 argon atoms on the brick path with a 0.02 nm skin: the neighbour structure is rebuilt inside the run."""
    sd = H.lj_fluid(6, seed=3, dtype=F64)
    s = H.make_system(sd, (mb.LennardJones(cutoff=mb.ShiftedForceCutoff(0.9), use_neighbors=True),), F64, r_list=0.92)
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


SYSTEMS = {"readme-allpairs": _readme, "lj-brick-rebuilds": _lj_brick, "molecular-brick": _molecular}


def _parity(sd, s, fe, path, T=300.0, friction=1.0, rcm=1, init_step=0, n=50, dt=0.002, wrap=None, seed=7):
    sim = mb.Langevin(dt=dt, temperature=T, friction=friction, remove_CM_motion=rcm)
    x_ref, v_ref = lo.simulate_langevin(fe, sd["coords"], sd["velocities"], sd["mass"], dt, n, KB * T, friction, _keys(seed),
                                        wrap or _box_wrap(sd["box"]), remove_cm_every=rcm, init_step=init_step)
    rb0 = s.stats()["n_rebuilds"] if s._ctx is not None else 0
    mb.simulate(s, sim, n, init_step=init_step, rng=np.random.default_rng(seed))
    st = s.stats()
    ex = _pos_err(s.coords, x_ref, sd["box"]) if wrap is None else np.abs(s.coords - x_ref).max()
    ev = np.abs(s.velocities - v_ref).max()
    print(f"[Langevin rcm={rcm} init={init_step} path={st['path']} graph={st['graph_mode']} rebuilds={st['n_rebuilds'] - rb0}] "
          f"dx={ex:.3e} dv={ev:.3e}")
    assert st["path"] == path
    assert ex < 1e-9 and ev < 1e-8
    return st["n_rebuilds"] - rb0


@pytest.mark.parametrize("name", list(SYSTEMS))
def test_parity_f64(name):
    sd, s, fe, path = SYSTEMS[name]()
    rebuilds = _parity(sd, s, fe, path, T=120.0 if name != "readme-allpairs" else 300.0)
    if name == "lj-brick-rebuilds":
        assert rebuilds > 1
    s.close()


def test_parity_6mrr_bonded(golden_6mrr):
    sd, s, fe, path = _sixmrr(golden_6mrr)
    _parity(sd, s, fe, path, n=20)
    s.close()


@pytest.mark.parametrize("rcm,init_step", [(0, 0), (3, 0), (1, 13), (3, 13)])
def test_parity_remove_cm_and_init_step(rcm, init_step):
    sd, s, fe, path = _readme()
    _parity(sd, s, fe, path, rcm=rcm, init_step=init_step)
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


@pytest.mark.parametrize("dtype", [F32, F64])
def test_o_step_statistics_free_particles(dtype):
    """All eps = 0: F = 0, so the velocity of every atom is an AR(1) process v_n = c v_{n-1} + sigma xi: E[v_n] = c^n v0 and
    Var[v_n] = (kT/m)(1 - c^(2n)). 24 000 atoms in four mass groups plus massless ones, remove_CM_motion = 0. The bars are 5
    standard errors of the sample mean and variance (N = 3 x 6000 components per group)."""
    n_grp, masses = 6000, [1.0, 12.0, 39.948, 200.0]
    n = n_grp * len(masses) + 50
    mass = np.concatenate([np.full(n_grp, m) for m in masses] + [np.zeros(50)])
    rng = np.random.default_rng(4)
    x = rng.random((n, 3)) * 10.0
    v0 = np.tile(np.array([0.7, -0.3, 0.2]), (n, 1))
    T, gamma, dt = 300.0, 5.0, 0.004
    kT, c = KB * T, math.exp(-gamma * dt)
    atoms = mb.atoms_from_arrays(mass, np.zeros(n), np.full(n, 0.3), np.zeros(n), dtype)
    s = mb.System(atoms=atoms, coords=x.astype(dtype), velocities=v0.astype(dtype), boundary=mb.CubicBoundary(10.0),
                  pairwise_inters=(mb.LennardJones(),), dtype=dtype)
    sim = mb.Langevin(dt=dt, temperature=T, friction=gamma, remove_CM_motion=0)
    done = 0
    for k in (1, 10, 60):
        mb.simulate(s, sim, k - done, init_step=done, rng=np.random.default_rng(11))
        done = k
        v = s.velocities.astype(np.float64)
        for g, m in enumerate(masses):
            vg = v[g * n_grp:(g + 1) * n_grp] - c ** k * v0[0]
            var = kT / m * (1 - c ** (2 * k))
            N = vg.size
            assert abs(vg.mean()) < 5 * math.sqrt(var / N), (k, m)
            assert abs(vg.var() / var - 1) < 5 * math.sqrt(2 / N), (k, m)
        np.testing.assert_allclose(v[-50:], np.tile(c ** k * v0[0], (50, 1)), rtol=1e-5 if dtype == F32 else 1e-12)
    s.close()


@pytest.mark.parametrize("dtype", [F32, F64])
def test_reference_simulation_protocol(dtype):
    """test/simulation.jl:770-800: 400 LJ atoms in a 10 nm box at 300 K, dt 2 fs, friction 1 ps^-1, 2000 steps,
    TemperatureLogger(10); the mean of the last 101 records lies in [280, 320] K."""
    n, box = 400, 10.0
    sd = H.readme_system(n, box, seed=9, min_dist=0.3)
    atoms = mb.atoms_from_arrays(np.full(n, 10.0), np.zeros(n), np.full(n, 0.3), np.full(n, 0.2), dtype)
    s = mb.System(atoms=atoms, coords=sd["coords"].astype(dtype), velocities=sd["velocities"].astype(dtype),
                  boundary=mb.CubicBoundary(box), pairwise_inters=(mb.LennardJones(cutoff=mb.DistanceCutoff(1.0), use_neighbors=True),),
                  neighbor_finder=mb.GPUNeighborFinder(dist_cutoff=1.2), dtype=dtype,
                  loggers={"temperature": mb.TemperatureLogger(10)})
    mb.simulate(s, mb.Langevin(dt=0.002, temperature=300.0, friction=1.0), 2000, rng=np.random.default_rng(3))
    temps = np.array(mb.values(s.loggers["temperature"]))
    assert len(temps) == 201
    print(f"[simulation.jl Langevin {np.dtype(dtype).name}] <T> over the last 101 = {temps[-101:].mean():.2f} K")
    assert 280.0 < temps[-101:].mean() < 320.0
    s.close()


def test_canonical_kinetic_energy():
    """2916 argon atoms at 90 K, friction 5 ps^-1. In the canonical ensemble <K> = Nf kT / 2, Var(K) = Nf (kT)^2 / 2 with
    Nf = 3N - 3 (CM removed every step). KE is logged every 10 steps; blocks of 50 records (1 ps, five relaxation times
    1/friction) give the standard errors; 4-sigma bars. The velocities lag the positions by half a step, so <K> carries an
    O((gamma dt)^2, (omega dt)^2) bias far below these bars at dt = 2 fs."""
    sd = H.lj_fluid(9, seed=21, dtype=F64, temp=90.0)
    s = H.make_system(sd, (mb.LennardJones(cutoff=mb.ShiftedForceCutoff(1.0), use_neighbors=True),), F64, r_list=1.2)
    s.loggers = {"ke": mb.KineticEnergyLogger(10)}
    T0 = 90.0
    mb.simulate(s, mb.Langevin(dt=0.002, temperature=T0, friction=5.0), 21_000, rng=np.random.default_rng(8))
    ke = np.array(s.loggers["ke"].history[101:])
    nf = 3 * sd["n"] - 3
    kbar = nf * KB * T0 / 2
    nb = len(ke) // 50
    blocks = ke[:nb * 50].reshape(nb, 50)
    mean, se_mean = blocks.mean(), blocks.mean(1).std(ddof=1) / math.sqrt(nb)
    dev2 = (blocks - mean) ** 2
    ratio = dev2.mean() / (2 * kbar * kbar / nf)
    se_ratio = dev2.mean(1).std(ddof=1) / math.sqrt(nb) / (2 * kbar * kbar / nf)
    print(f"[Langevin canonical] <K>/Kbar-1={mean / kbar - 1:.2e} (se {se_mean / kbar:.1e}); Var ratio={ratio:.3f} (se {se_ratio:.3f})")
    assert abs(mean - kbar) < 4 * se_mean + 2e-3 * kbar
    assert abs(ratio - 1) < 4 * se_ratio + 0.02


def _run(seed, friction=2.0, n=40, loggers=None, dtype=F64, device=False):
    sd, s, _, _ = _lj_brick()
    if dtype != F64:
        s = H.make_system(sd, (mb.LennardJones(cutoff=mb.ShiftedForceCutoff(0.9), use_neighbors=True),), dtype, r_list=0.92)
    if loggers:
        s.loggers = loggers
    if device:
        import torch
        s.coords = torch.from_numpy(s.coords).cuda()
        s.velocities = torch.from_numpy(s.velocities).cuda()
    mb.simulate(s, mb.Langevin(dt=0.002, temperature=120.0, friction=friction), n, rng=np.random.default_rng(seed))
    out = [a.cpu().numpy() if hasattr(a, "cpu") else a.copy() for a in (s.coords, s.velocities)] + [s.stats()["graph_mode"]]
    s.close()
    return out


def test_friction_zero_ignores_the_seed():
    x0, v0, _ = _run(1, friction=0.0)
    x1, v1, _ = _run(2, friction=0.0)
    assert np.array_equal(x0, x1) and np.array_equal(v0, v1)


def test_seeds():
    x0, v0, g = _run(9)
    x1, v1, _ = _run(9)
    x2, v2, _ = _run(10)
    assert g == 1
    assert np.array_equal(x0, x1) and np.array_equal(v0, v1)
    assert np.abs(v0 - v2).max() > 1e-3


def test_graph_and_stream_paths_bit_identical(monkeypatch):
    res = []
    for no_graph in ("0", "1"):
        monkeypatch.setenv("MOLLYB200_NO_GRAPH", no_graph)
        lg = {"ke": mb.KineticEnergyLogger(5)}
        x, v, g = _run(2, loggers=lg)
        res.append((x, v, list(lg["ke"].history), g))
    (xa, va, ka, ga), (xb, vb, kb, gb) = res
    assert (ga, gb) == (1, 0)
    assert np.array_equal(xa, xb) and np.array_equal(va, vb) and ka == kb


def test_host_and_device_buffers_identical():
    a, b = _run(6), _run(6, device=True)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


@pytest.mark.parametrize("dtype", [F32, F64])
def test_loggers_are_observers(dtype):
    x0, v0, _ = _run(4, n=30, dtype=dtype)
    lg = {"v": mb.VelocitiesLogger(7), "e": mb.TotalEnergyLogger(7), "pe": mb.PotentialEnergyLogger(7),
          "ke": mb.KineticEnergyLogger(7), "x": mb.CoordinatesLogger(10)}
    x1, v1, _ = _run(4, n=30, loggers=lg, dtype=dtype)
    assert np.array_equal(x0, x1) and np.array_equal(v0, v1)
    # a logged record equals an unlogged run stopped at that step
    for k, step in enumerate(mb.record_steps(7, 30)):
        if step == 0:
            continue
        xs, vs, _ = _run(4, n=step, dtype=dtype)
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


def test_chunked_calls_equal_one_call():
    """simulate(25) then simulate(15; init_step=25) == simulate(40): the draws are a function of (keys, step, atom), so with
    the same keys (a fresh generator of the same seed for every call) the chunked run takes the same draws."""
    sim = mb.Langevin(dt=0.002, temperature=120.0, friction=2.0)
    sd, a, _, _ = _lj_brick()
    _, b, _, _ = _lj_brick()
    mb.simulate(a, sim, 40, rng=np.random.default_rng(1))
    mb.simulate(b, sim, 25, rng=np.random.default_rng(1))
    mb.simulate(b, sim, 15, init_step=25, rng=np.random.default_rng(1))
    assert _pos_err(a.coords, b.coords, sd["box"]) < 1e-9
    assert np.abs(a.velocities - b.velocities).max() < 1e-8
    a.close(); b.close()


def test_refusals_leave_coordinates_untouched():
    sd, s, _, _ = _readme()
    ctx = s.engine()
    L = s._L
    x, v = s.coords.copy(), s.velocities.copy()
    P = mb.capi.MBLangevinParams
    bad = [P(0.0, 10, 0, 1, 2.0, 1.0, 1, 2), P(-0.002, 10, 0, 1, 2.0, 1.0, 1, 2), P(0.002, -1, 0, 1, 2.0, 1.0, 1, 2),
           P(0.002, 10, 0, 1, -2.0, 1.0, 1, 2), P(0.002, 10, 0, 1, math.nan, 1.0, 1, 2), P(0.002, 10, 0, 1, math.inf, 1.0, 1, 2),
           P(0.002, 10, 0, 1, 2.0, -1.0, 1, 2), P(0.002, 10, 0, 1, 2.0, math.nan, 1, 2), P(0.002, 10, 0, 1, 2.0, math.inf, 1, 2)]
    for p in bad:
        assert L.mb_simulate_langevin(ctx, s.coords.ctypes.data, s.velocities.ctypes.data, C.byref(p), None) == mb.capi.MB_ERR_INVALID
        assert np.array_equal(x, s.coords) and np.array_equal(v, s.velocities)
    # a velocity coupling set on the context
    assert L.mb_set_velocity_coupling(ctx, C.byref(mb.capi.MBVCoupling(mb.capi.MB_VC_IMMEDIATE, 0, 2.0, 0.0))) == 0
    p = P(0.002, 10, 0, 1, 2.0, 1.0, 1, 2)
    assert L.mb_simulate_langevin(ctx, s.coords.ctypes.data, s.velocities.ctypes.data, C.byref(p), None) == mb.capi.MB_ERR_INVALID
    assert b"velocity coupling" in L.mb_last_error()
    assert np.array_equal(x, s.coords) and np.array_equal(v, s.velocities)
    # simulate clears it: the run goes through
    mb.simulate(s, mb.Langevin(0.002, 300.0, 1.0), 5)
    s.close()


def test_velocity_verlet_after_langevin_equals_fresh_system():
    sd, s, _, _ = _lj_brick()
    mb.simulate(s, mb.Langevin(dt=0.002, temperature=120.0, friction=2.0), 20, rng=np.random.default_rng(3))
    ref = H.make_system(dict(sd, coords=s.coords.copy(), velocities=s.velocities.copy()), s.pairwise_inters, F64, r_list=0.92)
    mb.simulate(s, mb.VelocityVerlet(dt=0.002), 30, init_step=20)
    mb.simulate(ref, mb.VelocityVerlet(dt=0.002), 30, init_step=20)
    assert _pos_err(s.coords, ref.coords, sd["box"]) < 1e-12
    assert np.abs(s.velocities - ref.velocities).max() < 1e-12
    s.close(); ref.close()
