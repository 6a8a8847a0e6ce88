"""GPU tests of Verlet, StormerVerlet and OverdampedLangevin (src/simulators.jl:858-1063, :1400-1490): trajectory parity
with the numpy restatements of the reference loops (tests/verlet_oracle.py) on the all-pairs, brick, molecular, triclinic,
6mrr (bonded, PME) and GBN2 paths; the engine's own identities against its VelocityVerlet; Andersen with Verlet;
Euler-Maruyama statistics; determinism, loggers and refusals; and the reference's test/simulation.jl protocols."""
import ctypes as C
import math
import os
import socket

import numpy as np
import pytest

import mbhelpers as H
import mollyb200 as mb
import thermostat_oracle as tho
import verlet_oracle as vo
from test_gpu_nosehoover import _box_wrap, _lj_brick, _molecular, _readme, _sixmrr, _sixmrr_pme
from test_gpu_parity import _pos_err

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
KB = mb.BOLTZMANN_K
KINDS = ["verlet", "stormer", "overdamped"]
SYSTEMS = {"readme-allpairs": _readme, "lj-brick-rebuilds": _lj_brick, "molecular-brick": _molecular}


def _sim(kind, dt, rcm=1, T=120.0, friction=20.0):
    if kind == "verlet":
        return mb.Verlet(dt=dt, remove_CM_motion=rcm)
    if kind == "stormer":
        return mb.StormerVerlet(dt=dt)
    return mb.OverdampedLangevin(dt=dt, temperature=T, friction=friction, remove_CM_motion=rcm)


def _cubic_vector(box):
    def vec(a, b):
        d = b - a
        return d - box * np.round(d / box)
    return vec


def _parity(kind, sd, s, fe, path, rcm=1, init_step=0, n=40, dt=0.002, T=120.0, friction=5.0, wrap=None, vector=None,
            chunks=None, seed=7, label=""):
    """n steps in one call (chunks=None) or in calls of `chunks` steps against the oracle's restatement of the same calls;
    simulate draws one pair of keys per call from `rng`, as the oracle does here. The friction (OverdampedLangevin only)
    must keep Euler-Maruyama stable: k dt / (m gamma) < 2 for the stiffest bond k on the lightest atom m."""
    sim = _sim(kind, dt, rcm, T, friction)
    wrap = wrap or _box_wrap(sd["box"])
    vector = vector or _cubic_vector(np.asarray(sd["box"], np.float64))
    rng_o, rng_e = np.random.default_rng(seed), np.random.default_rng(seed)
    x_ref, v_ref, step = sd["coords"], sd["velocities"], init_step
    rb0 = s.stats()["n_rebuilds"] if s._ctx is not None else 0
    for k in (chunks or [n]):
        keys = tho.rng_words(int(rng_o.integers(0, 2 ** 63)), int(rng_o.integers(0, 2 ** 63)))
        if kind == "verlet":
            x_ref, v_ref = vo.simulate_verlet(fe, x_ref, v_ref, sd["mass"], dt, k, wrap, remove_cm_every=rcm, init_step=step)
        elif kind == "stormer":
            x_ref, v_ref = vo.simulate_stormer_verlet(fe, x_ref, v_ref, sd["mass"], dt, k, wrap, vector, init_step=step)
        else:
            x_ref, v_ref = vo.simulate_overdamped(fe, x_ref, v_ref, sd["mass"], dt, k, KB * T, friction, keys, wrap,
                                                  remove_cm_every=rcm, init_step=step)
        mb.simulate(s, sim, k, init_step=step, rng=rng_e)
        step += k
    st = s.stats()
    ex = np.abs(vector(x_ref, s.coords)).max()
    ev = np.abs(s.velocities - v_ref).max()
    print(f"[{kind} {label} rcm={rcm} init={init_step} chunks={chunks} path={st['path']} graph={st['graph_mode']} "
          f"rebuilds={st['n_rebuilds'] - rb0}] dx={ex:.3e} dv={ev:.3e}")
    assert path is None or st["path"] == path
    assert ex < 1e-9 and ev < 1e-8
    return st, st["n_rebuilds"] - rb0


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("name", list(SYSTEMS))
def test_parity_f64(name, kind):
    sd, s, fe, path = SYSTEMS[name]()
    # (the molecular system's bonds to light atoms need a large friction for a stable Euler-Maruyama step)
    st, rebuilds = _parity(kind, sd, s, fe, path, friction=2000.0 if name == "molecular-brick" else 5.0, label=name)
    assert st["graph_mode"] == 1
    if name == "lj-brick-rebuilds" and kind != "overdamped":
        assert rebuilds > 1
    s.close()


@pytest.mark.parametrize("kind", KINDS)
def test_parity_6mrr_bonded(golden_6mrr, kind):
    sd, s, fe, path = _sixmrr(golden_6mrr)
    _parity(kind, sd, s, fe, path, n=15, T=300.0, friction=2000.0, label="6mrr")
    s.close()


@pytest.mark.parametrize("kind", KINDS)
def test_parity_6mrr_pme_stream_path(golden_6mrr, kind):
    """PME runs the stream path (cuFFT stays outside the captured step)."""
    sd, s, fe, path = _sixmrr_pme(golden_6mrr)
    st, _ = _parity(kind, sd, s, fe, path, n=8, dt=0.0005, T=300.0, friction=2000.0, label="6mrr+PME")
    assert st["graph_mode"] == 0
    s.close()


@pytest.mark.parametrize("kind", KINDS)
def test_parity_implicit_solvent(kind):
    from test_gpu_implicit_solvent import ROOT, _full_oracle, _full_system
    g = np.load(os.path.join(ROOT, "tests", "golden", "6mrr_gb.npz"))
    v0 = np.random.default_rng(11).normal(0, 0.3, g["coords"].shape)
    s = _full_system(g, "gbn2", F64, velocities=v0)
    sd = dict(coords=g["coords"], velocities=v0, mass=g["mass"], box=np.asarray(g["box"], np.float64))
    st, _ = _parity(kind, sd, s, _full_oracle(g, "gbn2"), None, n=10, dt=0.001, T=300.0, friction=2000.0, label="gbn2")
    assert st["graph_mode"] == 1
    s.close()


@pytest.mark.parametrize("kind", KINDS)
def test_parity_triclinic_allpairs(kind):
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
    vector = lambda a, b: np.array([t.vector(p, q) for p, q in zip(a, b)])  # noqa: E731
    _parity(kind, sd, s, lambda y: tri.forces_energy(t, y, sig, eps, r_cut=1.2)[0], 0, wrap=wrap, vector=vector,
            label="triclinic")
    assert np.abs(vector(s.coords, wrap(s.coords))).max() < 1e-12
    s.close()


@pytest.mark.parametrize("kind,rcm,init_step", [(k, r, i) for k in ("verlet", "overdamped") for r in (0, 1, 3) for i in (0, 13)]
                         + [("stormer", 0, 0), ("stormer", 0, 13)])
def test_parity_remove_cm_and_init_step(kind, rcm, init_step):
    sd, s, fe, path = _readme()
    _parity(kind, sd, s, fe, path, rcm=rcm, init_step=init_step, T=250.0)
    s.close()


@pytest.mark.parametrize("kind", KINDS)
def test_parity_chunked_calls(kind):
    """Calls of 15, 11 and 14 steps on the brick path against the oracle's three calls: StormerVerlet's first-step rule
    applies in every call, and the state carried in the velocities survives the re-sorts in between."""
    sd, s, fe, path = _lj_brick()
    _parity(kind, sd, s, fe, path, chunks=[15, 11, 14], init_step=4, rcm=1 if kind != "stormer" else 0, label="chunked")
    s.close()


def _run(kind, n=40, loggers=None, dtype=F64, seed=5, rcm=1):
    sd, s, _, _ = _lj_brick(dtype)
    if loggers:
        s.loggers = loggers
    mb.simulate(s, _sim(kind, 0.002, rcm), n, rng=np.random.default_rng(seed))
    st = s.stats()
    out = (s.coords.copy(), s.velocities.copy(), st)
    s.close()
    return out


@pytest.mark.parametrize("kind", KINDS)
def test_graph_and_stream_paths_bit_identical(monkeypatch, kind):
    res = []
    for no_graph in ("0", "1"):
        monkeypatch.setenv("MOLLYB200_NO_GRAPH", no_graph)
        lg = {"ke": mb.KineticEnergyLogger(5)}
        x, v, st = _run(kind, loggers=lg)
        res.append((x, v, list(lg["ke"].history), st))
    (xa, va, ka, sa), (xb, vb, kb, sb) = res
    assert (sa["graph_mode"], sb["graph_mode"]) == (1, 0)
    assert np.array_equal(xa, xb) and np.array_equal(va, vb) and ka == kb


@pytest.mark.parametrize("kind", KINDS)
def test_one_force_evaluation_per_step(kind):
    sd, s, _, _ = _readme()
    mb.simulate(s, _sim(kind, 0.002), 5)
    e0 = s.stats()["n_force_evals"]
    mb.simulate(s, _sim(kind, 0.002), 30, init_step=5)
    assert s.stats()["n_force_evals"] - e0 == 31  # F0 and one per step
    s.close()


@pytest.mark.parametrize("kind", KINDS)
def test_same_keys_same_trajectory(kind):
    a, b = _run(kind, seed=9), _run(kind, seed=9)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    if kind == "overdamped":
        c = _run(kind, seed=10)
        assert np.abs(c[0] - a[0]).max() > 1e-4


def test_overdamped_split_run_takes_the_same_draws():
    """One 40-step call and 20 + 20 steps with the same keys (through the C ABI): the same draws, so the same trajectory
    up to the force summation order of the rebuilds at different points."""
    out = []
    for chunks in ([40], [20, 20]):
        sd, s, _, _ = _readme()
        ctx = s.engine()
        step = 0
        for k in chunks:
            p = mb.capi.MBLangevinParams(0.002, k, step, 0, KB * 200.0, 5.0, 0x1234567, 0x89ABCDEF)
            mb.capi.check(s._L.mb_simulate_overdamped_langevin(ctx, s.coords.ctypes.data, s.velocities.ctypes.data, C.byref(p), None))
            step += k
        out.append(s.coords.copy())
        s.close()
    assert _pos_err(out[0], out[1], sd["box"]) < 1e-12


def test_engine_stormer_and_shifted_verlet_equal_velocity_verlet():
    """In exact arithmetic StormerVerlet's positions are VelocityVerlet's, and so are those of Verlet started from
    v0 - a0 dt/2 (remove_CM_motion = 0 everywhere). The engine's three runs agree to f64 rounding over 100 steps."""
    dt, n = 0.002, 100
    sd, vv, _, _ = _readme()
    mb.simulate(vv, mb.VelocityVerlet(dt=dt, remove_CM_motion=0), n)
    _, sv, _, _ = _readme()
    mb.simulate(sv, mb.StormerVerlet(dt=dt), n)
    _, lf, _, _ = _readme()
    a0 = mb.forces(lf) / np.asarray(sd["mass"], np.float64)[:, None]
    lf.velocities[...] = lf.velocities - a0 * dt / 2
    mb.simulate(lf, mb.Verlet(dt=dt, remove_CM_motion=0), n)
    es, el = _pos_err(sv.coords, vv.coords, sd["box"]), _pos_err(lf.coords, vv.coords, sd["box"])
    print(f"[identities] stormer-vv {es:.3e} shifted verlet-vv {el:.3e}")
    assert es < 1e-9 and el < 1e-9
    for s in (vv, sv, lf):
        s.close()


def test_verlet_andersen_temperature():
    """Verlet with AndersenThermostat(150 K, 0.1 ps) on 864 argon atoms started at 90 K: the mean temperature of the last
    4000 of 6000 steps lies within 3 % of 150 K (the leapfrog's half-step velocities are biased by O(dt^2) only)."""
    T0 = 150.0
    sd = H.lj_fluid(6, seed=3, dtype=F64)
    s = H.make_system(sd, (mb.LennardJones(cutoff=mb.ShiftedForceCutoff(0.9), use_neighbors=True),), F64, r_list=1.0)
    s.loggers = {"t": mb.TemperatureLogger(10)}
    mb.simulate(s, mb.Verlet(dt=0.002, coupling=mb.AndersenThermostat(T0, 0.1)), 6000, rng=np.random.default_rng(3))
    temps = np.array(mb.values(s.loggers["t"]))[-400:]
    print(f"[Verlet + Andersen] <T> = {temps.mean():.2f} K (target {T0})")
    assert abs(temps.mean() - T0) < 0.03 * T0
    s.close()


def _free_system(n, box, mass, seed, restraint_k=None):
    rng = np.random.default_rng(seed)
    x = rng.uniform(0, box, (n, 3))
    atoms = mb.atoms_from_arrays(np.full(n, mass), np.zeros(n), np.full(n, 0.3), np.zeros(n), F64)  # eps = 0: no pair force
    s = mb.System(atoms=atoms, coords=x.copy(), velocities=np.zeros((n, 3)), boundary=mb.CubicBoundary(box),
                  pairwise_inters=(mb.LennardJones(cutoff=mb.DistanceCutoff(1.0)),), dtype=F64)
    if restraint_k is not None:
        s = mb.add_position_restraints(s, restraint_k)
    return s, x


def test_overdamped_free_diffusion():
    """Free particles: the displacement per component after n steps has variance 2 kT dt n / (m gamma). 3000 atoms x 3
    components: the sample variance has relative standard error sqrt(2 / 9000) = 1.5 %; the bound is 5 of those."""
    n, box, m, T, gamma, dt, steps = 3000, 30.0, 10.0, 300.0, 2.0, 0.002, 50
    s, x0 = _free_system(n, box, m, 1)
    mb.simulate(s, mb.OverdampedLangevin(dt=dt, temperature=T, friction=gamma, remove_CM_motion=0), steps,
                rng=np.random.default_rng(2))
    d = _cubic_vector(box)(x0, s.coords)
    var, expect = d.var(), 2 * KB * T * dt * steps / (m * gamma)
    print(f"[overdamped free] var {var:.5f} expected {expect:.5f}")
    assert abs(d.mean()) < 5 * math.sqrt(expect / d.size)
    assert abs(var / expect - 1) < 5 * math.sqrt(2 / d.size)
    s.close()


def test_overdamped_restraint_stationary_variance():
    """HarmonicPositionRestraint of constant k: Euler-Maruyama's stationary variance is exactly (kT/k) / (1 - k dt/(2 m gamma))
    (here 25 % above the continuous kT/k). Samples every 10 steps (correlation 0.6^10) over 20 calls, 60 000 values: the
    relative standard error of the variance is 0.6 %; the bound is 5 of those."""
    n, box, m, T, gamma, dt, k = 1000, 30.0, 1.0, 300.0, 1.0, 0.002, 200.0
    s, x0 = _free_system(n, box, m, 4, restraint_k=k)
    sim = mb.OverdampedLangevin(dt=dt, temperature=T, friction=gamma, remove_CM_motion=0)
    rng = np.random.default_rng(5)
    mb.simulate(s, sim, 50, rng=rng)
    samples = []
    for c in range(20):
        mb.simulate(s, sim, 10, init_step=50 + 10 * c, rng=rng)
        samples.append(_cubic_vector(box)(x0, s.coords))
    d = np.concatenate(samples)
    expect = (KB * T / k) / (1 - k * dt / (2 * m * gamma))
    print(f"[overdamped restraint] var {d.var():.6f} expected {expect:.6f} (continuous {KB * T / k:.6f})")
    assert abs(d.var() / expect - 1) < 5 * math.sqrt(2 / d.size)
    s.close()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("dtype", [F32, F64])
def test_loggers_are_observers(kind, dtype):
    x0, v0, _ = _run(kind, n=30, dtype=dtype)
    lg = {"v": mb.VelocitiesLogger(7), "x": mb.CoordinatesLogger(7), "ke": mb.KineticEnergyLogger(7)}
    x1, v1, _ = _run(kind, n=30, dtype=dtype, loggers=lg)
    assert np.array_equal(x0, x1) and np.array_equal(v0, v1)
    for j, step in enumerate(mb.record_steps(7, 30)):
        if step == 0:
            continue
        xs, vs, _ = _run(kind, n=step, dtype=dtype)
        assert np.array_equal(lg["v"].history[j], vs) and np.array_equal(lg["x"].history[j], xs)
        m = np.asarray(H.lj_fluid(6, seed=3, dtype=F64)["mass"], np.float64)[:, None]
        ke = 0.5 * float((m * vs.astype(np.float64) ** 2).sum())
        assert abs(lg["ke"].history[j] - ke) < 1e-6 * ke


def test_refusals_leave_coordinates_untouched():
    sd, s, _, _ = _readme()
    ctx = s.engine()
    L = s._L
    x, v = s.coords.copy(), s.velocities.copy()
    xp, vp = s.coords.ctypes.data, s.velocities.ctypes.data
    P, S, V = mb.capi.MBLangevinParams, mb.capi.MBStormerParams, mb.capi.MBVVParams
    bad_od = [P(0.0, 10, 0, 1, 2.0, 1.0), P(-0.002, 10, 0, 1, 2.0, 1.0), P(math.nan, 10, 0, 1, 2.0, 1.0),
              P(0.002, -1, 0, 1, 2.0, 1.0), P(0.002, 10, 0, 1, -2.0, 1.0), P(0.002, 10, 0, 1, math.nan, 1.0),
              P(0.002, 10, 0, 1, math.inf, 1.0), P(0.002, 10, 0, 1, 2.0, 0.0), P(0.002, 10, 0, 1, 2.0, -1.0),
              P(0.002, 10, 0, 1, 2.0, math.nan), P(0.002, 10, 0, 1, 2.0, math.inf)]
    calls = [(L.mb_simulate_overdamped_langevin, p) for p in bad_od]
    calls += [(L.mb_simulate_stormer_verlet, S(0.0, 10, 0)), (L.mb_simulate_stormer_verlet, S(math.nan, 10, 0)),
              (L.mb_simulate_stormer_verlet, S(0.002, -1, 0)), (L.mb_simulate_verlet, V(0.0, 10, 0, 1)),
              (L.mb_simulate_verlet, V(0.002, -1, 0, 1))]
    for fn, p in calls:
        assert fn(ctx, xp, vp, C.byref(p), None) == mb.capi.MB_ERR_INVALID
        assert np.array_equal(x, s.coords) and np.array_equal(v, s.velocities)
    for fn in (L.mb_simulate_verlet, L.mb_simulate_stormer_verlet, L.mb_simulate_overdamped_langevin):
        assert fn(ctx, xp, vp, None, None) == mb.capi.MB_ERR_INVALID
    assert L.mb_simulate_overdamped_langevin(ctx, xp, vp, C.byref(P(0.002, 10, 0, 1, 2.0, 0.0)), None) == mb.capi.MB_ERR_INVALID
    assert b"mb_simulate_overdamped_langevin" in L.mb_last_error() and b"friction" in L.mb_last_error()
    # a velocity coupling set on the context
    assert L.mb_set_velocity_coupling(ctx, C.byref(mb.capi.MBVCoupling(mb.capi.MB_VC_BERENDSEN, 0, 2.0, 0.1))) == 0
    good = [(L.mb_simulate_verlet, V(0.002, 10, 0, 1, 2.0, 0.01, 1, 2)), (L.mb_simulate_stormer_verlet, S(0.002, 10, 0)),
            (L.mb_simulate_overdamped_langevin, P(0.002, 10, 0, 1, 2.0, 1.0))]
    for fn, p in good:
        assert fn(ctx, xp, vp, C.byref(p), None) == mb.capi.MB_ERR_INVALID
        assert b"velocity coupling" in L.mb_last_error()
        assert np.array_equal(x, s.coords) and np.array_equal(v, s.velocities)
    mb.simulate(s, mb.Verlet(0.002), 5)  # simulate clears the coupling: the run goes through
    s.close()


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
    sd = H.lj_fluid(10, seed=9, dtype=F64, temp=120.0)
    atoms = mb.atoms_from_arrays(sd["mass"], sd["charge"], sd["sigma"], sd["eps"], F64)
    s = mb.System(atoms=atoms, coords=sd["coords"].copy(), boundary=mb.CubicBoundary(*sd["box"]),
                  velocities=sd["velocities"].copy(), pairwise_inters=(mb.LennardJones(cutoff=mb.ShiftedForceCutoff(1.0),
                                                                                        use_neighbors=True),),
                  neighbor_finder=mb.GPUNeighborFinder(dist_cutoff=1.15, n_steps=20), dtype=F64, device=rank)
    s.engine()
    uid = [mb.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    mb.comm_init(s, uid[0], rank, world)
    x0, out = s.coords.copy(), []
    for sim in (mb.Verlet(0.002), mb.StormerVerlet(0.002), mb.OverdampedLangevin(0.002, 100.0, 5.0)):
        try:
            mb.simulate(s, sim, 5)
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


def _verlet_protocol(dtype, sims):
    """test/simulation.jl:440-508 ("Verlet integrators on CPU and GPU"): 100 atoms (m 10, sigma 0.1 nm, eps 0.2 kJ/mol) in a
    4 nm box at least 0.2 nm apart, velocities at 298 K scaled by 0.01, LennardJones on neighbour lists with a 2 nm cutoff;
    1000 steps of each simulator in `sims`, one after the other, by the engine in `dtype` and by the f64 oracle. Returns the
    mean and largest |coordinate difference| (nm) and |energy difference| (kJ/mol) after every one."""
    from oracle import oracle as o
    n, box, T = 100, 4.0, 298.0
    sd = H.readme_system(n, box, seed=8, min_dist=0.2)
    rng = np.random.default_rng(9)
    sd = dict(sd, mass=np.full(n, 10.0), charge=np.zeros(n), sigma=np.full(n, 0.1), eps=np.full(n, 0.2),
              velocities=rng.normal(0.0, math.sqrt(KB * T / 10.0), (n, 3)) * 0.01)
    orc = H.make_oracle(sd, [o.Inter(o.LJ, o.CUT_DISTANCE, 2.0, use_neighbors=True)])
    fe = lambda x: orc.forces_allpairs(x, energy=False)[0]  # noqa: E731
    s = H.make_system(sd, (mb.LennardJones(cutoff=mb.DistanceCutoff(2.0)),), dtype)
    wrap, vec = _box_wrap(sd["box"]), _cubic_vector(np.asarray(sd["box"], np.float64))
    x, v, step, out = sd["coords"], sd["velocities"], 0, []
    for sim in sims:
        if isinstance(sim, mb.VelocityVerlet):
            x, v = vo.simulate_velocity_verlet(fe, x, v, sd["mass"], 0.002, 1000, wrap, remove_cm_every=1, init_step=step)
        elif isinstance(sim, mb.Verlet):
            x, v = vo.simulate_verlet(fe, x, v, sd["mass"], 0.002, 1000, wrap, init_step=step)
        else:
            x, v = vo.simulate_stormer_verlet(fe, x, v, sd["mass"], 0.002, 1000, wrap, vec, init_step=step)
        mb.simulate(s, sim, 1000, init_step=step)
        step += 1000
        d = np.abs(vec(x, s.coords.astype(np.float64)))
        out.append((d.sum() / (3 * n), d.max(), abs(mb.potential_energy(s) - orc.forces_allpairs(x)[1])))
        print(f"[simulation.jl Verlet integrators {np.dtype(dtype).name}] {type(sim).__name__}: mean |dx| {out[-1][0]:.3e} nm, "
              f"max |dx| {out[-1][1]:.3e} nm, |dE| {out[-1][2]:.3e} kJ/mol")
    s.close()
    return out


REFERENCE_SEQUENCE = (mb.VelocityVerlet(dt=0.002), mb.Verlet(dt=0.002), mb.StormerVerlet(dt=0.002))


def test_reference_verlet_integrators_protocol():
    """The reference's sequence in f64, the precision its CPU and GPU systems run it in: mean |coordinate difference|
    < 1e-4 nm and |energy difference| < 5e-4 kJ/mol after every integrator."""
    for dx, _, de in _verlet_protocol(F64, REFERENCE_SEQUENCE):
        assert dx < 1e-4 and de < 5e-4


def test_reference_verlet_integrators_protocol_f32():
    """The same sequence in f32 against the f64 oracle: the mean coordinate difference stays under the reference's 1e-4 nm
    after every integrator (measured 1.8e-5, 3.2e-5, 6.4e-5 nm). The energy bar of 5e-4 kJ/mol holds after the first two
    1000-step stages only. The f32 and f64 trajectories drift apart with time, and atoms near the steep LJ wall (sigma
    0.1 nm) turn a few 1e-4 nm of it into energy: after 3000 steps the StormerVerlet stage is 1.0e-2 kJ/mol off, and
    VelocityVerlet or Verlet run alone for 3000 steps miss the bar too (1.1e-3, 8.9e-4), while StormerVerlet alone meets it
    (1.6e-4). So the third stage is held to the coordinate bar."""
    out = _verlet_protocol(F32, REFERENCE_SEQUENCE)
    for dx, _, _ in out:
        assert dx < 1e-4
    for _, _, de in out[:2]:
        assert de < 5e-4


def test_reference_lennard_jones_simulators():
    """test/simulation.jl:388-437 ("Lennard-Jones simulators"): 100 atoms (m 10, sigma 0.3 nm, eps 0.2 kJ/mol) in a 2 nm box,
    velocities at 298 K, CoordinatesLogger(100); Verlet + Andersen(298 K, 10 ps), StormerVerlet, Langevin(1 ps^-1) and
    OverdampedLangevin(10 ps^-1), 20 000 steps of 2 fs each in turn, in f32. The state stays finite and in the box."""
    n, box, T = 100, 2.0, 298.0
    sd = H.readme_system(n, box, seed=2, min_dist=0.3)
    atoms = mb.atoms_from_arrays(np.full(n, 10.0), np.zeros(n), np.full(n, 0.3), np.full(n, 0.2), F32)
    s = mb.System(atoms=atoms, coords=sd["coords"].astype(F32), boundary=mb.CubicBoundary(box),
                  pairwise_inters=(mb.LennardJones(),), dtype=F32, loggers={"x": mb.CoordinatesLogger(100)})
    s.velocities[...] = mb.random_velocities(s, T, rng=np.random.default_rng(3))
    sims = [mb.Verlet(dt=0.002, coupling=(mb.AndersenThermostat(T, 10.0),)), mb.StormerVerlet(dt=0.002),
            mb.Langevin(dt=0.002, temperature=T, friction=1.0), mb.OverdampedLangevin(dt=0.002, temperature=T, friction=10.0)]
    for sim in sims:
        mb.simulate(s, sim, 20_000)
        assert np.isfinite(s.coords).all() and np.isfinite(s.velocities).all()
        assert (s.coords >= 0).all() and (s.coords <= box).all()
        print(f"[simulation.jl LJ simulators] {type(sim).__name__}: T = {mb.temperature(s):.1f} K")
    assert len(s.loggers["x"].history) == 4 * 201
    s.close()
