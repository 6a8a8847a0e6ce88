"""GPU tests of LangevinSplitting (src/simulators.jl:1212-1398): f64 trajectory parity with the numpy restatement of the
reference loop (tests/langevin_splitting_oracle.py) for six splittings on the all-pairs, brick, bonded, triclinic, PME and
implicit-solvent systems; remove_CM_motion x init_step and chunked calls; "BAB" = VelocityVerlet and the reference's
"Langevin splitting" testset (BAOA = Langevin); the force evaluations per step (host counter and profiler, graph and stream
paths); the O step's exact moments and canonical K for BAOAB; the determinism and observer properties of the step graph;
and the refusals."""
import ctypes as C
import math

import numpy as np
import pytest

import langevin_splitting_oracle as so
import mbhelpers as H
import mollyb200 as mb
import thermostat_oracle as tho
from oracle import oracle as o
from test_gpu_langevin import _lj_brick, _molecular, _readme
from test_gpu_parity import _pos_err

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
KB = mb.BOLTZMANN_K
SPLITTINGS = ["BAOAB", "OBABO", "ABOBA", "BAOA", "BABAB", "AB"]


def _keys(seed):
    r = np.random.default_rng(seed)
    return tho.rng_words(int(r.integers(0, 2 ** 63)), int(r.integers(0, 2 ** 63)))


def _box_wrap(box):
    return lambda x: x - np.floor(x / box) * box


def _lj_small_skin():
    """864 argon atoms on the brick path with a 0.01 nm skin at 300 K: rebuilds fall inside the run, also between the two
    evaluations of a BABAB step."""
    sd = H.lj_fluid(6, seed=3, dtype=F64, temp=300.0)
    s = H.make_system(sd, (mb.LennardJones(cutoff=mb.ShiftedForceCutoff(0.9), use_neighbors=True),), F64, r_list=0.91)
    orc = H.make_oracle(sd, [o.Inter(o.LJ, o.CUT_SHIFTED_FORCE, 0.9, use_neighbors=True)])
    return sd, s, lambda x: orc.forces_allpairs(x, energy=False)[0], 1


def _sixmrr(g):
    s = H.sixmrr_system(g, F64, r_list=1.05)
    orc, sd = H.sixmrr_oracle(g)
    return sd, s, lambda x: orc.forces_nl(x, orc.neighbor_list(x, 1.05), energy=False)[0] + H.bonded_forces_oracle(g, x)[0], 1


SYSTEMS = {"readme-allpairs": _readme, "lj-small-skin": _lj_small_skin, "molecular-brick": _molecular}


def _parity(sd, s, fe, path, splitting, T=120.0, friction=10.0, rcm=1, init_step=0, n=30, dt=0.002, wrap=None, seed=7,
            label=""):
    sim = mb.LangevinSplitting(dt=dt, temperature=T, friction=friction, splitting=splitting, remove_CM_motion=rcm)
    x_ref, v_ref = so.simulate_splitting(fe, sd["coords"], sd["velocities"], sd["mass"], dt, n, KB * T, friction, splitting,
                                         _keys(seed), wrap or _box_wrap(sd["box"]), remove_cm_every=rcm, init_step=init_step)
    rb0 = s.stats()["n_rebuilds"] if s._ctx is not None else 0
    mb.simulate(s, sim, n, init_step=init_step, rng=np.random.default_rng(seed))
    st = s.stats()
    ex = _pos_err(s.coords, x_ref, sd["box"]) if wrap is None else np.abs(s.coords - x_ref).max()
    ev = np.abs(s.velocities - v_ref).max()
    print(f"[{splitting} {label} rcm={rcm} init={init_step} path={st['path']} graph={st['graph_mode']} "
          f"rebuilds={st['n_rebuilds'] - rb0}] dx={ex:.3e} dv={ev:.3e}")
    assert path is None or st["path"] == path
    assert ex < 1e-9 and ev < 1e-8
    return st, st["n_rebuilds"] - rb0


@pytest.mark.parametrize("splitting", SPLITTINGS)
@pytest.mark.parametrize("name", list(SYSTEMS))
def test_parity_f64(name, splitting):
    sd, s, fe, path = SYSTEMS[name]()
    st, rebuilds = _parity(sd, s, fe, path, splitting, T=300.0 if name != "molecular-brick" else 120.0, label=name)
    assert st["graph_mode"] == 1
    if name == "lj-small-skin":
        assert rebuilds > 2
    s.close()


@pytest.mark.parametrize("splitting", SPLITTINGS)
def test_parity_6mrr_bonded(golden_6mrr, splitting):
    sd, s, fe, path = _sixmrr(golden_6mrr)
    _parity(sd, s, fe, path, splitting, T=300.0, n=15, label="6mrr")
    s.close()


@pytest.mark.parametrize("splitting", ["BAOAB", "BABAB"])
def test_parity_triclinic_allpairs(splitting):
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
    _parity(sd, s, lambda y: tri.forces_energy(t, y, sig, eps, r_cut=1.2)[0], 0, splitting, wrap=wrap, label="triclinic")
    d = np.array([t.vector(a, b) for a, b in zip(s.coords, wrap(s.coords))])
    assert np.abs(d).max() < 1e-12
    s.close()


@pytest.mark.parametrize("splitting", ["BAOAB", "BABAB"])
def test_parity_6mrr_pme_stream_path(golden_6mrr, splitting):
    from oracle import pme
    g = golden_6mrr
    s = H.sixmrr_pme_system(g, F64)
    sd = H.sixmrr_description(g)
    alpha = pme.pme_alpha(1.0)
    orc = H.make_oracle(sd, [o.Inter(o.LJ, o.CUT_DISTANCE, 1.0, weight_special=float(g["lj14scale"]), use_neighbors=True),
                             o.Inter(o.EWALD_REAL, o.CUT_DISTANCE, 1.0, weight_special=float(g["coulomb14scale"]), ewald_alpha=alpha,
                                     use_neighbors=True)])
    excl = np.concatenate([g["excluded"], g["special"]])

    def fe(x):
        f = orc.forces_nl(x, orc.neighbor_list(x, 1.2), energy=False)[0] + H.bonded_forces_oracle(g, x)[0]
        return f + pme.pme_reciprocal(x, g["charge"], sd["box"], r_cut=1.0, error_tol=0.0005, order=5)[0] + \
            pme.ewald_exclusion(x, g["charge"], sd["box"], excl)[0]
    st, _ = _parity(sd, s, fe, 1, splitting, T=300.0, n=8, label="6mrr+PME")
    assert st["graph_mode"] == 0
    s.close()


def test_parity_implicit_solvent():
    import os

    from test_gpu_implicit_solvent import ROOT, _full_oracle, _full_system
    g = np.load(os.path.join(ROOT, "tests", "golden", "6mrr_gb.npz"))
    v0 = np.random.default_rng(11).normal(0, 0.3, g["coords"].shape)
    s = _full_system(g, "gbn2", F64, velocities=v0)
    sd = dict(coords=g["coords"], velocities=v0, mass=g["mass"], box=np.asarray(g["box"], np.float64))
    st, _ = _parity(sd, s, _full_oracle(g, "gbn2"), None, "BAOAB", T=300.0, n=10, dt=0.001, label="gbn2")
    assert st["graph_mode"] == 1
    s.close()


@pytest.mark.parametrize("rcm,init_step", [(0, 0), (1, 0), (3, 0), (0, 13), (1, 13), (3, 13)])
def test_parity_remove_cm_and_init_step(rcm, init_step):
    sd, s, fe, path = _readme()
    _parity(sd, s, fe, path, "BAOAB", T=300.0, rcm=rcm, init_step=init_step)
    s.close()


@pytest.mark.parametrize("splitting", ["BAOAB", "BAOA", "BABAB"])
def test_chunked_calls_equal_one_call(splitting):
    """simulate(25) then simulate(25; init_step=25) == simulate(50) with the same keys: the draws are a function of (keys,
    step, j, atom), and a recomputing B at the top of a step is served by the same positions either way."""
    sim = mb.LangevinSplitting(dt=0.002, temperature=120.0, friction=20.0, splitting=splitting)
    sd, a, _, _ = _lj_brick()
    _, b, _, _ = _lj_brick()
    mb.simulate(a, sim, 50, rng=np.random.default_rng(1))
    mb.simulate(b, sim, 25, rng=np.random.default_rng(1))
    mb.simulate(b, sim, 25, init_step=25, rng=np.random.default_rng(1))
    assert _pos_err(a.coords, b.coords, sd["box"]) < 1e-9
    assert np.abs(a.velocities - b.velocities).max() < 1e-8
    a.close(); b.close()


def test_bab_is_velocity_verlet_lj(golden_6mrr):
    for make in (_lj_brick, lambda: _sixmrr(golden_6mrr)):
        sd, a, _, _ = make()
        _, b, _, _ = make()
        mb.simulate(a, mb.LangevinSplitting(0.002, 300.0, 10.0, "BAB"), 30, rng=np.random.default_rng(4))
        mb.simulate(b, mb.VelocityVerlet(0.002), 30)
        dx, dv = _pos_err(a.coords, b.coords, sd["box"]), np.abs(a.velocities - b.velocities).max()
        print(f"[BAB vs VelocityVerlet] dx={dx:.2e} dv={dv:.2e}")
        assert dx < 1e-10
        a.close(); b.close()


def _reference_testset(dtype):
    """test/simulation.jl:770-803: 400 atoms of 10 g/mol in a 10 nm box, velocities 0.01 x Maxwell-Boltzmann at 300 K, LJ on
    a neighbour list (cut at 1 nm as in test_gpu_langevin's protocol), TemperatureLogger(10), 2000 steps of 2 fs; Langevin
    with friction 1 ps^-1 and "BAOA" with friction 10 g mol^-1 ps^-1 from the same generator seed."""
    n, box = 400, 10.0
    sd = H.readme_system(n, box, seed=9, min_dist=0.3)
    v = np.random.default_rng(5).normal(0, math.sqrt(KB * 300.0 / 10.0), (n, 3)) * 0.01
    out = []
    for sim in (mb.Langevin(dt=0.002, temperature=300.0, friction=1.0),
                mb.LangevinSplitting(dt=0.002, temperature=300.0, friction=10.0, splitting="BAOA")):
        atoms = mb.atoms_from_arrays(np.full(n, 10.0), np.zeros(n), np.full(n, 0.3), np.full(n, 0.2), dtype)
        s = mb.System(atoms=atoms, coords=sd["coords"].astype(dtype), velocities=v.astype(dtype), boundary=mb.CubicBoundary(box),
                      pairwise_inters=(mb.LennardJones(cutoff=mb.DistanceCutoff(1.0), use_neighbors=True),),
                      neighbor_finder=mb.GPUNeighborFinder(dist_cutoff=1.2), dtype=dtype,
                      loggers={"temp": mb.TemperatureLogger(10)})
        mb.simulate(s, sim, 2000, rng=np.random.default_rng(2022))
        temps = np.array(mb.values(s.loggers["temp"]))
        out.append((s.coords.astype(np.float64).copy(), temps[-101:].mean()))
        s.close()
    return out, box


@pytest.mark.parametrize("dtype", [F32, F64])
def test_reference_langevin_splitting_testset(dtype):
    ((xa, ta), (xb, tb)), box = _reference_testset(dtype)
    dx = _pos_err(xa, xb, np.full(3, box))
    print(f"[simulation.jl Langevin splitting {np.dtype(dtype).name}] <T> Langevin {ta:.2f} K, BAOA {tb:.2f} K, max|dx| {dx:.2e} nm")
    assert 280.0 <= ta <= 320.0 and 280.0 <= tb <= 320.0
    if dtype == F64:
        assert dx < 1e-5


@pytest.mark.parametrize("no_graph", ["0", "1"])
@pytest.mark.parametrize("splitting", ["BAOAB", "BAOA", "BABAB", "O"])
def test_force_evaluations_per_step(monkeypatch, no_graph, splitting):
    """Unlogged: n_force_evals grows by n_steps x the reference's evaluations per step plus F0, and the profiler sees as many
    pair-kernel launches."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    monkeypatch.setenv("MOLLYB200_NO_GRAPH", no_graph)
    _, s, _, _ = _lj_brick()
    sim = mb.LangevinSplitting(0.002, 120.0, 10.0, splitting)
    mb.simulate(s, sim, 4)  # (first build and graph capture outside the window)
    n = 12
    ev0 = s.stats()["n_force_evals"]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        mb.simulate(s, sim, n)
        torch.cuda.synchronize()
    st = s.stats()
    pair = sum(1 for e in prof.events() if "brick_force_kernel<" in e.name)
    want = n * so.evaluations_per_step(splitting) + 1
    print(f"[{splitting} graph={st['graph_mode']}] force evals +{st['n_force_evals'] - ev0}, pair kernels {pair}, want {want}")
    assert st["graph_mode"] == (0 if no_graph == "1" else 1)
    assert st["n_force_evals"] - ev0 == want and pair == want
    s.close()


@pytest.mark.parametrize("dtype", [F32, F64])
def test_o_step_statistics_free_particles(dtype):
    """Splitting "O", all eps = 0 (F = 0): every velocity component is v_n = c_i v_{n-1} + sigma_i xi with
    c_i = exp(-friction dt / m_i), so E[v_n] = c_i^n v0 and Var[v_n] = (kT / m_i)(1 - c_i^(2n)). Four mass groups pin the
    mass-per-time friction; massless atoms keep their velocity. 5-standard-error bars."""
    n_grp, masses = 6000, [1.0, 12.0, 39.948, 200.0]
    n = n_grp * len(masses) + 50
    mass = np.concatenate([np.full(n_grp, m) for m in masses] + [np.zeros(50)])
    rng = np.random.default_rng(4)
    x = rng.random((n, 3)) * 10.0
    v0 = np.tile(np.array([0.7, -0.3, 0.2]), (n, 1))
    T, fr, dt = 300.0, 60.0, 0.004
    kT = KB * T
    atoms = mb.atoms_from_arrays(mass, np.zeros(n), np.full(n, 0.3), np.zeros(n), dtype)
    s = mb.System(atoms=atoms, coords=x.astype(dtype), velocities=v0.astype(dtype), boundary=mb.CubicBoundary(10.0),
                  pairwise_inters=(mb.LennardJones(),), dtype=dtype)
    sim = mb.LangevinSplitting(dt, T, fr, "O", remove_CM_motion=0)
    done = 0
    for k in (1, 10, 60):
        mb.simulate(s, sim, k - done, init_step=done, rng=np.random.default_rng(11))
        done = k
        v = s.velocities.astype(np.float64)
        for gi, m in enumerate(masses):
            c = math.exp(-fr * dt / m)
            vg = v[gi * n_grp:(gi + 1) * n_grp] - c ** k * v0[0]
            var = kT / m * (1 - c ** (2 * k))
            N = vg.size
            assert abs(vg.mean()) < 5 * math.sqrt(var / N), (k, m)
            assert abs(vg.var() / var - 1) < 5 * math.sqrt(2 / N), (k, m)
        np.testing.assert_array_equal(v[-50:], np.tile(v0[0].astype(dtype).astype(np.float64), (50, 1)))
        assert np.array_equal(s.coords, x.astype(dtype))
    s.close()


def test_canonical_kinetic_energy_baoab():
    """2916 argon atoms at 90 K under BAOAB, friction 200 g mol^-1 ps^-1 (5 ps^-1 for argon). <K> = Nf kT / 2 and
    Var(K) = Nf (kT)^2 / 2 with Nf = 3N - 3; blocks of 50 records every 10 steps; 4-sigma bars."""
    sd = H.lj_fluid(9, seed=21, dtype=F64, temp=90.0)
    s = H.make_system(sd, (mb.LennardJones(cutoff=mb.ShiftedForceCutoff(1.0), use_neighbors=True),), F64, r_list=1.2)
    s.loggers = {"ke": mb.KineticEnergyLogger(10)}
    T0 = 90.0
    mb.simulate(s, mb.LangevinSplitting(dt=0.002, temperature=T0, friction=200.0, splitting="BAOAB"), 21_000,
                rng=np.random.default_rng(8))
    ke = np.array(s.loggers["ke"].history[101:])
    nf = 3 * sd["n"] - 3
    kbar = nf * KB * T0 / 2
    nb = len(ke) // 50
    blocks = ke[:nb * 50].reshape(nb, 50)
    mean, se_mean = blocks.mean(), blocks.mean(1).std(ddof=1) / math.sqrt(nb)
    dev2 = (blocks - mean) ** 2
    ratio = dev2.mean() / (2 * kbar * kbar / nf)
    se_ratio = dev2.mean(1).std(ddof=1) / math.sqrt(nb) / (2 * kbar * kbar / nf)
    print(f"[BAOAB canonical] <K>/Kbar-1={mean / kbar - 1:.2e} (se {se_mean / kbar:.1e}); Var ratio={ratio:.3f} (se {se_ratio:.3f})")
    assert abs(mean - kbar) < 4 * se_mean + 2e-3 * kbar
    assert abs(ratio - 1) < 4 * se_ratio + 0.02
    s.close()


def _run(seed, splitting="BAOAB", friction=20.0, n=40, loggers=None, dtype=F64, device=False):
    sd, s, _, _ = _lj_brick()
    if dtype != F64:
        s = H.make_system(sd, (mb.LennardJones(cutoff=mb.ShiftedForceCutoff(0.9), use_neighbors=True),), dtype, r_list=0.92)
    if loggers:
        s.loggers = loggers
    if device:
        import torch
        s.coords = torch.from_numpy(s.coords).cuda()
        s.velocities = torch.from_numpy(s.velocities).cuda()
    mb.simulate(s, mb.LangevinSplitting(0.002, 120.0, friction, splitting), n, rng=np.random.default_rng(seed))
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


@pytest.mark.parametrize("splitting", ["BAOAB", "OBABO", "BABAB", "ABOBA"])
def test_graph_and_stream_paths_bit_identical(monkeypatch, splitting):
    res = []
    for no_graph in ("0", "1"):
        monkeypatch.setenv("MOLLYB200_NO_GRAPH", no_graph)
        lg = {"ke": mb.KineticEnergyLogger(5), "pe": mb.PotentialEnergyLogger(5)}
        x, v, g = _run(2, splitting=splitting, loggers=lg)
        res.append((x, v, list(lg["ke"].history), list(lg["pe"].history), g))
    (xa, va, ka, pa, ga), (xb, vb, kb, pb, gb) = res
    assert (ga, gb) == (1, 0)
    assert np.array_equal(xa, xb) and np.array_equal(va, vb) and ka == kb and pa == pb


def test_host_and_device_buffers_identical():
    a, b = _run(6), _run(6, device=True)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


@pytest.mark.parametrize("dtype", [F32, F64])
def test_loggers_are_observers(dtype):
    x0, v0, _ = _run(4, n=30, dtype=dtype)
    lg = {"v": mb.VelocitiesLogger(7), "pe": mb.PotentialEnergyLogger(7), "x": mb.CoordinatesLogger(10)}
    x1, v1, _ = _run(4, n=30, loggers=lg, dtype=dtype)
    assert np.array_equal(x0, x1) and np.array_equal(v0, v1)
    for k, step in enumerate(mb.record_steps(7, 30)):
        if step == 0:
            continue
        xs, vs, _ = _run(4, n=step, dtype=dtype)
        assert np.array_equal(lg["v"].history[k], vs)
        sd, s, _, _ = _lj_brick()
        ref = H.make_system(dict(sd, coords=xs, velocities=vs), s.pairwise_inters, dtype, r_list=0.92)
        s.close()
        pe = mb.potential_energy(ref)
        ref.close()
        assert abs(lg["pe"].history[k] - pe) < (1e-5 if dtype == F32 else 1e-10) * abs(pe)


def test_refusals_leave_coordinates_untouched():
    sd, s, _, _ = _readme()
    ctx = s.engine()
    L = s._L
    x, v = s.coords.copy(), s.velocities.copy()

    def P(dt=0.002, n=10, kT=2.0, fr=1.0, ops=b"BAOAB", n_ops=None):
        return mb.capi.MBSplittingParams(dt, n, 0, 1, kT, fr, 1, 2, len(ops) if n_ops is None else n_ops, ops)
    bad = [P(dt=0.0), P(dt=-0.002), P(n=-1), P(kT=-2.0), P(kT=math.nan), P(kT=math.inf), P(fr=-1.0), P(fr=math.nan),
           P(fr=math.inf), P(ops=b""), P(ops=b"BAXAB"), P(ops=b"baoab"), P(ops=b"BAOAB", n_ops=33), P(ops=b"BAOAB", n_ops=-1)]
    for p in bad:
        assert L.mb_simulate_langevin_splitting(ctx, s.coords.ctypes.data, s.velocities.ctypes.data, C.byref(p), None) == mb.capi.MB_ERR_INVALID
        assert np.array_equal(x, s.coords) and np.array_equal(v, s.velocities)
    assert L.mb_set_velocity_coupling(ctx, C.byref(mb.capi.MBVCoupling(mb.capi.MB_VC_IMMEDIATE, 0, 2.0, 0.0))) == 0
    p = P()
    assert L.mb_simulate_langevin_splitting(ctx, s.coords.ctypes.data, s.velocities.ctypes.data, C.byref(p), None) == mb.capi.MB_ERR_INVALID
    assert b"velocity coupling" in L.mb_last_error()
    assert np.array_equal(x, s.coords) and np.array_equal(v, s.velocities)
    mb.simulate(s, mb.LangevinSplitting(0.002, 300.0, 10.0, "BAOAB"), 5)  # (simulate clears it)
    s.close()


def test_velocity_verlet_after_langevin_splitting_equals_fresh_system():
    sd, s, _, _ = _lj_brick()
    mb.simulate(s, mb.LangevinSplitting(0.002, 120.0, 20.0, "BABAB"), 20, rng=np.random.default_rng(3))
    ref = H.make_system(dict(sd, coords=s.coords.copy(), velocities=s.velocities.copy()), s.pairwise_inters, F64, r_list=0.92)
    mb.simulate(s, mb.VelocityVerlet(dt=0.002), 30, init_step=20)
    mb.simulate(ref, mb.VelocityVerlet(dt=0.002), 30, init_step=20)
    assert _pos_err(s.coords, ref.coords, sd["box"]) < 1e-12
    assert np.abs(s.velocities - ref.velocities).max() < 1e-12
    s.close(); ref.close()
