"""GPU tests of the velocity-rescaling thermostats inside the VelocityVerlet step (ImmediateThermostat, BerendsenThermostat,
VelocityRescaleThermostat; src/coupling.jl:82-168, :227-238): trajectory parity with the numpy restatement of the reference
loop (tests/thermostat_oracle.py) on the all-pairs and brick paths, the reference's test/coupling.jl protocol, canonical
sampling of the kinetic energy by the Bussi thermostat, and the observer / determinism properties of the step graph."""
import ctypes as C
import math

import numpy as np
import pytest

import mbhelpers as H
import mollyb200 as mb
import thermostat_oracle as tho
from oracle import oracle as o
from test_gpu_parity import _pos_err

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
KB = mb.BOLTZMANN_K
THERMOSTATS = {
    "immediate": lambda: mb.ImmediateThermostat(300.0),
    "berendsen": lambda: mb.BerendsenThermostat(250.0, 0.05),
    "bussi": lambda: mb.VelocityRescaleThermostat(350.0, 0.05),
    "bussi5": lambda: mb.VelocityRescaleThermostat(350.0, 0.05, n_steps=5),
}


def _keys(seed):
    """The (rng_ctr1, rng_key) simulate(..., rng=np.random.default_rng(seed)) passes to the engine."""
    r = np.random.default_rng(seed)
    return tho.rng_words(int(r.integers(0, 2 ** 63)), int(r.integers(0, 2 ** 63)))


def _readme():
    sd = H.readme_system(100, 2.0, seed=1)
    return sd, H.make_system(sd, (mb.LennardJones(),), F64), H.make_oracle(sd, [o.Inter(o.LJ)])


def _lj_exceptions(dtype=F64, seed=3):
    """864 argon atoms on the brick path, with excluded and special (weight 0.5) pairs between near neighbours."""
    sd = H.lj_fluid(6, seed=seed, dtype=F64)
    hubs = np.arange(0, sd["n"], 9)
    excl = [(int(h), int(j)) for h in hubs for j in H.nearest_partners(sd, h, 2)]
    excluded = {frozenset(p) for p in excl}
    spec = [(int(h), int(j)) for h in hubs[::2] for j in H.nearest_partners(sd, h, 4) if frozenset((h, j)) not in excluded]
    sd["excluded"], sd["special"] = np.array(excl, np.int32), np.array(spec, np.int32)
    s = H.make_system(sd, (mb.LennardJones(cutoff=mb.ShiftedForceCutoff(0.9), use_neighbors=True, weight_special=0.5),),
                      dtype, r_list=1.0)
    orc = H.make_oracle(sd, [o.Inter(o.LJ, o.CUT_SHIFTED_FORCE, 0.9, weight_special=0.5, use_neighbors=True)])
    return sd, s, orc


def _parity(sd, s, orc, th, rcm, init_step=0, n=100, dt=0.002, path=None):
    x_ref, v_ref = tho.simulate_vv_coupled(orc, sd["coords"], sd["velocities"], sd["mass"], sd["box"], dt, n, th, KB, _keys(7),
                                           remove_cm_every=rcm, init_step=init_step)
    mb.simulate(s, mb.VelocityVerlet(dt=dt, coupling=th, remove_CM_motion=rcm), n, init_step=init_step, rng=np.random.default_rng(7))
    st = s.stats()
    ex, ev = _pos_err(s.coords, x_ref, sd["box"]), np.abs(s.velocities - v_ref).max()
    print(f"[{type(th).__name__} rcm={rcm} init={init_step} path={st['path']} graph={st['graph_mode']}] dx={ex:.3e} dv={ev:.3e}")
    if path is not None:
        assert st["path"] == path
    # the bars of test_vv_readme_allpairs_f64 / test_vv_chunked_equals_single_call
    assert ex < 1e-9 and ev < 1e-8
    s.close()


@pytest.mark.parametrize("rcm", [0, 1, 3])
@pytest.mark.parametrize("name", list(THERMOSTATS))
def test_parity_allpairs_f64(name, rcm):
    sd, s, orc = _readme()
    _parity(sd, s, orc, THERMOSTATS[name](), rcm, path=0)


@pytest.mark.parametrize("name,rcm", [("immediate", 1), ("berendsen", 1), ("bussi", 1), ("bussi5", 3), ("berendsen", 0)])
def test_parity_brick_exceptions_f64(name, rcm):
    sd, s, orc = _lj_exceptions()
    th = {"immediate": mb.ImmediateThermostat(120.0), "berendsen": mb.BerendsenThermostat(120.0, 0.05),
          "bussi": mb.VelocityRescaleThermostat(120.0, 0.05), "bussi5": mb.VelocityRescaleThermostat(120.0, 0.05, n_steps=5)}[name]
    _parity(sd, s, orc, th, rcm, path=1)


@pytest.mark.parametrize("name", ["berendsen", "bussi5"])
def test_parity_nonzero_init_step(name):
    sd, s, orc = _readme()
    _parity(sd, s, orc, THERMOSTATS[name](), 1, init_step=13)


@pytest.mark.parametrize("rcm", [0, 1])
def test_kinetic_energy_after_cm_removal(rcm):
    """K after the step's CM removal (K2's sum with the CM correction) against numpy's removal-then-sum: the Immediate
    thermostat rescales to exactly Nf k T0 / 2 by that K, so the logged KE / (Nf k T0 / 2) = K_numpy / K_engine."""
    sd = H.readme_system(100, 2.0, seed=1)
    v = sd["velocities"] + np.array([0.3, -0.2, 0.1])  # a CM velocity for the correction to remove
    s = H.make_system(dict(sd, velocities=v), (mb.LennardJones(),), F64)
    s.loggers = {"ke": mb.KineticEnergyLogger(1)}
    mb.simulate(s, mb.VelocityVerlet(dt=0.002, coupling=mb.ImmediateThermostat(300.0), remove_CM_motion=rcm), 20)
    kbar = (3 * 100 - 3) * KB * 300.0 / 2
    ke = np.array(s.loggers["ke"].history[1:])
    print(f"[K after CM removal rcm={rcm}] max |KE/Kbar - 1| = {np.abs(ke / kbar - 1).max():.3e}")
    assert np.abs(ke / kbar - 1).max() < 1e-11
    s.close()


def _protocol_system(dtype, seed):
    # test/coupling.jl: 100 atoms of mass 10, sigma 0.04 nm, eps 0.1 kJ/mol, 4 nm box, LJ with DistanceCutoff(1 nm)
    sd = H.readme_system(100, 4.0, seed=seed, min_dist=0.1)
    sd["sigma"], sd["eps"] = np.full(100, 0.04), np.full(100, 0.1)
    atoms = mb.atoms_from_arrays(sd["mass"], sd["charge"], sd["sigma"], sd["eps"], dtype)
    return mb.System(atoms=atoms, coords=sd["coords"].astype(dtype), boundary=mb.CubicBoundary(4.0),
                     pairwise_inters=(mb.LennardJones(cutoff=mb.DistanceCutoff(1.0)),), dtype=dtype,
                     loggers={"temperature": mb.TemperatureLogger(10)})


@pytest.mark.parametrize("dtype", [F32, F64])
@pytest.mark.parametrize("name", ["immediate", "berendsen", "bussi"])
def test_reference_coupling_protocol(name, dtype):
    temp = 10.0
    th = {"immediate": mb.ImmediateThermostat(temp), "berendsen": mb.BerendsenThermostat(temp, 0.1),
          "bussi": mb.VelocityRescaleThermostat(temp, 0.1)}[name]
    s = _protocol_system(dtype, seed=2)
    rng = np.random.default_rng(3)
    mb.random_velocities_(s, temp, rng=rng)
    mb.simulate(s, mb.VelocityVerlet(dt=0.001, coupling=(th,)), 40_000, rng=rng)
    temps = np.array(mb.values(s.loggers["temperature"])[2000:])
    print(f"[coupling.jl {name} {np.dtype(dtype).name}] <T>={temps.mean():.4f} std={temps.std():.4f} n={len(temps)}")
    assert len(temps) == 2001
    assert 9.5 < temps.mean() < 10.5 and temps.std() < 1.0
    s.close()


def test_bussi_samples_canonical_kinetic_energy():
    """2916 argon atoms on the brick path at 90 K. In the canonical ensemble K ~ Gamma(Nf/2, kT): <K> = Nf k T0 / 2 and
    Var(K) = 2 <K>^2 / Nf. KE is logged every 10 steps (0.02 ps); its correlation time under the thermostat is about
    tau / 2 = 0.05 ps, so blocks of 50 records (1 ps = 10 tau) are independent and the block averages give the standard
    errors; with ~40 blocks a 4-sigma bar on each moment."""
    sd = H.lj_fluid(9, seed=21, dtype=F64, temp=90.0)
    s = H.make_system(sd, (mb.LennardJones(cutoff=mb.ShiftedForceCutoff(1.0), use_neighbors=True),), F64, r_list=1.2)
    s.loggers = {"ke": mb.KineticEnergyLogger(10)}
    T0, dt = 90.0, 0.002
    mb.simulate(s, mb.VelocityVerlet(dt=dt, coupling=mb.VelocityRescaleThermostat(T0, 0.1)), 21_000, rng=np.random.default_rng(8))
    assert s.stats()["path"] == 1
    ke = np.array(s.loggers["ke"].history[101:])  # drop 2 ps (20 tau) of equilibration
    nf = 3 * sd["n"] - 3
    kbar = nf * KB * T0 / 2
    nb = len(ke) // 50
    blocks = ke[:nb * 50].reshape(nb, 50)
    mean, se_mean = blocks.mean(), blocks.mean(1).std(ddof=1) / math.sqrt(nb)
    dev2 = (blocks - mean) ** 2
    ratio = dev2.mean() / (2 * kbar * kbar / nf)
    se_ratio = dev2.mean(1).std(ddof=1) / math.sqrt(nb) / (2 * kbar * kbar / nf)
    print(f"[Bussi canonical] <K>/Kbar-1={mean / kbar - 1:.2e} (se {se_mean / kbar:.1e}); Var ratio={ratio:.3f} (se {se_ratio:.3f}); "
          f"{nb} blocks")
    assert abs(mean - kbar) < 4 * se_mean
    assert abs(ratio - 1) < 4 * se_ratio


def _bussi_run(seed, loggers=None, n=30, dtype=F64):
    sd, s, _ = _lj_exceptions(dtype)
    if loggers:
        s.loggers = loggers
    mb.simulate(s, mb.VelocityVerlet(dt=0.002, coupling=mb.VelocityRescaleThermostat(120.0, 0.05, n_steps=2)), n,
                rng=np.random.default_rng(seed))
    out = (s.coords.copy(), s.velocities.copy(), s.stats()["graph_mode"])
    s.close()
    return out


@pytest.mark.parametrize("dtype", [F32, F64])
def test_loggers_are_observers(dtype):
    x0, v0, g0 = _bussi_run(4, dtype=dtype)
    lg = {"v": mb.VelocitiesLogger(7), "ke": mb.KineticEnergyLogger(7), "x": mb.CoordinatesLogger(10)}
    x1, v1, g1 = _bussi_run(4, lg, dtype=dtype)
    assert g0 == g1 == 1
    assert np.array_equal(x0, x1) and np.array_equal(v0, v1)
    # a logged velocity frame (after the step's coupling) equals an unlogged run stopped at that step
    for k, step in enumerate(mb.record_steps(7, 30)):
        if step == 0:
            continue
        xs, vs, _ = _bussi_run(4, n=step, dtype=dtype)
        assert np.array_equal(lg["v"].history[k], vs)
        m = H.lj_fluid(6)["mass"].astype(dtype).astype(np.float64)[:, None]  # the masses the engine holds
        ke = 0.5 * float(np.sum(m * vs.astype(np.float64) ** 2))
        assert abs(lg["ke"].history[k] - ke) < 1e-12 * ke


@pytest.mark.parametrize("name", ["immediate", "berendsen", "bussi5"])
def test_graph_and_stream_paths_bit_identical(name, monkeypatch):
    res = []
    for no_graph in ("0", "1"):
        monkeypatch.setenv("MOLLYB200_NO_GRAPH", no_graph)
        _, s, _ = _lj_exceptions()
        th = {"immediate": mb.ImmediateThermostat(120.0), "berendsen": mb.BerendsenThermostat(120.0, 0.05),
              "bussi5": mb.VelocityRescaleThermostat(120.0, 0.05, n_steps=5)}[name]
        s.loggers = {"ke": mb.KineticEnergyLogger(5)}
        mb.simulate(s, mb.VelocityVerlet(dt=0.002, coupling=th), 40, rng=np.random.default_rng(2))
        res.append((s.coords.copy(), s.velocities.copy(), list(s.loggers["ke"].history), s.stats()["graph_mode"]))
        s.close()
    (xa, va, ka, ga), (xb, vb, kb, gb) = res
    assert (ga, gb) == (1, 0)
    assert np.array_equal(xa, xb) and np.array_equal(va, vb) and ka == kb


def test_host_and_device_buffers_identical():
    import torch
    out = []
    for device in (False, True):
        sd, s, _ = _lj_exceptions()
        if device:
            s.coords = torch.from_numpy(s.coords).cuda()
            s.velocities = torch.from_numpy(s.velocities).cuda()
        mb.simulate(s, mb.VelocityVerlet(dt=0.002, coupling=mb.VelocityRescaleThermostat(120.0, 0.05)), 25,
                    rng=np.random.default_rng(6))
        torch.cuda.synchronize()
        out.append([a.cpu().numpy() if hasattr(a, "cpu") else a.copy() for a in (s.coords, s.velocities)])
        s.close()
    assert np.array_equal(out[0][0], out[1][0]) and np.array_equal(out[0][1], out[1][1])


@pytest.mark.parametrize("name", ["immediate", "berendsen", "bussi"])
def test_chunked_calls_equal_one_call(name):
    """simulate!(25) then simulate!(15; init_step=25) == simulate!(40). The Bussi draws are a function of (keys, step) only,
    so with the same keys (a fresh generator of the same seed for every call) the chunked run takes the same draws."""
    th = {"immediate": mb.ImmediateThermostat(120.0), "berendsen": mb.BerendsenThermostat(120.0, 0.05),
          "bussi": mb.VelocityRescaleThermostat(120.0, 0.05)}[name]
    sim = mb.VelocityVerlet(dt=0.002, coupling=th)
    sd, a, _ = _lj_exceptions()
    _, b, _ = _lj_exceptions()
    mb.simulate(a, sim, 40, rng=np.random.default_rng(1))
    mb.simulate(b, sim, 25, rng=np.random.default_rng(1))
    mb.simulate(b, sim, 15, init_step=25, rng=np.random.default_rng(1))
    assert _pos_err(a.coords, b.coords, sd["box"]) < 1e-9
    assert np.abs(a.velocities - b.velocities).max() < 1e-8
    a.close(); b.close()


def test_bussi_seeds():
    x0, v0, _ = _bussi_run(9)
    x1, v1, _ = _bussi_run(9)
    x2, v2, _ = _bussi_run(10)
    assert np.array_equal(x0, x1) and np.array_equal(v0, v1)
    assert np.abs(v0 - v2).max() > 1e-6


def test_refusals_and_switching_off():
    sd, s, _ = _readme()
    ctx = s.engine()
    L = s._L
    bad = [(capi_kind, n, kT, tau) for capi_kind, n, kT, tau in (
        (7, 1, 1.0, 0.1), (-1, 1, 1.0, 0.1), (mb.capi.MB_VC_IMMEDIATE, 0, -1.0, 0.0), (mb.capi.MB_VC_IMMEDIATE, 0, math.nan, 0.0),
        (mb.capi.MB_VC_BERENDSEN, 0, 1.0, 0.0), (mb.capi.MB_VC_BERENDSEN, 0, 1.0, math.inf), (mb.capi.MB_VC_VRESCALE, 0, 1.0, 0.1),
        (mb.capi.MB_VC_VRESCALE, 1, 1.0, -0.1))]
    for b in bad:
        assert L.mb_set_velocity_coupling(ctx, C.byref(mb.capi.MBVCoupling(*b))) == mb.capi.MB_ERR_INVALID
    # Andersen and a velocity-rescaling thermostat in one call: refused before any work (coordinates untouched)
    assert L.mb_set_velocity_coupling(ctx, C.byref(mb.capi.MBVCoupling(mb.capi.MB_VC_IMMEDIATE, 0, 2.0, 0.0))) == 0
    p = mb.capi.MBVVParams(0.002, 10, 0, 1, 2.0, 0.02, 1, 2)
    x = s.coords.copy()
    assert L.mb_simulate_vv(ctx, s.coords.ctypes.data, s.velocities.ctypes.data, C.byref(p)) == mb.capi.MB_ERR_INVALID
    assert b"at most one thermostat" in L.mb_last_error()
    assert np.array_equal(x, s.coords)
    # simulate sets or clears the coupling on every call: a plain run after a thermostatted one is the plain trajectory
    mb.simulate(s, mb.VelocityVerlet(dt=0.002, coupling=mb.ImmediateThermostat(300.0)), 5)
    ref = H.make_system(dict(sd, coords=s.coords.copy(), velocities=s.velocities.copy()), (mb.LennardJones(),), F64)
    mb.simulate(s, mb.VelocityVerlet(dt=0.002), 10, init_step=5)
    mb.simulate(ref, mb.VelocityVerlet(dt=0.002), 10, init_step=5)
    assert np.array_equal(s.coords, ref.coords) and np.array_equal(s.velocities, ref.velocities)
    s.close(); ref.close()
