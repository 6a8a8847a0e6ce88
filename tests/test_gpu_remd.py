"""GPU tests of temperature replica exchange: mb_simulate_group gives what the same calls made one at a time give (graph
path on LJ, stream path on 6mrr with PME and on the GBN2 protein), and a member that overflows is retried alone;
simulate_remd follows tests/remd_oracle.py (every exchange decision, the state indices, the exchange logger and the f64
trajectories); the reference's "Temperature REMD" testset (test/simulation.jl:833-927); and the acceptance rate and
per-state energies against their closed forms on restrained atoms."""
import ctypes as C
import math
import os

import numpy as np
import pytest

import langevin_oracle as lo
import mbhelpers as H
import mollyb200 as mb
import nosehoover_oracle as nho
import remd_oracle as ro
import thermostat_oracle as tho
from molly_jl_b200.api import _Call
from oracle import oracle as o

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
KB = mb.BOLTZMANN_K
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _readme(r_list, seed):
    """The reference's 100-atom system; on the cell-list path (which needs a box of 2.5 r_list) 200 atoms in a 3 nm box."""
    return H.readme_system(200, 3.0, seed=seed) if r_list > 0 else H.readme_system(100, 2.0, seed=seed)


def _lj(dtype, r_list, seed):
    sd = _readme(r_list, seed)
    if r_list > 0:
        inters = (mb.LennardJones(cutoff=mb.DistanceCutoff(0.9), use_neighbors=True),)
    else:
        inters = (mb.LennardJones(),)
    s = H.make_system(sd, inters, dtype, r_list=r_list)
    s.loggers = dict(e=mb.TotalEnergyLogger(3), x=mb.CoordinatesLogger(7))
    return s


_SIMS = (lambda: mb.Langevin(dt=0.002, temperature=200.0, friction=1.0),
         lambda: mb.VelocityVerlet(dt=0.002, coupling=mb.BerendsenThermostat(150.0, 0.1)),
         lambda: mb.NoseHoover(dt=0.002, temperature=250.0),
         lambda: mb.Verlet(dt=0.002))


@pytest.mark.parametrize("R", [1, 3, 8])
@pytest.mark.parametrize("dtype", [F32, F64])
@pytest.mark.parametrize("r_list", [0.0, 1.1])
def test_group_equals_sequential(R, dtype, r_list):
    """Members with different integrators and step counts, loggers on: bit-identical to the single calls."""
    steps = [40 + 13 * i for i in range(R)]
    seq = [_lj(dtype, r_list, 10 + i) for i in range(R)]
    grp = [_lj(dtype, r_list, 10 + i) for i in range(R)]
    for i, s in enumerate(seq):
        mb.simulate(s, _SIMS[i % 4](), steps[i], rng=np.random.default_rng(i))
    calls = [_Call(s, _SIMS[i % 4](), steps[i], 0, np.random.default_rng(i), True) for i, s in enumerate(grp)]
    members = (mb.capi.MBGroupMember * R)()
    for m, s, call in zip(members, grp, calls):
        call.configure(s)
        m.ctx, m.coords, m.vels, m.kind = s.engine(), s.coords.ctypes.data, s.velocities.ctypes.data, call.kind
        m.params = C.addressof(call.p)
        m.log = C.addressof(call.plan.desc)
    rc = mb.capi.load().mb_simulate_group(R, members)
    assert rc == mb.capi.MB_OK, mb.capi.load().mb_last_error()
    for m, s, call in zip(members, grp, calls):
        call.run(s, 0, rc=m.status)
    for a, b in zip(seq, grp):
        np.testing.assert_array_equal(a.coords, b.coords)
        np.testing.assert_array_equal(a.velocities, b.velocities)
        for k in ("e", "x"):
            assert len(a.loggers[k].history) == len(b.loggers[k].history)
            for u, w in zip(a.loggers[k].history, b.loggers[k].history):
                np.testing.assert_array_equal(u, w)
    for s in seq + grp:
        s.close()


def test_group_refusals():
    L = mb.capi.load()
    a, b = _lj(F64, 0.0, 1), _lj(F32, 0.0, 2)
    p = mb.capi.MBLangevinParams(dt=0.002, n_steps=5, kT=1.0, friction=1.0)
    members = (mb.capi.MBGroupMember * 2)()
    for m, s in zip(members, (a, a)):
        m.ctx, m.coords, m.vels, m.kind, m.params = s.engine(), s.coords.ctypes.data, s.velocities.ctypes.data, \
            mb.capi.MB_INTEG_LANGEVIN, C.addressof(p)
    x0 = a.coords.copy()
    assert L.mb_simulate_group(2, members) == mb.capi.MB_ERR_INVALID
    assert b"same context" in L.mb_last_error()
    members[1].ctx, members[1].kind = b.engine(), 99
    assert L.mb_simulate_group(2, members) == mb.capi.MB_ERR_INVALID
    members[1].kind, members[1].params = mb.capi.MB_INTEG_LANGEVIN, None
    assert L.mb_simulate_group(2, members) == mb.capi.MB_ERR_INVALID
    np.testing.assert_array_equal(a.coords, x0)


def _oracle_setup(r_list):
    sd = _readme(r_list, 1)
    if r_list > 0:
        inter = o.Inter(o.LJ, o.CUT_DISTANCE, 0.9, use_neighbors=True)
        base = H.make_system(sd, (mb.LennardJones(cutoff=mb.DistanceCutoff(0.9), use_neighbors=True),), F64, r_list=r_list)
    else:
        inter = o.Inter(o.LJ)
        base = H.make_system(sd, (mb.LennardJones(),), F64)
    orc = H.make_oracle(sd, [inter])
    wrap = lambda x: x - np.floor(x / sd["box"]) * sd["box"]
    fe = lambda x: orc.forces_allpairs(np.asarray(x, F64), energy=False)[0]
    energy = lambda x: orc.forces_allpairs(np.asarray(x, F64))[1]
    return sd, base, wrap, fe, energy


@pytest.mark.parametrize("kind,r_list", [("nosehoover", 0.0), ("langevin", 0.0), ("vv_bussi", 0.0), ("langevin", 1.1)])
def test_trajectory_parity_with_oracle(kind, r_list):
    """4 replicas, 80 cycles of 5 steps, f64: every decision, state index, logger entry and the trajectories."""
    sd, base, wrap, fe, energy = _oracle_setup(r_list)
    temps = (120.0, 180.0, 240.0, 300.0)
    dt, n_steps, ex = 0.002, 400, 0.0099
    mk = {"nosehoover": lambda t: mb.NoseHoover(dt=dt, temperature=t),
          "langevin": lambda t: mb.Langevin(dt=dt, temperature=t, friction=2.0),
          "vv_bussi": lambda t: mb.VelocityVerlet(dt=dt, coupling=mb.VelocityRescaleThermostat(t, 0.05))}[kind]
    states = [mb.ThermoState(base, mk(t)) for t in temps]
    v0 = [_readme(r_list, 1 + i)["velocities"].astype(F64) for i in range(4)]
    rs = mb.ReplicaSystem(states, [sd["coords"].copy() for _ in temps], replica_velocities=[v.copy() for v in v0])
    mb.simulate(rs, mb.ReplicaExchangeMD(dt, ex), n_steps, rng=np.random.default_rng(5))

    def integrate(s, x, v, n, start, keys):
        kT = KB * temps[s]
        if kind == "nosehoover":
            return nho.simulate_nose_hoover(fe, x, v, sd["mass"], dt, n, kT, states[s].integrator.damping, wrap, 1, start)[:2]
        if kind == "langevin":
            return lo.simulate_langevin(fe, x, v, sd["mass"], dt, n, kT, 2.0, tho.rng_words(*keys), wrap, 1, start)
        orc = H.make_oracle(sd, [o.Inter(o.LJ)])
        return tho.simulate_vv_coupled(orc, x, v, sd["mass"], sd["box"], dt, n, states[s].integrator.coupling, KB,
                                       tho.rng_words(*keys), 1, start)[:2]

    xs = [sd["coords"].astype(F64).copy() for _ in temps]
    vs = [v.copy() for v in v0]
    si, log, _ = ro.simulate_remd(xs, vs, rs.betas, range(4), integrate, energy, n_steps, dt, ex, 0,
                                  np.random.default_rng(5), F64, draws=kind != "nosehoover")
    assert rs.state_indices == si
    xl = rs.exchange_logger
    assert xl.indices == log["indices"] and xl.steps == log["steps"] and xl.n_attempts == log["n_attempts"]
    np.testing.assert_allclose(xl.deltas, log["deltas"], rtol=1e-6, atol=1e-9)
    assert len(log["indices"]) > 0
    for i in range(4):
        d = rs.replica_coords[i] - xs[i]
        d -= sd["box"] * np.round(d / sd["box"])
        assert np.abs(d).max() < 1e-9, (i, np.abs(d).max())
        assert np.abs(rs.replica_velocities[i] - vs[i]).max() < 1e-8
    rs.close()


@pytest.mark.parametrize("dtype", [F32, F64])
def test_reference_temperature_remd(dtype):
    """test/simulation.jl:833-927: 100 atoms, 4 Langevin replicas at 120-300 K, dt 0.005 ps, exchanges every 2.5 ps,
    simulate called twice with 20 000 steps."""
    sd = H.readme_system(100, 2.0, seed=1)
    base = H.make_system(sd, (mb.LennardJones(),), dtype)
    temps = (120.0, 180.0, 240.0, 300.0)
    states = [mb.ThermoState(base, mb.Langevin(dt=0.005, temperature=t, friction=0.1), temperature=t) for t in temps]
    loggers = [dict(temp=mb.TemperatureLogger(10), coords=mb.CoordinatesLogger(10)) for _ in temps]
    rs = mb.ReplicaSystem(states, [sd["coords"].astype(dtype).copy() for _ in temps], replica_loggers=loggers)
    sim = mb.ReplicaExchangeMD(dt=0.005, exchange_time=2.5)
    n = 20_000
    rng = np.random.default_rng(10)
    mb.simulate(rs, sim, n, assign_velocities=True, rng=rng)
    mb.simulate(rs, sim, n, rng=rng)
    assert rs.current_step == 2 * n
    for lg in loggers:
        assert len(lg["temp"].history) == len(range(0, 2 * n + 1, 10))
        assert len(lg["coords"].history) == len(range(0, 2 * n + 1, 10))
    xl = rs.exchange_logger
    assert xl.steps == sorted(xl.steps) and all(0 < s <= rs.current_step for s in xl.steps)
    eff = xl.n_exchanges / xl.n_attempts
    assert 0.16 < eff < 1.0, eff
    for lg in loggers:
        mean_t = float(np.mean(lg["temp"].history))
        assert 0.9 * temps[0] < mean_t < 1.15 * temps[-1], mean_t
    rs.close()


def _group_vs_sequential(make, sims, steps, tol_x, tol_v, box):
    """The same calls through mb_simulate_group and one at a time, on systems make(i); trajectories within the bars."""
    R = len(sims)
    seq = [make(i) for i in range(R)]
    grp = [make(i) for i in range(R)]
    for i, s in enumerate(seq):
        mb.simulate(s, sims[i](), steps[i], rng=np.random.default_rng(i))
    calls = [_Call(s, sims[i](), steps[i], 0, np.random.default_rng(i), True) for i, s in enumerate(grp)]
    members = (mb.capi.MBGroupMember * R)()
    for m, s, call in zip(members, grp, calls):
        call.configure(s)
        m.ctx, m.coords, m.vels, m.kind = s.engine(), s.coords.ctypes.data, s.velocities.ctypes.data, call.kind
        m.params = C.addressof(call.p)
        m.log = C.addressof(call.plan.desc) if call.plan is not None else None
    rc = mb.capi.load().mb_simulate_group(R, members)
    assert rc == mb.capi.MB_OK, mb.capi.load().mb_last_error()
    for m, s, call in zip(members, grp, calls):
        call.run(s, 0, rc=m.status)
    for a, b in zip(seq, grp):
        d = a.coords - b.coords
        d -= box * np.round(d / box)
        print(f"[group vs sequential] max |dx| {np.abs(d).max():.3e} nm, max |dv| {np.abs(a.velocities - b.velocities).max():.3e}")
        assert np.abs(d).max() < tol_x
        assert np.abs(a.velocities - b.velocities).max() < tol_v
        for u, w in zip(a.loggers["e"].history, b.loggers["e"].history):
            assert abs(u - w) <= 1e-9 * max(1.0, abs(u))
    for s in seq + grp:
        s.close()


_STREAM_SIMS = (lambda: mb.Langevin(dt=0.001, temperature=300.0, friction=1.0),
                lambda: mb.VelocityVerlet(dt=0.001),
                lambda: mb.NoseHoover(dt=0.001, temperature=310.0))


def test_group_equals_sequential_6mrr_pme_f64():
    """6mrr with PME (graphs off: each step on the stream, cuFFT on each context's stream), f64, 3 members: within 1e-9 nm
    (bonded forces and PME spreading add with atomics, so runs agree to rounding, not bit for bit)."""
    g = dict(np.load(os.path.join(ROOT, "tests", "golden", "6mrr.npz")))

    def make(i):
        s = H.sixmrr_pme_system(g, F64, exact=True, velocities=g["velocities_300K"])
        s.loggers = dict(e=mb.PotentialEnergyLogger(5))
        return s
    _group_vs_sequential(make, _STREAM_SIMS, [20, 27, 34], 1e-9, 1e-6, g["box"])


def test_group_equals_sequential_gbn2_f64():
    """The 1170-atom GBN2 protein, f64, 3 members: within 1e-9 nm."""
    from test_gpu_implicit_solvent import _full_system
    g = np.load(os.path.join(ROOT, "tests", "golden", "6mrr_gb.npz"))

    def make(i):
        v = np.random.default_rng(20 + i).normal(0, 0.3, g["coords"].shape)
        return _full_system(g, "gbn2", F64, velocities=v, loggers=dict(e=mb.PotentialEnergyLogger(5)))
    _group_vs_sequential(make, _STREAM_SIMS, [20, 27, 34], 1e-9, 1e-6, g["box"])


def test_capacity_member_is_retried_alone(monkeypatch):
    """Two states of one droplet System: replica 0 drifts through a face and overflows the capacities its first build
    derived (MB_ERR_CAPACITY from the group), replica 1 stays put and succeeds. The driver restores replica 0 and reruns it
    through the single call; both replicas end where single simulate calls of the same runs end."""
    side, radius, dt, n = 12.0, 3.5, 0.002, 200
    box = np.array([side] * 3)
    sd = H.argon_droplet(radius, box, [side - 1.5 - radius, side / 2, side / 2], seed=11)
    v_drift = sd["velocities"] + np.array([12.0, 0.0, 0.0])
    inters = (mb.LennardJones(cutoff=mb.ShiftedForceCutoff(1.2), use_neighbors=True),)
    base = H.make_system(sd, inters, F64, r_list=1.3)
    vv = lambda: mb.VelocityVerlet(dt=dt, remove_CM_motion=0)
    states = [mb.ThermoState(base, vv(), temperature=t) for t in (90.0, 100.0)]
    rs = mb.ReplicaSystem(states, [sd["coords"].copy(), sd["coords"].copy()],
                          replica_velocities=[v_drift.copy(), sd["velocities"].copy()])
    L = mb.capi.load()
    group, seen = L.mb_simulate_group, []

    def recording(n_members, members):
        rc = group(n_members, members)
        seen.append([members[i].status for i in range(n_members)])
        return rc
    monkeypatch.setattr(L, "mb_simulate_group", recording)
    mb.simulate(rs, mb.ReplicaExchangeMD(dt, 10.0), n)  # (no exchange: one group call of n steps)
    assert seen == [[mb.capi.MB_ERR_CAPACITY, mb.capi.MB_OK]]
    for i, v0 in enumerate((v_drift, sd["velocities"])):
        s = H.make_system(dict(sd, velocities=v0), inters, F64, r_list=1.3)
        mb.simulate(s, vv(), n)
        d = rs.replica_coords[i] - s.coords
        d -= box * np.round(d / box)
        assert np.abs(d).max() < 1e-9, (i, np.abs(d).max())
        assert np.abs(rs.replica_velocities[i] - s.velocities).max() < 1e-8
        s.close()
    rs.close()


def test_exchange_statistics_closed_form():
    """Non-interacting atoms held by harmonic position restraints, Langevin (BAOAB, which samples a harmonic configuration
    exactly) without CM removal, at 300 and 330 K. U at state T is Gamma(3N/2, kT), so the acceptance rate must be
    E[min(1, exp(-Delta))] over the two Gamma laws (sampled with numpy) within 4 binomial standard errors, and the mean U
    at each state 3N/2 kT within 5 standard errors. Exchanges are 1.5 ps apart: 2.4 oscillation periods, and 3.75 decay
    times of the oscillation at friction 5/ps."""
    from molly_jl_b200.api import _EngineRunner
    N, k, m, box = 50, 1000.0, 10.0, 6.0
    temps, dt, cyc, n_cyc = (300.0, 330.0), 0.005, 300, 1600
    x0 = np.random.default_rng(4).uniform(1.0, box - 1.0, (N, 3))
    atoms = mb.atoms_from_arrays(np.full(N, m), np.zeros(N), np.full(N, 0.3), np.zeros(N), F64)  # eps = 0: no pair force
    base = mb.System(atoms=atoms, coords=x0.copy(), velocities=np.zeros((N, 3)), boundary=mb.CubicBoundary(box),
                     pairwise_inters=(mb.LennardJones(cutoff=mb.DistanceCutoff(1.0)),), dtype=F64)
    base = mb.add_position_restraints(base, k)
    states = [mb.ThermoState(base, mb.Langevin(dt=dt, temperature=t, friction=5.0, remove_CM_motion=0)) for t in temps]
    rs = mb.ReplicaSystem(states, [x0.copy(), x0.copy()])
    samples = {0: [], 1: []}

    class Recording(_EngineRunner):
        def energy(self, repsys, s, coords):
            u = super().energy(repsys, s, coords)
            samples[s].append(u)
            return u
    rng = np.random.default_rng(8)
    sim = mb.ReplicaExchangeMD(dt, cyc * dt * 0.999999)
    mb.simulate_remd(rs, sim, 4 * cyc, assign_velocities=True, rng=rng)  # equilibration
    samples[0].clear(), samples[1].clear()
    xl = rs.exchange_logger
    a0, e0 = xl.n_attempts, xl.n_exchanges
    mb.simulate_remd(rs, sim, n_cyc * cyc, rng=rng, runner=Recording())
    att, acc = xl.n_attempts - a0, xl.n_exchanges - e0
    kT = [KB * t for t in temps]
    g = np.random.default_rng(0)
    u0, u1 = g.gamma(1.5 * N, kT[0], 2_000_000), g.gamma(1.5 * N, kT[1], 2_000_000)
    delta = (1 / kT[1] - 1 / kT[0]) * (u0 - u1)
    p = np.minimum(1.0, np.exp(-delta)).mean()
    rate, se = acc / att, math.sqrt(p * (1 - p) / att)
    print(f"[closed form] acceptance {rate:.4f} expected {p:.4f} +- {se:.4f} over {att} attempts")
    assert att == n_cyc // 2
    assert abs(rate - p) < 4 * se
    for s in (0, 1):
        u = np.array(samples[s])
        mean, expect = u.mean(), 1.5 * N * kT[s]
        print(f"[closed form] state {s}: <U> {mean:.3f} expected {expect:.3f} ({len(u)} samples)")
        assert abs(mean - expect) < 5 * math.sqrt(1.5 * N) * kT[s] / math.sqrt(len(u))
    rs.close()
