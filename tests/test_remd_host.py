"""CPU tests of temperature replica exchange (mollyb200.simulate_remd): the driver's cycle split, pair parity, rng draw
order, state indices, exchange logger, current_step and logger steps against tests/remd_oracle.py, with the numpy Langevin
restatement run in place of the engine through the driver's runner seam; the argument refusals; and mb_simulate_group's
refusals, which need no GPU."""
import ctypes as C

import numpy as np
import pytest

import langevin_oracle as lo
import mbhelpers as H
import mollyb200 as mb
import remd_oracle as ro
import thermostat_oracle as tho
from oracle import oracle as o

F64 = np.float64
TEMPS = (120.0, 180.0, 240.0, 300.0)


def _setup(n=20, box=1.6):
    sd = H.readme_system(n, box, seed=3)
    orc = H.make_oracle(sd, [o.Inter(o.LJ)])
    base = H.make_system(sd, (mb.LennardJones(),), F64)
    wrap = lambda x: x - np.floor(x / sd["box"]) * sd["box"]
    fe = lambda x: orc.forces_allpairs(np.asarray(x, F64), energy=False)[0]
    energy = lambda x: orc.forces_allpairs(np.asarray(x, F64))[1]
    return sd, base, wrap, fe, energy


class _OracleRunner:
    """The runner seam: each call is run by the numpy Langevin loop with the keys the driver drew for it."""

    def __init__(self, sd, wrap, fe, energy):
        self.sd, self.wrap, self.fe, self.e = sd, wrap, fe, energy
        self.calls, self.log_steps = [], {}

    def run(self, repsys, calls, max_retries):
        for s, call in calls:
            st = repsys.state_system(s)
            p = call.p
            i = next(k for k in range(repsys.n_replicas) if repsys.replica_coords[k] is st.coords)
            x, v = lo.simulate_langevin(self.fe, st.coords, st.velocities, self.sd["mass"], p.dt, p.n_steps, p.kT, p.friction,
                                        tho.rng_words(p.rng_ctr1, p.rng_key), self.wrap, p.remove_cm_every, p.init_step)
            st.coords[...], st.velocities[...] = x, v
            self.calls.append((i, s, p.n_steps, p.init_step))
            if call.plan is not None:
                self.log_steps.setdefault(i, []).extend(call.plan.steps["energy"])

    def energy(self, repsys, s, coords):
        return self.e(coords)


def _repsys(base, sd, loggers=False):
    states = [mb.ThermoState(base, mb.Langevin(dt=0.005, temperature=t, friction=0.1)) for t in TEMPS]
    lgs = [dict(temp=mb.TemperatureLogger(10)) for _ in TEMPS] if loggers else None
    return mb.ReplicaSystem(states, [sd["coords"].copy() for _ in TEMPS], replica_loggers=lgs)


@pytest.mark.parametrize("n_steps,exchange_time", [(230, 0.25), (200, 0.25), (30, 0.5)])
def test_driver_matches_oracle(n_steps, exchange_time):
    """Cycle split with and without remainder (230 steps: 4 cycles of 57 and 2 more; 30 steps: no cycle at all)."""
    sd, base, wrap, fe, energy = _setup()
    rs = _repsys(base, sd)
    rng_k = [np.random.default_rng(11) for _ in range(2)]
    for i, v in enumerate(rs.replica_velocities):
        v[...] = np.random.default_rng(100 + i).normal(0, 0.5, v.shape)
    xs = [x.copy() for x in rs.replica_coords]
    vs = [v.copy() for v in rs.replica_velocities]
    runner = _OracleRunner(sd, wrap, fe, energy)
    mb.simulate_remd(rs, mb.ReplicaExchangeMD(0.005, exchange_time), n_steps, rng=rng_k[0], runner=runner)

    def integrate(s, x, v, n, start, keys):
        return lo.simulate_langevin(fe, x, v, sd["mass"], 0.005, n, mb.BOLTZMANN_K * TEMPS[s], 0.1, tho.rng_words(*keys), wrap,
                                    1, start)

    betas = [1.0 / (mb.BOLTZMANN_K * t) for t in TEMPS]
    si, log, calls = ro.simulate_remd(xs, vs, betas, range(4), integrate, energy, n_steps, 0.005, exchange_time, 0, rng_k[1], F64)
    assert runner.calls == calls
    assert rs.state_indices == si
    xl = rs.exchange_logger
    assert xl.indices == log["indices"] and xl.steps == log["steps"] and xl.deltas == log["deltas"]
    assert xl.n_attempts == log["n_attempts"] and xl.end_step == log["end_step"] == n_steps
    assert xl.n_exchanges == len(log["indices"])
    assert rs.current_step == n_steps
    for i in range(4):
        np.testing.assert_array_equal(rs.replica_coords[i], xs[i])
        np.testing.assert_array_equal(rs.replica_velocities[i], vs[i])
    # both generators were drawn from identically, the short-circuited uniforms included
    assert rng_k[0].random() == rng_k[1].random()
    n_cycles = int((n_steps * 0.005) // exchange_time)
    if n_cycles:
        L = n_steps // n_cycles
        # odd cycles pair (1, 2); even cycles (0, 1) and (2, 3)
        assert xl.n_attempts == sum(1 if c % 2 else 2 for c in range(1, n_cycles + 1))
        assert all(s % L == 0 for s in xl.steps)
        assert all((i, j) in ((1, 2),) if (s // L) % 2 else (i, j) in ((0, 1), (2, 3)) for (i, j), s in zip(xl.indices, xl.steps))


def test_two_calls_logger_steps_and_current_step():
    sd, base, wrap, fe, energy = _setup()
    rs = _repsys(base, sd, loggers=True)
    runner = _OracleRunner(sd, wrap, fe, energy)
    sim = mb.ReplicaExchangeMD(0.005, 0.25)
    n = 200
    mb.simulate_remd(rs, sim, n, rng=np.random.default_rng(1), runner=runner)
    mb.simulate_remd(rs, sim, n, rng=np.random.default_rng(2), runner=runner)
    assert rs.current_step == 2 * n
    for i in range(4):
        assert runner.log_steps[i] == list(range(0, 2 * n + 1, 10))
    assert rs.exchange_logger.end_step == 2 * n
    assert all(0 < s <= 2 * n for s in rs.exchange_logger.steps) and rs.exchange_logger.steps == sorted(rs.exchange_logger.steps)
    assert rs.exchange_logger.n_attempts == 2 * (2 + 1 + 2 + 1)


def test_refusals():
    sd, base, *_ = _setup()
    with pytest.raises(ValueError):
        mb.ReplicaExchangeMD(0.005, 0.005)
    with pytest.raises(ValueError):
        mb.ThermoState(base, mb.VelocityVerlet(dt=0.002))
    ts = mb.ThermoState(base, mb.VelocityVerlet(dt=0.002, coupling=mb.BerendsenThermostat(250.0, 0.1)))
    assert ts.temperature == 250.0 and ts.beta == pytest.approx(1 / (mb.BOLTZMANN_K * 250.0))
    assert mb.ThermoState(base, mb.NoseHoover(dt=0.002, temperature=200.0)).temperature == 200.0
    with pytest.raises(TypeError):
        mb.ThermoState(base, mb.Langevin(dt=0.005, temperature=300.0, friction=1.0), pressure=1.0)
    other = H.make_system(sd, (mb.LennardJones(),), F64)
    lv = lambda s, t: mb.ThermoState(s, mb.Langevin(dt=0.005, temperature=t, friction=0.1))
    with pytest.raises(TypeError, match="Hamiltonian"):
        mb.ReplicaSystem([lv(base, 100.0), lv(other, 200.0)], [sd["coords"]] * 2)
    with pytest.raises(ValueError):
        mb.ReplicaSystem([lv(base, 100.0), lv(base, 200.0)], [sd["coords"]] * 3)
    with pytest.raises(ValueError):
        mb.ReplicaSystem([lv(base, 100.0), lv(base, 200.0)], [sd["coords"]] * 2, replica_velocities=[sd["coords"]])
    with pytest.raises(TypeError):
        mb.ReplicaSystem([lv(base, 100.0), lv(base, 200.0)], [sd["coords"]] * 2, replica_boundaries=[base.boundary] * 2)
    with pytest.raises(TypeError):
        mb.ReplicaSystem([mb.ThermoState(base, mb.SteepestDescentMinimizer(), temperature=100.0)], [sd["coords"]])
    rs = mb.ReplicaSystem([lv(base, 100.0), lv(base, 200.0)], [sd["coords"]] * 2)
    with pytest.raises(TypeError):
        mb.simulate(rs, mb.Langevin(dt=0.005, temperature=100.0, friction=0.1), 10)
    with pytest.raises(TypeError):
        mb.simulate(base, mb.ReplicaExchangeMD(0.005, 0.1), 10)


def test_group_refusals_without_gpu():
    L = mb.capi.load()
    assert L.mb_simulate_group(0, None) == mb.capi.MB_ERR_INVALID
    assert b"mb_simulate_group" in L.mb_last_error()
    members = (mb.capi.MBGroupMember * 2)()
    assert L.mb_simulate_group(2, members) == mb.capi.MB_ERR_INVALID
    assert b"null context" in L.mb_last_error()
    assert [m.status for m in members] == [mb.capi.MB_ERR_INVALID] * 2  # (a refused group runs no member)
    assert L.mb_simulate_group(-1, members) == mb.capi.MB_ERR_INVALID
