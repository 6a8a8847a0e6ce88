"""Captured graphs follow the context they run on: a setter called between two runs on the same context (masses, box or
LJ cutoff through the C ABI, as a C or Julia caller would) must give the run a fresh context configured with the changed
state would give, bit for bit, on the all-pairs and cell-list paths and for the minimiser. So must a change of one
integrator or thermostat parameter between two runs on the same context."""
import ctypes as C

import numpy as np
import pytest

import mbhelpers as H
import mollyb200 as mb

pytestmark = pytest.mark.gpu

F64 = np.float64
N_STEPS = 20


def _lj(cutoff, nl=False):
    return (mb.LennardJones(cutoff=mb.DistanceCutoff(cutoff), use_neighbors=nl),)


def _masses(sd, s):
    """Every other atom 1.5 times heavier: the total mass and the momentum that K2 removes change, n does not."""
    sd = dict(sd, mass=sd["mass"] * np.where(np.arange(sd["n"]) % 2 == 0, 1.0, 1.5))
    atoms = mb.atoms_from_arrays(sd["mass"], sd["charge"], sd["sigma"], sd["eps"], F64)
    mb.capi.check(s._L.mb_set_atoms(s.engine(), sd["n"], atoms.ctypes.data))
    return sd, s.pairwise_inters


def _box(sd, s):
    """A 2 % larger box: the coordinates stay inside it."""
    sd = dict(sd, box=sd["box"] * 1.02)
    mb.capi.check(s._L.mb_set_box(s.engine(), (C.c_double * 3)(*sd["box"])))
    return sd, s.pairwise_inters


def _cutoff(sd, s):
    inters = _lj(0.9, s.pairwise_inters[0].use_neighbors)
    mb.capi.check(s._L.mb_set_inters(s.engine(), 1, (mb.capi.MBInter * 1)(inters[0].descriptor())))
    return sd, inters


ALLPAIRS = dict(make=lambda: H.readme_system(100, 2.0, seed=1), inters=_lj(1.0), r_list=0.0, path=0)
BRICK = dict(make=lambda: H.lj_fluid(6, dtype=F64), inters=_lj(1.0, nl=True), r_list=1.2, path=1)


def _fresh(sd, inters, r_list, x, v):
    return H.make_system(dict(sd, coords=x.copy(), velocities=v.copy()), inters, F64, r_list=r_list)


@pytest.mark.parametrize("system,change", [(ALLPAIRS, _masses), (ALLPAIRS, _box), (ALLPAIRS, _cutoff), (BRICK, _box)],
                         ids=["allpairs-masses", "allpairs-box", "allpairs-cutoff", "brick-box"])
def test_setter_between_simulate_calls(system, change):
    sd = system["make"]()
    s = H.make_system(sd, system["inters"], F64, r_list=system["r_list"])
    vv = mb.VelocityVerlet(dt=0.002)
    mb.simulate(s, vv, N_STEPS, rng=np.random.default_rng(0))
    st = s.stats()
    assert st["graph_mode"] == 1 and st["path"] == system["path"]
    sd2, inters2 = change(sd, s)
    ref = _fresh(sd2, inters2, system["r_list"], s.coords, s.velocities)
    # init_step > 0: no CM removal before the first step, so the first K2 removes the momentum of the new state
    for sys_ in (s, ref):
        mb.simulate(sys_, vv, N_STEPS, init_step=N_STEPS, rng=np.random.default_rng(1))
        assert sys_.stats()["graph_mode"] == 1
    assert np.array_equal(s.coords, ref.coords)
    assert np.array_equal(s.velocities, ref.velocities)
    s.close()
    ref.close()


def _readme():
    return H.make_system(H.readme_system(100, 2.0, seed=1), _lj(1.0), F64)


def _chains():
    """Chain molecules with bonded terms (test_gpu_mts): the bonded forces add with float atomics, so two contexts agree to
    1e-12 nm, not bit for bit. A graph replayed with the old fractions or friction is off by many orders more."""
    from test_gpu_mts import _molecules
    return _molecules()[1]


def _mts(si, friction=None):
    if friction is None:
        return mb.MTSIntegrator(0.002, pi_fractions=(1, 1), si_fractions=si)
    return mb.MTSLangevinIntegrator(0.002, 120.0, friction, pi_fractions=(1, 1), si_fractions=si)


# (system, the first call's integrator, the second call's): one parameter differs
INTEGRATOR_CHANGES = {
    "langevin-friction": (_readme, mb.Langevin(0.002, 300.0, 1.0), mb.Langevin(0.002, 300.0, 5.0)),
    "langevin-temperature": (_readme, mb.Langevin(0.002, 300.0, 1.0), mb.Langevin(0.002, 350.0, 1.0)),
    "nosehoover-damping": (_readme, mb.NoseHoover(0.002, 300.0, 0.2), mb.NoseHoover(0.002, 300.0, 0.05)),
    # every list keeps its level, so the context keeps its graphs and only the key tells the calls apart
    "mts-fractions": (_chains, _mts((2, 2, 1)), _mts((4, 4, 1))),
    "mtslangevin-friction": (_chains, _mts((4, 2, 1), 10.0), _mts((4, 2, 1), 5.0)),
    "andersen-coupling-const": (_readme, mb.VelocityVerlet(0.002, coupling=mb.AndersenThermostat(300.0, 0.1)),
                                mb.VelocityVerlet(0.002, coupling=mb.AndersenThermostat(300.0, 0.02))),
    "bussi-coupling-const": (_readme, mb.VelocityVerlet(0.002, coupling=mb.VelocityRescaleThermostat(300.0, 0.1)),
                             mb.VelocityVerlet(0.002, coupling=mb.VelocityRescaleThermostat(300.0, 0.02))),
}


@pytest.mark.parametrize("change", list(INTEGRATOR_CHANGES))
def test_integrator_parameter_between_simulate_calls(change):
    """A step graph keeps the integrator's parameters by value: the second call, with one of them changed, must not replay
    the first call's graph, and gives what a fresh context gives from the same state."""
    make, first, second = INTEGRATOR_CHANGES[change]
    s = make()
    mb.simulate(s, first, N_STEPS, rng=np.random.default_rng(0))
    assert s.stats()["graph_mode"] == 1
    ref = make()
    ref.coords[...], ref.velocities[...] = s.coords, s.velocities
    for sys_ in (s, ref):
        mb.simulate(sys_, second, N_STEPS, init_step=N_STEPS, rng=np.random.default_rng(1))
        assert sys_.stats()["graph_mode"] == 1
    if make is _chains:
        from test_gpu_mts import _close
        assert _close((s.coords, s.velocities), (ref.coords, ref.velocities))
    else:
        assert np.array_equal(s.coords, ref.coords)
        assert np.array_equal(s.velocities, ref.velocities)
    s.close()
    ref.close()


def test_minimize_after_set_box():
    sd = H.readme_system(100, 2.0, seed=1)
    s = H.make_system(sd, _lj(1.0), F64)
    sdm = mb.SteepestDescentMinimizer(max_steps=30, tol=0.0)
    mb.steepest_descent(s, sdm)
    assert s.stats()["graph_mode"] == 1
    sd2, _ = _box(sd, s)
    ref = _fresh(sd2, _lj(1.0), 0.0, s.coords, s.velocities)
    traces = []
    for sys_ in (s, ref):
        traces.append(mb.steepest_descent(sys_, sdm)[1])
        assert sys_.stats()["graph_mode"] == 1
    assert np.array_equal(traces[0], traces[1], equal_nan=True)  # (record 0 has no max force)
    assert np.array_equal(s.coords, ref.coords)
    s.close()
    ref.close()
