"""Captured graphs follow the context they run on: a setter called between two runs on the same context (masses, box or
LJ cutoff through the C ABI, as a C or Julia caller would) must give the run a fresh context configured with the changed
state would give, bit for bit, on the all-pairs and cell-list paths and for the minimiser."""
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
