"""CPU tests of the multiple-time-step integrators (MTSIntegrator, MTSLangevinIntegrator): the constructors against
setup_mts_integrator, the C-ABI parameter layout against the header, the list -> level mapping through the by-kind
concatenation, simulate's refusals, and the numpy restatement of the reference loop (tests/mts_oracle.py): one level is the
VelocityVerlet step, and two levels integrate a small molecule with an energy error of second order in the outer step.
The GPU counterpart is tests/test_gpu_mts.py."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import mollyb200 as mb
import mts_oracle as mo
from oracle import bonded as bd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("pi,si,gi,ordered", [((1,), (), (), (1,)), ((1, 1), (2, 4), (), (1, 2, 4)),
                                               ((), (4, 2, 1, 4), (1,), (1, 2, 4)), ((1,), (3, 3, 6), (), (1, 3, 6)),
                                               ((1,), (8, 4, 2), (), (1, 2, 4, 8)), ((1,), (np.int64(2),), (), (1, 2))])
def test_ordered_fractions(pi, si, gi, ordered):
    sim = mb.MTSIntegrator(0.002, pi_fractions=pi, si_fractions=si, gi_fractions=gi)
    assert sim.ordered_fractions == ordered
    assert mb.MTSLangevinIntegrator(0.002, 300.0, 1.0, pi_fractions=pi, si_fractions=si, gi_fractions=gi).ordered_fractions == ordered


@pytest.mark.parametrize("pi,si,gi,match", [((), (), (), "requires one of"), ((1.0,), (), (), "integers"),
                                            ((1,), (2.0,), (), "integers"), ((0, 1), (), (), "less than 1"),
                                            ((2,), (4,), (), "must include 1"), ((1,), (2, 3), (), "not a multiple"),
                                            ((1,), (4, 6), (), "not a multiple")])
def test_constructor_refusals_mirror_setup_mts_integrator(pi, si, gi, match):
    for make in (lambda: mb.MTSIntegrator(0.002, pi_fractions=pi, si_fractions=si, gi_fractions=gi),
                 lambda: mb.MTSLangevinIntegrator(0.002, 300.0, 1.0, pi_fractions=pi, si_fractions=si, gi_fractions=gi)):
        with pytest.raises(ValueError, match=match):
            make()


def test_constructor_arguments():
    for bad in (0.0, -0.001, math.inf, math.nan):
        with pytest.raises(ValueError):
            mb.MTSIntegrator(bad, pi_fractions=(1,))
    with pytest.raises(ValueError):
        mb.MTSIntegrator(0.002, pi_fractions=(1,), remove_CM_motion=-1)
    assert mb.MTSIntegrator(0.002, pi_fractions=(1,), remove_CM_motion=False).remove_CM_motion == 0
    for T, g in ((-1.0, 1.0), (math.nan, 1.0), (300.0, -1.0), (300.0, math.inf)):
        with pytest.raises(ValueError):
            mb.MTSLangevinIntegrator(0.002, T, g, pi_fractions=(1,))
    sim = mb.MTSLangevinIntegrator(0.004, 300.0, 10.0, pi_fractions=(1,), si_fractions=(4, 2))
    c = math.exp(-0.004 * 10.0 / 4)  # exp(-dt friction / last(ordered_fractions)), src/simulators.jl:1751-1753
    assert sim.vel_scale == c and sim.noise_scale == math.sqrt(1 - c * c)


def test_params_layout_matches_header(tmp_path):
    P = mb.capi.MBMTSParams
    fields = [f[0] for f in P._fields_]
    offsets = {f: getattr(P, f).offset for f in fields}
    assert mb.capi.MB_MTS_MAX_LEVELS == 8 and C.sizeof(P) == 104
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "mollyb200.h"\nint main(void) {\n'
                   + "".join(f'    printf("{f} %zu\\n", offsetof(mb_mts_params_t, {f}));\n' for f in fields)
                   + '    printf("size %zu max %d\\n", sizeof(mb_mts_params_t), MB_MTS_MAX_LEVELS);\n    return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    out = dict(line.split(" ", 1) for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert {f: int(out[f]) for f in fields} == offsets
    assert out["size"] == f"{C.sizeof(P)} max 8"


def test_exports():
    L = mb.capi.load()
    for name in ("mb_simulate_mts", "mb_set_specific_levels"):
        assert name in mb.capi.EXPORTED and hasattr(L, name)


def _chain(n=6, seed=0):
    """A zigzag chain of n carbon-like atoms in a 10 nm box: stiff bonds, soft angles and torsions (0-based indices)."""
    rng = np.random.default_rng(seed)
    x = np.array([[5.0 + 0.125 * i, 5.0 + 0.07 * (i % 2), 5.0 + 0.03 * (i % 3)] for i in range(n)])
    mass = np.full(n, 12.0)
    v = rng.normal(0, math.sqrt(mb.BOLTZMANN_K * 300.0 / 12.0), (n, 3))
    bonds = (np.array([[i, i + 1] for i in range(n - 1)]), np.tile([2.0e5, 0.15], (n - 1, 1)))
    angles = (np.array([[i, i + 1, i + 2] for i in range(n - 2)]), np.tile([400.0, 1.91], (n - 2, 1)))
    tors = (np.array([[i, i + 1, i + 2, i + 3] for i in range(n - 3)]), np.tile([3.0, 0.0, 2.0], (n - 3, 1)))
    return x, v, mass, np.full(3, 10.0), bonds, angles, tors


def _terms(box, *lists):
    fns = {2: bd.bond_forces, 3: bd.angle_forces, 4: bd.torsion_forces}

    def fe(x):
        f, e = np.zeros_like(x), 0.0
        for idx, par in lists:
            ff, ee = fns[idx.shape[1]](x, box, idx, par)
            f, e = f + ff, e + ee
        return f, e
    return fe


def _wrap(box):
    return lambda y: y - np.floor(y / box) * box


def test_one_level_is_velocity_verlet():
    """fractions (1,): mts_substeps! reduces to simulate!(sys, VelocityVerlet(dt)) (src/simulators.jl:547-668)."""
    x, v, mass, box, bonds, angles, tors = _chain()
    fe = _terms(box, bonds, angles, tors)
    for rcm, init in ((1, 0), (0, 0), (3, 13)):
        xm, vm = mo.simulate_mts([lambda y: fe(y)[0]], x, v, mass, 0.0005, 50, (1,), _wrap(box), remove_cm_every=rcm, init_step=init)
        xv, vv = _wrap(box)(x.copy()), v.copy()
        if init == 0 and rcm != 0:
            vv = mo.remove_cm(vv, mass)
        f = fe(xv)[0]
        for step in range(init + 1, init + 51):
            vv = vv + f / mass[:, None] * (0.0005 / 2)
            xv = _wrap(box)(xv + vv * 0.0005)
            f = fe(xv)[0]
            vv = vv + f / mass[:, None] * (0.0005 / 2)
            if rcm and step % rcm == 0:
                vv = mo.remove_cm(vv, mass)
        assert np.abs(xm - xv).max() < 1e-14 and np.abs(vm - vv).max() < 1e-14


def test_two_level_energy_error_is_second_order():
    """Bonds at level 1 (two substeps), angles and torsions at level 0. Over the same 0.2 ps, the largest deviation of the
    total energy from its start value falls by about 4x when the outer step halves."""
    x, v, mass, box, bonds, angles, tors = _chain()
    fast, slow = _terms(box, bonds), _terms(box, angles, tors)

    def drift(dt):
        xs, vs, es = x, v, []
        for _ in range(int(round(0.2 / dt))):
            xs, vs = mo.simulate_mts([lambda y: slow(y)[0], lambda y: fast(y)[0]], xs, vs, mass, dt, 1, (1, 2), _wrap(box),
                                     remove_cm_every=0, init_step=1)
            es.append(fast(xs)[1] + slow(xs)[1] + 0.5 * np.sum(mass[:, None] * vs * vs))
        e0 = fast(x)[1] + slow(x)[1] + 0.5 * np.sum(mass[:, None] * v * v)
        return np.abs(np.array(es) - e0).max()
    e1, e2 = drift(0.002), drift(0.001)
    print(f"[MTS energy error] dt 2 fs: {e1:.3e}  dt 1 fs: {e2:.3e}  ratio {e1 / e2:.2f}")
    assert 3.0 < e1 / e2 < 5.0


def test_counts_and_langevin_draws():
    """Level l > 0 is evaluated fractions[l] + fractions[l - 1] times per outer step, level 0 once (plus the start); the
    Langevin restatement draws once per innermost substep with the MTS counter."""
    x, v, mass, box, bonds, angles, tors = _chain()
    fe = [lambda y: _terms(box, angles)(y)[0], lambda y: _terms(box, tors)(y)[0], lambda y: _terms(box, bonds)(y)[0]]
    counts = []
    mo.simulate_mts(fe, x, v, mass, 0.002, 5, (1, 2, 4), _wrap(box), counts=counts)
    assert counts == [5 + 1, 5 * (2 + 1), 5 * (4 + 2)]
    rng = (11, 12, 13, 14)
    a = mo.normals(7, 3, 6, rng)
    b = mo.normals(7, 2, 6, rng)
    assert a.shape == (6, 3) and not np.allclose(a, b)
    # friction 0: the noise vanishes and the run equals MTSIntegrator
    xa, va = mo.simulate_mts(fe, x, v, mass, 0.002, 5, (1, 2, 4), _wrap(box), langevin=(2.5, 0.0, rng))
    xb, vb = mo.simulate_mts(fe, x, v, mass, 0.002, 5, (1, 2, 4), _wrap(box))
    assert np.abs(xa - xb).max() < 1e-13 and np.abs(va - vb).max() < 1e-10  # (two half drifts: rounding only)


def _protein_like():
    """bonds, angles, propers and impropers as four lists (the last two of one kind, as in a force field setup)."""
    x, v, mass, box, bonds, angles, tors = _chain(8)
    atoms = mb.atoms_from_arrays(mass, np.zeros(len(x)), np.full(len(x), 0.3), np.full(len(x), 0.2), np.float64)
    b, a, t = bonds[0] + 1, angles[0] + 1, tors[0] + 1
    lists = (mb.InteractionList2Atoms(b[:, 0], b[:, 1], bonds[1][:, 0], bonds[1][:, 1]),
             mb.InteractionList3Atoms(a[:, 0], a[:, 1], a[:, 2], angles[1][:, 0], angles[1][:, 1]),
             mb.InteractionList4Atoms(t[:3, 0], t[:3, 1], t[:3, 2], t[:3, 3], *tors[1][:3].T),
             mb.InteractionList4Atoms(t[3:, 0], t[3:, 1], t[3:, 2], t[3:, 3], *tors[1][3:].T))
    return mb.System(atoms=atoms, coords=x, velocities=v, boundary=mb.CubicBoundary(10.0),
                     pairwise_inters=(mb.LennardJones(cutoff=mb.DistanceCutoff(1.0)),), specific_inter_lists=lists,
                     general_inters=(mb.LJDispersionCorrection(1.0),), dtype=np.float64)


def test_list_levels_follow_the_by_kind_concatenation():
    s = _protein_like()
    sim = mb.MTSIntegrator(0.002, pi_fractions=(1,), si_fractions=(4, 2, 1, 2), gi_fractions=(8,))
    assert sim.ordered_fractions == (1, 2, 4, 8)
    lv = mb.mts_levels(s, sim)
    assert sorted(lv) == [0, 1, 2]
    assert lv[0].tolist() == [2] * 7                 # bonds: fraction 4
    assert lv[1].tolist() == [1] * 6                 # angles: fraction 2
    assert lv[2].tolist() == [0] * 3 + [1] * 2       # propers (fraction 1), then impropers (fraction 2)
    assert all(a.dtype == np.int32 and a.flags["C_CONTIGUOUS"] for a in lv.values())


def test_simulate_refusals_before_any_work():
    s = _protein_like()
    x, v = s.coords.copy(), s.velocities.copy()
    cases = [(ValueError, mb.MTSIntegrator(0.002, pi_fractions=(1, 1), si_fractions=(2, 2, 1, 1), gi_fractions=(1,))),
             (ValueError, mb.MTSIntegrator(0.002, pi_fractions=(1,), si_fractions=(2, 2, 1), gi_fractions=(1,))),
             (ValueError, mb.MTSIntegrator(0.002, pi_fractions=(1,), si_fractions=(2, 2, 1, 1))),
             (TypeError, mb.MTSIntegrator(0.002, pi_fractions=(2,), si_fractions=(2, 2, 1, 1), gi_fractions=(1,))),
             (TypeError, mb.MTSIntegrator(0.002, pi_fractions=(1,), si_fractions=(2, 2, 1, 1), gi_fractions=(1,),
                                          coupling=mb.AndersenThermostat(300.0, 0.1))),
             (TypeError, mb.MTSLangevinIntegrator(0.002, 300.0, 1.0, pi_fractions=(1,), si_fractions=(2, 2, 1, 1),
                                                  gi_fractions=(1,), coupling=mb.BerendsenThermostat(300.0, 0.1)))]
    for exc, sim in cases:
        with pytest.raises(exc):
            mb.simulate(s, sim, 10)
        assert s._ctx is None and np.array_equal(x, s.coords) and np.array_equal(v, s.velocities)
    with pytest.raises(TypeError):
        mb.simulate(s, mb.MTSIntegrator(0.002, pi_fractions=(1,), si_fractions=(2, 2, 1, 1), gi_fractions=(1,)))  # no n_steps
    # PME at an inner level
    pme = mb.System(atoms=s.atoms, coords=s.coords, velocities=s.velocities, boundary=s.boundary,
                    pairwise_inters=(mb.CoulombEwald(dist_cutoff=1.0),), general_inters=(mb.PME(dist_cutoff=1.0),), dtype=np.float64)
    with pytest.raises(TypeError, match="PME"):
        mb.simulate(pme, mb.MTSIntegrator(0.002, pi_fractions=(1,), gi_fractions=(2,)), 10)
    assert pme._ctx is None
