"""CPU tests of LangevinSplitting: the force evaluations per step of the numpy restatement (tests/langevin_splitting_oracle.py)
against counts derived by hand from the reference's rule, the constructor's validation, simulate's refusals, the C-ABI
parameter layout against the header, and the oracle's equivalences ("BAB" is VelocityVerlet, "BAOA" is Langevin). The GPU
counterpart is tests/test_gpu_langevin_splitting.py."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import langevin_oracle as lo
import langevin_splitting_oracle as so
import mollyb200 as mb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Forces are known at the start of a step unless an A follows the last B; an A makes them unknown; a B recomputes only when
# they are unknown.
EVALS = {"BAOAB": 1, "OBABO": 1, "ABOBA": 1, "BAOA": 1, "BAB": 1, "BABAB": 2, "AB": 1, "BA": 1, "O": 0, "A": 0, "AOA": 0,
         "B": 0, "OBO": 0, "ABAB": 2, "BBAA": 1, "AOBOA": 1}


@pytest.mark.parametrize("splitting", list(EVALS))
def test_evaluations_per_step(splitting):
    assert so.evaluations_per_step(splitting) == EVALS[splitting]
    calls, count = [0], []
    x0 = np.array([[0.5, 0.5, 0.5], [1.0, 1.2, 0.9]])

    def fe(x):
        calls[0] += 1
        return np.zeros_like(x)

    so.simulate_splitting(fe, x0, np.zeros_like(x0), [1.0, 2.0], 0.002, 5, 2.5, 1.0, splitting, (1, 2, 3, 4), lambda x: x,
                          count=count)
    assert count == [EVALS[splitting]] * 5
    assert calls[0] == 1 + 5 * EVALS[splitting]  # (the initial evaluation before the loop)


def test_recompute_letters():
    assert so.force_computation_steps("BAOAB") == [False, False, False, False, True]
    assert so.force_computation_steps("BAOA") == [True, False, False, False]
    assert so.force_computation_steps("BABAB") == [False, False, True, False, True]
    assert so.force_computation_steps("ABOBA") == [False, True, False, False, False]


def test_constructor():
    s = mb.LangevinSplitting(dt=0.002, temperature=300.0, friction=10.0, splitting="BAOAB")
    assert (s.splitting, s.remove_CM_motion) == ("BAOAB", 1)
    assert mb.LangevinSplitting(0.002, 300.0, 10.0, "O", remove_CM_motion=False).remove_CM_motion == 0
    assert mb.LangevinSplitting(0.002, 300.0, 0.0, "A" * 32).splitting == "A" * 32
    for bad in ("", "BAOAX", "baoab", "BA OA", "A" * 33):
        with pytest.raises(ValueError):
            mb.LangevinSplitting(0.002, 300.0, 10.0, bad)
    with pytest.raises(ValueError, match="only A, B, and O"):
        mb.LangevinSplitting(0.002, 300.0, 10.0, "BAC")
    for bad in (0.0, -0.001, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            mb.LangevinSplitting(bad, 300.0, 10.0, "BAOAB")
    for bad in (-1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            mb.LangevinSplitting(0.002, bad, 10.0, "BAOAB")
        with pytest.raises(ValueError):
            mb.LangevinSplitting(0.002, 300.0, bad, "BAOAB")
    with pytest.raises(ValueError):
        mb.LangevinSplitting(0.002, 300.0, 10.0, "BAOAB", remove_CM_motion=-1)
    with pytest.raises(ValueError):
        so.simulate_splitting(None, np.zeros((1, 3)), np.zeros((1, 3)), [1.0], 0.002, 1, 1.0, 1.0, "BAX", (0, 0, 0, 0), None)


def test_simulate_refusals():
    # checked before the engine is touched, so this needs no GPU
    sysd = dict(mass=[1.0, 1.0], charge=[0, 0], sigma=[0.3, 0.3], eps=[0.2, 0.2])
    s = mb.System(atoms=mb.atoms_from_arrays(**sysd, dtype=np.float64), coords=np.array([[0.1, 0.1, 0.1], [1.0, 1.0, 1.0]]),
                  boundary=mb.CubicBoundary(2.0), pairwise_inters=(mb.LennardJones(),), dtype=np.float64)
    with pytest.raises(TypeError):
        mb.simulate(s, mb.LangevinSplitting(0.001, 10.0, 1.0, "BAOAB"))  # n_steps
    with pytest.raises(ValueError):
        mb.simulate(s, mb.LangevinSplitting(0.001, 10.0, 1.0, "BAOAB"), 1, run_loggers="sometimes")


def test_exports():
    L = mb.capi.load()
    assert "mb_simulate_langevin_splitting" in mb.capi.EXPORTED and hasattr(L, "mb_simulate_langevin_splitting")


def test_params_layout_matches_header(tmp_path):
    P = mb.capi.MBSplittingParams
    fields = [f[0] for f in P._fields_]
    offsets = {f: getattr(P, f).offset for f in fields}
    assert mb.capi.MB_SPLIT_MAX_OPS == 32 and C.sizeof(P) == 104
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "mollyb200.h"\nint main(void) {\n'
                   + "".join(f'    printf("{f} %zu\\n", offsetof(mb_splitting_params_t, {f}));\n' for f in fields)
                   + '    printf("size %zu max %d\\n", sizeof(mb_splitting_params_t), MB_SPLIT_MAX_OPS);\n    return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    out = dict(line.split(" ", 1) for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert {f: int(out[f]) for f in fields} == offsets
    assert out["size"] == f"{C.sizeof(P)} max 32"


def _harmonic(x):
    """A stiff pair potential between neighbours of a short chain: a force field with real dynamics for the equivalences."""
    f = np.zeros_like(x)
    for i in range(len(x) - 1):
        d = x[i + 1] - x[i]
        r = np.linalg.norm(d)
        g = 500.0 * (r - 0.15) * d / r
        f[i] += g
        f[i + 1] -= g
    return f


def _chain():
    rng = np.random.default_rng(3)
    x = np.array([[1.0 + 0.15 * i, 1.0 + 0.02 * (i % 2), 1.0] for i in range(6)]) + rng.normal(0, 0.01, (6, 3))
    return x, rng.normal(0, 0.5, (6, 3)), np.array([12.0, 1.0, 16.0, 14.0, 12.0, 2.0])


def test_bab_is_velocity_verlet():
    x0, v0, m = _chain()
    ident = lambda y: y  # noqa: E731
    x, v = so.simulate_splitting(_harmonic, x0, v0, m, 0.001, 50, 2.5, 10.0, "BAB", (1, 2, 3, 4), ident, remove_cm_every=0)
    xr, vr = x0.copy(), v0.copy()
    f = _harmonic(xr)
    for _ in range(50):
        vr = vr + f / m[:, None] * 0.0005
        xr = xr + vr * 0.001
        f = _harmonic(xr)
        vr = vr + f / m[:, None] * 0.0005
    assert np.abs(x - xr).max() < 1e-13 and np.abs(v - vr).max() < 1e-12


def test_baoa_is_langevin_with_equal_masses():
    """friction gamma in ps^-1 for Langevin is m gamma for LangevinSplitting; with equal masses the two steps coincide."""
    x0, v0, _ = _chain()
    m = np.full(6, 10.0)
    ident = lambda y: y  # noqa: E731
    rng = (5, 6, 7, 8)
    xa, va = lo.simulate_langevin(_harmonic, x0, v0, m, 0.002, 40, 2.5, 1.0, rng, ident)
    xb, vb = so.simulate_splitting(_harmonic, x0, v0, m, 0.002, 40, 2.5, 10.0, "BAOA", rng, ident)
    assert np.abs(xa - xb).max() < 1e-12 and np.abs(va - vb).max() < 1e-10


def test_o_only_moments_exact():
    """Splitting "O" on free particles: v_n = c^n v_0 + noise with Var = kT/m (1 - c^(2n)), c = exp(-friction dt / m)."""
    n, m, kT, fr, dt = 20000, 4.0, 2.5, 10.0, 0.002
    v0 = np.tile([0.3, -0.2, 0.1], (n, 1))
    x, v = so.simulate_splitting(lambda y: np.zeros_like(y), np.zeros((n, 3)), v0, np.full(n, m), dt, 5, kT, fr, "O",
                                 (1, 0, 9, 9), lambda y: y, remove_cm_every=0)
    c = math.exp(-fr * dt / m)
    d = v - c ** 5 * v0
    var = kT / m * (1 - c ** 10)
    assert abs(d.mean()) < 5 * math.sqrt(var / d.size)
    assert abs(d.var() / var - 1) < 5 * math.sqrt(2 / d.size)
    assert not x.any()
