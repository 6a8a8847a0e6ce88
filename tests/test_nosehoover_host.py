"""The Nose-Hoover zeta update (nh_zeta_step, csrc/nosehoover.cuh) compiled for the HOST and checked against the numpy
restatement in tests/nosehoover_oracle.py; the NoseHoover constructor, the C-ABI parameter layout and simulate's refusals.
The GPU counterpart is tests/test_gpu_nosehoover.py."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import mollyb200 as mb
import nosehoover_oracle as nho

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = str(tmp_path_factory.mktemp("nosehooverh") / "libnosehooverh.so")
    p = subprocess.run([nvcc, "-std=c++17", "-O2", "-shared", "-Xcompiler", "-fPIC", "-ccbin", "/usr/bin/g++", "-gencode",
                        "arch=compute_90a,code=sm_90a", "-o", out, os.path.join(ROOT, "tests", "host", "nosehoover_host.cu")],
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-3000:]
    L = C.CDLL(out)
    L.nhh_zeta.argtypes = [C.c_double, C.c_longlong, C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_void_p]
    return L


@pytest.mark.parametrize("dt,damping,n_atoms,kT", [(0.002, 0.2, 256, 0.8314), (0.0005, 0.05, 2, 2.494), (0.004, 1.0, 10 ** 6, 0.1)])
def test_zeta_update_matches_numpy(hostlib, dt, damping, n_atoms, kT):
    """A sequence of 500 steps with kinetic sums scattered around equipartition (and far from it), zeta carried over from
    one step to the next: every value to 1e-15 relative (or 1e-15 of the step's coefficient where zeta crosses 0)."""
    rng = np.random.default_rng(n_atoms)
    count = 500
    nf_kT = (3 * n_atoms - 3) * kT
    mv2_old = nf_kT * rng.uniform(0.2, 3.0, count)
    mv2_half = mv2_old * rng.uniform(0.9, 1.1, count)
    out = np.zeros(count)
    coef = dt / (2 * damping * damping)
    hostlib.nhh_zeta(0.0, count, mv2_old.ctypes.data, mv2_half.ctypes.data, coef, nf_kT, out.ctypes.data)
    z, ref = 0.0, np.zeros(count)
    for k in range(count):
        z = ref[k] = nho.zeta_step(z, mv2_old[k], mv2_half[k], dt, damping, nf_kT)
    assert np.all(np.abs(out - ref) <= 1e-15 * np.maximum(np.abs(ref), coef))
    # at equipartition in both halves zeta does not move
    hostlib.nhh_zeta(0.25, 1, np.array([nf_kT]).ctypes.data, np.array([nf_kT]).ctypes.data, coef, nf_kT, out.ctypes.data)
    assert out[0] == 0.25


def test_constructor():
    s = mb.NoseHoover(dt=0.002, temperature=100.0)
    assert s.damping == 100 * 0.002 and (s.coupling, s.remove_CM_motion) == (None, 1)
    assert mb.NoseHoover(0.001, 10.0, 0.5).damping == 0.5
    assert mb.NoseHoover(0.001, 10.0, remove_CM_motion=False).remove_CM_motion == 0
    for bad in (0.0, -0.001, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            mb.NoseHoover(bad, 300.0)
        with pytest.raises(ValueError):
            mb.NoseHoover(0.002, 300.0, damping=bad)
    for bad in (0.0, -1.0, float("nan"), float("inf")):  # T0 = 0: T / T0 is infinite
        with pytest.raises(ValueError):
            mb.NoseHoover(0.002, bad)
    with pytest.raises(ValueError):
        mb.NoseHoover(0.002, 300.0, remove_CM_motion=-1)


def test_params_layout():
    P = mb.capi.MBNoseHooverParams
    assert C.sizeof(P) == 48
    assert [(f, getattr(P, f).offset) for f, _ in P._fields_] == [
        ("dt", 0), ("n_steps", 8), ("init_step", 16), ("remove_cm_every", 24), ("kT", 32), ("damping", 40)]
    assert "mb_simulate_nose_hoover" in mb.capi.EXPORTED


def test_simulate_refusals():
    # checked before the engine is touched, so this needs no GPU
    sysd = dict(mass=[1.0, 1.0], charge=[0, 0], sigma=[0.3, 0.3], eps=[0.2, 0.2])
    s = mb.System(atoms=mb.atoms_from_arrays(**sysd, dtype=np.float64), coords=np.array([[0.1, 0.1, 0.1], [1.0, 1.0, 1.0]]),
                  boundary=mb.CubicBoundary(2.0), pairwise_inters=(mb.LennardJones(),), dtype=np.float64)
    for coupling in (mb.BerendsenThermostat(10.0, 0.1), (mb.AndersenThermostat(10.0, 0.1),), mb.VelocityRescaleThermostat(10.0, 0.1),
                     [object()]):
        with pytest.raises(TypeError):
            mb.simulate(s, mb.NoseHoover(0.001, 10.0, coupling=coupling), 1)
    with pytest.raises(TypeError):
        mb.simulate(s, mb.NoseHoover(0.001, 10.0))  # n_steps
    with pytest.raises(ValueError):
        mb.simulate(s, mb.NoseHoover(0.001, 10.0), 1, run_loggers="sometimes")
    assert math.isclose(mb.NoseHoover(0.001, 10.0).damping, 0.1)
