"""The Langevin O step's draws (philox4x32_10 + box_muller3, csrc/common.cuh) compiled for the HOST and checked against the
numpy restatement in tests/langevin_oracle.py; the Langevin constructor and simulate's refusals. The GPU counterpart is
tests/test_gpu_langevin.py."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import langevin_oracle as lo
import mollyb200 as mb
import thermostat_oracle as tho

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = [(0, 0), (1, 2), (0x0123456789ABCDEF, 0x7EDCBA9876543210), (2 ** 63 - 1, 12345)]


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = str(tmp_path_factory.mktemp("langevinh") / "liblangevinh.so")
    p = subprocess.run([nvcc, "-std=c++17", "-O2", "-shared", "-Xcompiler", "-fPIC", "-ccbin", "/usr/bin/g++", "-gencode",
                        "arch=compute_90a,code=sm_90a", "-o", out, os.path.join(ROOT, "tests", "host", "langevin_host.cu")],
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-3000:]
    L = C.CDLL(out)
    L.lgh_draws.argtypes = [C.c_int, C.c_uint32, C.POINTER(C.c_uint32), C.c_double, C.c_void_p, C.c_void_p]
    return L


def _draws(L, n, step, ctr1, key, sd=1.0):
    words = np.zeros((n, 4), np.uint32)
    out = np.zeros((n, 3))
    L.lgh_draws(n, step, (C.c_uint32 * 4)(*tho.rng_words(ctr1, key)), sd, words.ctypes.data, out.ctypes.data)
    return words, out


@pytest.mark.parametrize("ctr1,key", KEYS)
def test_draws_match_numpy(hostlib, ctr1, key):
    rng = tho.rng_words(ctr1, key)
    n = 3000
    for step in (1, 2, 77, 2 ** 31 + 5, 2 ** 32 - 1):
        words, out = _draws(hostlib, n, step, ctr1, key, sd=0.37)
        idx = np.arange(1, n + 1, dtype=np.uint64)
        ref = tho.philox4x32_10([idx, np.full(n, step, np.uint64), np.full(n, rng[0], np.uint64), np.full(n, rng[1], np.uint64)],
                                rng[2], rng[3])
        assert np.array_equal(words, np.stack([np.asarray(r, np.uint32) for r in ref], 1))
        np.testing.assert_allclose(out, lo.normals(step, n, rng, 0.37), rtol=1e-12, atol=1e-12)


def test_draws_are_standard_normal(hostlib):
    from scipy import stats
    _, out = _draws(hostlib, 200_000, 5, 0x5EED, 0xC0FFEE)
    for k in range(3):
        assert stats.kstest(out[:, k], "norm").pvalue > 1e-4
    assert abs(np.corrcoef(out[:, 0], out[:, 1])[0, 1]) < 5 / math.sqrt(len(out))
    # sd = 0 (massless atoms): exactly zero noise
    assert not _draws(hostlib, 100, 3, 1, 2, sd=0.0)[1].any()


def test_constructor():
    s = mb.Langevin(dt=0.002, temperature=300.0, friction=1.0)
    assert s.vel_scale == math.exp(-0.002) and s.noise_scale == math.sqrt(1 - math.exp(-0.002) ** 2)
    assert (s.coupling, s.remove_CM_motion) == (None, 1)
    assert mb.Langevin(0.001, 10.0, 0.0).vel_scale == 1.0 and mb.Langevin(0.001, 10.0, 0.0).noise_scale == 0.0
    assert mb.Langevin(0.001, 10.0, 2.0, remove_CM_motion=False).remove_CM_motion == 0
    for bad in (0.0, -0.001, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            mb.Langevin(bad, 300.0, 1.0)
    for bad in (-1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            mb.Langevin(0.002, bad, 1.0)
        with pytest.raises(ValueError):
            mb.Langevin(0.002, 300.0, bad)
    with pytest.raises(ValueError):
        mb.Langevin(0.002, 300.0, 1.0, remove_CM_motion=-1)
    assert C.sizeof(mb.capi.MBLangevinParams) == 64


def test_simulate_refusals():
    # checked before the engine is touched, so this needs no GPU
    sysd = dict(mass=[1.0, 1.0], charge=[0, 0], sigma=[0.3, 0.3], eps=[0.2, 0.2])
    s = mb.System(atoms=mb.atoms_from_arrays(**sysd, dtype=np.float64), coords=np.array([[0.1, 0.1, 0.1], [1.0, 1.0, 1.0]]),
                  boundary=mb.CubicBoundary(2.0), pairwise_inters=(mb.LennardJones(),), dtype=np.float64)
    for coupling in (mb.BerendsenThermostat(10.0, 0.1), (mb.AndersenThermostat(10.0, 0.1),), [object()]):
        with pytest.raises(TypeError):
            mb.simulate(s, mb.Langevin(0.001, 10.0, 1.0, coupling=coupling), 1)
    with pytest.raises(TypeError):
        mb.simulate(s, mb.Langevin(0.001, 10.0, 1.0))  # n_steps
    with pytest.raises(ValueError):
        mb.simulate(s, mb.Langevin(0.001, 10.0, 1.0), 1, run_loggers="sometimes")
