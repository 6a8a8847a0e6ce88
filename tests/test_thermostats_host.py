"""The velocity-rescaling thermostats' device arithmetic (csrc/vrescale.cuh) compiled for the HOST and checked against the
numpy restatement in tests/thermostat_oracle.py and against the distributions it must sample; the Python constructors and
simulate's refusals. The GPU counterpart is tests/test_gpu_thermostats.py."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import mollyb200 as mb
import thermostat_oracle as tho

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = [(0, 0), (1, 2), (0x0123456789ABCDEF, 0x7EDCBA9876543210), (2 ** 63 - 1, 12345), (987654321987, 2 ** 40 + 17)]


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = str(tmp_path_factory.mktemp("thermoh") / "libthermoh.so")
    p = subprocess.run([nvcc, "-std=c++17", "-O2", "-shared", "-Xcompiler", "-fPIC", "-ccbin", "/usr/bin/g++", "-gencode",
                        "arch=compute_90a,code=sm_90a", "-o", out, os.path.join(ROOT, "tests", "host", "thermostat_host.cu")],
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-3000:]
    L = C.CDLL(out)
    u32p, dp = C.POINTER(C.c_uint32), C.POINTER(C.c_double)
    L.thh_block.argtypes = [C.c_uint32, C.c_uint32, u32p, u32p]
    L.thh_normal.argtypes = [C.c_uint32, C.c_uint32]
    L.thh_normal.restype = C.c_double
    L.thh_chi2.argtypes = [C.c_longlong, C.c_longlong, C.c_uint32, u32p, dp]
    L.thh_lambda.argtypes = [C.c_int, C.c_int, C.c_longlong, C.c_double, C.c_double, C.c_double, C.c_double, C.c_longlong,
                             C.c_longlong, u32p, dp]
    return L


def _rng(ctr1, key):
    return (C.c_uint32 * 4)(*tho.rng_words(ctr1, key))


def _chi2(L, k, count, step0, rng):
    out = np.zeros(count)
    L.thh_chi2(k, count, step0, rng, out.ctypes.data_as(C.POINTER(C.c_double)))
    return out


def _lambda(L, kind, nf, kT, dt, K, tau=0.0, n_steps=1, step0=0, count=1, rng=None):
    out = np.zeros(count)
    L.thh_lambda(kind, n_steps, nf, kT, dt, tau, K, step0, count, rng or _rng(0, 0), out.ctypes.data_as(C.POINTER(C.c_double)))
    return out


def test_philox_blocks_match_numpy_bit_for_bit(hostlib):
    steps = np.array([0, 1, 2, 77, 2 ** 31 + 5, 2 ** 32 - 1], np.uint64)
    for ctr1, key in KEYS:
        rng = _rng(ctr1, key)
        for j in (0, 1, 2, 63, 64):
            ref = tho.block(j, steps, tho.rng_words(ctr1, key))
            for i, s in enumerate(steps):
                w = (C.c_uint32 * 4)()
                hostlib.thh_block(j, int(s), rng, w)
                assert list(w) == [int(r[i]) for r in ref]
    # the Philox rounds themselves: the published known-answer vector of Philox4x32-10 (Random123, kat_vectors)
    w = tho.philox4x32_10([0xFFFFFFFF] * 4, 0xFFFFFFFF, 0xFFFFFFFF)
    assert [int(x) for x in w] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]


def test_normal_and_chi2_draws_match_numpy(hostlib):
    r = np.random.default_rng(0)
    for a, b in r.integers(0, 2 ** 32, (2000, 2)):
        assert abs(hostlib.thh_normal(int(a), int(b)) - tho.normal(a, b)) <= 1e-12 * max(1.0, abs(tho.normal(a, b)))
    for a, b in ((0xFFFFFFFF, 0), (0, 0), (0, 0x80000000)):  # the ends of the Box-Muller inputs are finite
        assert math.isfinite(hostlib.thh_normal(a, b))
    for ctr1, key in KEYS[1:4]:
        words = tho.rng_words(ctr1, key)
        for k in (1, 2, 3, 5, 40, 299, 767999):
            got = _chi2(hostlib, k, 300, 1000, _rng(ctr1, key))
            ref = np.array([tho.chi2(k, 1000 + i, words) for i in range(300)])
            np.testing.assert_allclose(got, ref, rtol=1e-12, atol=0)


@pytest.mark.parametrize("k", [1, 2, 5, 300, 767999])
def test_chi2_moments(hostlib, k):
    # 10^6 draws: sample mean within 5 sigma of k (sigma^2 = 2k / N) and sample variance within 5 sigma of 2k, the variance
    # of the sample variance being (mu4 - sigma^4) / N = (12 k (k + 4) - 4 k^2) / N for chi^2_k
    N = 1_000_000
    x = _chi2(hostlib, k, N, 3, _rng(0x5EED, 0xC0FFEE + k))
    assert (x >= 0).all() and np.isfinite(x).all()
    assert abs(x.mean() - k) < 5 * math.sqrt(2 * k / N)
    assert abs(x.var() - 2 * k) < 5 * math.sqrt((12 * k * (k + 4) - 4 * k * k) / N)


@pytest.mark.parametrize("k", [1, 2, 5])
def test_chi2_ks_small_k(hostlib, k):
    from scipy import stats
    x = _chi2(hostlib, k, 200_000, 11, _rng(97, 31 + k))
    assert stats.kstest(x, stats.chi2(k).cdf).pvalue > 1e-4


@pytest.mark.parametrize("nf,c_tau", [(297, 0.1), (2, 0.01), (3 * 864 - 3, 1.0)])
def test_bussi_kinetic_energy_moments(hostlib, nf, c_tau):
    # For fixed K, K' = lambda^2 K = c K + (1-c) (Kbar/Nf) chi^2_Nf + 2 sqrt(c (1-c) K Kbar / Nf) R with R^2 + S ~ chi^2_Nf and
    # E[R^3] = 0: E[K'] = c K + (1-c) Kbar, Var[K'] = 2 Nf (1-c)^2 (Kbar/Nf)^2 + 4 c (1-c) K Kbar / Nf
    N, dt, kT = 200_000, 0.002, 0.8
    kbar = nf * kT / 2
    K = 1.7 * kbar
    c = math.exp(-dt / c_tau)
    lam = _lambda(hostlib, tho.VRESCALE, nf, kT, dt, K, tau=c_tau, step0=1, count=N, rng=_rng(4242, nf))
    kp = lam * lam * K
    mean, var = c * K + (1 - c) * kbar, 2 * nf * (1 - c) ** 2 * (kbar / nf) ** 2 + 4 * c * (1 - c) * K * kbar / nf
    m4 = np.mean((kp - kp.mean()) ** 4)
    assert abs(kp.mean() - mean) < 5 * math.sqrt(var / N)
    assert abs(kp.var() - var) < 5 * math.sqrt((m4 - kp.var() ** 2) / N)


def test_lambda_edge_cases(hostlib):
    r = np.random.default_rng(5)
    rng = _rng(11, 22)
    words = tho.rng_words(11, 22)
    for _ in range(200):  # Immediate and Berendsen against numpy
        nf, kT, K, dt, tau = int(r.integers(1, 10 ** 6)), r.uniform(0.01, 5), r.uniform(0.01, 1e5), r.uniform(1e-4, 4e-3), r.uniform(0.01, 2)
        for kind in (tho.IMMEDIATE, tho.BERENDSEN):
            got = _lambda(hostlib, kind, nf, kT, dt, K, tau=tau, rng=rng)[0]
            assert abs(got - tho.lam(kind, K, nf, kT, dt, tau)) <= 1e-14 * got
    # K = 0 (or nf = 0) leaves the velocities unchanged, for every kind; so does a step Bussi skips
    for kind in (tho.IMMEDIATE, tho.BERENDSEN, tho.VRESCALE):
        assert _lambda(hostlib, kind, 297, 0.1, 0.001, 0.0, tau=0.1)[0] == 1.0
        assert _lambda(hostlib, kind, 0, 0.1, 0.001, 5.0, tau=0.1)[0] == 1.0
    assert (_lambda(hostlib, tho.VRESCALE, 297, 0.1, 0.001, 5.0, tau=0.1, n_steps=5, step0=1, count=4) == 1.0).all()
    # Nf = 1 (S = 0) and Nf = 2 (chi^2_1: the shape < 1 boost) against numpy
    for nf in (1, 2):
        got = _lambda(hostlib, tho.VRESCALE, nf, 0.1, 0.001, 0.07, tau=0.05, step0=40, count=200, rng=rng)
        ref = [tho.lam(tho.VRESCALE, 0.07, nf, 0.1, 0.001, 0.05, 1, 40 + i, words) for i in range(200)]
        np.testing.assert_allclose(got, ref, rtol=1e-12)
    # the floor: Nf = 1 makes lambda^2 = (sqrt(c) + sqrt((1-c) A) R)^2; choose A so that it cancels at a step with R < 0
    step = next(s for s in range(1, 100) if tho.normal(*tho.block(0, s, words)[:2]) < -0.5)
    R = tho.normal(*tho.block(0, step, words)[:2])
    dt, tau, kT = 0.001, 0.1, 0.2
    c = math.exp(-dt / tau)
    K = (kT / 2) * (1 - c) * R * R / c  # A = Kbar / K = c / ((1 - c) R^2)
    got = _lambda(hostlib, tho.VRESCALE, 1, kT, dt, K, tau=tau, step0=step, rng=rng)[0]
    assert math.sqrt(np.finfo(np.float64).eps) <= got < 1e-6
    assert math.sqrt(np.finfo(np.float64).eps) <= tho.lam(tho.VRESCALE, K, 1, kT, dt, tau, 1, step, words) < 1e-6


def test_constructors_validate():
    for bad in (-1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            mb.ImmediateThermostat(bad)
        with pytest.raises(ValueError):
            mb.BerendsenThermostat(bad, 0.1)
        with pytest.raises(ValueError):
            mb.VelocityRescaleThermostat(bad, 0.1)
    for bad in (0.0, -0.1, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            mb.BerendsenThermostat(10.0, bad)
        with pytest.raises(ValueError):
            mb.VelocityRescaleThermostat(10.0, bad)
    for bad in (0, -3, 1.5, True):
        with pytest.raises(ValueError):
            mb.VelocityRescaleThermostat(10.0, 0.1, n_steps=bad)
    t = mb.VelocityRescaleThermostat(300.0, 0.1)
    assert t.n_steps == 1
    d = t.descriptor(mb.BOLTZMANN_K)
    assert (d.kind, d.n_steps, d.kT, d.tau) == (mb.capi.MB_VC_VRESCALE, 1, mb.BOLTZMANN_K * 300.0, 0.1)
    assert C.sizeof(mb.capi.MBVCoupling) == 24
    assert mb.ImmediateThermostat(0.0).descriptor(mb.BOLTZMANN_K).kind == mb.capi.MB_VC_IMMEDIATE
    assert mb.BerendsenThermostat(10.0, 0.5).descriptor(mb.BOLTZMANN_K).kind == mb.capi.MB_VC_BERENDSEN


def test_simulate_refuses_combinations():
    # checked before the engine is touched, so this needs no GPU
    sysd = dict(mass=[1.0, 1.0], charge=[0, 0], sigma=[0.3, 0.3], eps=[0.2, 0.2])
    s = mb.System(atoms=mb.atoms_from_arrays(**sysd, dtype=np.float64), coords=np.array([[0.1, 0.1, 0.1], [1.0, 1.0, 1.0]]),
                  boundary=mb.CubicBoundary(2.0), pairwise_inters=(mb.LennardJones(),), dtype=np.float64)
    imm, ber, vr = mb.ImmediateThermostat(10.0), mb.BerendsenThermostat(10.0, 0.1), mb.VelocityRescaleThermostat(10.0, 0.1)
    for coupling in ((imm, mb.AndersenThermostat(10.0, 0.1)), (mb.AndersenThermostat(10.0, 0.1), vr), (vr, vr), [ber, imm],
                     (object(),)):
        with pytest.raises(TypeError):
            mb.simulate(s, mb.VelocityVerlet(dt=0.001, coupling=coupling), 1)
