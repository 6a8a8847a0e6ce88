"""The DPD pair term and pairwise draw (dpd_pair, dpd_normal of csrc/dpd.cuh) compiled for the HOST and checked against
the reference's "DPD interaction" testset (test/interactions.jl:1763-1868) and, to the last bit in f64, against
tests/dpd_oracle.py; the C-ABI layouts and the Python validation of DPDInteraction and DPDVelocityVerlet. The GPU
counterpart is tests/test_gpu_dpd.py."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import dpd_oracle as do
import mollyb200 as mb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = str(tmp_path_factory.mktemp("dpdh") / "libdpdh.so")
    p = subprocess.run([nvcc, "-std=c++17", "-O2", "-shared", "-Xcompiler", "-fPIC", "-ccbin", "/usr/bin/g++", "-gencode",
                        "arch=compute_90a,code=sm_90a", "-o", out, os.path.join(ROOT, "tests", "host", "dpd_host.cu")],
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-3000:]
    L = C.CDLL(out)
    for name in ("dh_pair_f64", "dh_pair_f32"):
        getattr(L, name).argtypes = [C.c_int] + [C.c_void_p] * 7
    L.dh_normal.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ulonglong, C.c_void_p]
    return L


def _pair(L, par, r, d, dv, xi, dtype=np.float64):
    r, xi = np.ascontiguousarray(np.atleast_1d(r), np.float64), np.ascontiguousarray(np.atleast_1d(xi), np.float64)
    d, dv = np.ascontiguousarray(np.reshape(d, (-1, 3)), np.float64), np.ascontiguousarray(np.reshape(dv, (-1, 3)), np.float64)
    pa = np.ascontiguousarray([par["a"], par["gamma"], par["sigma"], par["r_c"], par["dt"]], np.float64)
    fr, e = np.zeros(len(r), dtype), np.zeros(len(r), dtype)
    fn = L.dh_pair_f64 if dtype == np.float64 else L.dh_pair_f32
    fn(len(r), pa.ctypes.data, r.ctypes.data, d.ctypes.data, dv.ctypes.data, xi.ctypes.data, fr.ctypes.data, e.ctypes.data)
    return fr, e


def _normal(L, i, j, step, key):
    """xi of pairs (i, j) (0-based, broadcast together with step)"""
    i, j, step = np.broadcast_arrays(np.atleast_1d(i), np.atleast_1d(j), np.atleast_1d(step))
    i, j = np.ascontiguousarray(i, np.int32), np.ascontiguousarray(j, np.int32)
    st = np.ascontiguousarray(step, np.int64)
    out = np.zeros(len(i))
    L.dh_normal(len(i), i.ctypes.data, j.ctypes.data, st.ctypes.data, int(key), out.ctypes.data)
    return out


def _ref_force(L, par, c_i, c_j, v_i, v_j, step, i=0, j=1, box=10.0):
    """force(inter, dr, atom_i, atom_j, ..., velocity_i, velocity_j, step_n) of the reference: the vector f with
    fs[i] -= f, i.e. fr dr with dr = vector(c_i, c_j)."""
    dr = do.min_image(np.full(3, box))(np.asarray(c_i, float), np.asarray(c_j, float))
    r = math.sqrt(dr[0] * dr[0] + dr[1] * dr[1] + dr[2] * dr[2])
    xi = _normal(L, [i], [j], step, par["key"])
    fr, e = _pair(L, par, [r], -dr, np.subtract(v_i, v_j), xi)
    return fr[0] * dr, e[0]


# ---- the reference's "DPD interaction" testset ------------------------------------------------------------------------
R_C, A, GAMMA, SIGMA, DT = 2.5, 25.0, 4.5, 3.0, 0.01
INTER = dict(a=A, gamma=GAMMA, sigma=SIGMA, r_c=R_C, dt=DT, key=1)
C1, C2 = (1.0, 1.0, 1.0), (1.5, 1.0, 1.0)
ZERO = (0.0, 0.0, 0.0)


def test_conservative_force_and_energy(hostlib):
    cons = dict(INTER, sigma=0.0)
    f, pe = _ref_force(hostlib, cons, C1, C2, ZERO, ZERO, 0)
    dr = np.subtract(C2, C1)
    r = np.linalg.norm(dr)
    w = 1 - r / R_C
    assert np.allclose(f, A * w / r * dr, atol=1e-10)
    assert f[0] > 0.0
    assert abs(pe - (A / 2) * R_C * w ** 2) < 1e-10


@pytest.mark.parametrize("c", [(3.5, 1.0, 1.0), (4.0, 1.0, 1.0)])
def test_zero_at_and_beyond_cutoff(hostlib, c):
    f, pe = _ref_force(hostlib, INTER, C1, c, ZERO, ZERO, 0)
    assert np.all(f == 0.0) and pe == 0.0


def test_dissipative_signs(hostlib):
    nodiss = dict(INTER, a=0.0, sigma=0.0)
    f, _ = _ref_force(hostlib, nodiss, C1, C2, (1.0, 0.0, 0.0), ZERO, 0)  # approaching
    assert f[0] > 0.0 and abs(f[1]) < 1e-10 and abs(f[2]) < 1e-10
    f, _ = _ref_force(hostlib, nodiss, C1, C2, (-1.0, 0.0, 0.0), ZERO, 0)  # receding
    assert f[0] < 0.0


def test_pair_forces_equal_and_opposite_along_the_line(hostlib):
    c5, v5, v6 = (1.2, 1.3, 1.6), (0.5, -0.2, 0.1), (-0.3, 0.4, 0.2)
    f_ij, _ = _ref_force(hostlib, INTER, C1, c5, v5, v6, 7, 0, 1)
    f_ji, _ = _ref_force(hostlib, INTER, c5, C1, v6, v5, 7, 1, 0)
    assert np.array_equal(f_ij, -f_ji)
    assert np.any(f_ij != 0)
    dr = np.subtract(c5, C1)
    assert abs(abs(f_ij @ dr) - np.linalg.norm(f_ij) * np.linalg.norm(dr)) < 1e-10


def test_draw_symmetric(hostlib):
    for step in range(1, 11):  # dpd_gaussian(1, 2, step, 1) == dpd_gaussian(2, 1, step, 1), 1-based
        assert _normal(hostlib, [0], [1], step, 1)[0] == _normal(hostlib, [1], [0], step, 1)[0]
        assert _normal(hostlib, [4], [12], step, 1)[0] == _normal(hostlib, [12], [4], step, 1)[0]


def test_draw_covariance(hostlib):
    """The reference's 7 x 7 covariance check on the engine's draw (1-based indices of the reference minus one)."""
    n = 100000
    s = np.arange(1, n + 1)
    cols = [
        _normal(hostlib, 0, 1, s, 1), _normal(hostlib, 0, 2, s, 1), _normal(hostlib, 0, 1, s, 2),
        _normal(hostlib, np.arange(5, n + 5) - 1, 0, 1, 2),
        _normal(hostlib, np.arange(5, n + 5) - 1, 1, 1, 2),
        _normal(hostlib, s - 1, 9999999, 1, 2),
        _normal(hostlib, s - 1, 10000000, 1, 2),
    ]
    cov = np.cov(np.stack(cols))
    assert np.all(np.abs(np.diag(cov) - 1.0) < 0.02), np.diag(cov)
    off = cov - np.diag(np.diag(cov))
    assert np.all(np.abs(off) < 0.02), off


# ---- engine-specific checks ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_coincident_beads_give_zero(hostlib, dtype):
    fr, e = _pair(hostlib, INTER, [0.0], ZERO, (1.0, 2.0, 3.0), [0.7], dtype)
    assert fr[0] == 0.0 and e[0] == 0.0 and np.isfinite(fr[0])


def test_conservative_force_is_minus_gradient(hostlib):
    """gamma = sigma = 0: the force on i is -dE/dc_i by central differences."""
    par = dict(INTER, gamma=0.0, sigma=0.0)
    rng = np.random.default_rng(4)
    h = 1e-6
    for _ in range(20):
        d = rng.uniform(-1.4, 1.4, 3)
        r = np.linalg.norm(d)
        if r >= R_C or r < 0.05:
            continue
        fr, _ = _pair(hostlib, par, [r], d, ZERO, [0.0])
        grad = np.zeros(3)
        for k in range(3):
            dp, dm = d.copy(), d.copy()
            dp[k] += h
            dm[k] -= h
            ep = _pair(hostlib, par, [np.linalg.norm(dp)], dp, ZERO, [0.0])[1][0]
            em = _pair(hostlib, par, [np.linalg.norm(dm)], dm, ZERO, [0.0])[1][0]
            grad[k] = (ep - em) / (2 * h)  # dE/dd = dE/dc_i
        assert np.allclose(fr[0] * d, -grad, rtol=1e-6, atol=1e-7)


def test_pair_and_draw_match_oracle_bitwise(hostlib):
    """f64: the host-compiled pair term and draw equal the oracle's restatement to the last bit."""
    rng = np.random.default_rng(11)
    m = 4000
    par = dict(a=25.0, gamma=4.5, sigma=3.0, r_c=1.0, dt=0.04, key=0x9E3779B97F4A7C15)
    d = rng.uniform(-0.8, 0.8, (m, 3))
    r = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])
    r[:5] = 0.0
    dv = rng.normal(0, 1, (m, 3))
    i, j = rng.integers(0, 1 << 20, m), rng.integers(0, 1 << 20, m)
    for step in (0, 1, 12345, (1 << 32) + 7):
        xi_e = _normal(hostlib, i, j, step, par["key"])
        xi_o = do.normal(i, j, step, par["key"])
        assert np.array_equal(xi_e, xi_o)
    fr_e, e_e = _pair(hostlib, par, r, d, dv, xi_e)
    fr_o, e_o = do.pair(par, r, d, dv, xi_o)
    assert np.array_equal(fr_e, fr_o) and np.array_equal(e_e, e_o)
    fr32, _ = _pair(hostlib, par, r, d, dv, xi_e, np.float32)
    assert np.allclose(fr32, fr_o, rtol=2e-5, atol=2e-5 * np.abs(fr_o).max())


# ---- C ABI and Python validation -------------------------------------------------------------------------------------------
def test_abi_layouts():
    assert C.sizeof(mb.capi.MBDpd) == 56
    assert [f for f, _ in mb.capi.MBDpd._fields_] == ["a", "gamma", "sigma", "r_c", "dt", "key", "use_neighbors"]
    assert mb.capi.MBDpd.key.offset == 40 and mb.capi.MBDpd.use_neighbors.offset == 48
    assert C.sizeof(mb.capi.MBDpdVVParams) == 40
    assert [f for f, _ in mb.capi.MBDpdVVParams._fields_] == ["dt", "n_steps", "init_step", "remove_cm_every", "lambda_"]
    assert mb.capi.MBDpdVVParams.lambda_.offset == 32
    for name in ("mb_set_dpd", "mb_forces_energy_vel", "mb_simulate_dpd_vv"):
        assert name in mb.capi.EXPORTED
        assert name in open(os.path.join(ROOT, "include", "mollyb200.h")).read()


def test_python_validation():
    d = mb.DPDInteraction()
    assert (d.a, d.gamma, d.sigma, d.r_c, d.dt, d.use_neighbors) == (25.0, 4.5, 3.0, 1.0, 0.01, False)
    assert 0 <= d.key < 2 ** 64 and d.key != mb.DPDInteraction().key
    assert mb.DPDInteraction(key=2 ** 64 - 1).key == 2 ** 64 - 1
    for bad in (dict(r_c=0.0), dict(r_c=math.inf), dict(dt=0.0), dict(dt=-1.0), dict(gamma=-0.1), dict(sigma=math.nan),
                dict(a=math.inf), dict(key=-1), dict(key=2 ** 64), dict(key=1.5)):
        with pytest.raises(ValueError):
            mb.DPDInteraction(**bad)
    s = mb.DPDVelocityVerlet(dt=0.04)
    assert (s.lam, s.coupling, s.remove_CM_motion) == (0.65, None, 1)
    assert mb.DPDVelocityVerlet(dt=0.04, remove_CM_motion=False).remove_CM_motion == 0
    for bad in (dict(dt=0.0), dict(dt=math.nan), dict(dt=0.04, lam=math.inf), dict(dt=0.04, remove_CM_motion=-1)):
        with pytest.raises(ValueError):
            mb.DPDVelocityVerlet(**bad)


def test_oracle_without_dissipation_is_velocity_verlet():
    """gamma = sigma = 0: v_pred does not enter the forces, and the loop is VelocityVerlet's."""
    rng = np.random.default_rng(2)
    box = np.full(3, 4.0)
    x, v, m = rng.uniform(0, 4, (60, 3)), rng.normal(0, 1, (60, 3)), np.ones(60)
    p = dict(a=25.0, gamma=0.0, sigma=0.0, r_c=1.0, dt=0.02, key=5)
    x1, v1 = do.simulate_dpd_vv(x, v, m, box, p, 0.02, 0.65, 10)
    x2, v2 = do.simulate_dpd_vv(x, v, m, box, p, 0.02, 0.5, 10)
    assert np.array_equal(x1, x2) and np.array_equal(v1, v2)
