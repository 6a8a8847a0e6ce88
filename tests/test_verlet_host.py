"""The per-atom update of Verlet, StormerVerlet and OverdampedLangevin (verlet_update, csrc/verlet.cuh) compiled for the
HOST and checked against the numpy restatements in tests/verlet_oracle.py; two identities of the oracle; the constructors,
the C-ABI parameter layouts and simulate's refusals. The GPU counterpart is tests/test_gpu_verlet.py."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import langevin_oracle as lo
import mollyb200 as mb
import thermostat_oracle as tho
import verlet_oracle as vo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LEAPFROG, STORMER, OVERDAMPED = 0, 1, 2


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = str(tmp_path_factory.mktemp("verleth") / "libverleth.so")
    p = subprocess.run([nvcc, "-std=c++17", "-O2", "-shared", "-Xcompiler", "-fPIC", "-ccbin", "/usr/bin/g++", "-gencode",
                        "arch=compute_90a,code=sm_90a", "-o", out, os.path.join(ROOT, "tests", "host", "verlet_host.cu")],
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-3000:]
    L = C.CDLL(out)
    for name in ("vh_update_f64", "vh_update_f32"):
        getattr(L, name).argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 4 + [C.c_double, C.c_double, C.c_int, C.c_void_p]
    return L


def _update(L, kind, x, v, f, inv_m, dt, friction=0.0, first=False, g=None, dtype=np.float64):
    x, v = x.astype(dtype), v.astype(dtype)
    f, inv_m = f.astype(dtype), inv_m.astype(dtype)
    g = np.zeros(x.shape) if g is None else np.ascontiguousarray(g, np.float64)
    fn = L.vh_update_f64 if dtype == np.float64 else L.vh_update_f32
    fn(kind, len(x), x.ctypes.data, v.ctypes.data, f.ctypes.data, inv_m.ctypes.data, dt, friction, int(first), g.ctypes.data)
    return x, v


def _state(n=500, seed=3):
    r = np.random.default_rng(seed)
    mass = r.uniform(1.0, 40.0, n)
    mass[:3] = 0.0  # massless atoms
    inv_m = np.where(mass > 0, 1.0 / np.where(mass > 0, mass, 1.0), 0.0)
    return r.uniform(0, 3, (n, 3)), r.normal(0, 0.5, (n, 3)), r.normal(0, 300.0, (n, 3)), mass, inv_m


def _ident(y):
    return y


def _vec(a, b):
    return b - a


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_leapfrog_update_matches_oracle(hostlib, dtype):
    x, v, f, mass, inv_m = _state()
    dt = 0.002
    xe, ve = _update(hostlib, LEAPFROG, x, v, f, inv_m, dt, dtype=dtype)
    xr, vr = vo.simulate_verlet(lambda y: f, x, v, mass, dt, 1, _ident, remove_cm_every=0, init_step=5)
    tol = 1e-13 if dtype == np.float64 else 2e-6
    assert np.abs(xe - xr).max() < tol * 4 and np.abs(ve - vr).max() < tol * 10
    assert np.array_equal(ve[:3], v[:3].astype(dtype))  # massless: no kick


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("first", [True, False])
def test_stormer_update_matches_oracle(hostlib, dtype, first):
    """The engine's update from v = vector(x_last, x) / dt equals the reference's step from coords_last; on the first step
    of a call both start from the velocities with a dt^2 / 2."""
    x, v, f, mass, inv_m = _state()
    dt = 0.002
    xe, ve = _update(hostlib, STORMER, x, v, f, inv_m, dt, first=first, dtype=dtype)
    a = f * inv_m[:, None]
    if first:
        xr, vr = vo.simulate_stormer_verlet(lambda y: f, x, v, mass, dt, 1, _ident, _vec, init_step=3)
    else:
        xr = x + (x - (x - v * dt)) + a * dt * dt
        vr = (xr - x) / dt
    tol = 1e-13 if dtype == np.float64 else 2e-6
    assert np.abs(xe - xr).max() < tol * 4 and np.abs(ve - vr).max() < tol * 1e3


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_overdamped_update_matches_oracle(hostlib, dtype):
    x, v, f, mass, inv_m = _state()
    dt, friction, kT = 0.002, 5.0, 2.5
    rng = tho.rng_words(0x1234, 0x5678)
    g = np.sqrt(2 / friction * dt) * lo.normals(9, len(x), rng, np.sqrt(kT * inv_m))
    xe, ve = _update(hostlib, OVERDAMPED, x, v, f, inv_m, dt, friction=friction, g=g, dtype=dtype)
    xr, vr = vo.simulate_overdamped(lambda y: f, x, v, mass, dt, 1, kT, friction, rng, _ident, remove_cm_every=0, init_step=8)
    tol = 1e-13 if dtype == np.float64 else 2e-6
    assert np.abs(xe - xr).max() < tol * 4
    assert np.array_equal(ve, v.astype(dtype))  # the velocities are not touched
    assert np.array_equal(xe[:3], x[:3].astype(dtype))  # massless atoms do not move


def _smooth_forces(n=60, seed=5):
    """A smooth non-periodic force field (soft pair repulsion plus a weak harmonic well): no wrap, vector(a, b) = b - a."""
    r = np.random.default_rng(seed)
    x0 = r.uniform(0, 3, (n, 3))
    v0 = r.normal(0, 0.4, (n, 3))
    mass = r.uniform(5.0, 30.0, n)

    def fe(x):
        d = x[:, None, :] - x[None, :, :]
        r2 = (d * d).sum(-1) + np.eye(n)
        w = 2.0 * np.exp(-r2 / 0.2) / 0.2 * (1 - np.eye(n))
        return (w[:, :, None] * d).sum(1) - 0.5 * (x - 1.5)
    return fe, x0, v0, mass


def test_stormer_equals_velocity_verlet_positions():
    fe, x0, v0, mass = _smooth_forces()
    dt = 0.002
    xs, _ = vo.simulate_stormer_verlet(fe, x0, v0, mass, dt, 100, _ident, _vec)
    xv, _ = vo.simulate_velocity_verlet(fe, x0, v0, mass, dt, 100, _ident)
    assert np.abs(xs - xv).max() < 1e-12


def test_shifted_verlet_equals_velocity_verlet_positions():
    """Leapfrog started from v0 - a0 dt/2 is VelocityVerlet in positions."""
    fe, x0, v0, mass = _smooth_forces()
    dt = 0.002
    a0 = fe(x0) / mass[:, None]
    xl, _ = vo.simulate_verlet(fe, x0, v0 - a0 * dt / 2, mass, dt, 100, _ident, remove_cm_every=0)
    xv, _ = vo.simulate_velocity_verlet(fe, x0, v0, mass, dt, 100, _ident)
    assert np.abs(xl - xv).max() < 1e-12


def test_constructors():
    assert mb.Verlet(0.002) == mb.Verlet(dt=0.002, coupling=None, remove_CM_motion=1)
    assert mb.Verlet(0.002, remove_CM_motion=False).remove_CM_motion == 0
    assert mb.OverdampedLangevin(0.002, 300.0, 1.0).remove_CM_motion == 1
    assert mb.StormerVerlet(0.001).dt == 0.001
    for bad in (0.0, -0.001, float("nan"), float("inf")):
        for make in (lambda d: mb.Verlet(d), lambda d: mb.StormerVerlet(d), lambda d: mb.OverdampedLangevin(d, 300.0, 1.0)):
            with pytest.raises(ValueError):
                make(bad)
    for bad in (0.0, -1.0, float("nan"), float("inf")):  # friction 0: the noise prefactor is infinite
        with pytest.raises(ValueError):
            mb.OverdampedLangevin(0.002, 300.0, bad)
    for bad in (-1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            mb.OverdampedLangevin(0.002, bad, 1.0)
    for make in (lambda: mb.Verlet(0.002, remove_CM_motion=-1), lambda: mb.OverdampedLangevin(0.002, 1.0, 1.0, remove_CM_motion=-1)):
        with pytest.raises(ValueError):
            make()


def test_params_layout():
    P = mb.capi.MBStormerParams
    assert C.sizeof(P) == 24
    assert [(f, getattr(P, f).offset) for f, _ in P._fields_] == [("dt", 0), ("n_steps", 8), ("init_step", 16)]
    for name in ("mb_simulate_verlet", "mb_simulate_stormer_verlet", "mb_simulate_overdamped_langevin"):
        assert name in mb.capi.EXPORTED
    text = open(os.path.join(ROOT, "include", "mollyb200.h")).read()
    assert "int mb_simulate_verlet(mb_ctx* ctx, void* coords, void* vels, const mb_vv_params_t* p, mb_log_t* log);" in text
    assert ("int mb_simulate_overdamped_langevin(mb_ctx* ctx, void* coords, void* vels, const mb_langevin_params_t* p, "
            "mb_log_t* log);") in text


def test_simulate_refusals():
    # checked before the engine is touched, so this needs no GPU
    sysd = dict(mass=[1.0, 1.0], charge=[0, 0], sigma=[0.3, 0.3], eps=[0.2, 0.2])
    s = mb.System(atoms=mb.atoms_from_arrays(**sysd, dtype=np.float64), coords=np.array([[0.1, 0.1, 0.1], [1.0, 1.0, 1.0]]),
                  boundary=mb.CubicBoundary(2.0), pairwise_inters=(mb.LennardJones(),), dtype=np.float64)
    for coupling in (mb.BerendsenThermostat(10.0, 0.1), mb.ImmediateThermostat(10.0), mb.VelocityRescaleThermostat(10.0, 0.1),
                     (mb.AndersenThermostat(10.0, 0.1), mb.AndersenThermostat(10.0, 0.1)), [object()]):
        with pytest.raises(TypeError):
            mb.simulate(s, mb.Verlet(0.001, coupling=coupling), 1)
    for sim in (mb.Verlet(0.001), mb.StormerVerlet(0.001), mb.OverdampedLangevin(0.001, 10.0, 1.0)):
        with pytest.raises(TypeError):
            mb.simulate(s, sim)  # n_steps
        with pytest.raises(ValueError):
            mb.simulate(s, sim, 1, run_loggers="sometimes")
