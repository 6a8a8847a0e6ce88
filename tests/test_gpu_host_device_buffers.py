"""Host and device arrays at every C-ABI entry point that takes a caller's array (mb_forces with virial, mb_energy,
mb_forces_energy, mb_forces_energy_all, mb_remove_cm_motion, mb_kinetic_energy, mb_kinetic_energy_tensor,
mb_random_velocities, mb_simulate_vv): the same sequence of calls on a fresh context with numpy arrays, with torch CUDA
tensors and with a mix of both gives the same results, and outputs the caller pre-fills keep ADD semantics."""
import ctypes as C

import numpy as np
import pytest

import mbhelpers as H
import mollyb200 as mb
from test_gpu_parity import _pos_err

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
# results that bonded forces enter: the bonded kernel adds them with float atomics, so they are not bit-reproducible
BONDED_KEYS = ("f_all", "pe_all", "x_sim", "v_sim")


def _allpairs(dtype, g):
    """864 argon atoms without a neighbour list: the all-pairs kernel."""
    sd = H.lj_fluid(6, seed=3, dtype=dtype)
    return H.make_system(sd, (mb.LennardJones(cutoff=mb.ShiftedForceCutoff(1.0)),), dtype), sd["box"], 0.002


def _brick_bonded(dtype, g):
    """6mrr with bonds, angles, torsions and the LJ dispersion correction: the cell-list kernel plus the bonded kernel."""
    return H.sixmrr_system(g, dtype, r_list=1.2, dispersion=True), H.sixmrr_description(g)["box"], 0.0005


def _calls(s, dt_md, mode):
    """Every entry point with an array argument, in one fixed order. mode: "host" (numpy), "device" (torch CUDA) or "mixed"
    (every other array on the device, so pe and the virial also arrive one on each side)."""
    import torch
    ctx = s.engine()
    L, dt, n = s._L, s.dtype, s.n
    rng = np.random.default_rng(11)
    arrays = []

    def arr(a):
        on_dev = mode == "device" or (mode == "mixed" and len(arrays) % 2 == 1)
        a = np.ascontiguousarray(a, dtype=dt)
        arrays.append(torch.from_numpy(a.copy()).cuda() if on_dev else a.copy())
        return arrays[-1]

    def ptr(a):
        return a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data

    def val(a):
        if hasattr(a, "data_ptr"):
            torch.cuda.synchronize()
            return a.cpu().numpy()
        return a.copy()

    out = {}
    x, v = s.coords.astype(dt), s.velocities.astype(dt)
    pre_f, pre_v, pre_e = rng.normal(size=(n, 3)), rng.normal(size=9), 7.5
    # forces with virial, into pre-filled outputs and into zeros
    xa, fa, va = arr(x), arr(pre_f), arr(pre_v)
    mb.capi.check(L.mb_forces(ctx, ptr(xa), ptr(fa), ptr(va), 0))
    out["f"], out["vir"] = val(fa), val(va)
    fa, va = arr(np.zeros((n, 3))), arr(np.zeros(9))
    mb.capi.check(L.mb_forces(ctx, ptr(xa), ptr(fa), ptr(va), 0))
    out["f0"], out["vir0"] = val(fa), val(va)
    # energy
    pa = arr([pre_e])
    mb.capi.check(L.mb_energy(ctx, ptr(xa), ptr(pa), 0))
    out["pe"] = val(pa)
    pa = arr([0.0])
    mb.capi.check(L.mb_energy(ctx, ptr(xa), ptr(pa), 0))
    out["pe0"] = val(pa)
    # forces + energy + virial in one call
    fa, pa, va = arr(pre_f), arr([pre_e]), arr(pre_v)
    mb.capi.check(L.mb_forces_energy(ctx, ptr(xa), ptr(fa), ptr(pa), ptr(va), 0))
    out["f_fe"], out["pe_fe"], out["vir_fe"] = val(fa), val(pa), val(va)
    # with the specific (bonded) and general interactions
    fa, pa = arr(pre_f), arr([pre_e])
    mb.capi.check(L.mb_forces_energy_all(ctx, ptr(xa), ptr(fa), ptr(pa), 0))
    out["f_all"], out["pe_all"] = val(fa), val(pa)
    # velocities: centre-of-mass removal (in place), kinetic energy and its tensor (host outputs), random draw (output)
    vv = arr(v)
    mb.capi.check(L.mb_remove_cm_motion(ctx, ptr(vv)))
    out["v_cm"] = val(vv)
    ke, ket = C.c_double(), (C.c_double * 9)()
    mb.capi.check(L.mb_kinetic_energy(ctx, ptr(arr(v)), C.byref(ke)))
    mb.capi.check(L.mb_kinetic_energy_tensor(ctx, ptr(arr(v)), ket))
    out["ke"], out["ket"] = np.array([ke.value]), np.array(ket[:])
    vr = arr(rng.normal(size=(n, 3)))
    mb.capi.check(L.mb_random_velocities(ctx, ptr(vr), 1.5, 3, 99))
    out["v_rand"] = val(vr)
    # simulate: coordinates and velocities in and out
    p = mb.capi.MBVVParams()
    p.dt, p.n_steps, p.init_step, p.remove_cm_every = dt_md, 10, 0, 1
    xs, vs = arr(x), arr(v)
    mb.capi.check(L.mb_simulate_vv(ctx, ptr(xs), ptr(vs), C.byref(p)))
    out["x_sim"], out["v_sim"] = val(xs), val(vs)
    return out, pre_f, pre_v, pre_e


CASES = [("allpairs-f32", _allpairs, F32), ("allpairs-f64", _allpairs, F64),
         ("brick-bonded-f32", _brick_bonded, F32), ("brick-bonded-f64", _brick_bonded, F64)]


@pytest.mark.parametrize("name,make,dtype", CASES, ids=[c[0] for c in CASES])
def test_host_and_device_arrays_agree(name, make, dtype, golden_6mrr):
    pytest.importorskip("torch")
    res = {}
    for mode in ("host", "device", "mixed"):
        s, box, dt_md = make(dtype, {k: v.copy() for k, v in golden_6mrr.items()})
        res[mode], pre_f, pre_v, pre_e = _calls(s, dt_md, mode)
        s.close()
    h = res["host"]
    bonded = name.startswith("brick")
    eps = np.finfo(dtype).eps
    # ADD semantics: pre-filled outputs receive the sum (same rounding as the device's own +=)
    scale = np.abs(pre_f).max() + np.abs(h["f0"]).max()
    assert np.abs(h["f"] - (pre_f.astype(dtype) + h["f0"])).max() <= 4 * eps * scale
    assert np.abs(h["vir"] - (pre_v.astype(dtype) + h["vir0"])).max() <= 4 * eps * (np.abs(pre_v).max() + np.abs(h["vir0"]).max())
    assert abs(h["pe"][0] - (dtype(pre_e) + h["pe0"][0])) <= 4 * eps * (pre_e + abs(h["pe0"][0]))
    fmax = np.abs(h["f_all"]).max()
    for mode in ("device", "mixed"):
        d = res[mode]
        for k in h:
            if bonded and k in BONDED_KEYS:
                continue
            assert np.array_equal(h[k], d[k]), (mode, k)
        if bonded:
            ftol = 1e-12 * fmax if dtype == F64 else H.tol(F32, fmax)
            assert np.abs(h["f_all"] - d["f_all"]).max() <= ftol, mode
            assert abs(h["pe_all"][0] - d["pe_all"][0]) <= H.etol(dtype, h["pe_all"][0]), mode
            ex, ev = _pos_err(h["x_sim"], d["x_sim"], box), np.abs(h["v_sim"] - d["v_sim"]).max()
            print(f"[{name} {mode}] simulate dx={ex:.3e} dv={ev:.3e}")
            assert ex < (1e-9 if dtype == F64 else 1e-4) and ev < (1e-6 if dtype == F64 else 1e-3), mode
