"""Steepest-descent minimisation on the device (mb_minimize_sd): the reference's own minimisation test, per-iteration
parity with the numpy restatement (tests/sd_oracle.py) on the all-pairs and cell-list paths, rejected trials after a
rebuild, 6mrr as in test/protein.jl:695-699, edge cases, graph vs stream path, and the state a later simulate sees."""
import ctypes as C

import numpy as np
import pytest

import mbhelpers as H
import mollyb200 as mb
import sd_oracle as sdo
from test_gpu_parity import _pos_err

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64


def _run(s, **kw):
    _, trace = mb.steepest_descent(s, mb.SteepestDescentMinimizer(**kw))
    return trace, s.minimize_result


def _coords(s):
    c = s.coords
    return c.detach().cpu().numpy() if hasattr(c, "data_ptr") else np.array(c)


def _compare_traces(tr, ref, rtol=1e-9):
    """Per iteration: E_trial and max force to rtol; accept/reject identical wherever the decision is not a near tie."""
    assert tr.shape == ref.shape, (tr.shape, ref.shape)
    assert np.array_equal(tr[:, 0], ref[:, 0])
    assert abs(tr[0, 1] - ref[0, 1]) <= rtol * abs(ref[0, 1])
    e_kept = ref[0, 1]
    for k in range(1, len(ref)):
        for col in (1, 2):
            a, b = tr[k, col], ref[k, col]
            assert (np.isnan(a) and np.isnan(b)) or abs(a - b) <= rtol * max(abs(b), 1e-300), (k, col, a, b)
        if not abs(ref[k, 1] - e_kept) <= rtol * abs(e_kept):
            assert tr[k, 3] == ref[k, 3], (k, tr[k], ref[k])
        if ref[k, 3]:
            e_kept = ref[k, 1]


# ---- 1. the reference's own test (test/minimization.jl) ------------------------------------------------------------------
X3 = np.array([[1.0, 1.0, 1.0], [1.6, 1.0, 1.0], [1.4, 1.6, 1.0]])


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_reference_minimization(dtype):
    sig = 0.4 / 2 ** (1 / 6)
    atoms = mb.atoms_from_arrays(np.ones(3), np.zeros(3), np.full(3, sig), np.ones(3), dtype)
    s = mb.System(atoms=atoms, coords=X3.copy(), boundary=mb.CubicBoundary(5.0), pairwise_inters=(mb.LennardJones(),), dtype=dtype)
    mb.simulate(s, mb.SteepestDescentMinimizer(tol=1.0))
    x = _coords(s).astype(F64)
    d = [np.linalg.norm(x[j] - x[i]) for i, j in ((0, 1), (0, 2), (1, 2))]
    dtol, etol = (1e-3, 1e-4) if dtype == F64 else (1e-2, 1e-2)  # the reference's CPU / GPU bars
    assert np.all(np.abs(np.array(d) - 0.4) < dtol), d
    assert abs(mb.potential_energy(s) - (-3.0)) < etol
    assert s.minimize_result["converged"]
    if dtype == F64:  # same run as the restatement
        ref_x, ref = sdo.steepest_descent(X3, np.full(3, 5.0), lambda y: sdo.lj_energy_forces(y, np.full(3, 5.0), np.full(3, sig), np.ones(3)),
                                          tol=1.0)
        assert s.minimize_result["n_iterations"] == len(ref) - 1
        assert _pos_err(x, ref_x, np.full(3, 5.0)) < 1e-9
    s.close()


# ---- 2. trace parity with the oracle (f64) -------------------------------------------------------------------------------
def _readme():
    sd = H.readme_system()
    s = H.make_system(sd, (mb.LennardJones(cutoff=mb.DistanceCutoff(1.0)),), F64)
    orc = H.make_oracle(sd, [_o().Inter(_o().LJ, _o().CUT_DISTANCE, 1.0)])
    return s, sd, lambda x: orc.forces_allpairs(x)[:2], 0


def _molecular():
    sd = H.molecular_system(729, [5.1, 5.4, 5.8], seed=5, stable=True)
    o = _o()
    s = H.make_system(sd, (mb.LennardJones(cutoff=mb.ShiftedForceCutoff(1.0), use_neighbors=True, weight_special=0.5),
                           mb.CoulombReactionField(dist_cutoff=1.0, use_neighbors=True, weight_special=0.8333)), F64, r_list=1.15)
    orc = H.make_oracle(sd, [o.Inter(o.LJ, o.CUT_SHIFTED_FORCE, 1.0, weight_special=0.5, use_neighbors=True),
                             o.Inter(o.CRF, o.CUT_DISTANCE, 1.0, weight_special=0.8333, use_neighbors=True)])
    return s, sd, lambda x: orc.forces_nl(x, orc.neighbor_list(x, 1.15))[:2], 1


def _sixmrr(g):
    s = H.sixmrr_system(g, F64, r_list=1.2)
    orc, sd = H.sixmrr_oracle(g)

    def fe(x):
        f, e, _ = orc.forces_nl(x, orc.neighbor_list(x, 1.2))
        fb, eb = H.bonded_forces_oracle(g, x)
        return f + fb, e + eb
    return s, sd, fe, 1


def _o():
    from oracle import oracle as o
    return o


@pytest.mark.parametrize("name,steps", [("readme-allpairs", 40), ("molecular-brick", 25), ("6mrr-bonded", 8)])
def test_trace_matches_oracle(name, steps, golden_6mrr):
    s, sd, fe, path = {"readme-allpairs": _readme, "molecular-brick": _molecular}.get(name, lambda: _sixmrr(golden_6mrr))()
    tr, res = _run(s, step_size=0.01, max_steps=steps, tol=0.0)
    x_ref, ref = sdo.steepest_descent(sd["coords"].astype(F64), sd["box"], fe, step_size=0.01, max_steps=steps, tol=0.0)
    assert s.stats()["path"] == path
    print(f"[{name}] accepted {int(ref[1:, 3].sum())}/{steps}, E {ref[0, 1]:.6f} -> {res['energy']:.6f}")
    _compare_traces(tr, ref)
    assert np.array_equal(tr[1:, 3], ref[1:, 3])  # (no near ties in these runs: the coordinates below depend on it)
    assert _pos_err(_coords(s), x_ref, sd["box"]) < 1e-9
    s.close()


# ---- 3. rejected trials after a rebuild ------------------------------------------------------------------------------------
def test_rejected_trials_after_rebuilds_match_oracle():
    """Skin 0.02 nm and a step of 0.05 nm: trials rebuild the cell list, some of them are rejected, and the restored positions
    (saved in original order, put back into the frame of the re-sorted slots) continue the run exactly like the oracle's."""
    sd = H.lj_fluid(6, seed=3, dtype=F64)
    o = _o()
    s = H.make_system(sd, (mb.LennardJones(cutoff=mb.ShiftedForceCutoff(1.0), use_neighbors=True),), F64, r_list=1.02)
    orc = H.make_oracle(sd, [o.Inter(o.LJ, o.CUT_SHIFTED_FORCE, 1.0, use_neighbors=True)])
    mb.potential_energy(s)  # first build
    rb0 = s.stats()["n_rebuilds"]
    tr, _ = _run(s, step_size=0.05, max_steps=40, tol=0.0)
    st = s.stats()
    assert st["path"] == 1 and st["graph_mode"] == 1
    x_ref, ref = sdo.steepest_descent(sd["coords"].astype(F64), sd["box"], lambda x: orc.forces_allpairs(x)[:2],
                                      step_size=0.05, max_steps=40, tol=0.0)
    h, big_rejects = 0.05, 0
    for k in range(1, len(ref)):  # the trial of iteration k moves the atom with the largest force by h: > skin/2 rebuilds
        if not ref[k, 3] and h > 0.02:
            big_rejects += 1
        h = 6 * h / 5 if ref[k, 3] else h / 5
    print(f"[rebuild] rebuilds {st['n_rebuilds'] - rb0}, rejects {int((ref[1:, 3] == 0).sum())} ({big_rejects} with h > skin)")
    assert big_rejects > 0 and st["n_rebuilds"] - rb0 >= big_rejects
    _compare_traces(tr, ref)
    assert np.array_equal(tr[1:, 3], ref[1:, 3])
    assert _pos_err(_coords(s), x_ref, sd["box"]) < 1e-9
    s.close()


def test_triclinic_allpairs_matches_oracle():
    """A TriclinicBoundary box runs on the all-pairs kernel: trial moves are wrapped with wrap_coords of that boundary."""
    from oracle import triclinic as tri
    bv = np.array([[3.0, 0.0, 0.0], [0.8, 3.1, 0.0], [0.5, -0.6, 3.2]])
    t = tri.Triclinic(bv)
    rng = np.random.default_rng(21)
    pts = []
    while len(pts) < 40:
        c = rng.random(3) @ bv
        if all(np.linalg.norm(t.vector(c, q)) > 0.3 for q in pts):
            pts.append(c)
    x = np.array(pts)
    n = len(x)
    sig, eps = np.full(n, 0.3), np.full(n, 0.5)
    atoms = mb.atoms_from_arrays(np.ones(n), np.zeros(n), sig, eps, F64)
    s = mb.System(atoms=atoms, coords=x.copy(), boundary=mb.TriclinicBoundary(*bv),
                  pairwise_inters=(mb.LennardJones(cutoff=mb.DistanceCutoff(1.2)),), dtype=F64)
    tr, _ = _run(s, step_size=0.02, max_steps=20, tol=0.0)
    x_ref, ref = sdo.steepest_descent(x, np.diag(bv), lambda y: tri.forces_energy(t, y, sig, eps, r_cut=1.2)[:2],
                                      step_size=0.02, max_steps=20, tol=0.0, wrap_fn=lambda y: np.array([t.wrap(r) for r in y]))
    assert s.stats()["path"] == 0
    _compare_traces(tr, ref)
    assert np.array_equal(tr[1:, 3], ref[1:, 3])
    d = np.array([t.vector(a, b) for a, b in zip(_coords(s), x_ref)])
    assert np.abs(d).max() < 1e-9
    s.close()


# ---- 4. 6mrr, the analogue of test/protein.jl:695-699 ----------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["f64", "f32", "pme-f64"])
def test_6mrr_minimization(kind, golden_6mrr):
    g = golden_6mrr
    dtype = F32 if kind == "f32" else F64
    s = H.sixmrr_pme_system(g, dtype) if kind.startswith("pme") else H.sixmrr_system(g, dtype)
    box = H.sixmrr_description(g)["box"]
    x0 = _coords(s).astype(F64)
    e0 = mb.potential_energy(s)
    tr, res = _run(s, tol=400.0)
    assert s.stats()["graph_mode"] == (0 if kind.startswith("pme") else 1)
    acc = tr[tr[:, 3] == 1, 1]
    print(f"[6mrr {kind}] {res['n_iterations']} iterations, E {e0:.3f} -> {res['energy']:.3f}, max force {res['max_force']:.1f}")
    assert np.all(np.diff(acc) < 0)
    assert res["converged"] and tr[-1, 2] < 400.0
    assert res["energy"] < e0
    d = _coords(s).astype(F64) - x0
    d -= box * np.round(d / box)
    assert np.sqrt(np.mean(np.sum(d * d, 1))) < 0.1
    e1 = mb.potential_energy(s)
    fmax = np.sqrt(np.max(np.sum(mb.forces(s).astype(F64) ** 2, 1)))
    if dtype == F64:
        assert abs(res["energy"] - e1) <= 1e-9 * abs(e1)
        assert abs(res["max_force"] - fmax) <= 1e-9 * fmax
    else:
        assert abs(res["energy"] - e1) <= 1e-5 * abs(e1)
        assert abs(res["max_force"] - fmax) <= 1e-3 * fmax
    s.close()


# ---- 5. edge cases --------------------------------------------------------------------------------------------------------
def test_max_steps_zero_returns_wrapped_coordinates():
    sd = H.readme_system()
    x = sd["coords"].copy()
    x[::3] += sd["box"]
    x[1::3] -= 2 * sd["box"]
    sd = dict(sd, coords=x)
    s = H.make_system(sd, (mb.LennardJones(cutoff=mb.DistanceCutoff(1.0)),), F64)
    tr, res = _run(s, max_steps=0)
    assert tr.shape == (1, 4) and tr[0, 0] == 0 and np.isnan(tr[0, 2]) and tr[0, 3] == 1
    assert res["n_iterations"] == 0
    assert np.abs(_coords(s) - sdo.wrap(x, sd["box"])).max() < 1e-12
    assert abs(res["energy"] - mb.potential_energy(s)) <= 1e-12 * abs(res["energy"])
    s.close()


@pytest.mark.parametrize("r_list", [0.0, 1.2], ids=["allpairs", "brick"])
def test_zero_forces_reject_once_and_keep_coordinates(r_list):
    """Atoms beyond the cutoff of each other: m = 0, one rejected iteration with E_trial = NaN, unchanged coordinates."""
    x = np.array([[0.5 + 2.0 * i, 0.5 + 1.5 * j, 0.7 + 2.2 * k] for i in range(3) for j in range(4) for k in range(3)])
    sd = dict(box=np.full(3, 6.6))
    if r_list > 0:  # 72 atoms so that the cell-list path takes them; the pairs 0.017 nm apart are excluded
        x = np.concatenate([x, x + 0.01])
        sd["excluded"] = np.array([[i, i + 36] for i in range(36)], np.int32)
    n = len(x)
    sd.update(n=n, coords=x, velocities=np.zeros((n, 3)), mass=np.ones(n), charge=np.zeros(n), sigma=np.full(n, 0.3),
              eps=np.full(n, 0.5))
    s = H.make_system(sd, (mb.LennardJones(cutoff=mb.DistanceCutoff(1.0), use_neighbors=r_list > 0),), F64, r_list=r_list)
    tr, res = _run(s)
    assert s.stats()["path"] == (1 if r_list > 0 else 0)
    assert tr.shape == (2, 4) and tr[1, 3] == 0 and np.isnan(tr[1, 1]) and tr[1, 2] == 0.0
    assert res["converged"] and res["n_iterations"] == 1 and res["max_force"] == 0.0 and res["energy"] == 0.0
    out = _coords(s)
    assert np.all(np.isfinite(out)) and np.abs(out - x).max() < 1e-12
    s.close()


def test_huge_tol_takes_exactly_one_iteration():
    s, sd, fe, _ = _readme()
    tr, res = _run(s, tol=1e30)
    x_ref, ref = sdo.steepest_descent(sd["coords"].astype(F64), sd["box"], fe, tol=1e30)
    assert len(ref) == 2 and res["n_iterations"] == 1 and res["converged"]
    _compare_traces(tr, ref)
    assert _pos_err(_coords(s), x_ref, sd["box"]) < 1e-9
    s.close()


@pytest.mark.parametrize("make", ["readme", "molecular"])
def test_host_and_device_coordinates_agree(make):
    torch = pytest.importorskip("torch")
    out = []
    for device in (False, True):
        s, sd, _, _ = _readme() if make == "readme" else _molecular()
        if device:
            s.coords = torch.from_numpy(np.array(s.coords)).cuda()
        tr, res = _run(s, max_steps=20, tol=0.0)
        torch.cuda.synchronize()
        out.append((tr, _coords(s), res))
        s.close()
    assert np.array_equal(out[0][0], out[1][0], equal_nan=True)
    assert np.array_equal(out[0][1], out[1][1])
    assert out[0][2] == out[1][2]


def test_invalid_arguments_rejected():
    s, _, _, _ = _readme()
    ctx, L = s.engine(), s._L
    x = np.array(s.coords)
    trace = np.zeros((4, 4))
    for field, value in (("max_steps", -1), ("step_size", 0.0), ("step_size", -0.1), ("tol", -1.0), ("max_steps", 4)):
        p = mb.capi.MBSDParams(step_size=0.01, max_steps=3, tol=1.0, trace=trace.ctypes.data, trace_capacity=4)
        setattr(p, field, value)  # (max_steps 4 needs 5 records)
        assert L.mb_minimize_sd(ctx, x.ctypes.data, C.byref(p)) == mb.capi.MB_ERR_INVALID, field
    assert np.array_equal(x, np.array(s.coords)) and not trace.any()
    s.close()


# ---- 6. paths and state --------------------------------------------------------------------------------------------------
def _fluid(dtype):
    sd = H.lj_fluid(8, seed=4, dtype=dtype)
    return H.make_system(sd, (mb.LennardJones(cutoff=mb.ShiftedForceCutoff(1.0), use_neighbors=True),), dtype, r_list=1.1), sd


@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
def test_graph_and_stream_paths_are_bit_identical(dtype):
    out = []
    for profile in (False, False, True):  # graph, graph again, stream (profiling on)
        s, _ = _fluid(dtype)
        if profile:
            s.set_profiling(True)
        tr, res = _run(s, step_size=0.02, max_steps=60, tol=0.0)
        out.append((tr, _coords(s), res, s.stats()["graph_mode"]))
        s.close()
    assert [o[3] for o in out] == [1, 1, 0]
    for o in out[1:]:
        assert np.array_equal(out[0][0], o[0], equal_nan=True)
        assert np.array_equal(out[0][1], o[1])
        assert out[0][2] == o[2]
    assert 0 < out[0][0][1:, 3].sum() < 60  # the run accepts and rejects


def test_dynamics_after_minimization_start_clean():
    """simulate(VelocityVerlet) on the minimised System gives the trajectory of a fresh System built from its coordinates."""
    s, sd = _fluid(F64)
    _run(s, step_size=0.02, max_steps=30, tol=0.0)
    x_min = _coords(s).copy()
    mb.simulate(s, mb.VelocityVerlet(dt=0.002), 20)
    fresh = H.make_system(dict(sd, coords=x_min), (mb.LennardJones(cutoff=mb.ShiftedForceCutoff(1.0), use_neighbors=True),),
                          F64, r_list=1.1)
    mb.simulate(fresh, mb.VelocityVerlet(dt=0.002), 20)
    assert _pos_err(_coords(s), _coords(fresh), sd["box"]) < 1e-9
    assert np.abs(np.array(s.velocities) - np.array(fresh.velocities)).max() < 1e-7
    s.close()
    fresh.close()
