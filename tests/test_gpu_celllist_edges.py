"""Edge cases of the cell-list (brick) path against the f64 C oracle: brick shapes set by the caller, the smallest and a
strongly anisotropic cell grid, inhomogeneous systems (droplets, a slab, a sparse gas), capacity overflow and its recovery,
long and index-distant partner lists, and coordinates the caller did not wrap.

Bars are those of test_gpu_parity.py: per-atom force f64 1e-9 max|F| + 1e-9, f32 5e-5 max|F| + 2e-3 plus one F(rc) jump per
pair within f32 rounding of a cutoff; energy f64 rel 1e-11, f32 rel 2e-6; virial f64 rel 1e-9, f32 rel 1e-4.
"""
import ctypes as C

import numpy as np
import pytest

import mbhelpers as H
import mollyb200 as mb
from oracle import oracle as o
from test_gpu_parity import _pos_err

pytestmark = pytest.mark.gpu

F64, F32 = np.float64, np.float32


def _lj_inters(rc, shifted_force=False):
    cut, kind = (mb.ShiftedForceCutoff, o.CUT_SHIFTED_FORCE) if shifted_force else (mb.DistanceCutoff, o.CUT_DISTANCE)
    return (mb.LennardJones(cutoff=cut(rc), use_neighbors=True),), [o.Inter(o.LJ, kind, rc, use_neighbors=True)]


def _molecular_inters(rc):
    return ((mb.LennardJones(cutoff=mb.DistanceCutoff(rc), use_neighbors=True, weight_special=0.5),
             mb.CoulombReactionField(dist_cutoff=rc, use_neighbors=True, weight_special=0.8333)),
            [o.Inter(o.LJ, o.CUT_DISTANCE, rc, weight_special=0.5, use_neighbors=True),
             o.Inter(o.CRF, o.CUT_DISTANCE, rc, weight_special=0.8333, use_neighbors=True)])


def _wrap(x, box):
    return x - np.floor(x / box) * box


class _Reference:
    """f64 oracle forces, energy and virial on the coordinates as rounded to `dtype`. Systems of more than 6 000 atoms go
    through the oracle's neighbour list at the largest cutoff (widened by 3e-6, as for the full-size parity tests)."""

    def __init__(self, sd, o_inters, dtype):
        self.sd, self.o_inters, self.dtype = sd, o_inters, np.dtype(dtype)
        self.x64 = np.asarray(sd["coords"]).astype(dtype).astype(F64)
        self.orc = H.make_oracle(sd, o_inters)
        if sd["n"] > 6000:
            rc = max(it.r_cut for it in o_inters)
            self.f, self.e, self.vir = self.orc.forces_nl(self.x64, self.orc.neighbor_list(self.x64, rc * (1 + 3e-6)), virial=True)
        else:
            self.f, self.e, self.vir = self.orc.forces_allpairs(self.x64, virial=True)
        self.fmax = np.abs(self.f).max()

    def check(self, f, label, e=None, vir=None, st=None):
        per_atom = np.abs(f.astype(F64) - self.f).max(axis=1)
        allowed = H.tol(self.dtype, self.fmax)
        if self.dtype == F32 and per_atom.max() > allowed:
            # pairs sitting on a cutoff within f32 rounding may land on either side: one F(rc) jump each
            allowed = allowed + H.boundary_atoms(self.orc, self.x64, self.o_inters) * H.cutoff_force_bound(self.sd, self.o_inters)
        where = "" if st is None else f"path={st['path']} brick={st['brick_dims']} n_cells={st['n_cells']} "
        de = "" if e is None else f" dE={e - self.e:.3e} (E={self.e:.6e})"
        print(f"[{label}] n={self.sd['n']} {self.dtype.name} {where}max|dF|={per_atom.max():.3e} (max|F|={self.fmax:.3e}){de}")
        assert (per_atom <= allowed).all(), label
        if e is not None:
            assert abs(e - self.e) <= H.etol(self.dtype, self.e), label
        if vir is not None:
            vtol = (1e-9 if self.dtype == F64 else 1e-4) * max(np.abs(self.vir).max(), 1.0)
            assert np.abs(vir.astype(F64) - self.vir).max() <= vtol, label


def _evaluate(s):
    f = mb.forces(s)
    e = mb.potential_energy(s)
    f2, vir = mb.forces_virial(s)
    assert np.abs(f2.astype(F64) - f.astype(F64)).max() <= H.tol(s.dtype, np.abs(f).max())
    return f, e, vir


def _run(sd, mi, oi, dtype, r_list, label, expect_path=1):
    """Fresh System, one force / energy / virial evaluation against the oracle. Returns (System, forces, stats)."""
    sd = dict(sd, coords=np.asarray(sd["coords"]).astype(dtype))
    s = H.make_system(sd, mi, dtype, r_list=r_list)
    f, e, vir = _evaluate(s)
    st = s.stats()
    _Reference(sd, oi, dtype).check(f, label, e, vir, st)
    assert st["path"] == expect_path, st
    return s, f, st


# ---------------------------------------------------------------------------------------------------
# 1. brick shapes set by the caller
# ---------------------------------------------------------------------------------------------------
# For both systems below the cell grid at r_list 1.3 nm is 7 cells along x (7 x 8 x 8 and 7 x 7 x 7):
#   (1,5,5): a halo of 9 x 9 = 81 (y,z) runs, more than the 64 the producer warp prefetches;
#   (2,3,3): a partial last brick along every axis; (7,1,2): one brick spans the whole x axis;
#   (8,8,8): a halo beyond 4096 staged atoms, which the first build must shrink to a brick that fits.
SHAPES = [(1, 1, 1), (2, 1, 1), (1, 1, 3), (3, 3, 2), (1, 5, 5), (2, 3, 3), (7, 1, 2), (8, 8, 8)]


@pytest.mark.parametrize("kind,dtype", [("molecular", F64), ("molecular", F32), ("lj", F32), ("lj", F64)])
def test_forced_brick_shapes(kind, dtype):
    if kind == "molecular":  # 4000 atoms, LJ + CRF, exclusions and 1-4 specials
        sd = H.molecular_system(1000, [5.1, 5.4, 5.8], seed=5)
        mi, oi = _molecular_inters(1.0)
    else:  # 2916 argon atoms, box 5.17 nm: the uniform-LJ variants
        sd = H.lj_fluid(9, seed=42, dtype=F64)
        mi, oi = _lj_inters(1.2)
    sd = dict(sd, coords=sd["coords"].astype(dtype))
    ref = _Reference(sd, oi, dtype)
    s = H.make_system(sd, mi, dtype, r_list=1.3)
    first, pairs = None, set()
    for shape in SHAPES:
        s.set_launch_config(brick_dims=shape)
        f, e, vir = _evaluate(s)
        st = s.stats()
        ref.check(f, f"{kind} brick request {shape}", e, vir, st)
        assert st["path"] == 1
        assert all(b <= r for b, r in zip(st["brick_dims"], shape)), st["brick_dims"]
        pairs.add(st["n_pairs_in_list"])
        if first is None:
            first = f
        # a pair's image depends on the two atoms' cells only, so every shape evaluates the same pairs
        assert np.abs(f.astype(F64) - first.astype(F64)).max() <= H.tol(dtype, ref.fmax)
    print(f"    pairs in the list: {sorted(pairs)}")
    assert len(pairs) == 1
    if dtype == F64:  # full-shell list: every pair within r_list that is not excluded, twice
        assert pairs.pop() == 2 * len(ref.orc.neighbor_list(ref.x64, 1.3))
    s.close()


# ---------------------------------------------------------------------------------------------------
# 2. grid and path edges
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [F64, F32])
def test_smallest_cell_grid_and_path_switch(dtype):
    """A cubic box of exactly 2.5 r_list is the smallest the cell-list path takes (5 cells per axis); 1e-6 nm less runs
    on the no-list kernel. Both match the oracle."""
    rl = 1.3
    mi, oi = _lj_inters(1.2)
    for side, path in ((2.5 * rl, 1), (2.5 * rl - 1e-6, 0)):
        sd = H.fluid_in_box([side] * 3, seed=4)
        s, _, st = _run(sd, mi, oi, dtype, rl, f"cubic box {side:.7f} nm", expect_path=path)
        if path == 1:
            assert st["n_cells"] == [5, 5, 5]
        s.close()


@pytest.mark.parametrize("dtype", [F64, F32])
def test_anisotropic_cell_grid(dtype):
    # 10 800 atoms. Cells are at least r_list / 2 wide, so at r_list 1.3 the grid is 5 x 9 x 39 (26 / 40 = 0.65 is
    # exactly r_list / 2, which the grid treats as too narrow)
    sd = H.fluid_in_box([3.3, 6.0, 26.0], seed=6)
    s, _, st = _run(sd, *_lj_inters(1.2), dtype, 1.3, "anisotropic 3.3 x 6 x 26 nm")
    assert st["n_cells"] == [5, 9, 39]
    s.close()


def test_sparse_gas_forces_and_dynamics():
    """64 atoms (the smallest cell-list system) in a 6 nm box: 12^3 cells, nearly every brick empty."""
    sd = H.readme_system(64, 6.0, seed=3, min_dist=0.3)
    mi, oi = _lj_inters(0.9, shifted_force=True)
    _run(sd, mi, oi, F32, 1.0, "sparse gas")[0].close()
    s, _, _ = _run(sd, mi, oi, F64, 1.0, "sparse gas")
    x_ref, v_ref, _ = H.make_oracle(sd, oi).simulate_vv(sd["coords"], sd["velocities"], 0.002, 50, remove_cm_every=1,
                                                         r_list=1.0, nl_every=5)
    mb.simulate(s, mb.VelocityVerlet(dt=0.002), 50)
    ex, ev = _pos_err(s.coords, x_ref, sd["box"]), np.abs(s.velocities - v_ref).max()
    print(f"[sparse gas VV 50 steps] dx={ex:.3e} dv={ev:.3e} rebuilds={s.stats()['n_rebuilds']}")
    assert ex < 1e-7 and ev < 1e-5
    s.close()


# ---------------------------------------------------------------------------------------------------
# 3. inhomogeneous density
# ---------------------------------------------------------------------------------------------------
BOX30 = np.array([30.0, 30.0, 30.0])


def _droplets():
    """An argon droplet of radius 5 nm (11 000 atoms) centred in a 30 nm box, and the same droplet moved onto a box corner,
    where every atom has 1-7 ghost copies."""
    centred = H.argon_droplet(5.0, BOX30, BOX30 / 2)
    corner = dict(centred, coords=_wrap(centred["coords"] - BOX30 / 2, BOX30))
    return centred, corner


@pytest.mark.parametrize("dtype", [F64, F32])
def test_droplet_centred_and_on_a_corner(dtype):
    centred, corner = _droplets()
    mi, oi = _lj_inters(1.2)
    s1, f1, _ = _run(centred, mi, oi, dtype, 1.3, "droplet, centred")
    s2, f2, _ = _run(corner, mi, oi, dtype, 1.3, "droplet, on a corner")
    if dtype == F64:  # the same physical system translated by half a box
        fmax = np.abs(f1).max()
        print(f"    corner vs centred: max|dF|={np.abs(f2 - f1).max():.3e}")
        assert np.abs(f2 - f1).max() <= 1e-9 * fmax + 1e-9
    s1.close()
    s2.close()


@pytest.mark.parametrize("dtype", [F64, F32])
def test_liquid_slab(dtype):
    sd = H.argon_slab(6.0, [8.0, 8.0, 24.0])  # a 6 nm film with 18 nm of vacuum along z
    _run(sd, *_lj_inters(1.2), dtype, 1.3, "slab 8 x 8 x 24 nm")[0].close()


# ---------------------------------------------------------------------------------------------------
# 4. capacity overflow: the C ABI reports it, the next call re-derives the capacities, the Python API retries
# ---------------------------------------------------------------------------------------------------
def _raw_forces(s, x):
    fs = np.zeros((s.n, 3), s.dtype)
    x = np.ascontiguousarray(x, s.dtype)
    return s._L.mb_forces(s.engine(), x.ctypes.data, fs.ctypes.data, None, 0), fs


def _overflow_then_recover(start, target, label):
    mi, oi = _lj_inters(1.2)
    s = H.make_system(start, mi, F64, r_list=1.3)
    mb.forces(s)
    st0 = s.stats()
    rc, _ = _raw_forces(s, target["coords"])
    print(f"[{label}] capacities of the first configuration: halo {st0['halo_capacity']} stride {st0['list_stride']} "
          f"brick {st0['brick_dims']}; mb_forces on the second: rc={rc} ({mb.capi.load().mb_last_error().decode()})")
    assert rc == mb.capi.MB_ERR_CAPACITY
    rc, f = _raw_forces(s, target["coords"])  # the call after the error derives new capacities
    assert rc == mb.capi.MB_OK
    ref = _Reference(target, oi, F64)
    ref.check(f, f"{label}: next call", st=s.stats())
    s.close()
    # forces(sys) retries by itself
    s = H.make_system(start, mi, F64, r_list=1.3)
    mb.forces(s)
    s.coords[...] = target["coords"]
    f, e = mb.forces_energy(s)
    ref.check(f, f"{label}: forces_energy retried", e=e, st=s.stats())
    assert s.stats()["path"] == 1
    s.close()


def test_ghost_overflow_is_reported_then_recovered():
    """Capacities sized for a droplet without ghost copies; then the droplet on a corner (thousands of ghost copies)."""
    centred, corner = _droplets()
    _overflow_then_recover(centred, corner, "ghost overflow")


def test_halo_and_stride_overflow_is_reported_then_recovered():
    """Capacities sized for a dilute gas (no atom within r_list of another); then the same atoms gathered into a droplet:
    full halos, 190 neighbours per atom."""
    centred, _ = _droplets()
    m = int(np.ceil(centred["n"] ** (1 / 3)))
    g = np.stack(np.meshgrid(*[np.arange(m)] * 3, indexing="ij"), -1).reshape(-1, 3)[:centred["n"]]
    gas = dict(centred, coords=(g + 0.5) * (BOX30 / m))
    _overflow_then_recover(gas, centred, "halo/stride overflow")


def test_simulate_recovers_when_a_droplet_drifts_across_a_face():
    """A droplet (radius 3.5 nm, 3 800 atoms) 1.5 nm from a face, so without ghost copies, drifts through the face: about
    2 000 ghost copies at the end. The run overflows the first build's capacities; simulate restarts it with capacities
    for the state that overflowed and must match the oracle's trajectory."""
    side, radius = 12.0, 3.5
    box = np.array([side] * 3)
    sd = H.argon_droplet(radius, box, [side - 1.5 - radius, side / 2, side / 2], seed=11)
    sd["velocities"] = sd["velocities"] + np.array([12.0, 0.0, 0.0])  # common drift along x, nm/ps
    mi, oi = _lj_inters(1.2, shifted_force=True)
    dt, n = 0.002, 200  # 4.8 nm of drift
    raw = H.make_system(sd, mi, F64, r_list=1.3)
    p = mb.capi.MBVVParams()
    p.dt, p.n_steps, p.init_step, p.remove_cm_every = dt, n, 0, 0
    ctx = raw.engine()
    rc = raw._L.mb_simulate_vv(ctx, raw.coords.ctypes.data, raw.velocities.ctypes.data, C.byref(p))
    print(f"[drifting droplet] mb_simulate_vv: rc={rc} ({mb.capi.load().mb_last_error().decode()})")
    assert rc == mb.capi.MB_ERR_CAPACITY
    raw.close()
    s = H.make_system(sd, mi, F64, r_list=1.3)
    mb.simulate(s, mb.VelocityVerlet(dt=dt, remove_CM_motion=0), n)
    x_ref, v_ref, _ = H.make_oracle(sd, oi).simulate_vv(sd["coords"], sd["velocities"], dt, n, remove_cm_every=0,
                                                         r_list=1.3, nl_every=5)
    ex, ev = _pos_err(s.coords, x_ref, box), np.abs(s.velocities - v_ref).max()
    st = s.stats()
    print(f"[drifting droplet] simulate: dx={ex:.3e} dv={ev:.3e} rebuilds={st['n_rebuilds']} brick={st['brick_dims']} "
          f"halo capacity {st['halo_capacity']} stride {st['list_stride']}")
    assert ex < 1e-7 and ev < 1e-5
    assert (s.coords >= 0).all() and (s.coords < box).all()
    s.close()


# ---------------------------------------------------------------------------------------------------
# 5. partner lists: more than 32 partners, index-distant partners, the 255-special limit of the list path
# ---------------------------------------------------------------------------------------------------
def _partner_system(path):
    if path == 1:
        return H.molecular_system(1000, [5.1, 5.4, 5.8], seed=5), 1.0, 1.1
    return H.molecular_system(150, [3.0, 3.2, 3.4], seed=11), 1.2, 1.3  # 3.0 nm < 2.5 r_list: the no-list kernel


def _with_hub(sd, n_excluded, n_special):
    """Give the atom in the middle of the index range n_excluded extra excluded and n_special extra special partners, its
    nearest atoms first; also exclude the pair (0, n-1), which sit next to each other across the periodic boundary."""
    n = sd["n"]
    hub = n // 2 + 1
    own = {int(j) for p in np.concatenate([sd["excluded"], sd["special"]]) if hub in p for j in p}
    near = H.nearest_partners(sd, hub, n_excluded + n_special, skip=own | {0, n - 1})
    pairs = lambda js: np.array([(hub, j) for j in js], np.int32).reshape(-1, 2)
    excl = np.concatenate([sd["excluded"], pairs(near[:n_excluded]), [(0, n - 1)]]).astype(np.int32)
    spec = np.concatenate([sd["special"], pairs(near[n_excluded:])]).astype(np.int32)
    return dict(sd, excluded=excl, special=spec)


@pytest.mark.parametrize("dtype", [F64, F32])
@pytest.mark.parametrize("path", [0, 1])
def test_long_and_index_distant_partner_lists(path, dtype):
    sd, rc, rl = _partner_system(path)
    sd = _with_hub(sd, 40, 40)
    H.check(sd, *_molecular_inters(rc), dtype, r_list=rl, expect_path=path, label=f"40 + 40 partners, path {path}")


@pytest.mark.parametrize("dtype", [F64, F32])
@pytest.mark.parametrize("path", [0, 1])
def test_256_special_partners(path, dtype):
    sd, rc, rl = _partner_system(path)
    sd = _with_hub(sd, 0, 256)
    mi, oi = _molecular_inters(rc)
    if path == 1:  # special-list entries are 8-bit lengths in the task table
        s = H.make_system(dict(sd, coords=sd["coords"].astype(dtype)), mi, dtype, r_list=rl)
        with pytest.raises(mb.MollyB200Error, match="more than 255 special partners"):
            mb.forces(s)
        s.close()
    else:
        H.check(sd, mi, oi, dtype, r_list=rl, expect_path=0, label="256 special partners, no-list path")


# ---------------------------------------------------------------------------------------------------
# 6. coordinates the caller did not wrap
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [F64, F32])
def test_unwrapped_input_coordinates(dtype):
    sd = H.lj_fluid(9, seed=42, dtype=F64)
    box = sd["box"]
    x = sd["coords"].copy()
    for d in range(3):  # translate so that atom d sits exactly on the low face along axis d
        x[:, d] -= x[d, d]
    x = _wrap(x, box)
    assert x[0, 0] == 0 and x[1, 1] == 0 and x[2, 2] == 0
    sd = dict(sd, coords=x.astype(dtype))
    mi, oi = _lj_inters(1.2, shifted_force=True)
    s, f_w, _ = _run(sd, mi, oi, dtype, 1.3, "wrapped input")
    tol = H.tol(dtype, np.abs(f_w).max())
    k = np.random.default_rng(0).integers(-2, 3, x.shape)
    at_L, neg_zero = sd["coords"].copy(), sd["coords"].copy()
    for d in range(3):
        at_L[d, d] = box[d].astype(dtype)
        neg_zero[d, d] = -0.0
    variants = {"shifted by k L": (x + k * box).astype(dtype), "exactly L": at_L, "-0.0": neg_zero}
    for name, xv in variants.items():
        fresh = H.make_system(dict(sd, coords=xv), mi, dtype, r_list=1.3)
        f_fresh = mb.forces(fresh)
        s.coords[...] = xv  # and an engine that has seen the wrapped coordinates
        f_same = mb.forces(s)
        err = max(np.abs(f_fresh.astype(F64) - f_w).max(), np.abs(f_same.astype(F64) - f_w).max())
        print(f"[unwrapped input: {name}] max|dF| vs wrapped input = {err:.3e} (tol {tol:.3e})")
        assert err <= tol, name
        mb.simulate(fresh, mb.VelocityVerlet(dt=0.002), 10)
        assert (fresh.coords >= 0).all() and (fresh.coords < box.astype(dtype)).all(), name
        fresh.close()
    s.close()
