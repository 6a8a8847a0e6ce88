// cells.cuh — device-side neighbour structure: cell binning, deterministic cell sort, brick/halo
// tables and full-shell per-atom neighbour lists. Replaces CellListMap.jl on the host
// (src/neighbors.jl:552-693) and the O((N/32)^2) tile search + O(N^2/1024) mask table of the CUDA
// extension (ext/MollyCUDAExt.jl:1301-1568).
//
// Layout ("slot" = position in the cell-sorted order, x-fastest cell id):
//   pos4[slot]  = (x, y, z, q)            T4   positions are continuous (unwrapped) between rebuilds
//   lj2[slot]   = (sigma part, eps part)  T2   Lorentz: sigma/2, sqrt(eps)  (0,0 if LJ zero shortcut)
//   orig[slot]  = original atom index     int32
// A brick is a box of b[0] x b[1] x b[2] cells. Its halo is the brick plus h cells on every side.
// Positions are ALSO kept in an extended (ghost-padded) array pos4e: the cell grid grown by h cells on every side,
// x-fastest, the ghost cells holding the periodic images (coordinates already moved by +-L). Every (y,z) row of a
// brick's halo is then ONE contiguous run of pos4e, in the frame of the owned atoms, which the force kernel and the
// list builder stage into shared memory with 1-D bulk async copies (TMA) - no wrap splitting, no image arithmetic
// after the copy. The drift kernel (K1) keeps pos4e current: it stores every atom's new position at ext_of[slot] and
// at its ghost copies (a third of the atoms sit within h cells of a box face and have 1-7 of them).
// Neighbour list entries are 16-bit offsets into the staged halo.
//
// Every kernel of the rebuild pipeline is gated on ctl->rebuild so the whole sequence can be
// enqueued unconditionally (no host round trip when no atom moved more than skin/2).
#pragma once
#include "common.cuh"

namespace mb {

struct Control {
    int rebuild;        // gate: rebuild requested (set by the drift/ingest kernels or by the host)
    int disp;           // an atom moved more than skin/2 since the last build (fixed-interval policy)
    int overflow;       // bit0 halo capacity, bit1 list stride, bit2 special stride, bit3 task table, bit4 extended array / ghost table
    int violations;
    int max_icount;     // most atoms any brick owns (sizes the per-brick task table)
    int n_ghost;        // ghost copies in pos4e (extended array) of the last build
    unsigned long long n_rebuilds;
    unsigned long long n_pairs;  // real full-shell entries of the last build
    int max_neighbors;
    int max_halo;
    int max_special;
    int n_ext;          // atoms + ghost copies in the extended array of the last build
    // largest n_ghost / n_ext / max_halo / max_icount / max_neighbors of any rebuild since the first build. The counters
    // keep counting past a capacity, so after an overflow these size the next first build. (Five ints: they keep
    // rebuild_every .. call_max_disp2_bits a 48-byte tail the host uploads in one copy.)
    int peak_ghost, peak_ext, peak_halo, peak_icount, peak_neighbors;
    unsigned int ticket;  // last-block-done counter
    int rebuild_every;    // fixed-interval policy (0 = displacement-triggered)
    long long step;       // MD step counter (simulate!'s step_n), advanced on the device
    long long init_step;  // step_n at the start of the current mb_simulate_vv call
    unsigned int rng[4];  // Andersen thermostat: ctr1 lo/hi, key lo/hi
    // displacement bookkeeping (float bits of squared distances, non-negative floats order like unsigned ints)
    unsigned int max_disp2_bits;       // largest |x - x_ref|^2 since the last rebuild
    unsigned int call_max_disp2_bits;  // largest value any rebuild interval of the current call reached
};

// centre-of-mass velocity waiting to be subtracted by the next reader of the velocities (vv.cuh; published by the last CTA
// of K2, the Langevin step or NH2, or by the decomposed runs' v_cm kernels), and the velocity-rescaling thermostat's factor:
// the next reader applies v <- lam (v - v_cm), each part when its flag is set
template <typename T>
struct CmState {
    T v[3];
    int valid;
    T lam;
    int scaled;
    // v_cm = s / M from the momentum sum s = sum(m v) and inv_mass = 1 / M
    __device__ __forceinline__ void publish(const double s[3], double inv_mass) {
        for (int k = 0; k < 3; k++) v[k] = (T)(s[k] * inv_mass);
        valid = 1;
    }
    // the pending state applied to one velocity
    __device__ __forceinline__ void apply(typename VT<T>::T4& u) const {
        if (valid) { u.x -= v[0]; u.y -= v[1]; u.z -= v[2]; }
        if (scaled) { u.x *= lam; u.y *= lam; u.z *= lam; }
    }
};

struct BrickHdr {
    int halo_count;  // staged atoms incl. dummy + alignment pads
    int i_count;     // atoms owned by the brick
    unsigned int tx_pos, tx_lj;  // bytes the bulk copies deliver
    int any_shift;
    int pad[3];
};
struct Run {
    int gstart, count, soff, pad;  // gstart: index into the extended array pos4e; soff: index in the staged halo
};
struct IRow {
    int slot_begin, count, smem_begin, cum;
};

// TriclinicBoundary (src/spatial.jl:151-215): lower-triangular basis vectors, reciprocal heights and the projection
// constants of wrap_coords. Served by the no-list kernel only (boxes of this kind are small systems in the reference's
// tests); on = 0 for CubicBoundary.
template <typename T>
struct Tric {
    int on;
    T bv[3][3];
    T rs[3];
    T cot_bprojyz_cprojyz, cprojxy_x_over_z, cprojxy_y_over_z, cot_a_b;
};
// vector(c1, c2, ::TriclinicBoundary) with approx_images = true (src/spatial.jl:528-534): z, then y, then x
template <typename T>
__host__ __device__ inline void tric_vector(const Tric<T>& t, T& dx, T& dy, T& dz) {
    T k = ffloor(dz * t.rs[2] + (T)0.5);
    dx -= t.bv[2][0] * k; dy -= t.bv[2][1] * k; dz -= t.bv[2][2] * k;
    k = ffloor(dy * t.rs[1] + (T)0.5);
    dx -= t.bv[1][0] * k; dy -= t.bv[1][1] * k; dz -= t.bv[1][2] * k;
    k = ffloor(dx * t.rs[0] + (T)0.5);
    dx -= t.bv[0][0] * k; dy -= t.bv[0][1] * k; dz -= t.bv[0][2] * k;
}
// wrap_coords(v, ::TriclinicBoundary) (src/spatial.jl:584-600)
template <typename T>
__host__ __device__ inline void tric_wrap(const Tric<T>& t, T& x, T& y, T& z) {
    T k = ffloor(z * t.rs[2]);
    x -= t.bv[2][0] * k; y -= t.bv[2][1] * k; z -= t.bv[2][2] * k;
    k = ffloor((y - z * t.cot_bprojyz_cprojyz) * t.rs[1]);
    x -= t.bv[1][0] * k; y -= t.bv[1][1] * k; z -= t.bv[1][2] * k;
    const T ddx = z * t.cprojxy_x_over_z, ddy = z * t.cprojxy_y_over_z;
    k = ffloor((x - ddx - (y - ddy) * t.cot_a_b) * t.rs[0]);
    x -= t.bv[0][0] * k; y -= t.bv[0][1] * k; z -= t.bv[0][2] * k;
}

template <typename T>
struct Geom {
    T L[3], invL[3];
    T inv_cell[3];
    double Ld[3], celld[3];
    int nc[3], ncells;
    int b[3], nb[3], nbricks;
    int h, H[3];
    int max_runs, hcells, n_irows;
    int halo_cap, stride, sstride;
    int task_cap;  // entries per brick of the task table (even; 0 while the capacities are being measured)
    int nce[3], necells, nerows;  // extended grid: nc + 2h cells per dimension, rows = nce[1] * nce[2]
    int ext_cap, ghost_cap;       // capacities of pos4e / the ghost table (0 while they are being measured)
    Tric<T> tric;                 // no-list path only
    int n;        // atoms
    int align;    // atoms per 16 bytes of the lj2 array (2 for float, 1 for double)
    T rlist2;
    T skin_half2;
};

__device__ __forceinline__ int floor_div(int a, int b) { return (a >= 0) ? a / b : -((-a + b - 1) / b); }

// ---- R1: wrap into [0,L), cell id, count ------------------------------------------------------
template <typename T>
__global__ void bin_count_kernel(const Control* __restrict__ ctl, Geom<T> g, typename VT<T>::T4* __restrict__ pos4,
                                 int* __restrict__ cid_of, int* __restrict__ cell_count) {
    if (!ctl->rebuild) return;
    int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= g.n) return;
    typename VT<T>::T4 p = pos4[s];
    T x[3] = {p.x, p.y, p.z};
    int c[3];
#pragma unroll
    for (int d = 0; d < 3; d++) {
        T v = x[d] - ffloor(x[d] * g.invL[d]) * g.L[d];  // wrap_coord_1D, src/spatial.jl:573-579
        if (v >= g.L[d]) v -= g.L[d];
        if (v < (T)0) v = (T)0;
        x[d] = v;
        int ci = (int)(v * g.inv_cell[d]);
        c[d] = min(max(ci, 0), g.nc[d] - 1);
    }
    p.x = x[0]; p.y = x[1]; p.z = x[2];
    pos4[s] = p;
    int cid = (c[2] * g.nc[1] + c[1]) * g.nc[0] + c[0];
    cid_of[s] = cid;
    atomicAdd(&cell_count[cid], 1);
}

// ---- R2: exclusive scan of cell counts (single CTA) --------------------------------------------
// Every warp owns a contiguous chunk of cells and walks it in coalesced tiles of 32: chunk sums (lanes accumulate
// independently, one warp reduction) -> scan of the 32 chunk sums -> tile-by-tile shuffle scan with a register carry.
// Two block barriers in total (a tile-by-tile scan across the whole CTA cost four barriers per 1024 cells, 45 us at
// C2's 45 k cells).
__global__ void cell_scan_kernel(const Control* __restrict__ ctl, int ncells, int n, const int* __restrict__ cell_count,
                                 int* __restrict__ cell_start, int* __restrict__ cell_fill) {
    if (!ctl->rebuild) return;
    __shared__ int s_warp[32];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nw = blockDim.x >> 5;
    const int per = (((ncells + nw - 1) / nw) + 31) & ~31;  // cells per warp, whole tiles
    const int c0 = min(wid * per, ncells), c1 = min(c0 + per, ncells);
    int sum = 0;
#pragma unroll 4
    for (int c = c0 + lane; c < c1; c += 32) sum += cell_count[c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (lane == 0) s_warp[wid] = sum;
    __syncthreads();
    if (wid == 0) {
        int w = (lane < nw) ? s_warp[lane] : 0;
        int wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int t = __shfl_up_sync(0xffffffffu, wi, o);
            if (lane >= o) wi += t;
        }
        s_warp[lane] = wi - w;  // exclusive chunk offsets
    }
    __syncthreads();
    int carry = s_warp[wid];
    for (int base = c0; base < c1; base += 32) {
        const int c = base + lane;
        const int v = (c < c1) ? cell_count[c] : 0;
        int incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (c < c1) {
            cell_start[c] = carry + incl - v;
            cell_fill[c] = 0;
        }
        carry += __shfl_sync(0xffffffffu, incl, 31);
    }
    // n >= 0: the caller knows the total; n < 0: the last warp's carry is the total
    if (n >= 0) { if (tid == 0) cell_start[ncells] = n; }
    else if (wid == nw - 1 && lane == 0) cell_start[ncells] = carry;
}

// ---- R3: scatter old slots into their cell segment (order inside the cell fixed up by R4a) -----
__global__ void cell_scatter_kernel(const Control* __restrict__ ctl, int n, const int* __restrict__ cid_of,
                                    const int* __restrict__ cell_start, int* __restrict__ cell_fill,
                                    int* __restrict__ perm) {
    if (!ctl->rebuild) return;
    int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    int c = cid_of[s];
    int r = atomicAdd(&cell_fill[c], 1);
    perm[cell_start[c] + r] = s;
}

// ---- R4a: sort each cell segment by old slot (deterministic order), reset counts ---------------
__global__ void cell_sort_kernel(const Control* __restrict__ ctl, int ncells, const int* __restrict__ cell_start,
                                 int* __restrict__ perm, int* __restrict__ cell_count) {
    if (!ctl->rebuild) return;
    int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= ncells) return;
    int a = cell_start[c], b = cell_start[c + 1];
    for (int i = a + 1; i < b; i++) {
        int v = perm[i];
        int j = i - 1;
        while (j >= a && perm[j] > v) {
            perm[j + 1] = perm[j];
            j--;
        }
        perm[j + 1] = v;
    }
    cell_count[c] = 0;
}

// ---- R4b/R4c: permute the per-slot state into the new order ------------------------------------
template <typename T>
__global__ void permute_gather_kernel(const Control* __restrict__ ctl, int n, const int* __restrict__ perm,
                                      const typename VT<T>::T4* __restrict__ pos4,
                                      const typename VT<T>::T4* __restrict__ vel4,
                                      const typename VT<T>::T2* __restrict__ lj2, const int* __restrict__ orig,
                                      const T* __restrict__ mass, typename VT<T>::T4* __restrict__ pos4_t,
                                      typename VT<T>::T4* __restrict__ vel4_t, typename VT<T>::T2* __restrict__ lj2_t,
                                      int* __restrict__ orig_t, T* __restrict__ mass_t) {
    if (!ctl->rebuild) return;
    int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    int o = perm[s];
    pos4_t[s] = pos4[o];
    vel4_t[s] = vel4[o];
    lj2_t[s] = lj2[o];
    orig_t[s] = orig[o];
    mass_t[s] = mass[o];
}
template <typename T>
__global__ void permute_commit_kernel(const Control* __restrict__ ctl, int n,
                                      const typename VT<T>::T4* __restrict__ pos4_t,
                                      const typename VT<T>::T4* __restrict__ vel4_t,
                                      const typename VT<T>::T2* __restrict__ lj2_t, const int* __restrict__ orig_t,
                                      const T* __restrict__ mass_t, typename VT<T>::T4* __restrict__ pos4,
                                      typename VT<T>::T4* __restrict__ vel4, typename VT<T>::T2* __restrict__ lj2,
                                      int* __restrict__ orig, T* __restrict__ mass,
                                      typename VT<T>::T4* __restrict__ xref4, int* __restrict__ inv_orig) {
    if (!ctl->rebuild) return;
    int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    typename VT<T>::T4 p = pos4_t[s];
    pos4[s] = p;
    xref4[s] = p;
    vel4[s] = vel4_t[s];
    lj2[s] = lj2_t[s];
    int o = orig_t[s];
    orig[s] = o;
    inv_orig[o] = s;
    mass[s] = mass_t[s];
}

// ---- R4d: extended (ghost-padded) grid ---------------------------------------------------------------------
// Extended cell (ex, ey, ez), 0 <= e_d < nc_d + 2h, shows primary cell ((e_d - h) mod nc_d); cells outside [h, h + nc_d)
// are ghosts whose atoms are stored with their coordinates moved by +-L_d. An extended x-row is
// [last h cells of the primary row | the primary row | its first h cells], so its length and the offset of every cell
// in it follow from cell_start; only the row starts need a scan (nerows = nce[1] * nce[2] entries).
template <typename T>
__device__ __forceinline__ int ext_row_first_cell(const Geom<T>& g, int ey, int ez) {
    int py = ey - g.h, pz = ez - g.h;
    py += (py < 0) ? g.nc[1] : 0; py -= (py >= g.nc[1]) ? g.nc[1] : 0;
    pz += (pz < 0) ? g.nc[2] : 0; pz -= (pz >= g.nc[2]) ? g.nc[2] : 0;
    return (pz * g.nc[1] + py) * g.nc[0];
}
template <typename T>
__global__ void ext_row_totals_kernel(const Control* __restrict__ ctl, Geom<T> g, const int* __restrict__ cell_start,
                                      int* __restrict__ erow_total) {
    if (!ctl->rebuild) return;
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= g.nerows) return;
    const int c0 = ext_row_first_cell(g, r % g.nce[1], r / g.nce[1]);
    const int a = cell_start[c0], b = cell_start[c0 + g.nc[0]];
    erow_total[r] = (b - a) + (b - cell_start[c0 + g.nc[0] - g.h]) + (cell_start[c0 + g.h] - a);
}
template <typename T>
__global__ void ext_cells_kernel(Control* __restrict__ ctl, Geom<T> g, const int* __restrict__ cell_start,
                                 const int* __restrict__ erow_start, int* __restrict__ ecell_start) {
    if (!ctl->rebuild) return;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e > g.necells) return;
    if (e == g.necells) {
        const int total = erow_start[g.nerows];
        ecell_start[e] = total;
        ctl->n_ext = total;
        ctl->n_ghost = 0;
        if (g.ext_cap > 0 && total > g.ext_cap) atomicOr(&ctl->overflow, 16);
        return;
    }
    const int ex = e % g.nce[0], r = e / g.nce[0];
    const int c0 = ext_row_first_cell(g, r % g.nce[1], r / g.nce[1]);
    const int a = cell_start[c0], b = cell_start[c0 + g.nc[0]];
    const int left = b - cell_start[c0 + g.nc[0] - g.h];
    int off;
    if (ex < g.h) off = cell_start[c0 + g.nc[0] - g.h + ex] - cell_start[c0 + g.nc[0] - g.h];
    else if (ex < g.h + g.nc[0]) off = left + cell_start[c0 + ex - g.h] - a;
    else off = left + (b - a) + cell_start[c0 + ex - g.h - g.nc[0]] - a;
    ecell_start[e] = erow_start[r] + off;
}

// Map from slots to the extended array: ext_of[slot] = the atom's own entry; gptr[slot] = first ghost entry | count << 28;
// ghost table entry = (index in the extended array, image code), code = (sx+1) | (sy+1)<<2 | (sz+1)<<4, s_d in {-1,0,1}.
template <typename T>
struct ExtMap {
    const int* ext_of;
    const unsigned int* gptr;
    const int2* ghosts;
    typename VT<T>::T4* pos4e;
    double Ld[3];
};
template <typename T>
__device__ __forceinline__ typename VT<T>::T4 image_of(const double Ld[3], typename VT<T>::T4 p, int code) {
    // +-L in double, one rounding: the staged atom is in the frame of the brick's owned atoms
    p.x = (T)((double)p.x + (double)((code & 3) - 1) * Ld[0]);
    p.y = (T)((double)p.y + (double)(((code >> 2) & 3) - 1) * Ld[1]);
    p.z = (T)((double)p.z + (double)(((code >> 4) & 3) - 1) * Ld[2]);
    return p;
}
// store position p of slot s into an extended array (this rank's or a peer's): the atom's own entry and its ghost copies
template <typename T>
__device__ __forceinline__ void ext_store_at(const ExtMap<T>& m, int e_own, unsigned int gp, typename VT<T>::T4 p,
                                             typename VT<T>::T4* __restrict__ dst) {
    dst[e_own] = p;
    const int ng = (int)(gp >> 28);
    const int2* ge = m.ghosts + (gp & 0x0fffffffu);
    for (int k = 0; k < ng; k++) {
        const int2 e = ge[k];
        dst[e.x] = image_of<T>(m.Ld, p, e.y);
    }
}
template <typename T>
__device__ __forceinline__ void ext_store(const ExtMap<T>& m, int s, typename VT<T>::T4 p, typename VT<T>::T4* __restrict__ dst) {
    ext_store_at<T>(m, m.ext_of[s], m.gptr[s], p, dst);
}
// R4e: per-atom extended index + ghost table; also fills pos4e / lj2e for the positions of the rebuild
template <typename T>
__global__ void ext_atoms_kernel(Control* __restrict__ ctl, Geom<T> g, const int* __restrict__ cell_start,
                                 const int* __restrict__ ecell_start, const typename VT<T>::T4* __restrict__ pos4,
                                 const typename VT<T>::T2* __restrict__ lj2, int* __restrict__ ext_of,
                                 unsigned int* __restrict__ gptr, int2* __restrict__ ghosts,
                                 typename VT<T>::T4* __restrict__ pos4e, typename VT<T>::T2* __restrict__ lj2e,
                                 const int* __restrict__ orig, int* __restrict__ orig_e) {
    if (!ctl->rebuild) return;
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= g.n) return;
    if (g.ext_cap <= 0) {  // capacities are being measured: count the ghosts only
        const typename VT<T>::T4 p = pos4[s];
        const T x[3] = {p.x, p.y, p.z};
        int ng = 1;
        for (int d = 0; d < 3; d++) {
            const int c = min(max((int)(x[d] * g.inv_cell[d]), 0), g.nc[d] - 1);
            if (c < g.h || c >= g.nc[d] - g.h) ng *= 2;
        }
        if (ng > 1) atomicAdd(&ctl->n_ghost, ng - 1);
        return;
    }
    const typename VT<T>::T4 p = pos4[s];
    const T x[3] = {p.x, p.y, p.z};
    int c[3], ne[3], eo[3][2], sh[3][2];
#pragma unroll
    for (int d = 0; d < 3; d++) {
        c[d] = min(max((int)(x[d] * g.inv_cell[d]), 0), g.nc[d] - 1);  // same arithmetic as bin_count_kernel (positions are wrapped)
        eo[d][0] = c[d] + g.h; sh[d][0] = 0;
        ne[d] = 1;
        if (c[d] < g.h) { eo[d][1] = c[d] + g.h + g.nc[d]; sh[d][1] = 1; ne[d] = 2; }           // beyond the high face: +L
        else if (c[d] >= g.nc[d] - g.h) { eo[d][1] = c[d] + g.h - g.nc[d]; sh[d][1] = -1; ne[d] = 2; }  // below the low face: -L
    }
    const int cid = (c[2] * g.nc[1] + c[1]) * g.nc[0] + c[0];
    const int k = s - cell_start[cid];
    const int ng = ne[0] * ne[1] * ne[2] - 1;
    unsigned int base = 0;
    bool ok = true;
    if (ng > 0) {
        base = (unsigned int)atomicAdd(&ctl->n_ghost, ng);
        if ((int)base + ng > g.ghost_cap) { atomicOr(&ctl->overflow, 16); ok = false; }
    }
    const typename VT<T>::T2 lj = lj2 ? lj2[s] : make2<T>((T)0, (T)0);
    const int oa = orig_e ? orig[s] : 0;
    int w = 0;
    for (int iz = 0; iz < ne[2]; iz++)
        for (int iy = 0; iy < ne[1]; iy++)
            for (int ix = 0; ix < ne[0]; ix++) {
                const int e = (eo[2][iz] * g.nce[1] + eo[1][iy]) * g.nce[0] + eo[0][ix];
                const int ei = ecell_start[e] + k;
                if (ei >= g.ext_cap) continue;  // (overflow is flagged by ext_cells_kernel)
                const int code = (sh[0][ix] + 1) | ((sh[1][iy] + 1) << 2) | ((sh[2][iz] + 1) << 4);
                if (ix + iy + iz == 0) {
                    ext_of[s] = ei;
                    pos4e[ei] = p;
                } else {
                    if (ok) ghosts[base + w] = make_int2(ei, code);
                    w++;
                    pos4e[ei] = image_of<T>(g.Ld, p, code);
                }
                if (lj2e) lj2e[ei] = lj;
                if (orig_e) orig_e[ei] = oa;
            }
    gptr[s] = ok ? (base | ((unsigned int)ng << 28)) : 0u;
}
// refresh pos4e from pos4 for slots [s0, s0 + n) (after an ingest without a rebuild, or after a halo exchange over NCCL)
template <typename T>
__global__ void ext_fill_kernel(ExtMap<T> m, int s0, int n, const typename VT<T>::T4* __restrict__ pos4) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    ext_store<T>(m, s0 + k, pos4[s0 + k], m.pos4e);
}

// Task table: one int2 per owned atom of a brick, [brick * task_cap + task] = (slot, staged index | main-list length << 12 |
// special-list length << 24). brick_tables_kernel writes (slot, staged index), build_lists_kernel adds the lengths. The
// force kernel's producer warp copies a brick's entries into shared memory together with the halo.
constexpr int TASK_MAX_MAIN = 4095, TASK_MAX_SPECIAL = 255;
__host__ __device__ inline int task_pack(int si, int n_main, int n_spec) { return si | (n_main << 12) | (n_spec << 24); }


// ---- R5: brick tables ---------------------------------------------------------------------------
// One CTA per brick. Outputs: hdr, runs[max_runs] (one per (y,z) row of the halo: a contiguous range of the extended
// array), irows[n_irows], hcs[hcells] (start,end per halo cell in the staged halo), task table.
template <typename T>
__global__ void brick_tables_kernel(Control* __restrict__ ctl, Geom<T> g, const int* __restrict__ cell_start,
                                    const int* __restrict__ ecell_start, BrickHdr* __restrict__ hdrs,
                                    Run* __restrict__ runs, IRow* __restrict__ irows, ushort2* __restrict__ hcs,
                                    int2* __restrict__ task_tab, int uniform_lj) {
    if (!ctl->rebuild) return;
    extern __shared__ int s_mem[];
    int* s_len = s_mem;                  // max_runs
    int* s_base = s_mem + g.max_runs;    // max_runs
    __shared__ int s_total;
    const int b = blockIdx.x;
    const int tid = threadIdx.x;
    int B[3] = {b % g.nb[0], (b / g.nb[0]) % g.nb[1], b / (g.nb[0] * g.nb[1])};
    int c0[3], e[3], He[3];
#pragma unroll
    for (int d = 0; d < 3; d++) {
        c0[d] = B[d] * g.b[d];  // = extended coordinate of the halo's first cell (primary c0 - h, shifted by the h ghost cells)
        e[d] = min(g.b[d], g.nc[d] - c0[d]);
        He[d] = e[d] + 2 * g.h;
    }
    Run* my_runs = runs + (size_t)b * g.max_runs;
    const int A = g.align;
    // pass 1: run extents
    for (int r = tid; r < g.max_runs; r += blockDim.x) {
        const int ry = r % g.H[1], rz = r / g.H[1];
        Run run = {0, 0, 0, 0};
        int len = 0;
        if (ry < He[1] && rz < He[2]) {
            const int e_lo = ((c0[2] + rz) * g.nce[1] + (c0[1] + ry)) * g.nce[0] + c0[0];
            run.gstart = ecell_start[e_lo];
            run.count = ecell_start[e_lo + He[0]] - run.gstart;
            if (run.count > 0) len = ((run.gstart % A) + run.count + A - 1) / A * A;
        }
        my_runs[r] = run;
        s_len[r] = len;
    }
    __syncthreads();
    // serial-in-chunks exclusive scan of s_len (max_runs <= a few hundred): warp 0, 32 at a time
    if (tid < 32) {
        int carry = A;  // slots [0, A) hold the dummy atom
        for (int base = 0; base < g.max_runs; base += 32) {
            int r = base + tid;
            int v = (r < g.max_runs) ? s_len[r] : 0;
            int incl = v;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                int t = __shfl_up_sync(0xffffffffu, incl, o);
                if (tid >= o) incl += t;
            }
            if (r < g.max_runs) s_base[r] = carry + incl - v;
            carry += __shfl_sync(0xffffffffu, incl, 31);
        }
        if (tid == 0) s_total = carry;
    }
    __syncthreads();
    unsigned int tx_pos = 0, tx_lj = 0;
    for (int r = tid; r < g.max_runs; r += blockDim.x) {
        Run run = my_runs[r];
        if (run.count > 0) {
            run.soff = s_base[r] + (run.gstart % A);
            my_runs[r].soff = run.soff;
            tx_pos += (unsigned int)run.count * (unsigned int)sizeof(typename VT<T>::T4);
            if (!uniform_lj) tx_lj += (unsigned int)s_len[r] * (unsigned int)sizeof(typename VT<T>::T2);
        }
    }
    // block reduce tx through shared atomics
    __shared__ unsigned int s_tx_pos, s_tx_lj;
    if (tid == 0) { s_tx_pos = 0; s_tx_lj = 0; }
    __syncthreads();
    if (tx_pos) atomicAdd(&s_tx_pos, tx_pos);
    if (tx_lj) atomicAdd(&s_tx_lj, tx_lj);
    __syncthreads();
    // halo cell table
    ushort2* my_hcs = hcs + (size_t)b * g.hcells;
    for (int hc = tid; hc < g.hcells; hc += blockDim.x) {
        int rx = hc % g.H[0], ry = (hc / g.H[0]) % g.H[1], rz = hc / (g.H[0] * g.H[1]);
        ushort2 se = make_ushort2(0, 0);
        if (rx < He[0] && ry < He[1] && rz < He[2]) {
            const int ec = ((c0[2] + rz) * g.nce[1] + (c0[1] + ry)) * g.nce[0] + c0[0] + rx;
            const Run run = my_runs[rz * g.H[1] + ry];
            const int cs = ecell_start[ec], ce = ecell_start[ec + 1];
            int st = run.soff + (cs - run.gstart);
            int en = st + (ce - cs);
            st = min(st, 65535);
            en = min(en, 65535);
            se = make_ushort2((unsigned short)st, (unsigned short)en);
        }
        my_hcs[hc] = se;
    }
    __syncthreads();
    __shared__ int s_icount;
    IRow* my_rows = irows + (size_t)b * g.n_irows;
    if (tid == 0) {
        int cum = 0;
        for (int q = 0; q < g.n_irows; q++) {
            int iy = q % g.b[1], iz = q / g.b[1];
            IRow row = {0, 0, 0, cum};
            if (iy < e[1] && iz < e[2]) {
                int cid0 = ((c0[2] + iz) * g.nc[1] + (c0[1] + iy)) * g.nc[0] + c0[0];
                row.slot_begin = cell_start[cid0];
                row.count = cell_start[cid0 + e[0]] - row.slot_begin;
                int hc = ((iz + g.h) * g.H[1] + (iy + g.h)) * g.H[0] + g.h;
                row.smem_begin = my_hcs[hc].x;
            }
            my_rows[q] = row;
            cum += row.count;
        }
        BrickHdr hd;
        hd.halo_count = s_total;
        hd.i_count = (g.ext_cap > 0 && ecell_start[g.necells] > g.ext_cap) ? 0 : cum;  // extended array overflow: nothing may be staged
        hd.tx_pos = s_tx_pos;
        hd.tx_lj = s_tx_lj;
        hd.any_shift = 0;
        hd.pad[0] = hd.pad[1] = hd.pad[2] = 0;
        hdrs[b] = hd;
        s_icount = cum;
        atomicMax(&ctl->max_halo, s_total);
        atomicMax(&ctl->max_icount, cum);
        if (s_total > g.halo_cap) atomicOr(&ctl->overflow, 1);
        if (g.task_cap > 0 && cum > g.task_cap) atomicOr(&ctl->overflow, 8);
    }
    __syncthreads();
    // task table: (slot, staged index) of every owned atom, rows in order (the list builder adds the list lengths)
    if (task_tab != nullptr && g.task_cap > 0) {
        const int nt = min(s_icount, g.task_cap);
        for (int t = tid; t < nt; t += blockDim.x) {
            int q = 0;
            while (q + 1 < g.n_irows && my_rows[q + 1].cum <= t) q++;
            const IRow row = my_rows[q];
            task_tab[(size_t)b * g.task_cap + t] = make_int2(row.slot_begin + (t - row.cum), task_pack(row.smem_begin + (t - row.cum), 0, 0));
        }
    }
}

// ---- halo staging of the list builder (the force kernel's producer warp has its own pipelined copy loop) ---------
// Stages the pos4e runs of brick b into shared memory with bulk async copies and waits for them. The staged atoms are
// already in one frame (ghost cells hold shifted images), so nothing is touched after the copy.
template <typename T>
__device__ __forceinline__ void stage_halo(const Geom<T>& g, const BrickHdr& hd, const Run* __restrict__ my_runs,
                                           const typename VT<T>::T4* __restrict__ pos4e, typename VT<T>::T4* s_pos,
                                           uint64_t* bar) {
    using T4 = typename VT<T>::T4;
    const int tid = threadIdx.x;
    if (tid == 0) {
        mbar_init(bar, 1);
        mbar_fence_init();
    }
    if (tid < g.align) s_pos[tid] = make4<T>((T)1.0e6, (T)1.0e6, (T)1.0e6, (T)0);  // dummy atom: far away, no charge
    __syncthreads();
    if (tid == 0) mbar_arrive_expect_tx(bar, hd.tx_pos);
    __syncthreads();
    for (int r = tid; r < g.max_runs; r += blockDim.x) {
        Run run = my_runs[r];
        if (run.count > 0) bulk_g2s(&s_pos[run.soff], &pos4e[run.gstart], (uint32_t)run.count * (uint32_t)sizeof(T4), bar);
    }
    mbar_wait(bar, 0);
    __syncthreads();
}

// Main-list entries are stored as halo index << LIST_SHIFT (= byte offset of a float4 position in shared memory): the
// force kernel saves a shift per entry. 16-bit entries therefore address at most LIST_MAX_HALO staged atoms per brick.
constexpr int LIST_SHIFT = 4;
constexpr int LIST_MAX_HALO = 65536 >> LIST_SHIFT;
// ---- R6: full-shell neighbour lists --------------------------------------------------------------
// One CTA per brick, one warp per owned atom. Entries are 16-bit halo indices written in the lane-
// swizzled order the force kernel reads (see force.cuh). Excluded pairs are dropped here; special
// (1-4) pairs go to a separate short list (SURVEY Appendix A.2).
template <typename T, bool COUNT_ONLY, bool HAS_EX>
__global__ void __launch_bounds__(256)
    build_lists_kernel(Control* __restrict__ ctl, Geom<T> g, const BrickHdr* __restrict__ hdrs,
                       const Run* __restrict__ runs, const IRow* __restrict__ irows, const ushort2* __restrict__ hcs,
                       const typename VT<T>::T4* __restrict__ pos4e, const int* __restrict__ orig_e,
                       const int* __restrict__ ex_ptr, const int* __restrict__ ex_idx, const int* __restrict__ sp_ptr,
                       const int* __restrict__ sp_idx, unsigned short* __restrict__ list,
                       unsigned short* __restrict__ slist, ushort2* __restrict__ counts, int2* __restrict__ task_tab,
                       int brick0, int split) {
    if (!ctl->rebuild) return;
    using T4 = typename VT<T>::T4;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int b = (int)blockIdx.x / split + brick0;  // `split` CTAs share a brick: CTA k takes the tasks k, k + split, ... of each warp
    const BrickHdr hd = hdrs[b];
    if (hd.i_count == 0 || hd.halo_count > g.halo_cap) return;
    T4* s_pos = reinterpret_cast<T4*>(smem_raw);
    int* s_orig = reinterpret_cast<int*>(s_pos + g.halo_cap);
    ushort2* s_hcs = reinterpret_cast<ushort2*>(s_orig + g.halo_cap);
    IRow* s_rows = reinterpret_cast<IRow*>(s_hcs + ((g.hcells + 3) & ~3));
    __shared__ uint64_t s_bar;
    const Run* my_runs = runs + (size_t)b * g.max_runs;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nw = blockDim.x >> 5;
    // far-away fill for every slot (covers alignment pads), then stage
    for (int k = tid; k < hd.halo_count; k += blockDim.x) {
        s_pos[k] = make4<T>((T)1.0e6, (T)1.0e6, (T)1.0e6, (T)0);
        s_orig[k] = -1;
    }
    for (int k = tid; k < g.hcells; k += blockDim.x) s_hcs[k] = hcs[(size_t)b * g.hcells + k];
    for (int k = tid; k < g.n_irows; k += blockDim.x) s_rows[k] = irows[(size_t)b * g.n_irows + k];
    __syncthreads();
    fence_proxy_async();
    stage_halo<T>(g, hd, my_runs, pos4e, s_pos, &s_bar);
    if (HAS_EX) {
        for (int r = wid; r < g.max_runs; r += nw) {
            Run run = my_runs[r];
            for (int k = lane; k < run.count; k += 32) s_orig[run.soff + k] = orig_e[run.gstart + k];
        }
    }
    __syncthreads();
    // brick corner (the row trimming below works in coordinates relative to it; distances are frame-independent)
    double org[3];
    {
        const int B[3] = {b % g.nb[0], (b / g.nb[0]) % g.nb[1], b / (g.nb[0] * g.nb[1])};
#pragma unroll
        for (int d = 0; d < 3; d++) org[d] = (double)(B[d] * g.b[d]) * g.celld[d];
    }

    int my_max = 0;
    unsigned long long my_pairs = 0;
    for (int task = wid * split + (int)blockIdx.x % split; task < hd.i_count; task += nw * split) {
        // locate the owned atom
        int q = 0;
        while (q + 1 < g.n_irows && s_rows[q + 1].cum <= task) q++;
        IRow row = s_rows[q];
        int k_in_row = task - row.cum;
        int slot = row.slot_begin + k_in_row;
        int si = row.smem_begin + k_in_row;
        int iy = q % g.b[1], iz = q / g.b[1];
        // which cell of the row holds it
        int ix = 0;
        {
            int hc0 = ((iz + g.h) * g.H[1] + (iy + g.h)) * g.H[0] + g.h;
            while (ix + 1 < g.b[0] && si >= (int)s_hcs[hc0 + ix].y) ix++;
        }
        const T4 pi = s_pos[si];
        const T lx = (T)((double)pi.x - org[0]), ly = (T)((double)pi.y - org[1]), lz = (T)((double)pi.z - org[2]);
        int oi = HAS_EX ? s_orig[si] : 0;
        // exclusion / special partner lists of atom oi into lanes
        int ex_a = ex_ptr ? ex_ptr[oi] : 0, ex_n = ex_ptr ? ex_ptr[oi + 1] - ex_a : 0;
        int sp_a = sp_ptr ? sp_ptr[oi] : 0, sp_n = sp_ptr ? sp_ptr[oi + 1] - sp_a : 0;
        int my_ex = (lane < ex_n) ? ex_idx[ex_a + lane] : -2;
        int my_sp = (lane < sp_n) ? sp_idx[sp_a + lane] : -2;
        // Partners are bonded neighbours, so their original indices lie within a short span of oi. A step of 32 candidates
        // that holds no atom inside that span skips both partner loops (most steps: the partner lists are checked for a
        // few candidates per atom only).
        int span_lo = 0x7fffffff, span_hi = -1;
        if (HAS_EX) {
            for (int kk = lane; kk < ex_n; kk += 32) { const int v = ex_idx[ex_a + kk]; span_lo = min(span_lo, v); span_hi = max(span_hi, v); }
            for (int kk = lane; kk < sp_n; kk += 32) { const int v = sp_idx[sp_a + kk]; span_lo = min(span_lo, v); span_hi = max(span_hi, v); }
            span_lo = __reduce_min_sync(0xffffffffu, span_lo);
            span_hi = __reduce_max_sync(0xffffffffu, span_hi);
        }
        int count = 0, scount = 0;
        unsigned short* my_list = list + (size_t)slot * g.stride;
        unsigned short* my_slist = slist + (size_t)slot * g.sstride;
        // Only the part of each halo row that can hold a neighbour is scanned: with dy, dz the distance from the
        // atom to the row's (y,z) cell slab, candidates need |dx| <= sqrt(r_list^2 - dy^2 - dz^2). The (2h+1)^2 rows
        // are handled 32 at a time: lane r trims row r, a warp scan turns the row lengths into offsets, and the
        // candidates of all rows are then walked as ONE flattened range (every lane busy; a 5-step shuffle search
        // maps a flattened index back to its row). Entry order = row-major, as a row-by-row scan would give.
        const T cyv = (T)g.celld[1], czv = (T)g.celld[2];
        const T inv_cx = g.inv_cell[0];
        const T rl2 = g.rlist2 * (T)1.0001;
        const int side = 2 * g.h + 1, nrows = side * side;
        for (int rb = 0; rb < nrows; rb += 32) {
            const int r = rb + lane;
            int ra = 0, rlen = 0;
            if (r < nrows) {
                const int rz = iz + r / side, ry = iy + r % side;
                const T zlo = (T)(rz - g.h) * czv;
                const T dzm = fmax(fmax(zlo - lz, lz - (zlo + czv)), (T)0);
                const T ylo = (T)(ry - g.h) * cyv;
                const T dym = fmax(fmax(ylo - ly, ly - (ylo + cyv)), (T)0);
                const T rem = rl2 - dym * dym - dzm * dzm;
                if (rem >= (T)0) {
                    const T wx = fsqrt(rem) + (T)1e-4;
                    int rx_lo = (int)ffloor((lx - wx) * inv_cx) + g.h;
                    int rx_hi = (int)ffloor((lx + wx) * inv_cx) + g.h;
                    rx_lo = max(rx_lo, ix);
                    rx_hi = min(rx_hi, ix + 2 * g.h);
                    const int hcrow = (rz * g.H[1] + ry) * g.H[0];
                    ra = s_hcs[hcrow + rx_lo].x;
                    rlen = max((int)s_hcs[hcrow + rx_hi].y - ra, 0);
                }
            }
            int inc = rlen;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                int v = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += v;
            }
            const int roff = inc - rlen;  // exclusive offset of this lane's row in the flattened range
            const int total = __shfl_sync(0xffffffffu, inc, 31);
            // Compact the non-empty rows into lanes 0 .. nnz-1 (start index, flattened offset): the walk below then maps a
            // flattened position to its row with one warp OR-reduction and two shuffles instead of a 5-step shuffle search.
            const unsigned int nz = __ballot_sync(0xffffffffu, rlen > 0);
            const int nnz = __popc(nz);
            int src = 0;
            {
                unsigned int m = nz;
                int o = lane;  // position of the (lane+1)-th set bit of nz
#pragma unroll
                for (int sh = 16; sh > 0; sh >>= 1) {
                    const int cnt = __popc(m & ((1u << sh) - 1u));
                    if (o >= cnt) { o -= cnt; m >>= sh; src += sh; }
                }
            }
            const int cra = __shfl_sync(0xffffffffu, ra, src & 31);
            const int croff_all = __shfl_sync(0xffffffffu, roff, src & 31);  // (every lane takes part in the shuffle)
            const int croff = (lane < nnz) ? croff_all : 0x3fffffff;
            int starts_before = 0;  // compacted rows that start before k0
            for (int k0 = 0; k0 < total; k0 += 32) {
                const int k = k0 + lane;
                const unsigned int rel = (unsigned int)(croff - k0);
                const unsigned int mask = __reduce_or_sync(0xffffffffu, rel < 32u ? (1u << rel) : 0u);  // row starts inside this step
                const int ord = starts_before + __popc(mask & (0xffffffffu >> (31 - lane))) - 1;    // last row starting at or before k
                starts_before += __popc(mask);
                const int c = __shfl_sync(0xffffffffu, cra, ord & 31) + (k - __shfl_sync(0xffffffffu, croff, ord & 31));
                bool in = false, special = false;
                if (k < total && c != si) {
                    T4 pj = s_pos[c];
                    T dx = pi.x - pj.x, dy = pi.y - pj.y, dz = pi.z - pj.z;
                    T d2 = dx * dx + dy * dy + dz * dz;
                    in = d2 <= g.rlist2;
                }
                int oj = (HAS_EX && in) ? s_orig[c] : -1;
                const bool near_partner = HAS_EX && __any_sync(0xffffffffu, in && oj >= span_lo && oj <= span_hi);
                // exclusions (warp-uniform loops over the partner lists)
                if (HAS_EX && near_partner && ex_n > 0) {
                    int nn = min(ex_n, 32);
                    for (int kk = 0; kk < nn; kk++) {
                        int v = __shfl_sync(0xffffffffu, my_ex, kk);
                        if (v == oj) in = false;
                    }
                    for (int kk = 32; kk < ex_n; kk++)
                        if (ex_idx[ex_a + kk] == oj) in = false;
                }
                if (HAS_EX && near_partner && sp_n > 0) {
                    int nn = min(sp_n, 32);
                    for (int kk = 0; kk < nn; kk++) {
                        int v = __shfl_sync(0xffffffffu, my_sp, kk);
                        if (in && v == oj) special = true;
                    }
                    for (int kk = 32; kk < sp_n; kk++)
                        if (in && sp_idx[sp_a + kk] == oj) special = true;
                }
                bool main_hit = in && !special;
                bool spec_hit = in && special;
                unsigned int mb_ = __ballot_sync(0xffffffffu, main_hit);
                unsigned int sb_ = __ballot_sync(0xffffffffu, spec_hit);
                unsigned int lt = (1u << lane) - 1u;
                if (!COUNT_ONLY) {
                    if (main_hit) {
                        int m = count + __popc(mb_ & lt);
                        if (m < g.stride) {
                            int phys = (m & ~31) + ((m & 7) << 2) + ((m & 31) >> 3);
                            my_list[phys] = (unsigned short)(c << LIST_SHIFT);
                        }
                    }
                    if (spec_hit) {
                        int m = scount + __popc(sb_ & lt);
                        if (m < g.sstride) my_slist[m] = (unsigned short)c;
                    }
                }
                count += __popc(mb_);
                scount += __popc(sb_);
            }
        }
        if (!COUNT_ONLY) {
            // pad the last group of 32 with the dummy atom (halo slot 0)
            int padded = min((count + 31) & ~31, g.stride);
            for (int m = count + lane; m < padded; m += 32) {
                int phys = (m & ~31) + ((m & 7) << 2) + ((m & 31) >> 3);
                my_list[phys] = 0;
            }
            if (lane == 0) {
                counts[slot] = make_ushort2((unsigned short)min(count, g.stride), (unsigned short)min(scount, g.sstride));
                if (task < g.task_cap)
                    task_tab[(size_t)b * g.task_cap + task] = make_int2(slot, task_pack(si, min(count, g.stride), min(scount, g.sstride)));
                if (count > g.stride) atomicOr(&ctl->overflow, 2);
                if (scount > g.sstride) atomicOr(&ctl->overflow, 4);
            }
        }
        my_max = max(my_max, count);
        if (lane == 0) {
            my_pairs += (unsigned long long)(count + scount);
            atomicMax(&ctl->max_special, scount);
        }
    }
    if (lane == 0) {
        atomicMax(&ctl->max_neighbors, my_max);
        atomicAdd(&ctl->n_pairs, my_pairs);
    }
}

// ---- R7: finish ------------------------------------------------------------------------------
__global__ void rebuild_finish_kernel(Control* ctl) {
    if (!ctl->rebuild) return;
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        if (ctl->disp) ctl->violations++;
        ctl->disp = 0;
        ctl->rebuild = 0;
        ctl->n_rebuilds++;
        ctl->peak_ghost = max(ctl->peak_ghost, ctl->n_ghost);
        ctl->peak_ext = max(ctl->peak_ext, ctl->n_ext);
        ctl->peak_halo = max(ctl->peak_halo, ctl->max_halo);
        ctl->peak_icount = max(ctl->peak_icount, ctl->max_icount);
        ctl->peak_neighbors = max(ctl->peak_neighbors, ctl->max_neighbors);
        if (ctl->max_disp2_bits > ctl->call_max_disp2_bits) ctl->call_max_disp2_bits = ctl->max_disp2_bits;
        ctl->max_disp2_bits = 0;
    }
}
__global__ void rebuild_begin_kernel(Control* ctl) {
    if (!ctl->rebuild) return;
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        ctl->n_pairs = 0;
        ctl->max_neighbors = 0;
        ctl->max_halo = 0;
        ctl->max_special = 0;
        ctl->max_icount = 0;
    }
}

}  // namespace mb
