// pme.cuh — smooth particle-mesh Ewald reciprocal space and the Ewald exclusion correction (SURVEY.md §8(f)-3).
//
// Replaces the reference's `PME` general interaction (src/interactions/ewald.jl:363-958: grid placement :489-498,
// order-5 B-splines :518-556, charge spreading :598-617, reciprocal convolution :676-732, force interpolation
// :838-873, self / neutralising-background energy :947-956) and the `EwaldExclusion` specific interaction
// (:1016-1055). The pair-space term (`CoulombEwald`) is COUL_EWALD in force.cuh. Grid layout: complex, index
// (ix * K1 + iy) * K2 + iz, transformed in place by cuFFT (C2C / Z2Z, unnormalised both ways like fft! / bfft!).
// Checker: oracle/pme.py, pinned against OpenMM's forces_all_pme_exact (tests/test_oracle.py).
//
// Validation. Every kernel is a thin loop over a __host__ __device__ per-item function. tests/test_pme_host.py compiles
// those functions for the host and checks the chain spread -> FFT -> convolution -> inverse FFT -> interpolation ->
// exclusion against oracle/pme.py and the OpenMM goldens. On the device, tests/test_zz_gpu_pme.py matches OpenMM for 6mrr
// (f64) and the three waters (f64, f32). tests/test_gpu_pme_matrix.py compares PME-only systems with oracle/pme.py in
// f64 (1e-9) and f32: cubic, anisotropic and K = 6 meshes with odd and even K, error_tol 1e-3 to 1e-5, net charge,
// uncharged atoms, eps_r != 1, coordinates outside the box, edge exclusion pairs, both force paths, 6mrr, a finite-
// difference check, and mb_set_box / mb_set_atoms on a live context. tests/test_pme_direct_ewald.py pins oracle/pme.py
// against a direct Ewald sum on the same shapes. Nothing calls into this file unless mb_set_pme was.
#pragma once
#include "common.cuh"

namespace mb {

#ifndef MB_HD
#define MB_HD __host__ __device__ __forceinline__
#endif

constexpr int PME_ORDER = 5;
constexpr int PME_THREADS = 128;

struct PmeGeom {
    int K[3];
    double L[3];
};

// order-5 cardinal B-spline weights th[0..4] and derivatives dth[0..4] at grid fraction dr (ewald.jl:518-556)
template <typename T>
MB_HD void pme_bspline(T dr, T* th, T* dth) {
    constexpr int order = PME_ORDER;
    th[order - 1] = (T)0;
    th[1] = dr;
    th[0] = (T)1 - dr;
#pragma unroll
    for (int k = 3; k < order; k++) {
        const T d = (T)1 / (T)(k - 1);
        th[k - 1] = d * dr * th[k - 2];
#pragma unroll
        for (int l = 1; l <= k - 2; l++) th[k - l - 1] = d * ((dr + (T)l) * th[k - l - 2] + ((T)(k - l) - dr) * th[k - l - 1]);
        th[0] *= d * ((T)1 - dr);
    }
    dth[0] = -th[0];
#pragma unroll
    for (int k = 1; k < order; k++) dth[k] = th[k - 1] - th[k];
    const T d = (T)1 / (T)(order - 1);
    th[order - 1] = d * dr * th[order - 2];
#pragma unroll
    for (int l = 1; l <= order - 2; l++)
        th[order - l - 1] = d * ((dr + (T)l) * th[order - l - 2] + ((T)(order - l) - dr) * th[order - l - 1]);
    th[0] *= d * ((T)1 - dr);
}

// grid_placement (ewald.jl:489-498): first grid index and fraction per dimension
template <typename T>
MB_HD void pme_place(const typename VT<T>::T4& p, const PmeGeom& g, int* i0, T* fr) {
    const double c[3] = {(double)p.x, (double)p.y, (double)p.z};
#pragma unroll
    for (int d = 0; d < 3; d++) {
        double t = c[d] / g.L[d];
        t = (t - floor(t)) * (double)g.K[d];
        const int ti = (int)floor(t);
        fr[d] = (T)(t - (double)ti);
        i0[d] = ti % g.K[d];
    }
}

template <typename T>
MB_HD void pme_grid_add(T* addr, T v) {
#ifdef __CUDA_ARCH__
    atomicAdd(addr, v);
#else
    *addr += v;
#endif
}

// spread_charge (ewald.jl:598-617) for one atom: 125 adds into the real part of the grid
template <typename T>
MB_HD void pme_spread_atom(int s, const PmeGeom& g, const typename VT<T>::T4* pos4, typename VT<T>::T2* grid) {
    const typename VT<T>::T4 p = pos4[s];
    if (p.w == (T)0) return;
    int i0[3];
    T fr[3], th[3][PME_ORDER], dth[PME_ORDER];
    pme_place<T>(p, g, i0, fr);
#pragma unroll
    for (int d = 0; d < 3; d++) pme_bspline<T>(fr[d], th[d], dth);
    for (int a = 0; a < PME_ORDER; a++) {
        const int ix = (i0[0] + a) % g.K[0];
        const T qx = p.w * th[0][a];
        for (int b = 0; b < PME_ORDER; b++) {
            const int iy = (i0[1] + b) % g.K[1];
            const T qxy = qx * th[1][b];
            for (int c = 0; c < PME_ORDER; c++) {
                const int iz = (i0[2] + c) % g.K[2];
                pme_grid_add<T>(&grid[((size_t)ix * g.K[1] + iy) * g.K[2] + iz].x, qxy * th[2][c]);
            }
        }
    }
}

// recip_conv (ewald.jl:676-732) for one mesh point: S(k) *= eterm(k); returns eterm |S|^2 (0 at k = 0, which stays
// untouched like in the reference)
template <typename T>
MB_HD double pme_conv_point(size_t idx, const PmeGeom& g, double f_div_eps, double factor, double boxfactor,
                            const double* bsm_x, const double* bsm_y, const double* bsm_z, typename VT<T>::T2* grid) {
    if (idx == 0) return 0.0;
    const int kz = (int)(idx % g.K[2]);
    const int ky = (int)((idx / g.K[2]) % g.K[1]);
    const int kx = (int)(idx / ((size_t)g.K[2] * g.K[1]));
    const int mx = (kx < 0.5 * (g.K[0] + 1)) ? kx : kx - g.K[0];
    const int my = (ky < 0.5 * (g.K[1] + 1)) ? ky : ky - g.K[1];
    const int mz = (kz < 0.5 * (g.K[2] + 1)) ? kz : kz - g.K[2];
    const double hx = mx / g.L[0], hy = my / g.L[1], hz = mz / g.L[2];
    const double m2 = hx * hx + hy * hy + hz * hz;
    const double denom = m2 * boxfactor * bsm_x[kx] * bsm_y[ky] * bsm_z[kz];
    const double eterm = f_div_eps * exp(-factor * m2) / denom;
    typename VT<T>::T2 v = grid[idx];
    const double e = eterm * ((double)v.x * (double)v.x + (double)v.y * (double)v.y);
    v.x = (T)((double)v.x * eterm);
    v.y = (T)((double)v.y * eterm);
    grid[idx] = v;
    return e;
}

// interpolate_force (ewald.jl:838-873) for one atom: F_i -= q (fx K0/L0, fy K1/L1, fz K2/L2); one writer per slot
template <typename T>
MB_HD void pme_interp_atom(int s, const PmeGeom& g, const typename VT<T>::T4* pos4, const typename VT<T>::T2* grid,
                           typename VT<T>::T4* f4) {
    const typename VT<T>::T4 p = pos4[s];
    if (p.w == (T)0) return;
    int i0[3];
    T fr[3], th[3][PME_ORDER], dth[3][PME_ORDER];
    pme_place<T>(p, g, i0, fr);
#pragma unroll
    for (int d = 0; d < 3; d++) pme_bspline<T>(fr[d], th[d], dth[d]);
    T fx = (T)0, fy = (T)0, fz = (T)0;
    for (int a = 0; a < PME_ORDER; a++) {
        const int ix = (i0[0] + a) % g.K[0];
        for (int b = 0; b < PME_ORDER; b++) {
            const int iy = (i0[1] + b) % g.K[1];
            const T dtx_ty = dth[0][a] * th[1][b], tx_dty = th[0][a] * dth[1][b], txy = th[0][a] * th[1][b];
            for (int c = 0; c < PME_ORDER; c++) {
                const int iz = (i0[2] + c) % g.K[2];
                const T gv = grid[((size_t)ix * g.K[1] + iy) * g.K[2] + iz].x;
                fx += dtx_ty * th[2][c] * gv;
                fy += tx_dty * th[2][c] * gv;
                fz += txy * dth[2][c] * gv;
            }
        }
    }
    typename VT<T>::T4 f = f4[s];
    f.x -= p.w * fx * (T)((double)g.K[0] / g.L[0]);
    f.y -= p.w * fy * (T)((double)g.K[1] / g.L[1]);
    f.z -= p.w * fz * (T)((double)g.K[2] / g.L[2]);
    f4[s] = f;
}

// EwaldExclusion (ewald.jl:1016-1055) for one excluded-or-special pair: removes the erf(alpha r)/r part that the
// reciprocal sum contains for pairs the pair kernel does not treat with the Ewald real-space term. Returns the energy.
template <typename T>
MB_HD double ewald_exclusion_pair(int t, const int* pairs, const int* slot_of, const typename VT<T>::T4* pos4,
                                  typename VT<T>::T4* f4, const double* L, double alpha, double f_div_eps) {
    int i = pairs[2 * t], j = pairs[2 * t + 1];
    if (slot_of) { i = slot_of[i]; j = slot_of[j]; }
    const typename VT<T>::T4 pi = pos4[i], pj = pos4[j];
    // vector(c_i, c_j) = c_j - c_i, minimum image
    T v[3] = {pj.x - pi.x, pj.y - pi.y, pj.z - pi.z};
#pragma unroll
    for (int d = 0; d < 3; d++) v[d] -= (T)L[d] * (T)rint((double)(v[d] * (T)(1.0 / L[d])));
    const double r = sqrt((double)(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]));
    const double qq = (double)pi.w * (double)pj.w;
    const double ar = alpha * r;
    const double erf_ar = erf(ar);
    if (!(erf_ar > 1e-6)) return -alpha * 2.0 * f_div_eps * qq / 1.7724538509055160273;
    const double inv_r = 1.0 / r;
    const double de_dr = f_div_eps * qq * inv_r * inv_r * inv_r * (erf_ar - 2.0 * ar * exp(-ar * ar) / 1.7724538509055160273);
    T* fi = reinterpret_cast<T*>(&f4[i]);
    T* fj = reinterpret_cast<T*>(&f4[j]);
#pragma unroll
    for (int d = 0; d < 3; d++) {  // SpecificForce2Atoms(F, -F) with F = dE_dr * vec_ij
        pme_grid_add<T>(fi + d, (T)de_dr * v[d]);
        pme_grid_add<T>(fj + d, -((T)de_dr * v[d]));
    }
    return -f_div_eps * qq * inv_r * erf_ar;
}

#ifdef __CUDACC__
template <typename T>
__global__ void __launch_bounds__(PME_THREADS)
    pme_spread_kernel(int n, PmeGeom g, const typename VT<T>::T4* __restrict__ pos4, typename VT<T>::T2* __restrict__ grid) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < n) pme_spread_atom<T>(s, g, pos4, grid);
}

template <typename T, bool ENERGY>
__global__ void __launch_bounds__(PME_THREADS)
    pme_conv_kernel(PmeGeom g, double f_div_eps, double factor, double boxfactor, const double* __restrict__ bsm_x,
                    const double* __restrict__ bsm_y, const double* __restrict__ bsm_z, typename VT<T>::T2* __restrict__ grid,
                    double* __restrict__ partial) {
    const size_t total = (size_t)g.K[0] * g.K[1] * g.K[2];
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    double e = 0.0;
    if (idx < total) e = pme_conv_point<T>(idx, g, f_div_eps, factor, boxfactor, bsm_x, bsm_y, bsm_z, grid);
    if (ENERGY) {
        e = block_sum<PME_THREADS>(e);
        if (threadIdx.x == 0) partial[blockIdx.x] = 0.5 * e;  // the mesh holds k and -k: E = 1/2 sum
    }
}

template <typename T>
__global__ void __launch_bounds__(PME_THREADS)
    pme_interp_kernel(int n, PmeGeom g, const typename VT<T>::T4* __restrict__ pos4,
                      const typename VT<T>::T2* __restrict__ grid, typename VT<T>::T4* __restrict__ f4) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < n) pme_interp_atom<T>(s, g, pos4, grid, f4);
}

template <typename T, bool ENERGY>
__global__ void __launch_bounds__(PME_THREADS)
    ewald_exclusion_kernel(int n_pairs, const int* __restrict__ pairs, const int* __restrict__ slot_of,
                           const typename VT<T>::T4* __restrict__ pos4, typename VT<T>::T4* __restrict__ f4, PmeGeom g,
                           double alpha, double f_div_eps, double* __restrict__ partial) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    double e = 0.0;
    if (t < n_pairs) e = ewald_exclusion_pair<T>(t, pairs, slot_of, pos4, f4, g.L, alpha, f_div_eps);
    if (ENERGY) {
        e = block_sum<PME_THREADS>(e);
        if (threadIdx.x == 0) partial[blockIdx.x] = e;
    }
}

__global__ void add_const_kernel(double* acc, double v) { *acc += v; }
#endif  // __CUDACC__

}  // namespace mb
