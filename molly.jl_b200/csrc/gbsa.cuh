// gbsa.cuh — generalized-Born implicit solvent: ImplicitSolventOBC and ImplicitSolventGBN2
// (src/interactions/implicit_solvent.jl). Three dependent all-pairs passes, each needing every atom's result of the pass
// before it:
//   gb_born_kernel         I_i = sum_j the OBC integral (+ the GBN2 neck term), then per atom B_i, B'_i and the ACE seed
//                          (born_radii_loop_OBC / _GBN2, born_radii_sum, forces! :623-725, :1082-1088)
//   gb_pair_kernel<ENERGY> dG/dr forces and the Born forces bf_i = sum_j dG/d(alpha^2_ij) B_j, then b_i = bf_i B_i^2 B'_i;
//                          with ENERGY also gb_energy_loop (gb_force_loop_1, :839-876, :1095-1130)
//   gb_chain_kernel        F_k -= sum_j (x_j - x_k) (de_kj + de_jk), de_ij = b_i (t3_ij - I'_ij) / r (gb_force_loop_2,
//                          :878-898); the neck derivative I'_ij is recomputed here, so nothing n x n is stored
// No atomics: CTA (x, y) owns the atoms [128 x, 128 x + 128) (one per thread) and sums over the j split y, so every pair is
// evaluated from both of its sides. Per-split partials go to a buffer, and the last CTA of a column (per-column ticket)
// adds them in split order and finishes its atoms; with ENERGY the last CTA of the grid adds the per-CTA energies in index
// order. Same inputs, same bits. Per-pair arithmetic is in T, as in the reference; I, the Born forces and the energy are
// summed in double, the forces in T. Atoms are walked in slot order (the cell-list path's sort); the per-atom GB
// parameters stay in original order and are read through orig. Forces are added to f4 (one writer per slot).
#pragma once
#include "bonded.cuh"

namespace mb {

constexpr int GB_THREADS = 128;     // owned atoms per CTA, and atoms per staged j tile
constexpr int GB_CHUNK = 32;        // granularity of the j split
constexpr int GB_MAX_CLASSES = 32;  // MB_GB_MAX_NECK_CLASSES

template <typename T>
struct GbParams {
    int n, n_cls;
    int chunk;  // j atoms per split (a multiple of GB_CHUNK); gridDim.y splits
    int use_ace;
    T rc, rc2;  // 0: no cutoff
    T offset, neck_scale, neck_cut, kappa, f_solute, f_solvent;
    double offset_d, probe, sa_factor;
};

template <typename T>
struct GbArgs {
    using T4 = typename VT<T>::T4;
    const T4* par;     // original order: (offset radius, scaled offset radius, radius = offset radius + offset, neck class)
    const T4* abg;     // original order: (alpha, beta, gamma, 0)
    const T* d0;       // n_cls^2, entry [c_i n_cls + c_j] = the reference's d0s[i, j]
    const T* m0;
    const int* orig;   // slot -> original index
    const T4* pos4;    // slot order (x, y, z, q)
    T4* f4;            // slot order, forces added
    T* B;              // slot order: Born radius
    T* b;              // slot order: b_i = bf_i B_i^2 B'_i
    dbl4* st;          // slot order: (ACE seed of the Born force, B_i^2 B'_i, B_i, the ACE term sa_i), in double
    double* pd;        // [split][n] double partials (I, then the Born forces)
    T4* pf;            // [split][n] force partials
    double* pe;        // [gridDim.x gridDim.y] pair energies, then [gridDim.x] self energies
    unsigned int* tk;  // [gridDim.x] column tickets, then one grid ticket
    double* acc;       // energy accumulator (ENERGY)
};

// True in every thread of the CTA that takes the last of `count` tickets on *ticket (wraps back to 0): last_cta for a
// ticket other than the grid's.
__device__ __forceinline__ bool gb_last_of(unsigned int* ticket, unsigned int count) {
    __shared__ bool s_last;
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        s_last = (atomicInc(ticket, count - 1) == count - 1);
    }
    __syncthreads();
    return s_last;
}

// a force partial written by another CTA of this launch (L2, not a possibly stale L1 line)
template <typename T>
__device__ __forceinline__ Vec3<T> gb_ld_partial(const typename VT<T>::T4* p) {
    const T* q = reinterpret_cast<const T*>(p);
    return v3(__ldcg(q), __ldcg(q + 1), __ldcg(q + 2));
}

// the OBC integral of one ordered pair (born_radii_loop_OBC :629-637)
template <typename T>
__device__ __forceinline__ T gb_obc_integral(T r, T ori, T srj) {
    T I = 0;
    const T U = r + srj;
    if (ori < U) {
        const T D = fabs(r - srj);
        const T L = fmax(ori, D);
        I += ((T)1 / L - (T)1 / U + (r - (srj * srj) / r) * ((T)1 / (U * U) - (T)1 / (L * L)) / (T)4 + log(L / U) / ((T)2 * r)) / (T)2;
        if (ori < (srj - r)) I += (T)2 * ((T)1 / ori - (T)1 / L);
    }
    return I;
}
// the GBN2 neck term of one ordered pair and its derivative (born_radii_loop_GBN2 :711-723); d0, m0 of (c_i, c_j)
template <typename T>
__device__ __forceinline__ void gb_neck(T r, T d0, T m0, T neck_scale, T& I, T& I_grad) {
    const T s = (T)10 * (r - d0);  // the integral uses Angstrom
    const T s2 = s * s, s4 = s2 * s2;
    const T denom = (T)1 + s2 + (T)3 * (s4 * s2) / (T)10;
    I = neck_scale * m0 / denom;
    const T numer = (T)2 * s + (T)9 * (s4 * s) / (T)5;
    I_grad = -((T)10 * neck_scale * m0 * numer / (denom * denom));
}
// t3 of gb_force_loop_2 (:885-891), for a pair with ori < r + srj
template <typename T>
__device__ __forceinline__ T gb_t3(T r, T ori, T srj, T r2inv) {
    const T L = (T)1 / fmax(ori, fabs(r - srj));
    const T U = (T)1 / (r + srj);
    return ((T)1 + (srj * srj) * r2inv) * (L * L - U * U) / (T)8 + log(U / L) * r2inv / (T)4;
}
// pre_factor of gb_force_loop_1 (:856-861)
template <typename T>
__device__ __forceinline__ T gb_force_pre(const GbParams<T>& P, T den) {
    if (P.kappa == (T)0) return P.f_solute + P.f_solvent;
    const T ek = exp(-P.kappa * den);
    return P.f_solute + ek * P.f_solvent + P.kappa * den * ek * P.f_solvent;
}
// dGpol/dr and dGpol/d(alpha^2_ij) of one pair at squared distance r2 (:851-864); returns the GB distance
// f_ij = sqrt(r2 + B_i B_j exp(-r2 / (4 B_i B_j))), which gb_energy_loop uses too
template <typename T>
__device__ __forceinline__ T gb_pair_terms(const GbParams<T>& P, T r2, T Bi, T Bj, T qi, T qj, T& dGdr, T& dGda) {
    const T a2 = Bi * Bj;
    const T D = r2 / ((T)4 * a2);
    const T ex = exp(-D);
    const T den2 = r2 + a2 * ex;
    const T den = sqrt(den2);
    const T G = (gb_force_pre(P, den) * qi * qj) / den;
    dGdr = -G * ((T)1 - ex / (T)4) / den2;
    dGda = -G * ex * ((T)1 + D) / ((T)2 * den2);
    return den;
}

template <typename T>
__device__ __forceinline__ void gb_load_tables(const GbParams<T>& P, const GbArgs<T>& a, T* s_d0, T* s_m0) {
    for (int k = threadIdx.x; k < P.n_cls * P.n_cls; k += GB_THREADS) {
        s_d0[k] = a.d0[k];
        s_m0[k] = a.m0[k];
    }
}

// ---- pass 1: Born radii ------------------------------------------------------------------------------------------------
template <typename T, typename Box>
__global__ void __launch_bounds__(GB_THREADS) gb_born_kernel(const GbParams<T> P, const GbArgs<T> a, const Box box) {
    using T4 = typename VT<T>::T4;
    __shared__ T4 s_pos[GB_THREADS], s_par[GB_THREADS];
    __shared__ T s_d0[GB_MAX_CLASSES * GB_MAX_CLASSES], s_m0[GB_MAX_CLASSES * GB_MAX_CLASSES];
    gb_load_tables(P, a, s_d0, s_m0);
    const Mic<T, Box> mic(box);
    const int i = blockIdx.x * GB_THREADS + threadIdx.x;
    const bool own = i < P.n;
    const T4 zero = make4<T>(0, 0, 0, 0);
    const T4 pi = own ? a.pos4[i] : zero, gi = own ? a.par[a.orig[i]] : zero;
    const int ci = (int)gi.w;
    double I = 0;
    const int j0 = blockIdx.y * P.chunk, j1 = min(j0 + P.chunk, P.n);
    for (int t0 = j0; t0 < j1; t0 += GB_THREADS) {
        const int m = min(GB_THREADS, j1 - t0);
        __syncthreads();
        if ((int)threadIdx.x < m) {
            s_pos[threadIdx.x] = a.pos4[t0 + threadIdx.x];
            s_par[threadIdx.x] = a.par[a.orig[t0 + threadIdx.x]];
        }
        __syncthreads();
        if (own)
            for (int k = 0; k < m; k++) {
                if (t0 + k == i) continue;
                const Vec3<T> dr = mic(pi, s_pos[k]);
                const T r = fsqrt(dot(dr, dr));
                if (r == (T)0 || (P.rc > (T)0 && r > P.rc)) continue;
                const T4 gj = s_par[k];
                T Iij = gb_obc_integral(r, gi.x, gj.y);
                if (P.n_cls > 0 && r < (gi.z + gj.z + P.neck_cut)) {
                    const int c = ci * P.n_cls + (int)gj.w;
                    T In, Ig;
                    gb_neck(r, s_d0[c], s_m0[c], P.neck_scale, In, Ig);
                    Iij += In;
                }
                I += (double)Iij;
            }
    }
    if (own) a.pd[(size_t)blockIdx.y * P.n + i] = I;
    if (!gb_last_of(&a.tk[blockIdx.x], gridDim.y)) return;
    __threadfence();
    if (!own) return;
    double s = 0;
    for (int y = 0; y < (int)gridDim.y; y++) s += __ldcg(&a.pd[(size_t)y * P.n + i]);
    // born_radii_sum (:649-658) and the ACE seed (:1082-1088), in double
    const T4 abg = a.abg[a.orig[i]];
    const double orr = (double)gi.x, radius = orr + P.offset_d;
    const double psi = s * orr, psi2 = psi * psi;
    const double th = tanh((double)abg.x * psi - (double)abg.y * psi2 + (double)abg.z * psi2 * psi);
    const double B = 1.0 / (1.0 / orr - th / radius);
    const double Bg = (1.0 - th * th) * (orr * ((double)abg.x - 2.0 * (double)abg.y * psi + 3.0 * (double)abg.z * psi2)) / radius;
    double seed = 0, sa = 0;
    if (P.use_ace && B > 0) {
        const double rr = radius / B, rr2 = rr * rr;
        sa = P.sa_factor * (radius + P.probe) * (radius + P.probe) * (rr2 * rr2 * rr2);
        seed = -6.0 * sa / B;
    }
    a.B[i] = (T)B;
    a.st[i] = dbl4{seed, B * B * Bg, B, sa};
}

// ---- pass 2: dG/dr forces and Born forces (+ energy) -------------------------------------------------------------------
template <typename T, bool ENERGY, typename Box>
__global__ void __launch_bounds__(GB_THREADS) gb_pair_kernel(const GbParams<T> P, const GbArgs<T> a, const Box box) {
    using T4 = typename VT<T>::T4;
    __shared__ T4 s_pos[GB_THREADS];
    __shared__ T s_B[GB_THREADS];
    const Mic<T, Box> mic(box);
    const int i = blockIdx.x * GB_THREADS + threadIdx.x;
    const bool own = i < P.n;
    const T4 pi = own ? a.pos4[i] : make4<T>(0, 0, 0, 0);
    const T Bi = own ? a.B[i] : (T)1;
    T fx = 0, fy = 0, fz = 0;
    double bf = 0, e = 0;
    const int j0 = blockIdx.y * P.chunk, j1 = min(j0 + P.chunk, P.n);
    for (int t0 = j0; t0 < j1; t0 += GB_THREADS) {
        const int m = min(GB_THREADS, j1 - t0);
        __syncthreads();
        if ((int)threadIdx.x < m) {
            s_pos[threadIdx.x] = a.pos4[t0 + threadIdx.x];
            s_B[threadIdx.x] = a.B[t0 + threadIdx.x];
        }
        __syncthreads();
        if (own)
            for (int k = 0; k < m; k++) {
                if (t0 + k == i) continue;
                const T4 pj = s_pos[k];
                const Vec3<T> dr = mic(pi, pj);
                const T r2 = dot(dr, dr);
                if (P.rc > (T)0 && r2 > P.rc2) continue;
                const T Bj = s_B[k];
                T dGdr, dGda;
                const T f = gb_pair_terms(P, r2, Bi, Bj, pi.w, pj.w, dGdr, dGda);
                fx += dr.x * dGdr;
                fy += dr.y * dGdr;
                fz += dr.z * dGdr;
                bf += (double)(dGda * Bj);
                if (ENERGY) {  // gb_energy_loop (:1110-1126) over ordered pairs, each half of the pair's term
                    const T fc = (P.rc > (T)0) ? ((T)1 / f - (T)1 / P.rc) : (T)1 / f;
                    const T pre = (P.kappa == (T)0) ? P.f_solute + P.f_solvent : P.f_solute + exp(-P.kappa * f) * P.f_solvent;
                    e += 0.5 * (double)(pre * pi.w * pj.w * fc);
                }
            }
    }
    if (own) {
        a.pd[(size_t)blockIdx.y * P.n + i] = bf;
        a.pf[(size_t)blockIdx.y * P.n + i] = make4<T>(fx, fy, fz, (T)0);
    }
    if (ENERGY) {
        e = block_sum<GB_THREADS>(e);
        if (threadIdx.x == 0) a.pe[(size_t)blockIdx.y * gridDim.x + blockIdx.x] = e;
    }
    if (gb_last_of(&a.tk[blockIdx.x], gridDim.y)) {
        __threadfence();
        double es = 0;
        if (own) {
            double s = 0;
            T gx = 0, gy = 0, gz = 0;
            for (int y = 0; y < (int)gridDim.y; y++) {
                s += __ldcg(&a.pd[(size_t)y * P.n + i]);
                const Vec3<T> f = gb_ld_partial<T>(&a.pf[(size_t)y * P.n + i]);
                gx += f.x; gy += f.y; gz += f.z;
            }
            T4 f = a.f4[i];
            f.x += gx; f.y += gy; f.z += gz;
            a.f4[i] = f;
            // the self pair (r = 0) feeds the Born force only
            T dGdr, dGda;
            gb_pair_terms(P, (T)0, Bi, Bi, pi.w, pi.w, dGdr, dGda);
            const dbl4 st = a.st[i];
            a.b[i] = (T)((st.x + s + (double)(dGda * Bi)) * st.y);
            if (ENERGY) {  // self term and ACE term of gb_energy_loop (:1098-1109), in double
                const double q = (double)pi.w;
                const double pre = (P.kappa == (T)0) ? (double)P.f_solute + (double)P.f_solvent
                                                     : (double)P.f_solute + exp(-(double)P.kappa * st.z) * (double)P.f_solvent;
                es = pre * q * q / (2.0 * st.z) + st.w;
            }
        }
        if (ENERGY) {
            es = block_sum<GB_THREADS>(es);
            if (threadIdx.x == 0) a.pe[(size_t)gridDim.x * gridDim.y + blockIdx.x] = es;
        }
    }
    if (ENERGY && gb_last_of(&a.tk[gridDim.x], gridDim.x * gridDim.y)) {
        __threadfence();
        const int np = (int)(gridDim.x * gridDim.y + gridDim.x);
        double s = 0;
        for (int k = threadIdx.x; k < np; k += GB_THREADS) s += __ldcg(&a.pe[k]);
        s = block_sum<GB_THREADS>(s);
        if (threadIdx.x == 0) *a.acc += s;
    }
}

// ---- pass 3: the chain rule through the Born radii ---------------------------------------------------------------------
template <typename T, typename Box>
__global__ void __launch_bounds__(GB_THREADS) gb_chain_kernel(const GbParams<T> P, const GbArgs<T> a, const Box box) {
    using T4 = typename VT<T>::T4;
    __shared__ T4 s_pos[GB_THREADS], s_par[GB_THREADS];
    __shared__ T s_b[GB_THREADS];
    __shared__ T s_d0[GB_MAX_CLASSES * GB_MAX_CLASSES], s_m0[GB_MAX_CLASSES * GB_MAX_CLASSES];
    gb_load_tables(P, a, s_d0, s_m0);
    const Mic<T, Box> mic(box);
    const int i = blockIdx.x * GB_THREADS + threadIdx.x;
    const bool own = i < P.n;
    const T4 zero = make4<T>(0, 0, 0, 0);
    const T4 pi = own ? a.pos4[i] : zero, gi = own ? a.par[a.orig[i]] : zero;
    const T bi = own ? a.b[i] : (T)0;
    const int ci = (int)gi.w;
    T fx = 0, fy = 0, fz = 0;
    const int j0 = blockIdx.y * P.chunk, j1 = min(j0 + P.chunk, P.n);
    for (int t0 = j0; t0 < j1; t0 += GB_THREADS) {
        const int m = min(GB_THREADS, j1 - t0);
        __syncthreads();
        if ((int)threadIdx.x < m) {
            s_pos[threadIdx.x] = a.pos4[t0 + threadIdx.x];
            s_par[threadIdx.x] = a.par[a.orig[t0 + threadIdx.x]];
            s_b[threadIdx.x] = a.b[t0 + threadIdx.x];
        }
        __syncthreads();
        if (own)
            for (int k = 0; k < m; k++) {
                if (t0 + k == i) continue;
                const Vec3<T> dr = mic(pi, s_pos[k]);
                const T r = fsqrt(dot(dr, dr));
                if (r == (T)0 || (P.rc > (T)0 && r > P.rc)) continue;
                const T4 gj = s_par[k];
                const int cj = (int)gj.w;
                const T rinv = (T)1 / r, r2inv = rinv * rinv;
                const bool neck = P.n_cls > 0 && r < (gi.z + gj.z + P.neck_cut);
                T de = 0;
                if (gi.x < r + gj.y) {  // de_ij: i's Born force through I_i
                    T ig = 0, In;
                    if (neck) gb_neck(r, s_d0[ci * P.n_cls + cj], s_m0[ci * P.n_cls + cj], P.neck_scale, In, ig);
                    de += bi * (gb_t3(r, gi.x, gj.y, r2inv) - ig) * rinv;
                }
                if (gj.x < r + gi.y) {  // de_ji: j's Born force through I_j
                    T ig = 0, In;
                    if (neck) gb_neck(r, s_d0[cj * P.n_cls + ci], s_m0[cj * P.n_cls + ci], P.neck_scale, In, ig);
                    de += s_b[k] * (gb_t3(r, gj.x, gi.y, r2inv) - ig) * rinv;
                }
                fx -= dr.x * de;
                fy -= dr.y * de;
                fz -= dr.z * de;
            }
    }
    if (own) a.pf[(size_t)blockIdx.y * P.n + i] = make4<T>(fx, fy, fz, (T)0);
    if (!gb_last_of(&a.tk[blockIdx.x], gridDim.y)) return;
    __threadfence();
    if (!own) return;
    T gx = 0, gy = 0, gz = 0;
    for (int y = 0; y < (int)gridDim.y; y++) {
        const Vec3<T> f = gb_ld_partial<T>(&a.pf[(size_t)y * P.n + i]);
        gx += f.x; gy += f.y; gz += f.z;
    }
    T4 f = a.f4[i];
    f.x += gx; f.y += gy; f.z += gz;
    a.f4[i] = f;
}

}  // namespace mb
