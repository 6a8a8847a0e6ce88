// dpd.cuh — dissipative particle dynamics: the DPDInteraction pair term (src/interactions/dpd.jl:57-142), its pairwise
// draw, and the predicted-velocity buffer the pair kernels read.
//
// Data layout on a DPD context: the w component of every position record (pos4, pos4e, the staged halo) holds the atom's
// original index as an exact value (T)orig instead of a charge; every kernel that moves or copies positions copies w through.
// The predicted velocities v_pred (xyz) live in vpred4[orig], in original atom order, so cell-list re-sorts never permute them
// and ghost images need no velocity copies. A pair evaluation gathers vpred4[orig_j] from global memory only for pairs
// inside r_c.
#pragma once
#include "cells.cuh"

namespace mb {

// The kernel constants of a DPDInteraction, digested on the host (mb_set_dpd), plus the buffers the pair kernels read. The
// all-pairs kernel takes it as an argument; the brick kernel reads it from device memory (dpd_args_of).
// inv_sqrt_dt = 1 / sqrt(dt) of the interaction's dt (not the integrator's); e_pre = (a / 2) r_c.
template <typename T>
struct DpdArgs {
    T a, gamma, sigma, rc, inv_sqrt_dt, e_pre;
    uint32_t key_lo, key_hi;
    int nl;                                  // use_neighbors: exclusions apply (the all-pairs kernel; lists never hold them)
    int dissipative;                         // gamma or sigma != 0: gather v_j and draw xi (0: the conservative force only)
    const typename VT<T>::T4* vpred;         // predicted velocities, original order (xyz)
    const long long* step;                   // step_n the draws are keyed by (Control::step)
};

// The DpdArgs the brick kernel's DPD variant reads through its LJ-parameter pointer, which no other part of that variant
// uses: it stages positions only (brick_force_kernel static_asserts the instantiation). The engine passes the address of a
// DpdArgs in device memory there (Engine::dpd_args_as_lj2e). A kernel argument of its own would change the code of every
// other brick_force_kernel instantiation.
template <typename T>
__device__ __forceinline__ const DpdArgs<T>& dpd_args_of(const typename VT<T>::T2* p) {
    return *reinterpret_cast<const DpdArgs<T>*>(p);
}

// What the DPD drift (vv_kick_drift_kernel<T, TH_DPD>) adds to VelocityVerlet's K1: v_pred = v_half + (lambda - 1/2) dt F / m
// into vpred[orig] (lam_dt = (lambda - 1/2) dt)
template <typename T>
struct DpdDrift {
    typename VT<T>::T4* vpred;
    T lam_dt;
};

// xi_ij of step `step`: one Philox4x32-10 block with counter (min(i, j) + 1, max(i, j) + 1, step_lo, step_hi) and key
// (key_lo, key_hi), i and j 0-based original indices (the reference's 1-based atom.index, dpd.jl:92-98). One N(0, 1) value
// from words 0 and 1 by the first output of box_muller3, in double. Symmetric in (i, j), so f_ij = -f_ji exactly. The
// reference draws through PhiloxRNG.jl's randn; the two agree in distribution only.
__host__ __device__ __forceinline__ double dpd_normal(int i, int j, long long step, uint32_t key_lo, uint32_t key_hi) {
    uint32_t c[4] = {(uint32_t)((i < j ? i : j) + 1), (uint32_t)((i < j ? j : i) + 1), (uint32_t)(unsigned long long)step,
                     (uint32_t)((unsigned long long)step >> 32)};
    philox4x32_10(c, key_lo, key_hi);
    const double u1 = ((double)c[0] + 1.0) * (1.0 / 4294967296.0), u2 = (double)c[1] * (1.0 / 4294967296.0);
    return sqrt(-2.0 * log(u1)) * cos(6.283185307179586 * u2);
}

// One pair at distance r (r = |d|, d = c_i - c_j) with dv = v_i - v_j and the pair's draw xi: fr such that the force on i is
// fr d, and the conservative energy e. Zero for r >= r_c and for r == 0 (beads on top of each other). In the reference's
// terms (dr = c_j - c_i = -d, fs[i] -= f dr): fr = f_C + f_D + f_R with
//   w = 1 - r / r_c, f_C = a w / r, f_D = gamma w^2 (dr . dv) / r^2, f_R = sigma w xi dt^(-1/2) / r,  e = (a / 2) r_c w^2.
template <typename T>
__host__ __device__ __forceinline__ void dpd_pair(const DpdArgs<T>& P, T r, T dx, T dy, T dz, T dvx, T dvy, T dvz, T xi, T& fr,
                                                  T& e) {
    if (!(r < P.rc) || r == (T)0) {
        fr = (T)0;
        e = (T)0;
        return;
    }
    const T w = (T)1 - r / P.rc;
    const T inv_r = (T)1 / r;
    const T f_c = P.a * w * inv_r;
    const T rdotv = -(dx * dvx + dy * dvy + dz * dvz) * inv_r * inv_r;  // dr . dv / r^2
    const T f_d = P.gamma * (w * w) * rdotv;
    const T f_r = P.sigma * w * xi * P.inv_sqrt_dt * inv_r;
    fr = f_c + f_d + f_r;
    e = P.e_pre * w * w;
}

// dpd_normal out of line: the pair kernels call it from the main-list and the special-list loop, and an inlined copy in
// each would not fit the registers of the f64 energy variant
static __device__ __noinline__ double dpd_normal_call(int i, int j, long long step, uint32_t key_lo, uint32_t key_hi) {
    return dpd_normal(i, j, step, key_lo, key_hi);
}

// One pair as the force kernels evaluate it: orig_i, orig_j from the position records' w, v_i = vi (the i atom's predicted
// velocity, loaded once per atom), v_j gathered and xi drawn only inside r_c, and only when gamma or sigma is non-zero.
template <typename T>
__device__ __forceinline__ void dpd_eval(const DpdArgs<T>& P, long long step, int oi, const typename VT<T>::T4& vi, T r2, T dx, T dy,
                                         T dz, T wj, T& fr, T& e) {
    const T r = sqrt(r2);
    fr = (T)0;
    e = (T)0;
    if (r < P.rc && r > (T)0) {
        T dvx = (T)0, dvy = (T)0, dvz = (T)0, xi = (T)0;
        if (P.dissipative) {
            const int oj = (int)wj;
            const typename VT<T>::T4 vj = P.vpred[oj];
            dvx = vi.x - vj.x;
            dvy = vi.y - vj.y;
            dvz = vi.z - vj.z;
            xi = (T)dpd_normal_call(oi, oj, step, P.key_lo, P.key_hi);
        }
        dpd_pair<T>(P, r, dx, dy, dz, dvx, dvy, dvz, xi, fr, e);
    }
}

// vpred4[orig[s]] = v of slot s after the pending v_cm (the prologue's F0 uses the current velocities)
template <typename T>
__global__ void dpd_vpred_init_kernel(int n, const typename VT<T>::T4* __restrict__ vel4, const int* __restrict__ orig,
                                      const CmState<T>* __restrict__ cm, typename VT<T>::T4* __restrict__ vpred) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    typename VT<T>::T4 v = vel4[s];
    cm->apply(v);
    vpred[orig[s]] = v;
}

// vpred4[i] = the caller's velocity of atom i (n x 3, original order): mb_forces_energy_vel
template <typename T>
__global__ void dpd_vpred_from_kernel(int n, const T* __restrict__ vels, typename VT<T>::T4* __restrict__ vpred) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    vpred[i] = make4<T>(vels[3 * (size_t)i], vels[3 * (size_t)i + 1], vels[3 * (size_t)i + 2], (T)0);
}

}  // namespace mb
