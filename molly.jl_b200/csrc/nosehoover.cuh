// nosehoover.cuh — the Nosé-Hoover integrator (Evans and Holian 1985; src/simulators.jl:1491-1614) as two passes per atom
// around the force evaluation:
//   NH1  v -= v_cm (pending);  sum m|v|^2;  v_half = v + (F/m - v zeta) dt/2;  sum m|v_half|^2;  x += v_half dt;
//        displacement check; the last CTA updates zeta from both kinetic sums
//   F    forces at the new x
//   NH2  v = (v_half + F/m dt/2) / (1 + zeta dt/2);  sum(m v) -> v_cm (last CTA, fixed order)
// zeta and the kinetic sums are double; the per-atom arithmetic stays in T, in the reference's order of operations.
#pragma once
#include "vv.cuh"

namespace mb {

// The thermostat variable of one simulate call: zeroed in the call's prologue (the reference keeps zeta as a local of
// simulate!, so every call starts from 0), written by NH1's last CTA, read by NH2 and the next NH1.
struct NhState {
    double zeta;  // ps^-1
};

struct NhCoef {
    double coef;   // dt / (2 Q^2), Q = damping
    double nf_kT;  // Nf k T0 with Nf = 3N - 3: T / T0 = sum m|v|^2 / (Nf k T0)
};

// zeta after one step from sum m|v|^2 of the full-step velocities (mv2_old, before the step's kick) and of the half-step
// velocities (mv2_half): zeta_half = zeta + coef (T(v) / T0 - 1), zeta' = zeta_half + coef (T(v_half) / T0 - 1)
// (src/simulators.jl:1575-1579).
__host__ __device__ inline double nh_zeta_step(double zeta, double mv2_old, double mv2_half, NhCoef c) {
    const double zeta_half = zeta + c.coef * (mv2_old / c.nf_kT - 1.0);
    return zeta_half + c.coef * (mv2_half / c.nf_kT - 1.0);
}

// NH1: one atom per thread (grid-stride). (sum m|v|^2, sum m|v_half|^2) go through grid_sum; the last CTA updates zeta and does
// the step bookkeeping (step_advance). zeta and the step counter read below are overwritten by that CTA (last_cta orders every
// CTA's reads before its ticket). Four CTAs per SM: left to itself, ptxas squeezes the f32 instantiation into 48 registers and
// spills in the ghost-copy loop.
template <typename T>
__global__ void __launch_bounds__(VV_THREADS, 4)
    nh_kick_drift_kernel(int n, T dt, T dt_half, T skin_half2, NhCoef nc, NhState* __restrict__ nh, const CmState<T>* cm,
                         const typename VT<T>::T4* __restrict__ f4, const typename VT<T>::T4* __restrict__ xref4,
                         typename VT<T>::T4* __restrict__ pos4, typename VT<T>::T4* __restrict__ vel4, const T* __restrict__ mass,
                         double* __restrict__ partial, int* __restrict__ flag, Control* __restrict__ ctl,
                         cudaGraphConditionalHandle handle, int use_handle, ExtMap<T> ext) {
    const double zeta = nh->zeta;
    const T z = (T)zeta;
    const bool cmv = cm->valid != 0;
    const T cx = cm->v[0], cy = cm->v[1], cz = cm->v[2];
    bool moved = false;
    double k2[2] = {0, 0};  // sum m|v|^2 of the full-step velocities, of the half-step velocities
    for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x) {
        typename VT<T>::T4 v = vel4[s], p = pos4[s];
        const typename VT<T>::T4 f = f4[s], r = xref4[s];
        const T m = mass[s];
        int e_own = 0;
        unsigned int e_gp = 0;
        if (ext.pos4e) { e_own = ext.ext_of[s]; e_gp = ext.gptr[s]; }
        if (cmv) { v.x -= cx; v.y -= cy; v.z -= cz; }
        k2[0] += (double)m * ((double)v.x * v.x + (double)v.y * v.y + (double)v.z * v.z);
        const T im = v.w;  // 1/m (massless atoms: 0, no kick)
        v.x = v.x + (f.x * im - v.x * z) * dt_half;
        v.y = v.y + (f.y * im - v.y * z) * dt_half;
        v.z = v.z + (f.z * im - v.z * z) * dt_half;
        k2[1] += (double)m * ((double)v.x * v.x + (double)v.y * v.y + (double)v.z * v.z);
        p.x += v.x * dt; p.y += v.y * dt; p.z += v.z * dt;
        vel4[s] = v;
        pos4[s] = p;
        if (ext.pos4e) ext_store_at<T>(ext, e_own, e_gp, p, ext.pos4e);
        const T dx = p.x - r.x, dy = p.y - r.y, dz = p.z - r.z;
        moved |= (dx * dx + dy * dy + dz * dz > skin_half2);
    }
    if (moved) *flag = 1;
    if (!grid_sum<VV_THREADS, 2>(k2, partial, &ctl->ticket) || threadIdx.x != 0) return;
    nh->zeta = nh_zeta_step(zeta, k2[0], k2[1], nc);
    step_advance(ctl, handle, use_handle);  // (last: nothing stays live across its conditional-node call)
}

// NH2: one atom per thread (grid-stride). NH1 consumed the pending v_cm. When do_cm, sum(m v) goes through grid_sum and the last
// CTA publishes v_cm = sum(m v) / sum(m), applied lazily by the next reader of the velocities; otherwise v_cm is marked
// consumed.
template <typename T>
__global__ void __launch_bounds__(VV_THREADS)
    nh_kick2_kernel(int n, T dt_half, int do_cm, double inv_total_mass, const NhState* __restrict__ nh,
                    const typename VT<T>::T4* __restrict__ f4, const T* __restrict__ mass, typename VT<T>::T4* __restrict__ vel4,
                    double* __restrict__ partial, Control* __restrict__ ctl, CmState<T>* __restrict__ cm) {
    const T den = (T)1 + (T)nh->zeta * dt_half;
    double mv[3] = {0, 0, 0};
    for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x) {
        typename VT<T>::T4 v = vel4[s];
        const typename VT<T>::T4 f = f4[s];
        const T im = v.w;
        v.x = (v.x + f.x * im * dt_half) / den;
        v.y = (v.y + f.y * im * dt_half) / den;
        v.z = (v.z + f.z * im * dt_half) / den;
        vel4[s] = v;
        if (do_cm) {
            const T m = mass[s];
            mv[0] += (double)(v.x * m); mv[1] += (double)(v.y * m); mv[2] += (double)(v.z * m);
        }
    }
    if (!do_cm) {
        if (blockIdx.x == 0 && threadIdx.x == 0) cm->valid = 0;
        return;
    }
    if (grid_sum<VV_THREADS, 3>(mv, partial, &ctl->ticket) && threadIdx.x == 0) cm->publish(mv, inv_total_mass);
}

}  // namespace mb
