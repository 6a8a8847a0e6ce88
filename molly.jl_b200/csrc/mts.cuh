// mts.cuh — the multiple-time-step integrators MTSIntegrator (rRESPA, Tuckerman et al. 1992) and MTSLangevinIntegrator
// (BAOAB-RESPA, Lagardère et al. 2019), src/simulators.jl:1616-1940. The interactions are split into levels l = 0, 1, ...
// with ordered fractions f_0 = 1 < f_1 < ..., each a multiple of the one before; level l is applied f_l times per outer step
// with dt_x = dt / f_l and dt_v = dt_x / 2. One outer step is the recursion of mts_substeps!, unrolled by the host (the
// levels are static): per substep of level l
//   [F_l]  kick_l  (innermost: drift | other levels: the substeps of level l + 1)  F_l  kick_l
// The passes here are the kicks and the innermost kick + drift; the closing kick of level 0 is K2 (vv_kick2_kernel), which
// also sums m v for the CM removal.
#pragma once
#include "langevin.cuh"

namespace mb {

constexpr int MTS_MAX_LEVELS = 8;  // MB_MTS_MAX_LEVELS

// v += F (1/m) dt_v over one level's force buffer. apply_cm: the first kick of an outer step subtracts the pending v_cm first,
// as K1 does (it does not clear it: the closing K2 overwrites it, or the host clears it after this launch).
template <typename T>
__global__ void __launch_bounds__(VV_THREADS)
    mts_kick_kernel(int n, T dt_v, int apply_cm, const CmState<T>* __restrict__ cm, const typename VT<T>::T4* __restrict__ f4,
                    typename VT<T>::T4* __restrict__ vel4) {
    const bool cmv = apply_cm && cm->valid != 0;
    const T cx = cm->v[0], cy = cm->v[1], cz = cm->v[2];
    for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x) {
        typename VT<T>::T4 v = vel4[s];
        const typename VT<T>::T4 f = f4[s];
        if (cmv) { v.x -= cx; v.y -= cy; v.z -= cz; }
        const T a = v.w * dt_v;  // (1/m) dt_v; massless atoms: 1/m = 0
        v.x += f.x * a; v.y += f.y * a; v.z += f.z * a;
        vel4[s] = v;
    }
}

// The innermost level's kick and drift in one pass: v += F (1/m) dt_v, then x += v dt_x (MTSIntegrator) or, for
// MTSLangevinIntegrator, x += v dt_x/2; v = c v + sigma_i xi; x += v dt_x/2 with c = exp(-dt friction / f_last) and
// sigma_i = sqrt(1 - c^2) sqrt(kT / m_i), c v + sigma xi formed in double and rounded once.
// Draws: Philox4x32-10 with counter (original atom index + 1, outer step, substep, ctr1_lo) and key (key_lo, key_hi), one
// block per atom and innermost substep (substep = 0 .. f_last - 1 within the outer step), Box-Muller of its four words
// (box_muller3): a function of (keys, outer step, substep, atom) only.
// Only the last innermost drift of an outer step (last = 1) writes the extended array (own entry and ghosts), takes the
// displacement test against xref4 and does the step bookkeeping (step_advance: ctl->step counts outer steps); the earlier
// ones write pos4 only, which is all the bonded terms read. So the neighbour structure, and with it the slot order, changes
// only between the last drift and the pair evaluation of an outer step. The step counter read below is advanced by the last
// CTA of the last drift's own launch (last_cta orders every CTA's reads before its ticket). Four CTAs per SM: without that
// bound ptxas fits the f32 MTSIntegrator instantiation into 32 registers and spills in the ghost-copy loop.
template <typename T, bool LANGEVIN>
__global__ void __launch_bounds__(VV_THREADS, 4)
    mts_kick_drift_kernel(int n, T dt_v, T dt_x, T dt_xh, T skin_half2, LangevinCoef lc, int substep, int apply_cm, int last,
                          const CmState<T>* __restrict__ cm, const typename VT<T>::T4* __restrict__ f4,
                          const typename VT<T>::T4* __restrict__ xref4, typename VT<T>::T4* __restrict__ pos4,
                          typename VT<T>::T4* __restrict__ vel4, const int* __restrict__ orig, int* __restrict__ flag,
                          Control* __restrict__ ctl, cudaGraphConditionalHandle handle, int use_handle, ExtMap<T> ext) {
    const bool cmv = apply_cm && cm->valid != 0;
    const T cx = cm->v[0], cy = cm->v[1], cz = cm->v[2];
    uint32_t step_lo = 0, c0 = 0, k0 = 0, k1 = 0;
    if (LANGEVIN) { step_lo = (uint32_t)(ctl->step + 1); c0 = ctl->rng[0]; k0 = ctl->rng[2]; k1 = ctl->rng[3]; }
    const bool ext_on = last && ext.pos4e;
    bool moved = false;
    for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x) {
        typename VT<T>::T4 v = vel4[s], p = pos4[s];
        const typename VT<T>::T4 f = f4[s];
        int e_own = 0;
        unsigned int e_gp = 0;
        if (ext_on) { e_own = ext.ext_of[s]; e_gp = ext.gptr[s]; }
        if (cmv) { v.x -= cx; v.y -= cy; v.z -= cz; }
        const T a = v.w * dt_v;
        v.x += f.x * a; v.y += f.y * a; v.z += f.z * a;
        if (LANGEVIN) {
            p.x += v.x * dt_xh; p.y += v.y * dt_xh; p.z += v.z * dt_xh;
            uint32_t w[4] = {(uint32_t)(orig[s] + 1), step_lo, (uint32_t)substep, c0};
            philox4x32_10(w, k0, k1);
            double g[3];
            box_muller3(w, lc.noise_scale * sqrt(lc.kT * (double)v.w), g);  // massless atoms: no noise
            v.x = (T)(lc.vel_scale * (double)v.x + g[0]);
            v.y = (T)(lc.vel_scale * (double)v.y + g[1]);
            v.z = (T)(lc.vel_scale * (double)v.z + g[2]);
            p.x += v.x * dt_xh; p.y += v.y * dt_xh; p.z += v.z * dt_xh;
        } else {
            p.x += v.x * dt_x; p.y += v.y * dt_x; p.z += v.z * dt_x;
        }
        vel4[s] = v;
        pos4[s] = p;
        if (last) {
            if (ext_on) ext_store_at<T>(ext, e_own, e_gp, p, ext.pos4e);
            const typename VT<T>::T4 r = xref4[s];
            const T dx = p.x - r.x, dy = p.y - r.y, dz = p.z - r.z;
            moved |= (dx * dx + dy * dy + dz * dz > skin_half2);
        }
    }
    if (!last) return;  // (uniform over the launch)
    if (moved) *flag = 1;
    if (!last_cta(&ctl->ticket) || threadIdx.x != 0) return;
    step_advance(ctl, handle, use_handle);
}

}  // namespace mb
