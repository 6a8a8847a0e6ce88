// langevin.cuh — the Langevin integrator (Molly's port of OpenMM's LangevinMiddleIntegrator, Zhang et al. 2019;
// src/simulators.jl:1065-1210, O step src/kernels.jl:723-756) as one pass per atom:
//   v -= v_cm (pending);  v += (F/m) dt;  x += v dt/2;  v = c v + sigma_i xi;  x += v dt/2;  displacement check
// with c = exp(-friction dt), sigma_i = sqrt(1 - c^2) sqrt(kT / m_i) and xi ~ N(0, 1)^3. The reference evaluates the forces at
// the top of its step, so one step here is this kernel followed by the force launch that the next step's kick reads.
#pragma once
#include "vv.cuh"

namespace mb {

struct LangevinCoef {
    double vel_scale;    // c = exp(-friction dt)
    double noise_scale;  // sqrt(1 - c^2)
    double kT;           // kJ/mol
};

// O step draws: Philox4x32-10 with counter (original atom index + 1, step, ctr1_lo, ctr1_hi) and key (key_lo, key_hi), one
// block per atom and step, Box-Muller of its four words (box_muller3). A function of (keys, step, atom) only.
// When do_cm, sum(m v) of the new velocities goes through grid_sum and the last CTA publishes v_cm = sum(m v) / sum(m);
// otherwise the last CTA marks v_cm as consumed. The pending v_cm and the step counter read below are overwritten by the last
// CTA of this same launch (last_cta orders every CTA's reads before its ticket).
template <typename T>
__global__ void __launch_bounds__(VV_THREADS)
    langevin_step_kernel(int n, T dt, T dt_half, T skin_half2, LangevinCoef lc, int do_cm, double inv_total_mass,
                         CmState<T>* cm, const typename VT<T>::T4* __restrict__ f4, const typename VT<T>::T4* __restrict__ xref4,
                         typename VT<T>::T4* __restrict__ pos4, typename VT<T>::T4* __restrict__ vel4, const int* __restrict__ orig,
                         const T* __restrict__ mass, double* __restrict__ partial, int* __restrict__ flag, Control* __restrict__ ctl,
                         cudaGraphConditionalHandle handle, int use_handle, ExtMap<T> ext) {
    const bool cmv = cm->valid != 0;
    const T cx = cm->v[0], cy = cm->v[1], cz = cm->v[2];
    const uint32_t step_lo = (uint32_t)(ctl->step + 1);  // the step this launch takes
    const uint32_t c0 = ctl->rng[0], c1 = ctl->rng[1], k0 = ctl->rng[2], k1 = ctl->rng[3];
    bool moved = false;  // (the largest displacement K1 also records serves decomposed runs only)
    double mv[3] = {0, 0, 0};
    for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x) {
        typename VT<T>::T4 v = vel4[s], p = pos4[s];
        const typename VT<T>::T4 f = f4[s], r = xref4[s];
        const int o = orig[s];
        int e_own = 0;
        unsigned int e_gp = 0;
        if (ext.pos4e) { e_own = ext.ext_of[s]; e_gp = ext.gptr[s]; }
        if (cmv) { v.x -= cx; v.y -= cy; v.z -= cz; }
        const T a = v.w * dt;  // (1/m) dt; massless atoms: 1/m = 0, no kick and no noise
        v.x += f.x * a; v.y += f.y * a; v.z += f.z * a;
        p.x += v.x * dt_half; p.y += v.y * dt_half; p.z += v.z * dt_half;
        uint32_t w[4] = {(uint32_t)(o + 1), step_lo, c0, c1};
        philox4x32_10(w, k0, k1);
        double g[3];
        box_muller3(w, lc.noise_scale * sqrt(lc.kT * (double)v.w), g);
        // c v + sigma xi in double, one rounding to T
        v.x = (T)(lc.vel_scale * (double)v.x + g[0]);
        v.y = (T)(lc.vel_scale * (double)v.y + g[1]);
        v.z = (T)(lc.vel_scale * (double)v.z + g[2]);
        p.x += v.x * dt_half; p.y += v.y * dt_half; p.z += v.z * dt_half;
        vel4[s] = v;
        pos4[s] = p;
        if (ext.pos4e) ext_store_at<T>(ext, e_own, e_gp, p, ext.pos4e);
        const T dx = p.x - r.x, dy = p.y - r.y, dz = p.z - r.z;
        moved |= (dx * dx + dy * dy + dz * dz > skin_half2);
        if (do_cm) {
            const T m = mass[s];
            mv[0] += (double)(v.x * m); mv[1] += (double)(v.y * m); mv[2] += (double)(v.z * m);
        }
    }
    if (moved) *flag = 1;
    if (!(do_cm ? grid_sum<VV_THREADS, 3>(mv, partial, &ctl->ticket) : last_cta(&ctl->ticket)) || threadIdx.x != 0) return;
    if (do_cm) cm->publish(mv, inv_total_mass);
    else cm->valid = 0;
    step_advance(ctl, handle, use_handle);  // (last: nothing stays live across its conditional-node call)
}

}  // namespace mb
