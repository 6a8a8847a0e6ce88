// verlet.cuh — the plain single-system integrators as one pass per atom (src/simulators.jl:858-1063, :1400-1490):
//   VERLET_LEAPFROG    Verlet:             v += (F/m) dt;  x += v dt
//   VERLET_STORMER     StormerVerlet:      d = v dt + (F/m) dt^2 (first step of a call: dt^2 / 2);  x += d;  v = d / dt
//   VERLET_OVERDAMPED  OverdampedLangevin: x += (F/m) dt/gamma + sqrt(2 dt/gamma) sqrt(kT/m) xi  (Euler-Maruyama)
// each preceded by v -= v_cm (pending) and followed by the displacement check. As for the Langevin step, the forces are
// evaluated at the top of the reference's step, so one step here is this kernel followed by the force launch that the next
// step reads.
//
// StormerVerlet keeps no second coordinate buffer: at the end of a step v dt equals vector(x_last, x) up to rounding, so
// the previous displacement travels as the velocity and survives the cell list's re-sorts and chunked calls. The reference
// takes `vector` of wrapped coordinates instead, so f32 rounding differs at the ulp level.
#pragma once
#include "vv.cuh"

#ifndef MB_HD
#define MB_HD __host__ __device__ __forceinline__
#endif

namespace mb {

enum { VERLET_LEAPFROG = 0, VERLET_STORMER = 1, VERLET_OVERDAMPED = 2 };

struct VerletCoef {
    double dt2;    // StormerVerlet: dt^2
    double dt_g;   // OverdampedLangevin: dt / gamma
    double noise;  // OverdampedLangevin: sqrt(2 dt / gamma)
    double kT;     // OverdampedLangevin: kJ/mol
};

// The update of one atom: p, v with v.w = 1/m (massless atoms: 0, so they neither feel a force nor move by noise), f the
// forces at p. first: StormerVerlet's first step of a call. g: OverdampedLangevin's noise sqrt(2 dt/gamma) sqrt(kT/m) xi.
template <typename T, int KIND>
MB_HD void verlet_update(typename VT<T>::T4& p, typename VT<T>::T4& v, const typename VT<T>::T4& f, T dt, const VerletCoef& c,
                         bool first, const double g[3]) {
    const T im = v.w;
    if (KIND == VERLET_LEAPFROG) {
        const T a = im * dt;
        v.x += f.x * a; v.y += f.y * a; v.z += f.z * a;
        p.x += v.x * dt; p.y += v.y * dt; p.z += v.z * dt;
    } else if (KIND == VERLET_STORMER) {
        const T a = im * (T)(first ? c.dt2 / 2 : c.dt2);
        const T dx = v.x * dt + f.x * a, dy = v.y * dt + f.y * a, dz = v.z * dt + f.z * a;
        p.x += dx; p.y += dy; p.z += dz;
        v.x = dx / dt; v.y = dy / dt; v.z = dz / dt;
    } else {
        // drift and noise in double, one rounding to T
        const double a = (double)im * c.dt_g;
        p.x = (T)((double)p.x + (double)f.x * a + g[0]);
        p.y = (T)((double)p.y + (double)f.y * a + g[1]);
        p.z = (T)((double)p.z + (double)f.z * a + g[2]);
    }
}

// One atom per thread (grid-stride). OverdampedLangevin's xi: Philox4x32-10 with counter (original atom index + 1, step,
// ctr1_lo, ctr1_hi) and key (key_lo, key_hi), Box-Muller of its four words (box_muller3): the Langevin step's draw. When
// do_cm, sum(m v) of the new velocities goes through grid_sum and the last CTA publishes v_cm = sum(m v) / sum(m); otherwise
// the last CTA marks v_cm as consumed. The pending v_cm and the step counter read below are overwritten by the last CTA of
// this same launch (last_cta orders every CTA's reads before its ticket).
template <typename T, int KIND>
__global__ void __launch_bounds__(VV_THREADS)
    verlet_step_kernel(int n, T dt, T skin_half2, VerletCoef vc, int do_cm, double inv_total_mass, CmState<T>* cm,
                       const typename VT<T>::T4* __restrict__ f4, const typename VT<T>::T4* __restrict__ xref4,
                       typename VT<T>::T4* __restrict__ pos4, typename VT<T>::T4* __restrict__ vel4, const int* __restrict__ orig,
                       const T* __restrict__ mass, double* __restrict__ partial, int* __restrict__ flag, Control* __restrict__ ctl,
                       cudaGraphConditionalHandle handle, int use_handle, ExtMap<T> ext) {
    const bool cmv = cm->valid != 0;
    const T cx = cm->v[0], cy = cm->v[1], cz = cm->v[2];
    const bool first = KIND == VERLET_STORMER && ctl->step == ctl->init_step;
    uint32_t step_lo = 0, c0 = 0, c1 = 0, k0 = 0, k1 = 0;
    if (KIND == VERLET_OVERDAMPED) {
        step_lo = (uint32_t)(ctl->step + 1);  // the step this launch takes
        c0 = ctl->rng[0]; c1 = ctl->rng[1]; k0 = ctl->rng[2]; k1 = ctl->rng[3];
    }
    bool moved = false;
    double mv[3] = {0, 0, 0};
    for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x) {
        typename VT<T>::T4 v = vel4[s], p = pos4[s];
        const typename VT<T>::T4 f = f4[s], r = xref4[s];
        int e_own = 0;
        unsigned int e_gp = 0;
        if (ext.pos4e) { e_own = ext.ext_of[s]; e_gp = ext.gptr[s]; }
        if (cmv) { v.x -= cx; v.y -= cy; v.z -= cz; }
        double g[3] = {0, 0, 0};
        if (KIND == VERLET_OVERDAMPED) {
            uint32_t w[4] = {(uint32_t)(orig[s] + 1), step_lo, c0, c1};
            philox4x32_10(w, k0, k1);
            box_muller3(w, vc.noise * sqrt(vc.kT * (double)v.w), g);
        }
        verlet_update<T, KIND>(p, v, f, dt, vc, first, g);
        if (KIND != VERLET_OVERDAMPED || cmv) vel4[s] = v;
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
