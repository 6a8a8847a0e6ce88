// splitting.cuh — LangevinSplitting (src/simulators.jl:1212-1398; Leimkuhler and Matthews 2013, Fass et al. 2018): a step
// is a string over A, B and O, each letter applied with its effective step dt / count(letter, splitting):
//   A  x += v dt_A                           B  v += (F/m) dt_B
//   O  v = vel_scale_i v + noise_scale_i xi  with vel_scale_i = exp(-friction dt_O / m_i), noise_scale_i =
//      sqrt(kT / m_i (1 - vel_scale_i^2)) (friction in mass per time, unlike Langevin's)
// The host cuts the step into passes at its force evaluations (engine.cu, SplitPlan); one pass is one launch of
// split_pass_kernel, which applies the pass's letters to each atom in one trip through vel4 / pos4.
#pragma once
#include "langevin.cuh"

namespace mb {

constexpr int SPLIT_MAX_OPS = 32;  // MB_SPLIT_MAX_OPS
enum { SPLIT_A = 0, SPLIT_B = 1, SPLIT_O = 2 };

// One pass as a by-value program: its letters in order as 2-bit codes (letter k in bits 2k, 2k + 1; a word rather than a
// byte array, which a loop could only index through a local copy) and the index j, among the O's of the step, of its first O
// (the O's of a pass are consecutive in j)
struct SplitProg {
    unsigned long long ops;  // SPLIT_* of letter k at bit 2k
    int n_ops;
    int o_base;              // j of the pass's first O (its draws use ctr1 + j)
    int has_a, has_b, has_o;
    int apply_cm;  // the step's first pass: subtract the pending v_cm first
    int last;      // the step's last pass: momentum sum or v_cm consumed, step counter advanced
};

// the letters' coefficients (StepCfg): dt_A, dt_B in the dtype; o_rate = -friction dt / n_O and kT in double
template <typename T>
struct SplitCoef {
    T dt_a, dt_b;
    double o_rate, kT;
};

// The pass's letters for each atom (one atom per thread, grid-stride), each op a warp-uniform branch on the program.
// O: vel_scale_i and noise_scale_i are formed in double from vel4.w (1/m; massless atoms: 1/m = 0, so no kick and no
// noise); the draws of the j-th O of step n are the Box-Muller transform (box_muller3) of one Philox4x32-10 block with counter
// (original atom index + 1, n, ctr1 + j as a 64-bit sum) and key rng_key. For j = 0 this is langevin_step_kernel's draw.
// c v + sigma xi is formed in double and rounded once.
// A pass that holds an A writes pos4 and also the extended array (own entry and ghosts), takes the displacement test against
// xref4 and has its last CTA publish the rebuild decision to the conditional node that follows it (every such pass is
// followed by a force evaluation or is the step's last pass that moves the atoms, so each pair evaluation, and a log step's
// energy, reads current lists).
// The last pass of the step sums m v through grid_sum and publishes v_cm (do_cm), or marks v_cm consumed, and its last CTA
// advances the step counter (step_count): every pass of step n reads ctl->step = n - 1, so every O of step n draws with step
// n. The pending v_cm and the step counter read below are overwritten only by the last CTA of the last pass's own launch
// (last_cta orders every CTA's reads before its ticket).
template <typename T>
__global__ void __launch_bounds__(VV_THREADS)
    split_pass_kernel(int n, SplitProg pg, SplitCoef<T> sc, T skin_half2, int do_cm, double inv_total_mass, CmState<T>* cm,
                      const typename VT<T>::T4* __restrict__ f4, const typename VT<T>::T4* __restrict__ xref4,
                      typename VT<T>::T4* __restrict__ pos4, typename VT<T>::T4* __restrict__ vel4, const int* __restrict__ orig,
                      const T* __restrict__ mass, double* __restrict__ partial, int* __restrict__ flag, Control* __restrict__ ctl,
                      cudaGraphConditionalHandle handle, int use_handle, ExtMap<T> ext) {
    const bool cmv = pg.apply_cm && cm->valid != 0;
    const T cx = cm->v[0], cy = cm->v[1], cz = cm->v[2];
    uint32_t step_lo = 0, k0 = 0, k1 = 0;
    uint64_t ctr1 = 0;
    if (pg.has_o) {
        step_lo = (uint32_t)(ctl->step + 1);  // the step this pass belongs to
        ctr1 = (uint64_t)ctl->rng[0] | ((uint64_t)ctl->rng[1] << 32);
        k0 = ctl->rng[2]; k1 = ctl->rng[3];
    }
    const bool ext_on = pg.has_a && ext.pos4e;
    const bool sum_mv = pg.last && do_cm;
    bool moved = false;
    double mv[3] = {0, 0, 0};
    for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x) {
        typename VT<T>::T4 v = vel4[s], p = {}, f = {};
        if (pg.has_a) p = pos4[s];
        if (pg.has_b) f = f4[s];
        int o = 0, e_own = 0;
        unsigned int e_gp = 0;
        if (pg.has_o) o = orig[s];
        if (ext_on) { e_own = ext.ext_of[s]; e_gp = ext.gptr[s]; }
        if (cmv) { v.x -= cx; v.y -= cy; v.z -= cz; }
        uint64_t ctr = ctr1 + (uint64_t)pg.o_base;
        for (int k = 0; k < pg.n_ops; k++) {
            const int op = (int)(pg.ops >> (2 * k)) & 3;
            if (op == SPLIT_A) {
                p.x += v.x * sc.dt_a; p.y += v.y * sc.dt_a; p.z += v.z * sc.dt_a;
            } else if (op == SPLIT_B) {
                const T a = v.w * sc.dt_b;  // (1/m) dt_B
                v.x += f.x * a; v.y += f.y * a; v.z += f.z * a;
            } else {
                const double im = (double)v.w;
                const double c = exp(sc.o_rate * im);
                uint32_t w[4] = {(uint32_t)(o + 1), step_lo, (uint32_t)ctr, (uint32_t)(ctr >> 32)};
                philox4x32_10(w, k0, k1);
                double g[3];
                box_muller3(w, sqrt(sc.kT * im * (1.0 - c * c)), g);
                v.x = (T)(c * (double)v.x + g[0]);
                v.y = (T)(c * (double)v.y + g[1]);
                v.z = (T)(c * (double)v.z + g[2]);
                ctr++;
            }
        }
        vel4[s] = v;
        if (pg.has_a) {
            pos4[s] = p;
            if (ext_on) ext_store_at<T>(ext, e_own, e_gp, p, ext.pos4e);
            const typename VT<T>::T4 r = xref4[s];
            const T dx = p.x - r.x, dy = p.y - r.y, dz = p.z - r.z;
            moved |= (dx * dx + dy * dy + dz * dz > skin_half2);
        }
        if (sum_mv) {
            const T m = mass[s];
            mv[0] += (double)(v.x * m); mv[1] += (double)(v.y * m); mv[2] += (double)(v.z * m);
        }
    }
    if (!pg.has_a && !pg.last) return;  // (uniform over the launch)
    if (moved) *flag = 1;
    if (!(sum_mv ? grid_sum<VV_THREADS, 3>(mv, partial, &ctl->ticket) : last_cta(&ctl->ticket)) || threadIdx.x != 0) return;
    if (!pg.last) {  // a rebuild point inside the step: publish the decision, the step goes on
        __threadfence();
        publish_rebuild(handle, use_handle, *(volatile int*)&ctl->rebuild);
        return;
    }
    if (sum_mv) cm->publish(mv, inv_total_mass);
    else cm->valid = 0;
    const int rb = step_count(ctl);
    if (pg.has_a) publish_rebuild(handle, use_handle, rb);  // (no A: the next rebuild point reads ctl->rebuild)
}

}  // namespace mb
