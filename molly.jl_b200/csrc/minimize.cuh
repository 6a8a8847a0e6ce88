// minimize.cuh — steepest-descent minimisation on the device (mb_minimize_sd).
//
// Reference: simulate!(sys, ::SteepestDescentMinimizer) src/simulators.jl:183-274. One iteration here is
//   trial    x_saved = x;  x += h F / m;  pos4e own entry + ghost copies;  displacement check     (one pass)
//   [rebuild when an atom moved more than skin/2 from its position at the last build]
//   evaluate forces + energy at the trial positions (ENERGY variants, bonded, PME)
//   decide   E_trial < E ? (accept, h = 6h/5) : (reject, h = h/5); trace record; continue flag      (one CTA)
//   accept   accept: F = F_trial;  reject: x = x_saved;  m = max |F| of the kept forces            (one pass)
// The kept forces and the saved positions live in ORIGINAL atom order (indexed through orig), so a rebuild that a trial
// triggered, which re-sorts the slots, leaves them valid. A rejected trial puts the saved position back in the periodic
// frame of the atom's current slot (the rebuild wrapped the trial position) by whole box vectors.
#pragma once
#include "cells.cuh"

namespace mb {

// Device state of one minimisation (the host uploads it, the kernels advance it, the host reads it back at the end).
struct SdState {
    double E;          // energy of the kept coordinates
    double h;          // step size
    double m;          // max |F_i| of the kept forces (the F of the next trial)
    double tol;
    double pe_const;   // energy terms without a kernel (LJDispersionCorrection)
    long long init_step, max_steps, iter;
    double* trace;     // (max_steps + 1) x 4 records (step, E or E_trial, max force, accepted), or null
    unsigned long long max_f2_bits;  // max |F_i|^2 of the accept pass (non-negative doubles order like their bits)
    int move_ok;       // the trial moved the atoms (m finite and > 0)
    int accepted;      // decision of the current iteration
    int cont;          // another iteration follows
    int converged;     // the last iteration's m was below tol
};

constexpr int SD_THREADS = 256;

// Trial move x <- x + h F / m (formed in double, one rounding into T) of every slot, after saving x. With m = 0 or not finite
// the positions stay where they are and the decide kernel records the trial as rejected (the reference's x + h F / m is NaN
// then). On the cell-list path (ext.pos4e != null) the move is also stored into the extended array (own entry + ghost
// copies, as K1 does) and tested against xref4; the last CTA sets the graph's conditional rebuild node.
template <typename T>
__global__ void __launch_bounds__(SD_THREADS)
    sd_trial_kernel(int n, const int* __restrict__ orig, const typename VT<T>::T4* __restrict__ fkeep,
                    typename VT<T>::T4* __restrict__ pos4, typename VT<T>::T4* __restrict__ xsave,
                    const typename VT<T>::T4* __restrict__ xref4, T skin_half2, ExtMap<T> ext, Control* __restrict__ ctl,
                    SdState* __restrict__ st, cudaGraphConditionalHandle handle, int use_handle) {
    const double h = st->h, m = st->m;
    const bool ok = m > 0.0 && m <= 1.7976931348623157e308;
    bool moved = false;
    for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x) {
        const int o = orig ? orig[s] : s;
        typename VT<T>::T4 p = pos4[s];
        xsave[o] = p;
        if (!ok) continue;
        const typename VT<T>::T4 f = fkeep[o];
        p.x = (T)((double)p.x + h * (double)f.x / m);
        p.y = (T)((double)p.y + h * (double)f.y / m);
        p.z = (T)((double)p.z + h * (double)f.z / m);
        pos4[s] = p;
        if (ext.pos4e) {
            ext_store<T>(ext, s, p, ext.pos4e);
            const typename VT<T>::T4 r = xref4[s];
            const T dx = p.x - r.x, dy = p.y - r.y, dz = p.z - r.z;
            moved |= (dx * dx + dy * dy + dz * dz > skin_half2);
        }
    }
    if (moved) ctl->rebuild = 1;
    if (last_cta(&ctl->ticket) && threadIdx.x == 0) {
        __threadfence();
        st->move_ok = ok ? 1 : 0;
        if (use_handle) cudaGraphSetConditional(handle, *(volatile int*)&ctl->rebuild ? 1u : 0u);
    }
}

// Energy of the trial positions (pair partials in index order with sum_partials, then the specific terms and the constant),
// the decision, the step-size update, the trace record and the continue flag. One CTA of SD_THREADS. init: the evaluation
// at the starting coordinates (record 0 = (init_step, E0, NaN, 1)).
__global__ void __launch_bounds__(SD_THREADS)
    sd_decide_kernel(SdState* __restrict__ st, const double* __restrict__ pe_partial, int n_pe, const double* __restrict__ sp_energy,
                     int init, cudaGraphConditionalHandle handle, int use_handle) {
    double s[1];
    sum_partials<SD_THREADS, 1>(pe_partial, n_pe, s);
    if (threadIdx.x != 0) return;
    double pe = s[0];
    if (sp_energy) pe += *sp_energy;
    pe += st->pe_const;
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    int acc, cont;
    double* rec = nullptr;
    if (init) {
        st->E = pe;
        st->iter = 0;
        st->converged = 0;
        acc = 1;
        cont = st->max_steps > 0;
        if (st->trace) { rec = st->trace; rec[0] = (double)st->init_step; rec[1] = pe; rec[2] = nan; rec[3] = 1.0; }
    } else {
        const double m = st->m;
        if (!st->move_ok) pe = nan;
        acc = pe < st->E;  // (false for NaN)
        if (acc) { st->h = 6.0 * st->h / 5.0; st->E = pe; }
        else st->h = st->h / 5.0;
        const long long k = ++st->iter;
        if (st->trace) { rec = st->trace + 4 * k; rec[0] = (double)(st->init_step + k); rec[1] = pe; rec[2] = m; rec[3] = acc; }
        const bool conv = m < st->tol;  // tested after the trial, as the reference does
        st->converged = conv;
        cont = !conv && k < st->max_steps;
    }
    st->accepted = acc;
    st->cont = cont;
    if (use_handle) cudaGraphSetConditional(handle, cont ? 1u : 0u);
}

// Accept: the trial's forces (slot order) become the kept forces (original order). Reject: the saved position goes back into
// pos4 (and pos4e with its ghost copies), moved by whole box vectors into the frame of the atom's current slot. Either way
// the max |F_i|^2 of the kept forces is taken (a max does not depend on the order); the last CTA stores m = its root.
template <typename T>
__global__ void __launch_bounds__(SD_THREADS)
    sd_accept_kernel(int n, const int* __restrict__ orig, const typename VT<T>::T4* __restrict__ ftrial,
                     typename VT<T>::T4* __restrict__ fkeep, const typename VT<T>::T4* __restrict__ xsave,
                     typename VT<T>::T4* __restrict__ pos4, ExtMap<T> ext, Control* __restrict__ ctl, SdState* __restrict__ st) {
    const bool acc = st->accepted != 0;
    unsigned long long f2max = 0;
    for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x) {
        const int o = orig ? orig[s] : s;
        typename VT<T>::T4 f;
        if (acc) {
            f = ftrial[s];
            fkeep[o] = f;
        } else {
            f = fkeep[o];
            typename VT<T>::T4 p = xsave[o];
            if (ext.pos4e) {
                const typename VT<T>::T4 c = pos4[s];
                const double k0 = rint(((double)p.x - (double)c.x) / ext.Ld[0]);
                const double k1 = rint(((double)p.y - (double)c.y) / ext.Ld[1]);
                const double k2 = rint(((double)p.z - (double)c.z) / ext.Ld[2]);
                if (k0 != 0.0) p.x = (T)((double)p.x - k0 * ext.Ld[0]);
                if (k1 != 0.0) p.y = (T)((double)p.y - k1 * ext.Ld[1]);
                if (k2 != 0.0) p.z = (T)((double)p.z - k2 * ext.Ld[2]);
                ext_store<T>(ext, s, p, ext.pos4e);
            }
            pos4[s] = p;
        }
        const double fx = f.x, fy = f.y, fz = f.z;
        const unsigned long long b = (unsigned long long)__double_as_longlong(fx * fx + fy * fy + fz * fz);
        f2max = b > f2max ? b : f2max;  // (a NaN has larger bits than +inf: it propagates)
    }
    for (int k = 16; k > 0; k >>= 1) {
        const unsigned long long v = __shfl_xor_sync(0xffffffffu, f2max, k);
        f2max = v > f2max ? v : f2max;
    }
    __shared__ unsigned long long s_max[SD_THREADS / 32];
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = f2max;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long mx = 0;
        for (int w = 0; w < SD_THREADS / 32; w++) mx = s_max[w] > mx ? s_max[w] : mx;
        atomicMax(&st->max_f2_bits, mx);  // one atomic per CTA
    }
    if (last_cta(&ctl->ticket) && threadIdx.x == 0) {
        __threadfence();
        const unsigned long long mx = atomicExch(&st->max_f2_bits, 0ull);
        st->m = sqrt(__longlong_as_double((long long)mx));
    }
}

}  // namespace mb
