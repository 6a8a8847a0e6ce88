// vv.cuh — fused VelocityVerlet kernels and the original-order <-> slot-order movers.
//
// Reference: simulate!(sys, ::VelocityVerlet, n) src/simulators.jl:547-668 runs the update as five
// separate broadcasts + two CM-removal kernels per step; here it is
//   K1  v -= v_cm (pending);  v += (F/m) dt/2;  x += v dt;  displacement check     (one pass)
//   F   brick_force_kernel
//   K2  v += (F/m) dt/2;  sum(m v) -> v_cm (last CTA, fixed order)                  (one pass)
// Positions stay continuous (unwrapped) between neighbour rebuilds; wrap_coords (src/spatial.jl:573-586)
// is applied at every rebuild and on export, which is equivalent under the minimum-image convention.
#pragma once
#include "cells.cuh"
#include "dpd.cuh"
#include "peer.cuh"
#include "vrescale.cuh"

namespace mb {


// ---- first-touch initialisation: slot order = original order -------------------------------------
template <typename T>
__global__ void init_slots_kernel(int n, const T* __restrict__ coords, const T* __restrict__ charge,
                                  const typename VT<T>::T2* __restrict__ ljp, const T* __restrict__ mass_in,
                                  typename VT<T>::T4* __restrict__ pos4, typename VT<T>::T4* __restrict__ vel4,
                                  typename VT<T>::T2* __restrict__ lj2, int* __restrict__ orig, int* __restrict__ inv_orig,
                                  T* __restrict__ mass, typename VT<T>::T4* __restrict__ xref4) {
    int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    typename VT<T>::T4 p = make4<T>(coords[3 * s], coords[3 * s + 1], coords[3 * s + 2], charge[s]);
    pos4[s] = p;
    xref4[s] = p;
    T m = mass_in[s];
    vel4[s] = make4<T>((T)0, (T)0, (T)0, (m == (T)0) ? (T)0 : (T)1 / m);  // calc_accels: massless -> 0
    lj2[s] = ljp[s];
    orig[s] = s;
    inv_orig[s] = s;
    mass[s] = m;
}

// ---- ingest coordinates (and velocities) from original order into the current slot order ------
// The caller's coordinates may have been wrapped by Molly since the last call, so the displacement
// from the reference position is taken modulo the box and the slot position continued from xref.
template <typename T>
__global__ void ingest_kernel(int n, Geom<T> g, const T* __restrict__ coords, const T* __restrict__ vels,
                              const int* __restrict__ orig, const typename VT<T>::T4* __restrict__ xref4,
                              typename VT<T>::T4* __restrict__ pos4, typename VT<T>::T4* __restrict__ vel4,
                              int* __restrict__ flag) {
    int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    int o = orig[s];
    typename VT<T>::T4 ref = xref4[s];
    typename VT<T>::T4 p = pos4[s];
    T x[3] = {coords[3 * (size_t)o], coords[3 * (size_t)o + 1], coords[3 * (size_t)o + 2]};
    T r[3] = {ref.x, ref.y, ref.z};
    T d2 = (T)0;
#pragma unroll
    for (int d = 0; d < 3 && !g.tric.on; d++) {  // (triclinic boxes run the no-list path: the caller's coordinates are taken as they are)
        T dd = x[d] - r[d];
        dd -= g.L[d] * frint(dd * g.invL[d]);
        d2 += dd * dd;
        // keep the caller's value when it is the same image (exact), otherwise continue from xref
        T cont = r[d] + dd;
        x[d] = (fabs((double)(x[d] - cont)) < 0.25 * (double)g.L[d]) ? x[d] : cont;
    }
    p.x = x[0]; p.y = x[1]; p.z = x[2];
    pos4[s] = p;
    if (vels) {
        typename VT<T>::T4 v = vel4[s];
        v.x = vels[3 * (size_t)o]; v.y = vels[3 * (size_t)o + 1]; v.z = vels[3 * (size_t)o + 2];
        vel4[s] = v;
    }
    if (d2 > g.skin_half2) *flag = 1;
}

// ---- export: slot order -> original order, wrapped coordinates, pending CM velocity applied ----
// position p wrapped into the box, stored at dst[0..2] (exported coordinates and the logger's coordinate frames)
template <typename T>
__device__ __forceinline__ void store_wrapped(const Geom<T>& g, typename VT<T>::T4 p, T* dst) {
    T x[3] = {p.x, p.y, p.z};
    if (g.tric.on) {
        tric_wrap<T>(g.tric, x[0], x[1], x[2]);
        for (int d = 0; d < 3; d++) dst[d] = x[d];
    } else {
#pragma unroll
        for (int d = 0; d < 3; d++) {
            T v = x[d] - ffloor(x[d] * g.invL[d]) * g.L[d];
            if (v >= g.L[d]) v -= g.L[d];
            if (v < (T)0) v = (T)0;
            dst[d] = v;
        }
    }
}
template <typename T>
__global__ void export_kernel(int n, Geom<T> g, const typename VT<T>::T4* __restrict__ pos4,
                              const typename VT<T>::T4* __restrict__ vel4, const int* __restrict__ orig,
                              const CmState<T>* __restrict__ cm, T* __restrict__ coords, T* __restrict__ vels) {
    int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    int o = orig[s];
    if (coords) store_wrapped<T>(g, pos4[s], coords + 3 * (size_t)o);
    if (vels) {
        typename VT<T>::T4 v = vel4[s];
        if (cm) cm->apply(v);
        vels[3 * (size_t)o] = v.x;
        vels[3 * (size_t)o + 1] = v.y;
        vels[3 * (size_t)o + 2] = v.z;
    }
}

// wrap positions into [0, L) (all-pairs path: the minimum-image select chain needs wrapped coordinates)
template <typename T>
__global__ void wrap_kernel(int n, Geom<T> g, typename VT<T>::T4* __restrict__ pos4) {
    int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    typename VT<T>::T4 p = pos4[s];
    T x[3] = {p.x, p.y, p.z};
    if (g.tric.on) {
        tric_wrap<T>(g.tric, x[0], x[1], x[2]);
    } else {
#pragma unroll
        for (int d = 0; d < 3; d++) x[d] = x[d] - ffloor(x[d] / g.L[d]) * g.L[d];  // wrap_coord_1D
    }
    p.x = x[0]; p.y = x[1]; p.z = x[2];
    pos4[s] = p;
}

// forces: slot order -> ADD into fs_mat (original order, 3 x n column-major)
template <typename T>
__global__ void scatter_forces_kernel(int n, const typename VT<T>::T4* __restrict__ f4, const int* __restrict__ orig,
                                      T* __restrict__ fs_mat) {
    int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    int o = orig ? orig[s] : s;
    typename VT<T>::T4 f = f4[s];
    fs_mat[3 * (size_t)o] += f.x;
    fs_mat[3 * (size_t)o + 1] += f.y;
    fs_mat[3 * (size_t)o + 2] += f.z;
}

// ---- Andersen thermostat arithmetic (src/coupling.jl:197-212, GPU kernel src/kernels.jl:705-721) ------------------------
// Philox4x32-10 keyed by the two rand(rng, UInt64) of the reference, counter = (original atom index, step): the draw for an
// atom does not depend on which kernel or rank evaluates it. Statistical parity only (SURVEY.md section 8c).
template <typename T>
struct Thermo {
    int on;            // apply the thermostat of the PREVIOUS step at the top of the drift kernel (step loop of one GPU)
    int n;             // atoms in the system (second counter block)
    T kT;
    double prob;
    const int* orig;
    const T* mass;
};
template <typename T>
__device__ __forceinline__ void andersen_apply(typename VT<T>::T4& v, int orig_index, int n, T m, T kT, double prob, uint32_t step_lo,
                                               uint32_t ctr1_lo, uint32_t ctr1_hi, uint32_t key_lo, uint32_t key_hi) {
    uint32_t c[4] = {(uint32_t)(orig_index + 1), step_lo, ctr1_lo, ctr1_hi};
    philox4x32_10(c, key_lo, key_hi);
    double u = ((double)c[0] * 4294967296.0 + (double)c[1]) * (1.0 / 18446744073709551616.0);
    if (u < prob) {
        uint32_t d[4] = {(uint32_t)(orig_index + 1 + n), step_lo, ctr1_lo, ctr1_hi};
        philox4x32_10(d, key_lo, key_hi);
        double g[3];
        box_muller3(d, (m > (T)0) ? sqrt((double)kT / (double)m) : 0.0, g);
        v.x = (T)g[0];
        v.y = (T)g[1];
        v.z = (T)g[2];
    }
}

// The step bookkeeping of a drift pass (K1, the Langevin step), done by one thread of the last CTA to finish: advance step_n,
// apply the fixed-interval neighbour policy (find_neighbors every n_steps, src/neighbors.jl:671) and publish the rebuild
// decision to the CUDA graph's conditional node (when the step runs as a graph). The two halves are separate for
// LangevinSplitting, whose passes may publish a decision without advancing the step or advance it without a rebuild node.
__device__ __forceinline__ int step_count(Control* __restrict__ ctl) {  // returns the rebuild decision
    __threadfence();
    const long long step_n = ++ctl->step;
    const long long kk = step_n - ctl->init_step;
    int rb = *(volatile int*)&ctl->rebuild;
    if (ctl->rebuild_every > 0 && kk > 1 && (step_n - 1) % ctl->rebuild_every == 0) { rb = 1; ctl->rebuild = 1; }
    return rb;
}
__device__ __forceinline__ void publish_rebuild(cudaGraphConditionalHandle handle, int use_handle, int rb) {
    if (use_handle) cudaGraphSetConditional(handle, rb ? 1u : 0u);
}
__device__ __forceinline__ void step_advance(Control* __restrict__ ctl, cudaGraphConditionalHandle handle, int use_handle) {
    publish_rebuild(handle, use_handle, step_count(ctl));
}

// ---- K1: first half kick + drift + displacement check; the last CTA to finish does the step bookkeeping (step_advance).
// THERMO: the variants that also apply the previous step's thermostat are separate instantiations so that the plain kernel
// keeps its register count (one atom per thread, latency-bound: occupancy matters): TH_ANDERSEN resamples (Philox +
// Box-Muller inlined), TH_SCALE applies the pending velocity-rescaling factor after the pending v_cm. TH_DPD is the
// DPDVelocityVerlet drift: K1 unchanged plus the predicted velocity of dd (dpd.cuh) stored by the original index in p.w.
enum { TH_NONE = 0, TH_ANDERSEN = 1, TH_SCALE = 2, TH_DPD = 3 };
template <typename T, int THERMO>
__global__ void vv_kick_drift_kernel(int s0, int n, T dt, T dt_half, T skin_half2, const CmState<T>* __restrict__ cm,
                                     const typename VT<T>::T4* __restrict__ f4,
                                     const typename VT<T>::T4* __restrict__ xref4, typename VT<T>::T4* __restrict__ pos4,
                                     typename VT<T>::T4* __restrict__ vel4, int* __restrict__ flag, Control* __restrict__ ctl,
                                     cudaGraphConditionalHandle handle, int use_handle, PeerPush<T> push, ExtMap<T> ext,
                                     Thermo<T> th, DpdDrift<T> dd) {
    bool cmv = cm->valid != 0;
    // thermostat of the step that just ended, folded in here (the standalone kernel would be one more launch per step):
    // same order of operations on v - subtract the pending v_cm, resample, then this step's first kick
    bool thermo = false;
    uint32_t t_step = 0, t_c0 = 0, t_c1 = 0, t_k0 = 0, t_k1 = 0;
    if (THERMO == TH_ANDERSEN && th.on) {  // (no loads from the control block on the path without a thermostat)
        thermo = ctl->step > ctl->init_step;
        t_step = (uint32_t)ctl->step; t_c0 = ctl->rng[0]; t_c1 = ctl->rng[1]; t_k0 = ctl->rng[2]; t_k1 = ctl->rng[3];
    }
    T cx = cm->v[0], cy = cm->v[1], cz = cm->v[2];
    const bool scl = THERMO == TH_SCALE && cm->scaled != 0;
    const T lam = THERMO == TH_SCALE ? cm->lam : (T)1;
    if (push.n_peer > 0 || push.cm_nranks > 0) {  // decomposed run over peer memory (peer.cuh)
        __shared__ double s_cm[3];
        // the neighbours must be done with the previous halo data before it is overwritten ...
        if ((int)threadIdx.x < push.n_peer) spin_until(push.wait_flag[threadIdx.x], push.epoch - 1);
        // ... and v_cm of the previous step is the rank-ordered sum of what every rank's K2 stored here
        const int par = (int)(push.cm_epoch & 1ull);
        const int r = (int)threadIdx.x - 32;
        if (r >= 0 && r < push.cm_nranks) spin_until(&push.cm_comm->mom_epoch[par][r], push.cm_epoch);
        __syncthreads();
        if (push.cm_nranks > 0) {
            if (threadIdx.x == 0) {
                double a = 0, b = 0, c = 0;
                for (int q = 0; q < push.cm_nranks; q++) {
                    const volatile double* m = push.cm_comm->mom[par][q];
                    a += m[0]; b += m[1]; c += m[2];
                }
                s_cm[0] = a * push.cm_inv_mass; s_cm[1] = b * push.cm_inv_mass; s_cm[2] = c * push.cm_inv_mass;
            }
            __syncthreads();
            cmv = true;
            cx = (T)s_cm[0]; cy = (T)s_cm[1]; cz = (T)s_cm[2];
        }
    }
    bool moved = false;
    float d2max = 0.f;
    // Two atoms per thread and iteration, all loads of both requested before any arithmetic: the kernel is bound by memory
    // latency (one wave of CTAs, ~130 B per atom), so the second atom's round trip hides behind the first one's.
    constexpr int UNR = 2;
    const int stride = gridDim.x * blockDim.x;
    for (int k0 = blockIdx.x * blockDim.x + threadIdx.x; k0 < n; k0 += UNR * stride) {
        typename VT<T>::T4 v[UNR], f[UNR], p[UNR], r[UNR];
        int e_own[UNR];
        unsigned int e_gp[UNR];
        bool ok[UNR];
#pragma unroll
        for (int u = 0; u < UNR; u++) {
            const int k = k0 + u * stride;
            ok[u] = k < n;
            const int s = s0 + (ok[u] ? k : k0);  // [s0, s0 + n): the slots this rank owns
            v[u] = vel4[s];
            f[u] = f4[s];
            p[u] = pos4[s];
            r[u] = xref4[s];
            // map into the extended array, requested together with the state so that no load waits behind the arithmetic
            e_own[u] = 0;
            e_gp[u] = 0;
            if (ext.pos4e) { e_own[u] = ext.ext_of[s]; e_gp[u] = ext.gptr[s]; }
        }
#pragma unroll
        for (int u = 0; u < UNR; u++) {
            if (!ok[u]) continue;
            const int s = s0 + k0 + u * stride;
            if (cmv) { v[u].x -= cx; v[u].y -= cy; v[u].z -= cz; }
            if (THERMO == TH_SCALE && scl) { v[u].x *= lam; v[u].y *= lam; v[u].z *= lam; }
            if (THERMO == TH_ANDERSEN && thermo) andersen_apply<T>(v[u], th.orig[s], th.n, th.mass[s], th.kT, th.prob, t_step, t_c0, t_c1, t_k0, t_k1);
            const T a = v[u].w * dt_half;  // (1/m) dt/2
            v[u].x += f[u].x * a; v[u].y += f[u].y * a; v[u].z += f[u].z * a;
            p[u].x += v[u].x * dt; p[u].y += v[u].y * dt; p[u].z += v[u].z * dt;
            if (THERMO == TH_DPD) {
                const T b = v[u].w * dd.lam_dt;  // (1/m) (lambda - 1/2) dt
                dd.vpred[(int)p[u].w] = make4<T>(v[u].x + f[u].x * b, v[u].y + f[u].y * b, v[u].z + f[u].z * b, (T)0);
            }
            vel4[s] = v[u];
            pos4[s] = p[u];
            if (ext.pos4e) {
                // extended (ghost-padded) array the force kernel stages from: own entry + periodic-image copies
                ext_store_at<T>(ext, e_own[u], e_gp[u], p[u], ext.pos4e);
                for (int q = 0; q < push.n_seg; q++)  // halo exchange fused into the drift: mirror boundary slots into the peers
                    if ((unsigned int)(s - push.start[q]) < (unsigned int)push.count[q]) ext_store_at<T>(ext, e_own[u], e_gp[u], p[u], push.dst[q]);
            }
            const T dx = p[u].x - r[u].x, dy = p[u].y - r[u].y, dz = p[u].z - r[u].z;
            const T d2 = dx * dx + dy * dy + dz * dz;
            moved |= (d2 > skin_half2);
            d2max = fmaxf(d2max, (float)d2);
        }
    }
    if (moved) *flag = 1;
    for (int o = 16; o > 0; o >>= 1) d2max = fmaxf(d2max, __shfl_xor_sync(0xffffffffu, d2max, o));
    __shared__ float s_d2[32];
    __shared__ bool s_last;
    if ((threadIdx.x & 31) == 0) s_d2[threadIdx.x >> 5] = d2max;
    __syncthreads();
    if (threadIdx.x == 0) {
        float m = 0.f;
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) m = fmaxf(m, s_d2[w]);
        if (m > 0.f) atomicMax(&ctl->max_disp2_bits, __float_as_uint(m));  // one atomic per CTA
        // the CTA barrier above ordered every thread's stores before this fence (cumulativity); at system scope when
        // some of them went to a peer GPU
        if (push.n_peer > 0) __threadfence_system();
        else __threadfence();
        unsigned int t = atomicInc(&ctl->ticket, gridDim.x - 1);
        s_last = (t == gridDim.x - 1);
    }
    __syncthreads();
    if (s_last && threadIdx.x == 0) {
        step_advance(ctl, handle, use_handle);
        if (push.n_peer > 0) {  // every CTA's peer stores are ordered before its ticket: publish the epoch
            __threadfence_system();
            for (int q = 0; q < push.n_peer; q++) st_release_sys(push.signal_flag[q], push.epoch);
        }
    }
}

// ---- K2: second half kick + centre-of-mass momentum -------------------------------------------
// sum(m v) over the grid (grid_sum); the last CTA publishes v_cm = sum(m v) / sum(m) (src/spatial.jl:901-916). The
// subtraction is applied lazily by the next reader of the velocities (K1, the thermostat or export).
// COUPLE: the variant for the velocity-rescaling thermostats (single GPU) also sums m v.v in double alongside sum(m v); the
// last CTA takes K after this step's CM removal, K - u.sum(m v) + M |u|^2 / 2 with u the v_cm as stored, and stores the
// thermostat's factor next to v_cm (vrescale.cuh).
constexpr int VV_THREADS = 256;
// the thermostat's factor for kinetic energy ke after this step's CM removal, stored as pending
template <typename T>
__device__ __forceinline__ void vcouple_store(CmState<T>* cm, const VCouple& vc, double ke, const Control* ctl) {
    const uint32_t rng[4] = {ctl->rng[0], ctl->rng[1], ctl->rng[2], ctl->rng[3]};
    cm->lam = (T)vcouple_lambda(vc, ke, ctl->step, rng);
    cm->scaled = 1;
}
// k + m |v|^2 with its roundings spelled out: fma(m, fma(z, z, fma(y, y, x x)), k). Left to the compiler, which of the
// products gets fused depends on the surrounding code, and in f64 that moves the last bits of the thermostat's K.
template <typename T4>
__device__ __forceinline__ double add_mvv(double k, double m, const T4& v) {
    return fma(m, fma((double)v.z, (double)v.z, fma((double)v.y, (double)v.y, (double)v.x * (double)v.x)), k);
}
template <typename T, bool COUPLE>
__global__ void __launch_bounds__(VV_THREADS)
    vv_kick2_kernel(int s0, int n, T dt_half, int do_cm, double inv_total_mass, const typename VT<T>::T4* __restrict__ f4,
                    const T* __restrict__ mass, typename VT<T>::T4* __restrict__ vel4, double* __restrict__ partial,
                    Control* __restrict__ ctl, CmState<T>* __restrict__ cm, double* __restrict__ mom_out, PeerSignal sig,
                    VCouple vc) {
    constexpr int W = COUPLE ? 4 : 3;
    double px = 0, py = 0, pz = 0, kk = 0;
    const int stride = gridDim.x * blockDim.x;
    for (int sa = s0 + blockIdx.x * blockDim.x + threadIdx.x; sa < s0 + n; sa += 2 * stride) {  // two atoms in flight per thread
        const int sb = sa + stride;
        const bool okb = sb < s0 + n;
        typename VT<T>::T4 va = vel4[sa], vb = vel4[okb ? sb : sa];
        const typename VT<T>::T4 fa = f4[sa], fb = f4[okb ? sb : sa];
        const T ma = mass[sa], mb_ = mass[okb ? sb : sa];
        const T aa = va.w * dt_half, ab = vb.w * dt_half;
        va.x += fa.x * aa; va.y += fa.y * aa; va.z += fa.z * aa;
        vb.x += fb.x * ab; vb.y += fb.y * ab; vb.z += fb.z * ab;
        vel4[sa] = va;
        px += (double)(va.x * ma); py += (double)(va.y * ma); pz += (double)(va.z * ma);
        if (COUPLE) kk = add_mvv(kk, ma, va);
        if (okb) {
            vel4[sb] = vb;
            px += (double)(vb.x * mb_); py += (double)(vb.y * mb_); pz += (double)(vb.z * mb_);
            if (COUPLE) kk = add_mvv(kk, mb_, vb);
        }
    }
    if (!COUPLE && !do_cm && sig.n_peer == 0) return;
    double s[W] = {px, py, pz};
    if constexpr (COUPLE) s[W - 1] = kk;
    if (!grid_sum<VV_THREADS, W>(s, partial, &ctl->ticket) || threadIdx.x != 0) return;
    const double a = s[0], b = s[1], c = s[2];
    // peer-memory transport: the force kernel in front of this one is done with the halo data ...
    for (int q = 0; q < sig.n_peer; q++) st_release_sys(sig.read_flag[q], sig.epoch);
    if (!do_cm) {
        if constexpr (COUPLE) vcouple_store<T>(cm, vc, 0.5 * s[W - 1], ctl);
        return;
    }
    if (sig.n_mom > 0) {  // ... and sum(m v) goes to every rank (peer_cm_kernel adds them in rank order)
        for (int r = 0; r < sig.n_mom; r++) {
            volatile double* d = sig.mom_dst[r];
            d[0] = a; d[1] = b; d[2] = c;
        }
        __threadfence_system();
        for (int r = 0; r < sig.n_mom; r++) st_release_sys(sig.mom_flag[r], sig.epoch);
    } else if (mom_out) {  // decomposed run over NCCL: the all-reduce and cm_from_sum_kernel finish it
        mom_out[0] = a; mom_out[1] = b; mom_out[2] = c;
    } else {
        cm->publish(s, inv_total_mass);
    }
    if constexpr (COUPLE) {  // (single GPU: v_cm was stored just above)
        const double ux = cm->v[0], uy = cm->v[1], uz = cm->v[2];
        vcouple_store<T>(cm, vc, 0.5 * s[W - 1] + 0.5 * vc.total_mass * (ux * ux + uy * uy + uz * uz) - (ux * a + uy * b + uz * c), ctl);
    }
}

// sqrt-free displacement summary of a call for the interval adaptation of decomposed runs: max(current interval, earlier ones)
__global__ void max_disp_kernel(const Control* __restrict__ ctl, float* __restrict__ out) {
    const unsigned int m = max(ctl->max_disp2_bits, ctl->call_max_disp2_bits);
    out[0] = __uint_as_float(m);
}

template <typename T>
__global__ void cm_from_sum_kernel(const double* __restrict__ mom_sum, double inv_total_mass, CmState<T>* cm) {
    cm->publish(mom_sum, inv_total_mass);
}

// v_cm from the nranks partial sums of the peer-memory all-to-all, added in rank order (see peer.cuh)
template <typename T>
__global__ void peer_cm_kernel(const PeerComm* __restrict__ comm, int nranks, unsigned long long epoch, double inv_total_mass,
                               CmState<T>* __restrict__ cm) {
    const int par = (int)(epoch & 1ull);
    if ((int)threadIdx.x < nranks) spin_until(&comm->mom_epoch[par][threadIdx.x], epoch);
    __syncwarp();
    if (threadIdx.x == 0) {
        double s[3] = {0, 0, 0};
        for (int r = 0; r < nranks; r++) {
            const volatile double* m = comm->mom[par][r];
            s[0] += m[0]; s[1] += m[1]; s[2] += m[2];
        }
        cm->publish(s, inv_total_mass);
    }
}

// no pending v_cm or scale factor: the state at the start of every simulate call
template <typename T>
__global__ void clear_cm_kernel(CmState<T>* cm) {
    cm->v[0] = cm->v[1] = cm->v[2] = (T)0;
    cm->valid = 0;
    cm->scaled = 0;
}

// ---- Andersen thermostat (src/coupling.jl:184-212; GPU kernel src/kernels.jl:705-721) -----------
// Each atom independently, with probability p per step, gets a velocity drawn from the
// Maxwell-Boltzmann distribution, sigma_v = sqrt(kT/m). Philox4x32-10 keyed by (key, ctr1), counter
// = atom index (original order, 1-based as in the reference) so the stream does not depend on the slot
// order; normals by Box-Muller. Statistical parity only (the reference's normal transform lives in
// the un-vendored PhiloxRNG.jl). Consumes the pending v_cm.
template <typename T>
__global__ void andersen_kernel(int s0, int n_own, int n, T kT, double prob, const int* __restrict__ orig,
                                const T* __restrict__ mass, typename VT<T>::T4* __restrict__ vel4,
                                CmState<T>* __restrict__ cm, Control* __restrict__ ctl) {
    int s = s0 + blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t ctr1_lo = ctl->rng[0], ctr1_hi = ctl->rng[1], key_lo = ctl->rng[2], key_hi = ctl->rng[3];
    const uint32_t step_lo = (uint32_t)ctl->step;
    if (s < s0 + n_own) {
        typename VT<T>::T4 v = vel4[s];
        cm->apply(v);
        andersen_apply<T>(v, orig[s], n, mass[s], kT, prob, step_lo, ctr1_lo, ctr1_hi, key_lo, key_hi);
        vel4[s] = v;
    }
    if (last_cta(&ctl->ticket) && threadIdx.x == 0) cm->valid = 0;  // the last CTA clears the pending v_cm
}

// ---- device-side loggers (mb_simulate_vv_log) -----------------------------------------------------------------
// What one logged step records; which of the three a step records is the launch's mask (LOG_*).
enum { LOG_ENERGY = 1, LOG_COORDS = 2, LOG_VELS = 4 };
template <typename T>
struct LogDesc {
    double* rec;                  // energy records (step, pe, ke), one per logged step
    T* frames[2];                 // coordinate / velocity frames (n x 3, original order): the output or a staging ring
    long long ring[2];            // frames the ring holds (the output's capacity when it is the output itself)
    unsigned long long count[3];  // energy records, coordinate frames, velocity frames written in this call
    double pe_const;              // energy terms without a kernel (LJDispersionCorrection)
};
constexpr int LOG_THREADS = 256;
// A read-only observer of the state after step ctl->step: applies the pending v_cm and scale factor and previews the Andersen draw that the
// next drift kernel (or the standalone thermostat closing the call) will apply, with the same operations, so the logged
// velocities are those export_kernel would return after this step. KE = 1/2 sum m v.v in double (grid_sum); the last CTA
// also adds the pair-energy partials of the ENERGY force launch in index order (sum_partials) and writes the record.
template <typename T>
__global__ void __launch_bounds__(LOG_THREADS)
    log_kernel(int n, int mask, Geom<T> g, const typename VT<T>::T4* __restrict__ pos4, const typename VT<T>::T4* __restrict__ vel4,
               const int* __restrict__ orig, const T* __restrict__ mass, const CmState<T>* __restrict__ cm, Control* __restrict__ ctl,
               Thermo<T> th, const double* __restrict__ pe_partial, int n_pe, const double* __restrict__ sp_energy,
               LogDesc<T>* __restrict__ d, double* __restrict__ ke_partial) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    double k = 0;
    if (s < n) {
        const int o = orig[s];
        typename VT<T>::T4 v = vel4[s];
        cm->apply(v);
        if (th.on && ctl->step > ctl->init_step)
            andersen_apply<T>(v, o, th.n, mass[s], th.kT, th.prob, (uint32_t)ctl->step, ctl->rng[0], ctl->rng[1], ctl->rng[2], ctl->rng[3]);
        const double vx = v.x, vy = v.y, vz = v.z;
        k = 0.5 * (double)mass[s] * (vx * vx + vy * vy + vz * vz);
        if (mask & LOG_COORDS)
            store_wrapped<T>(g, pos4[s], d->frames[0] + ((size_t)(d->count[1] % d->ring[0]) * n + o) * 3);
        if (mask & LOG_VELS) {
            T* dst = d->frames[1] + ((size_t)(d->count[2] % d->ring[1]) * n + o) * 3;
            dst[0] = v.x; dst[1] = v.y; dst[2] = v.z;
        }
    }
    double ke[1] = {k};
    if (!grid_sum<LOG_THREADS, 1>(ke, ke_partial, &ctl->ticket)) return;
    double pe[1];
    __syncthreads();  // block_sum's scratch is reused
    sum_partials<LOG_THREADS, 1>(pe_partial, (mask & LOG_ENERGY) ? n_pe : 0, pe);
    if (threadIdx.x == 0) {
        if (mask & LOG_ENERGY) {
            if (sp_energy) pe[0] += *sp_energy;
            pe[0] += d->pe_const;
            double* r = d->rec + 3 * (size_t)d->count[0];
            r[0] = (double)ctl->step; r[1] = pe[0]; r[2] = ke[0];
            d->count[0]++;
        }
        if (mask & LOG_COORDS) d->count[1]++;
        if (mask & LOG_VELS) d->count[2]++;
    }
}

// kinetic energy: 1/2 sum m v.v (src/energy.jl:56-70), partials per CTA then host sum
template <typename T>
__global__ void kinetic_kernel(int n, const T* __restrict__ vels, const T* __restrict__ mass, double* __restrict__ partial) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    double k = 0;
    if (i < n) {
        double vx = vels[3 * (size_t)i], vy = vels[3 * (size_t)i + 1], vz = vels[3 * (size_t)i + 2];
        k = 0.5 * (double)mass[i] * (vx * vx + vy * vy + vz * vz);
    }
    k = block_sum<SUM_THREADS>(k);
    if (threadIdx.x == 0) partial[blockIdx.x] = k;
}

// kinetic energy tensor K = 1/2 sum m v (x) v (src/energy.jl:56-70): xx, yy, zz, xy, xz, yz partials per CTA
template <typename T>
__global__ void kinetic_tensor_kernel(int n, const T* __restrict__ vels, const T* __restrict__ mass, double* __restrict__ partial) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    double k[6] = {0, 0, 0, 0, 0, 0};
    if (i < n) {
        const double m = 0.5 * (double)mass[i];
        const double vx = vels[3 * (size_t)i], vy = vels[3 * (size_t)i + 1], vz = vels[3 * (size_t)i + 2];
        k[0] = m * vx * vx; k[1] = m * vy * vy; k[2] = m * vz * vz; k[3] = m * vx * vy; k[4] = m * vx * vz; k[5] = m * vy * vz;
    }
    block_sum<SUM_THREADS, 6>(k);
    if (threadIdx.x == 0)
        for (int d = 0; d < 6; d++) partial[6 * (size_t)blockIdx.x + d] = k[d];
}

// random_velocities! (src/spatial.jl:803-831; GPU kernel src/kernels.jl:688-703): every atom gets a Maxwell-Boltzmann
// velocity, sigma_v = sqrt(kT / m) per component (massless / virtual sites: zero). Philox4x32-10, counter = 1-based atom
// index, (ctr1, key) = the caller's two rand(rng, UInt64); normals by Box-Muller. Statistical parity only (SURVEY §8c:
// the reference's uniform -> normal transform lives in the un-vendored PhiloxRNG.jl).
template <typename T>
__global__ void random_velocities_kernel(int n, T kT, const T* __restrict__ mass, uint32_t ctr1_lo, uint32_t ctr1_hi,
                                         uint32_t key_lo, uint32_t key_hi, T* __restrict__ vels) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t d[4] = {(uint32_t)(i + 1), 0u, ctr1_lo, ctr1_hi};
    philox4x32_10(d, key_lo, key_hi);
    const T m = mass[i];
    double g[3];
    box_muller3(d, (m > (T)0) ? sqrt((double)kT / (double)m) : 0.0, g);
    for (int k = 0; k < 3; k++) vels[3 * (size_t)i + k] = (T)g[k];
}

// sum(m v) partials over an original-order velocity array (mb_remove_cm_motion)
template <typename T>
__global__ void momentum_kernel(int n, const T* __restrict__ vels, const T* __restrict__ mass, double* __restrict__ partial) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    double p[3] = {0, 0, 0};
    if (i < n) {
        T m = mass[i];
        for (int d = 0; d < 3; d++) p[d] = (double)(vels[3 * (size_t)i + d] * m);
    }
    block_sum<SUM_THREADS, 3>(p);
    if (threadIdx.x == 0)
        for (int d = 0; d < 3; d++) partial[3 * (size_t)blockIdx.x + d] = p[d];
}
template <typename T>
__global__ void subtract_velocity_kernel(int n, T vx, T vy, T vz, T* __restrict__ vels) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    vels[3 * (size_t)i] -= vx;
    vels[3 * (size_t)i + 1] -= vy;
    vels[3 * (size_t)i + 2] -= vz;
}

}  // namespace mb
