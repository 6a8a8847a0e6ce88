// force.cuh — the non-bonded force/energy kernels.
//
// brick_force_kernel: the production path. Persistent CTAs (two per SM) work through the bricks of cells: a
// producer warp stages each brick's halo (all atoms within r_list of any owned atom) into a ring of shared-
// memory stages with the TMA engine (cp.async.bulk + mbarrier) as float4 (x,y,z,q) [+ float2 LJ parameters],
// periodic images moved into the owned atoms' frame; 15 consumer warps process the owned atoms, 8 lanes per
// atom walking its full-shell neighbour list (16-bit halo offsets, read as coalesced 8-byte words) with four
// independent pair evaluations in flight per lane. Partial forces are reduced with warp shuffles; there are no
// atomics on forces and no Newton-3 scatter, so results are bitwise reproducible run to run. Replaces force_kernel!/energy_kernel!
// (ext/MollyCUDAExt.jl:1595-2045, :2062-2294) and pairwise_force_kernel_nl! (src/kernels.jl:114-140).
//
// allpairs_force_kernel: O(N^2) minimum-image kernel for systems without a usable neighbour list
// (use_neighbors=false / NoCutoff / boxes smaller than 2.5 r_list); replaces
// pairwise_force_kernel_nonl! (ext/MollyCUDAExt.jl:2305-2371).
#pragma once
#include "cells.cuh"
#include "dpd.cuh"
#include "pair.cuh"
#include "peer.cuh"

namespace mb {

// ---- launch shape of the persistent brick kernel ---------------------------------------------------------------
// 16 warps per CTA: 15 consumer warps evaluate pairs, 1 producer warp feeds them through a ring of up to FORCE_MAX_STAGES
// shared-memory stages (one stage = one brick's halo + its task table), filled by the TMA engine.
constexpr int FORCE_THREADS = 512;
constexpr int FORCE_CTAS_F32 = 2;  // resident CTAs per SM the f32 variants are compiled for (register cap = 64K / (CTAs x threads))
constexpr int FORCE_CONSUMER_WARPS = FORCE_THREADS / 32 - 1;
constexpr int FORCE_MAX_STAGES = 3;

template <typename T>
struct ForceOut {
    typename VT<T>::T4* f4;   // per-slot force (w unused)
    double* pe_partial;       // [gridDim.x] (ENERGY)
    double* vir_partial;      // [gridDim.x*6] xx,yy,zz,xy,xz,yz (ENERGY)
    PeerWait gate;            // decomposed run over peer memory: epoch flags the halo data of this step arrives under
};

struct __align__(16) StageMeta {
    int brick;    // global brick index staged here
    int icount;   // owned atoms (tasks) of the brick; -1 = no more work for this CTA
    int nq;       // quads of 4 tasks
    int next_q;   // next quad to hand out (force-only launches; energy launches assign quads statically)
};

// bytes of one stage: positions [+ LJ parameters] of the halo, then the task table
template <typename T>
__host__ __device__ inline size_t force_stage_bytes(int halo_cap, int task_cap, bool uniform) {
    size_t b = (size_t)halo_cap * sizeof(typename VT<T>::T4);
    if (!uniform) b += (size_t)halo_cap * sizeof(typename VT<T>::T2);
    b = (b + 127) & ~(size_t)127;
    b += ((size_t)task_cap * sizeof(int2) + 127) & ~(size_t)127;
    return b;
}

// brick_force_kernel — persistent, warp-specialised.
//   producer warp: takes the next brick (atomic ticket; static round-robin for ENERGY launches so that the per-CTA energy
//     partials are reproducible), reads its header and run table, issues one bulk async copy (TMA) per (y,z) row of the
//     halo - a contiguous range of the extended array pos4e, periodic images included - and one for the task table into
//     the next free stage, and publishes the stage (mbarrier ready[s]) once the bytes have landed. It runs up to
//     nbuf-1 bricks ahead of the consumers.
//   consumer warps: take quads (4 consecutive owned atoms, 8 lanes each) of the published stages, walk the four
//     neighbour rows (software-pipelined: the next quad's first index words are requested while the current one is
//     evaluated, across stage boundaries), reduce with shuffles and store. A warp releases a stage (mbarrier empty[s])
//     once it holds no quad in it; there is no CTA-wide barrier in the steady state.
//   DPD: the DPDInteraction variant (dpd.cuh; instantiated with COUL_NONE, UNIFORM, CUTM_PLAIN): the staged w is the
//     original index, v_j is gathered from the predicted velocities and the pair's draw is keyed by the device step counter.
//     Special-list entries get the full force. No virial: the ENERGY variant sums the conservative energy only. One CTA per
//     SM: the draw's double-precision Box-Muller needs more than 64 registers.
template <typename T, int COUL, bool UNIFORM, int CUTM, bool ENERGY, bool DPD = false>
__global__ void __launch_bounds__(FORCE_THREADS, (sizeof(T) == 8 || DPD) ? 1 : FORCE_CTAS_F32)
    brick_force_kernel(Geom<T> g, PairParams<T> P, const BrickHdr* __restrict__ hdrs, const Run* __restrict__ runs,
                       const int2* __restrict__ task_tab, const typename VT<T>::T4* __restrict__ pos4e,
                       const typename VT<T>::T2* __restrict__ lj2e, const unsigned short* __restrict__ list,
                       const unsigned short* __restrict__ slist, ForceOut<T> out, int brick0, int nbr, int nbuf,
                       unsigned int* __restrict__ sched) {
    // DPD stages positions only, so the LJ-parameter pointer carries the address of its constants (DpdArgs in device
    // memory, dpd_args_of): the parameter list, and with it the code of every other variant, stays as it is
    static_assert(!DPD || (COUL == COUL_NONE && UNIFORM && CUTM == CUTM_PLAIN),
                  "the DPD variant stages positions only: its LJ-parameter pointer carries the DpdArgs (dpd_args_of)");
    using T4 = typename VT<T>::T4;
    using T2 = typename VT<T>::T2;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ uint64_t s_ready[FORCE_MAX_STAGES], s_empty[FORCE_MAX_STAGES], s_full[FORCE_MAX_STAGES];
    __shared__ StageMeta s_meta[FORCE_MAX_STAGES];
    constexpr int NW = FORCE_CONSUMER_WARPS;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const size_t lj_off = (size_t)g.halo_cap * sizeof(T4);
    const size_t task_off = ((lj_off + (UNIFORM ? 0 : (size_t)g.halo_cap * sizeof(T2))) + 127) & ~(size_t)127;
    const size_t stage_bytes = force_stage_bytes<T>(g.halo_cap, g.task_cap, UNIFORM);
    const int A = g.align;
    if (tid == 0) {
        for (int s = 0; s < nbuf; s++) {
            mbar_init(&s_ready[s], 1);
            mbar_init(&s_empty[s], NW);
            mbar_init(&s_full[s], 1);
        }
        mbar_fence_init();
    }
    if (tid < A * nbuf) {  // dummy atom of every stage (pads of the neighbour rows point at it): far away, no charge, no LJ
        unsigned char* st = smem_raw + (size_t)(tid / A) * stage_bytes;
        reinterpret_cast<T4*>(st)[tid % A] = make4<T>((T)1.0e6, (T)1.0e6, (T)1.0e6, (T)0);
        if (!UNIFORM) reinterpret_cast<T2*>(st + lj_off)[tid % A] = make2<T>((T)0, (T)0);
    }
    if (out.gate.n > 0) {  // the neighbours' drift kernels store this step's halo positions into pos4 (peer.cuh)
        if (tid < out.gate.n) spin_until(out.gate.flag[tid], out.gate.epoch);
    }
    __syncthreads();
    if (out.gate.n > 0) fence_proxy_async_all();  // the TMA engine reads them next

    T e_acc = (T)0;
    T vir[6] = {(T)0, (T)0, (T)0, (T)0, (T)0, (T)0};

    if (w == NW) {
        // =============================== producer warp ===============================
        int pend = 0, p_s = 0, p_par = 0, p_b = 0, p_icount = 0;  // stage issued but not yet published
        unsigned int full_bits = 0;  // phase parity of s_full[s] (a stage is only armed when its brick owns atoms)
        auto publish = [&]() {
            if (p_icount > 0) mbar_wait(&s_full[p_s], (uint32_t)p_par);  // the stage's bytes have landed
            __syncwarp();
            if (lane == 0) {
                StageMeta mt;
                mt.brick = p_b;
                mt.icount = p_icount;
                mt.nq = (p_icount + 3) >> 2;
                mt.next_q = 0;
                s_meta[p_s] = mt;
                mbar_arrive(&s_ready[p_s]);
            }
            pend = 0;
        };
        for (int seq = 0, s = 0, use = 0;; seq++, s = (s + 1 == nbuf) ? 0 : s + 1, use += (s == 0) ? 1 : 0) {
            // (1) next brick: the first one of a CTA is its block index (no ticket latency in front of the first stage), the
            //     others are drawn from the global ticket counter; static round-robin for ENERGY launches
            int bi;
            if (ENERGY) {
                bi = (int)blockIdx.x + seq * (int)gridDim.x;
            } else if (seq == 0) {
                bi = (int)blockIdx.x;
            } else {
                bi = 0;
                if (lane == 0) bi = (int)gridDim.x + (int)atomicAdd(sched, 1u);
                bi = __shfl_sync(0xffffffffu, bi, 0);
            }
            const bool last = bi >= nbr;
            const int c_b = brick0 + (last ? 0 : bi);
            BrickHdr hd = {0, 0, 0u, 0u, 0, {0, 0, 0}};
            // header and this lane's first run entries: requested together, in flight while the previous stage lands
            const Run* my_runs = runs + (size_t)c_b * g.max_runs;
            Run pre[2] = {{0, 0, 0, 0}, {0, 0, 0, 0}};
            if (!last) {
                hd = hdrs[c_b];
                if (lane < g.max_runs) pre[0] = my_runs[lane];
                if (lane + 32 < g.max_runs) pre[1] = my_runs[lane + 32];
            }
            // (2) publish the stage issued one round earlier. This comes BEFORE waiting for a free stage: a consumer may hold
            //     stage k while it waits for stage k + nbuf - 1 to be published.
            if (pend) publish();
            // (3) a free stage
            if (use > 0) mbar_wait(&s_empty[s], (uint32_t)((use - 1) & 1));
            fence_proxy_async();  // generic-proxy accesses of the stage's previous use before the async-proxy writes below
            if (last) {
                if (lane == 0) {
                    StageMeta mt = {0, -1, 0, 0};
                    s_meta[s] = mt;
                    mbar_arrive(&s_ready[s]);
                }
                break;
            }
            // (4) issue the copies
            const bool skip = hd.i_count == 0 || hd.halo_count > g.halo_cap;
            const int c_icount = skip ? 0 : min(hd.i_count, g.task_cap);
            int c_par = 0;
            if (c_icount > 0) {
                unsigned char* st = smem_raw + (size_t)s * stage_bytes;
                T4* sp = reinterpret_cast<T4*>(st);
                T2* sl = reinterpret_cast<T2*>(st + lj_off);
                const uint32_t tbytes = ((uint32_t)c_icount * (uint32_t)sizeof(int2) + 15u) & ~15u;
                c_par = (int)((full_bits >> s) & 1u);
                full_bits ^= 1u << s;
                if (lane == 0) mbar_arrive_expect_tx(&s_full[s], hd.tx_pos + (UNIFORM ? 0u : hd.tx_lj) + tbytes);
                __syncwarp();
                for (int r = lane, k = 0; r < g.max_runs; r += 32, k++) {
                    const Run run = (k == 0) ? pre[0] : ((k == 1) ? pre[1] : my_runs[r]);
                    if (run.count > 0) {
                        bulk_g2s(&sp[run.soff], &pos4e[run.gstart], (uint32_t)run.count * (uint32_t)sizeof(T4), &s_full[s]);
                        if (!UNIFORM) {
                            const int mis = run.gstart % A;
                            const int len = (mis + run.count + A - 1) / A * A;
                            bulk_g2s(&sl[run.soff - mis], &lj2e[run.gstart - mis], (uint32_t)len * (uint32_t)sizeof(T2), &s_full[s]);
                        }
                    }
                }
                if (lane == 0) bulk_g2s(st + task_off, task_tab + (size_t)c_b * g.task_cap, tbytes, &s_full[s]);
            }
            pend = 1; p_s = s; p_par = c_par; p_b = c_b; p_icount = c_icount;
        }
    } else {
        // =============================== consumer warps ===============================
        const int sub4 = lane >> 3, l = lane & 7;
        constexpr int LIST_HALF = 4;  // list words (4 entries each) per lane and half batch: 8 words in flight
        // per-quad state (the stage changes from quad to quad): shared-memory addresses of the staged positions / LJ pairs
        uint32_t s_pos_u32 = 0, s_lj_u32 = 0;
        T4 pi = make4<T>(0, 0, 0, 0);
        T lj_s_i = (T)0, lj_e_i = (T)0, kq_i = (T)0;
        T fx = (T)0, fy = (T)0, fz = (T)0;
        // DPD: the step the draws are keyed by, and the quad's atom: original index and predicted velocity
        long long dstep = 0;
        int oi = 0;
        T4 vi;
        if constexpr (DPD) dstep = *dpd_args_of<T>(lj2e).step;
        auto eval = [&](int j, auto special_tag) {
            constexpr bool SPECIAL = decltype(special_tag)::value;
            (void)SPECIAL;  // (the DPD variant gives special pairs the full force)
            const T4 pj = lds_pos(s_pos_u32 + (uint32_t)j * (uint32_t)sizeof(T4), (T)0);
            T lj_s_j = (T)0, lj_e_j = (T)0;
            if (!UNIFORM) {
                T2 t = lds_pair(s_lj_u32 + (uint32_t)j * (uint32_t)sizeof(T2), (T)0);
                lj_s_j = t.x;
                lj_e_j = t.y;
            }
            const T dx = pi.x - pj.x, dy = pi.y - pj.y, dz = pi.z - pj.z;
            const T r2 = dx * dx + dy * dy + dz * dz;
            T fr, e;
            if constexpr (DPD) dpd_eval<T>(dpd_args_of<T>(lj2e), dstep, oi, vi, r2, dx, dy, dz, pj.w, fr, e);
            else pair_eval<T, COUL, UNIFORM, CUTM, ENERGY, SPECIAL>(P, r2, lj_s_i, lj_e_i, lj_s_j, lj_e_j, kq_i, pj.w, fr, e);
            const T gx = fr * dx, gy = fr * dy, gz = fr * dz;
            fx += gx;
            fy += gy;
            fz += gz;
            if (ENERGY) {
                e_acc += e;
                if constexpr (!DPD) {
                    vir[0] += dx * gx; vir[1] += dy * gy; vir[2] += dz * gz;
                    vir[3] += dx * gy; vir[4] += dx * gz; vir[5] += dy * gz;
                }
            }
        };
        // four neighbours at once, stage by stage, so the four shared-memory loads and the four reciprocal
        // chains are independent and in flight together
        auto eval4 = [&](uint2 wd) {
            // entries are byte offsets of float4 records (halo index << LIST_SHIFT)
            if constexpr (DPD) {
                // one neighbour at a time: four draws (Philox and a Box-Muller in double each) in flight do not fit the registers
#pragma unroll 1
                for (int u = 0; u < 4; u++) {
                    const uint32_t w32 = (u < 2) ? wd.x : wd.y;
                    const uint32_t j = (u & 1) ? (w32 >> 16) : (w32 & 0xffffu);
                    const T4 pj = lds_pos(s_pos_u32 + j * (uint32_t)(sizeof(T4) >> LIST_SHIFT), (T)0);
                    const T dx = pi.x - pj.x, dy = pi.y - pj.y, dz = pi.z - pj.z;
                    T fr, e;
                    dpd_eval<T>(dpd_args_of<T>(lj2e), dstep, oi, vi, dx * dx + dy * dy + dz * dz, dx, dy, dz, pj.w, fr, e);
                    const T gx = fr * dx, gy = fr * dy, gz = fr * dz;
                    fx += gx;
                    fy += gy;
                    fz += gz;
                    if (ENERGY) e_acc += e;
                }
                return;
            }
            const int j[4] = {(int)(wd.x & 0xffffu), (int)(wd.x >> 16), (int)(wd.y & 0xffffu), (int)(wd.y >> 16)};
            T4 pj[4];
            T2 lj[4];
#pragma unroll
            for (int u = 0; u < 4; u++) {
                pj[u] = lds_pos(s_pos_u32 + (uint32_t)j[u] * (uint32_t)(sizeof(T4) >> LIST_SHIFT), (T)0);
                if (!UNIFORM) lj[u] = lds_pair(s_lj_u32 + (((uint32_t)j[u] * (uint32_t)sizeof(T2)) >> LIST_SHIFT), (T)0);
            }
            T dx[4], dy[4], dz[4], r2[4], fr[4], e[4];
#pragma unroll
            for (int u = 0; u < 4; u++) {
                dx[u] = pi.x - pj[u].x;
                dy[u] = pi.y - pj[u].y;
                dz[u] = pi.z - pj[u].z;
                r2[u] = dx[u] * dx[u] + dy[u] * dy[u] + dz[u] * dz[u];
            }
#pragma unroll
            for (int u = 0; u < 4; u++)
                pair_eval<T, COUL, UNIFORM, CUTM, ENERGY, false>(P, r2[u], lj_s_i, lj_e_i, UNIFORM ? (T)0 : lj[u].x,
                                                                  UNIFORM ? (T)0 : lj[u].y, kq_i, pj[u].w, fr[u], e[u]);
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const T gx = fr[u] * dx[u], gy = fr[u] * dy[u], gz = fr[u] * dz[u];
                fx += gx;
                fy += gy;
                fz += gz;
                if (ENERGY) {
                    e_acc += e[u];
                    vir[0] += dx[u] * gx; vir[1] += dy[u] * gy; vir[2] += dz[u] * gz;
                    vir[3] += dx[u] * gy; vir[4] += dx[u] * gz; vir[5] += dy[u] * gz;
                }
            }
        };

        // ---- quad hand-out ------------------------------------------------------------------------------------
        // The cursor (look_*) walks the stages in publication order; (seq, s, par) = sequence number, ring index and
        // mbarrier phase parity of a stage, advanced together (no division in the loop). held_* = earliest stage this
        // warp has not released yet.
        int look_seq = 0, look_s = 0;
        uint32_t look_par = 0;
        int held_seq = 0, held_s = 0;
        int k_local = 0;   // static hand-out: quads this warp already took from stage look_seq
        struct QD { int seq, slot, packed; uint32_t base; };  // packed = staged index | rows' lengths (task_pack); base = stage address
        auto release_upto = [&](int upto) {  // this warp holds no quad in the stages before `upto` any more
            __syncwarp();
            while (held_seq < upto) {
                if (lane == 0) mbar_arrive(&s_empty[held_s]);
                held_s = (held_s + 1 == nbuf) ? 0 : held_s + 1;
                held_seq++;
            }
        };
        // returns 1: quad found, 0: no more work, -1: the cursor would run more than the ring depth ahead of a held stage.
        // holding: a quad of this warp is still in flight in stage held_seq (stages are then released after that quad).
        auto lookup = [&](int max_seq, bool holding, QD& o) -> int {
            for (;;) {
                if (look_seq > max_seq) return -1;
                if (!mbar_try_wait(&s_ready[look_s], look_par)) mbar_wait_slow(&s_ready[look_s], look_par);
                const int4 mt = *reinterpret_cast<const int4*>(&s_meta[look_s]);  // brick, icount, nq, next_q
                if (mt.y < 0) return 0;
                int q;
                if (ENERGY) {
                    q = w + NW * k_local;
                    k_local++;
                } else {
                    q = 0;
                    if (lane == 0) q = atomicAdd(&s_meta[look_s].next_q, 1);
                    q = __shfl_sync(0xffffffffu, q, 0);
                }
                if (q < mt.z) {
                    const int t = 4 * q + sub4;
                    int2 e = make_int2(-1, 0);
                    if (t < mt.y) e = reinterpret_cast<const int2*>(smem_raw + (size_t)look_s * stage_bytes + task_off)[t];
                    o.seq = look_seq;
                    o.base = smem_u32(smem_raw) + (uint32_t)look_s * (uint32_t)stage_bytes;
                    o.slot = e.x;
                    o.packed = e.y;
                    return 1;
                }
                look_seq++;
                look_s++;
                if (look_s == nbuf) { look_s = 0; look_par ^= 1u; }
                k_local = 0;
                if (!holding) release_upto(look_seq);  // nothing in flight: pass exhausted stages on right away
            }
        };
        uint2 wa[LIST_HALF];
        auto request_first = [&](const QD& qd) {
            // only the groups this row was written with: a row shorter than the quad's longest one feeds zero words (the
            // dummy atom) for the rest. The part of the row beyond its padded length holds entries of earlier builds.
            const int ng = (((qd.packed >> 12) & 0xfff) + 31) >> 5;
            const uint2* p2 = reinterpret_cast<const uint2*>(list + (size_t)max(qd.slot, 0) * g.stride) + l;
#pragma unroll
            for (int u = 0; u < LIST_HALF; u++)
                wa[u] = (qd.slot >= 0 && u < ng) ? ldg_stream_u2(p2 + (size_t)u * 8) : make_uint2(0u, 0u);
        };
        QD cur, nxt;
        int r = lookup(0x7fffffff, false, cur);
        if (r == 1) request_first(cur);
        while (r == 1) {
            s_pos_u32 = cur.base;
            s_lj_u32 = cur.base + (uint32_t)lj_off;
            const bool valid = cur.slot >= 0;
            const int slot = max(cur.slot, 0);
            const int cur_si = cur.packed & 0xfff, cur_n_main = (cur.packed >> 12) & 0xfff;
            const int cur_n_spec = (int)((unsigned int)cur.packed >> 24);
            pi = lds_pos(s_pos_u32 + (uint32_t)cur_si * (uint32_t)sizeof(T4), (T)0);
            if (!valid) pi = make4<T>((T)-1.0e6, (T)-1.0e6, (T)-1.0e6, (T)0);  // idle lane group: far from the dummy atom its zero words point at
            if (!UNIFORM) {
                T2 t = lds_pair(s_lj_u32 + (uint32_t)cur_si * (uint32_t)sizeof(T2), (T)0);
                lj_s_i = t.x;
                lj_e_i = t.y;
            }
            kq_i = P.ke * pi.w;
            if constexpr (DPD) {
                oi = (int)pi.w;
                vi = dpd_args_of<T>(lj2e).vpred[oi];
            }
            fx = (T)0; fy = (T)0; fz = (T)0;
            // main list: groups of 32 entries; each of the 8 lanes owns 4 entries (one 8-byte word) per group
            const int n_groups = (cur_n_main + 31) >> 5;
            // the four atoms of the quad run the same number of group iterations (the longest row's); shorter rows feed zero
            // words, i.e. the dummy atom, so the loop control is warp-uniform
            int gmax = max(n_groups, __shfl_xor_sync(0xffffffffu, n_groups, 8));
            gmax = max(gmax, __shfl_xor_sync(0xffffffffu, gmax, 16));
            const uint2* lp2 = reinterpret_cast<const uint2*>(list + (size_t)slot * g.stride) + l;
            // second half of this quad's first batch
            uint2 wb[LIST_HALF];
#pragma unroll
            for (int u = 0; u < LIST_HALF; u++)
                wb[u] = (LIST_HALF + u < n_groups) ? ldg_stream_u2(lp2 + (size_t)(LIST_HALF + u) * 8) : make_uint2(0u, 0u);
            // the next quad (possibly in a later stage): descriptor now, its first index words after the first half below
            r = lookup(cur.seq + nbuf - 1, true, nxt);
#pragma unroll
            for (int u = 0; u < LIST_HALF; u++)
                if (u < gmax) eval4(wa[u]);
            if (r == 1) request_first(nxt);
#pragma unroll
            for (int u = 0; u < LIST_HALF; u++)
                if (LIST_HALF + u < gmax) eval4(wb[u]);
            // rows longer than one batch
            for (int g0 = 2 * LIST_HALF; g0 < gmax; g0 += LIST_HALF) {
                uint2 wc[LIST_HALF];
#pragma unroll
                for (int u = 0; u < LIST_HALF; u++)
                    wc[u] = (g0 + u < n_groups) ? ldg_stream_u2(lp2 + (size_t)(g0 + u) * 8) : make_uint2(0u, 0u);
#pragma unroll
                for (int u = 0; u < LIST_HALF; u++)
                    if (g0 + u < gmax) eval4(wc[u]);
            }
            // special (1-4) pairs
            for (int m = l; m < cur_n_spec; m += 8) eval((int)slist[(size_t)slot * g.sstride + m], std::true_type{});
            // reduce the 8 partial forces of every atom
            __syncwarp();
#pragma unroll
            for (int o = 4; o > 0; o >>= 1) {
                fx += shfl_xor(fx, o);
                fy += shfl_xor(fy, o);
                fz += shfl_xor(fz, o);
            }
            if (l == 0 && valid) out.f4[slot] = make4<T>(fx, fy, fz, (T)0);
            // release the stages this warp no longer holds a quad in
            release_upto((r == 1) ? nxt.seq : look_seq);
            if (r == -1) {  // the cursor stopped at the ring depth: nothing is held now, so waiting is safe
                r = lookup(0x7fffffff, false, nxt);
                if (r == 1) request_first(nxt);
            }
            cur = nxt;
        }
    }

    if (ENERGY) {
        // full shell: every pair was visited from both ends -> 1/2. The order is block_sum's (common.cuh), written out here:
        // calling the helper changes the register assignment of some of the plain (!ENERGY) instantiations.
        __shared__ double s_red[FORCE_THREADS / 32][7];
        double v[7] = {(double)e_acc, (double)vir[0], (double)vir[1], (double)vir[2],
                       (double)vir[3], (double)vir[4], (double)vir[5]};
#pragma unroll
        for (int k = 0; k < 7; k++) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
        }
        if (lane == 0)
            for (int k = 0; k < 7; k++) s_red[w][k] = v[k];
        __syncthreads();
        if (tid < 7) {
            double s = 0.0;
            for (int ww = 0; ww < FORCE_THREADS / 32; ww++) s += s_red[ww][tid];
            s *= 0.5;
            if (tid == 0) out.pe_partial[blockIdx.x] = s;
            else out.vir_partial[(size_t)blockIdx.x * 6 + (tid - 1)] = s;
        }
    }
    if (!ENERGY && tid == FORCE_THREADS - 32) {
        // the last CTA to get here re-arms the brick ticket for the next launch (every CTA has drawn its last ticket)
        __threadfence();
        const unsigned int t = atomicInc(sched + 1, gridDim.x - 1);
        if (t == gridDim.x - 1) {  // (tickets count from gridDim.x: every CTA's first brick is its block index)
            sched[0] = 0u;
            __threadfence();
        }
    }
}

// deterministic final reduction of per-CTA partials (one CTA of SUM_THREADS): pe_out[0] += sum, vir_out (3x3, T) += sum
template <typename T>
__global__ void reduce_partials_kernel(int n, const double* __restrict__ pe_partial, const double* __restrict__ vir_partial,
                                       T* pe_out, T* vir_out) {
    double s[7] = {0, 0, 0, 0, 0, 0, 0};
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        s[0] += pe_partial[i];
        if (vir_partial)
            for (int k = 0; k < 6; k++) s[1 + k] += vir_partial[(size_t)i * 6 + k];
    }
    block_sum<SUM_THREADS, 7>(s);
    if (threadIdx.x == 0) {
        if (pe_out) pe_out[0] += (T)s[0];
        if (vir_out) {
            // column-major 3x3: W[a,b] += dr[a] f[b]; symmetric here
            vir_out[0] += (T)s[1]; vir_out[4] += (T)s[2]; vir_out[8] += (T)s[3];
            vir_out[1] += (T)s[4]; vir_out[3] += (T)s[4];
            vir_out[2] += (T)s[5]; vir_out[6] += (T)s[5];
            vir_out[5] += (T)s[6]; vir_out[7] += (T)s[6];
        }
    }
}

// ---------------------------------------------------------------------------------------------
// All-pairs path (no neighbour list). Atoms in original order; minimum image by the reference's
// select chain (src/spatial.jl:491-500). One thread per i atom, j tiles through shared memory.
// Exclusions / specials through the per-atom CSR partner lists.
// ---------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ T mic_1d(T ci, T cj, T L) {
    // vector_1D(c1=ci, c2=cj): returns c_j - c_i minimum image
    T v = cj - ci;
    T vp = v + L, vm = v - L;
    return (v > (T)0) ? ((v < -vm) ? v : vm) : ((-v < vp) ? v : vp);
}

constexpr int AP_THREADS = 128;

// DPD: the DPDInteraction variant (dpd.cuh; instantiated with COUL_NONE, CUTM_PLAIN): the position records' w is the atom's
// index, v_j is gathered from dpd.vpred; exclusions apply when the interaction uses the neighbour list (dpd.nl). No virial.
template <typename T, int COUL, int CUTM, bool ENERGY, bool DPD = false>
__global__ void __launch_bounds__(AP_THREADS)
    allpairs_force_kernel(int n, PairParams<T> P, T Lx, T Ly, T Lz, Tric<T> tric, const typename VT<T>::T4* __restrict__ posq,
                          const typename VT<T>::T2* __restrict__ lj2, const int* __restrict__ ex_ptr,
                          const int* __restrict__ ex_idx, const int* __restrict__ sp_ptr,
                          const int* __restrict__ sp_idx, typename VT<T>::T4* __restrict__ f4,
                          double* __restrict__ pe_partial, double* __restrict__ vir_partial, DpdArgs<T> dpd) {
    using T4 = typename VT<T>::T4;
    using T2 = typename VT<T>::T2;
    __shared__ T4 s_pos[AP_THREADS];
    __shared__ T2 s_lj[AP_THREADS];
    const int tid = threadIdx.x;
    const int i = blockIdx.x * AP_THREADS + tid;
    const bool active = i < n;
    T4 pi = active ? posq[i] : make4<T>(0, 0, 0, 0);
    T2 li = active ? lj2[i] : make2<T>(0, 0);
    const T kq_i = P.ke * pi.w;
    int ex_a = 0, ex_n = 0, sp_a = 0, sp_n = 0;
    if (active && ex_ptr) { ex_a = ex_ptr[i]; ex_n = ex_ptr[i + 1] - ex_a; }
    if (active && sp_ptr) { sp_a = sp_ptr[i]; sp_n = sp_ptr[i + 1] - sp_a; }
    T fx = 0, fy = 0, fz = 0, e_acc = 0;
    T vir[6] = {0, 0, 0, 0, 0, 0};
    const long long dstep = DPD ? *dpd.step : 0;
    const T4 vi = (DPD && active) ? dpd.vpred[i] : make4<T>(0, 0, 0, 0);
    for (int j0 = 0; j0 < n; j0 += AP_THREADS) {
        int jj = j0 + tid;
        __syncthreads();
        s_pos[tid] = (jj < n) ? posq[jj] : make4<T>(0, 0, 0, 0);
        s_lj[tid] = (jj < n) ? lj2[jj] : make2<T>(0, 0);
        __syncthreads();
        int lim = min(AP_THREADS, n - j0);
        if (!active) continue;
        for (int k = 0; k < lim; k++) {
            int j = j0 + k;
            if (j == i) continue;
            bool excluded = false, special = false;
            for (int m = 0; m < ex_n; m++) excluded |= (ex_idx[ex_a + m] == j);
            for (int m = 0; m < sp_n; m++) special |= (sp_idx[sp_a + m] == j);
            T4 pj = s_pos[k];
            T2 lj = s_lj[k];
            // d = c_i - c_j = -vector(c_i, c_j)
            T dx, dy, dz;
            if (tric.on) {  // TriclinicBoundary: dr = vector(c_i, c_j), d = -dr
                T ex = pj.x - pi.x, ey = pj.y - pi.y, ez = pj.z - pi.z;
                tric_vector<T>(tric, ex, ey, ez);
                dx = -ex; dy = -ey; dz = -ez;
            } else {
                dx = -mic_1d(pi.x, pj.x, Lx); dy = -mic_1d(pi.y, pj.y, Ly); dz = -mic_1d(pi.z, pj.z, Lz);
            }
            T r2 = dx * dx + dy * dy + dz * dz;
            T fr, e;
            if constexpr (DPD) {
                if (excluded && dpd.nl) { fr = (T)0; e = (T)0; }
                else dpd_eval<T>(dpd, dstep, i, vi, r2, dx, dy, dz, pj.w, fr, e);
            } else {
                pair_eval_rt<T, COUL, CUTM, ENERGY>(P, r2, li.x, li.y, lj.x, lj.y, kq_i, pj.w, excluded, special, fr, e);
            }
            T gx = fr * dx, gy = fr * dy, gz = fr * dz;
            fx += gx; fy += gy; fz += gz;
            if (ENERGY) {
                e_acc += e;
                if constexpr (!DPD) {  // (DPD has no virial)
                    vir[0] += dx * gx; vir[1] += dy * gy; vir[2] += dz * gz;
                    vir[3] += dx * gy; vir[4] += dx * gz; vir[5] += dy * gz;
                }
            }
        }
    }
    if (active) f4[i] = make4<T>(fx, fy, fz, (T)0);
    if (ENERGY) {
        // full shell -> 1/2
        double v[7] = {(double)e_acc, (double)vir[0], (double)vir[1], (double)vir[2],
                       (double)vir[3], (double)vir[4], (double)vir[5]};
        __syncthreads();
        block_sum<AP_THREADS, 7>(v);
        if (tid == 0) {
            pe_partial[blockIdx.x] = v[0] * 0.5;
            for (int k = 0; k < 6; k++) vir_partial[(size_t)blockIdx.x * 6 + k] = v[1 + k] * 0.5;
        }
    }
}

}  // namespace mb
