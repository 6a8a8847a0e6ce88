// common.cuh — shared device helpers for libmollyb200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

namespace mb {

// ---------------------------------------------------------------------------------------------
// vector-type traits: T4 = (x, y, z, w) with 16-byte alignment, T2 = pair
// ---------------------------------------------------------------------------------------------
struct __align__(16) dbl4 {
    double x, y, z, w;
};
struct __align__(16) dbl2 {
    double x, y;
};

template <typename T>
struct VT;
template <>
struct VT<float> {
    using T4 = float4;
    using T2 = float2;
};
template <>
struct VT<double> {
    using T4 = dbl4;
    using T2 = dbl2;
};

template <typename T>
__host__ __device__ inline typename VT<T>::T4 make4(T x, T y, T z, T w) {
    typename VT<T>::T4 r;
    r.x = x; r.y = y; r.z = z; r.w = w;
    return r;
}
template <typename T>
__host__ __device__ inline typename VT<T>::T2 make2(T x, T y) {
    typename VT<T>::T2 r;
    r.x = x; r.y = y;
    return r;
}

// fast reciprocal / rsqrt: approx for float (<= 1-2 ulp), IEEE for double
__device__ __forceinline__ float frcp(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ double frcp(double x) { return 1.0 / x; }
__device__ __forceinline__ float frsqrt(float x) {
    float r;
    asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ double frsqrt(double x) { return 1.0 / sqrt(x); }
__device__ __forceinline__ float fsqrt(float x) { return sqrtf(x); }
__device__ __forceinline__ double fsqrt(double x) { return sqrt(x); }
__host__ __device__ __forceinline__ float ffloor(float x) { return floorf(x); }
__host__ __device__ __forceinline__ double ffloor(double x) { return floor(x); }
__device__ __forceinline__ float frint(float x) { return rintf(x); }
__device__ __forceinline__ double frint(double x) { return rint(x); }

// ---------------------------------------------------------------------------------------------
// mbarrier + 1-D bulk async copy (TMA engine; SASS: UBLKCP / SYNCS)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// generic-proxy accesses (incl. an acquire of data a peer GPU stored) before async-proxy (TMA) accesses, all state spaces
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a transaction-count mismatch would otherwise hang the SM forever; after ~2 s trap so the
// host sees a launch failure instead of a wedged GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > 4000000000LL) {
            printf("mollyb200: mbarrier wait timed out (block %d)\n", (int)blockIdx.x);
            __trap();
        }
    }
}
// slow path of a wait whose first try failed (kept out of line: the hot loops only carry the try)
__device__ __noinline__ void mbar_wait_slow(uint64_t* bar, uint32_t parity) { mbar_wait(bar, parity); }
// global -> shared bulk copy; src/dst 16-byte aligned, bytes a multiple of 16
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// position record (x, y, z, q) at a 32-bit shared-memory address: explicit ld.shared, so the address is a plain
// register + uniform base instead of a generic pointer that is converted at every use
__device__ __forceinline__ float4 lds_pos(uint32_t addr, float) {
    float4 r;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "r"(addr));
    return r;
}
__device__ __forceinline__ dbl4 lds_pos(uint32_t addr, double) {
    dbl4 r;
    asm volatile("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(r.x), "=d"(r.y) : "r"(addr));
    asm volatile("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(r.z), "=d"(r.w) : "r"(addr + 16u));
    return r;
}

// LJ parameter pair (sigma part, eps part) at a 32-bit shared-memory address
__device__ __forceinline__ float2 lds_pair(uint32_t addr, float) {
    float2 r;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(r.x), "=f"(r.y) : "r"(addr));
    return r;
}
__device__ __forceinline__ dbl2 lds_pair(uint32_t addr, double) {
    dbl2 r;
    asm volatile("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(r.x), "=d"(r.y) : "r"(addr));
    return r;
}

// streaming (read-once) global loads that do not pollute L1
__device__ __forceinline__ uint2 ldg_stream_u2(const uint2* p) {
    uint2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0, %1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}

// warp helpers
template <typename T>
__device__ __forceinline__ T shfl_xor(T v, int m) {
    return __shfl_xor_sync(0xffffffffu, v, m);
}

// ---------------------------------------------------------------------------------------------
// Deterministic CTA sums of doubles (energies, virials, momenta, kinetic sums): the same inputs give the same bits on
// every run, whatever order the warps finish in.
// ---------------------------------------------------------------------------------------------
// v[0..W) of every thread summed over the CTA, each component on its own: an xor butterfly within each warp (offsets 16, 8,
// 4, 2, 1), then the warp sums added to 0 in warp-index order. NT = blockDim.x. The result is valid in thread 0 only. The
// scratch is NT/32 x W doubles, one array per (NT, W) and kernel; a second call with the same (NT, W) reuses it, so a
// barrier must lie between thread 0's read of the first result and the second call.
constexpr int SUM_THREADS = 256;  // block size of the kernels that do nothing but such a sum (velocity sums, single-CTA sums of partials)
template <int NT, int W>
__device__ __forceinline__ void block_sum(double (&v)[W]) {
    static_assert(NT % 32 == 0 && NT <= 1024, "NT: whole warps of one CTA");
    __shared__ double s_red[NT / 32][W];
#pragma unroll
    for (int k = 0; k < W; k++)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    if ((threadIdx.x & 31) == 0)
#pragma unroll
        for (int k = 0; k < W; k++) s_red[threadIdx.x >> 5][k] = v[k];
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < W; k++) {
            double s = 0;
            for (int w = 0; w < NT / 32; w++) s += s_red[w][k];
            v[k] = s;
        }
    }
}
template <int NT>
__device__ __forceinline__ double block_sum(double v) {
    double a[1] = {v};
    block_sum<NT, 1>(a);
    return a[0];
}

// True in every thread of the CTA that takes the last of gridDim.x tickets (atomicInc wraps *ticket back to 0 for the next
// launch). It opens with a CTA barrier, so every thread of the CTA has finished its loads and stores before the CTA takes its
// ticket: the last CTA may overwrite what the other CTAs read (v_cm, the step counter, zeta), and the global stores of every
// thread are ordered before thread 0's fence, hence visible to the last CTA, which fences again before it reads them.
__device__ __forceinline__ bool last_cta(unsigned int* ticket) {
    __shared__ bool s_last;
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned int t = atomicInc(ticket, gridDim.x - 1);
        s_last = (t == gridDim.x - 1);
    }
    __syncthreads();
    return s_last;
}

// s = partial[0..n) of width W (W doubles per entry, component k at W i + k) summed per component in index order by one CTA
// of NT threads: thread t adds entries t, t + NT, ... in turn, then block_sum. The result is valid in thread 0 only; block_sum's
// rule on its scratch applies.
template <int NT, int W>
__device__ __forceinline__ void sum_partials(const double* __restrict__ partial, int n, double (&s)[W]) {
#pragma unroll
    for (int k = 0; k < W; k++) s[k] = 0;
    for (int i = threadIdx.x; i < n; i += NT)
#pragma unroll
        for (int k = 0; k < W; k++) s[k] += partial[W * (size_t)i + k];
    block_sum<NT, W>(s);
}

// v[0..W) of every thread summed over the grid, each component on its own and with the same bits on every run: each CTA's
// block_sum goes to partial[W blockIdx.x + k] (W gridDim.x doubles), and the CTA that takes the last ticket adds them in
// index order (sum_partials). Returns true in every thread of that CTA, with the totals in v of thread 0; false elsewhere.
template <int NT, int W>
__device__ __forceinline__ bool grid_sum(double (&v)[W], double* __restrict__ partial, unsigned int* ticket) {
    block_sum<NT, W>(v);
    if (threadIdx.x == 0)
#pragma unroll
        for (int k = 0; k < W; k++) partial[W * (size_t)blockIdx.x + k] = v[k];
    if (!last_cta(ticket)) return false;
    __threadfence();
    sum_partials<NT, W>(partial, gridDim.x, v);  // (last_cta's barriers lie between block_sum's two uses of its scratch)
    return true;
}

// ---------------------------------------------------------------------------------------------
// Philox4x32-10 counter RNG (public algorithm; Salmon et al. 2011) for the Andersen thermostat
// (reference: src/kernels.jl:688-721 via PhiloxRNG.jl — statistical parity only, SURVEY §8c).
// ---------------------------------------------------------------------------------------------
__host__ __device__ inline void philox4x32_10(uint32_t c[4], uint32_t k0, uint32_t k1) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
    for (int r = 0; r < 10; r++) {
        uint64_t p0 = (uint64_t)M0 * c[0];
        uint64_t p1 = (uint64_t)M1 * c[2];
        uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0;
        uint32_t hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
        uint32_t n0 = hi1 ^ c[1] ^ k0;
        uint32_t n1 = lo1;
        uint32_t n2 = hi0 ^ c[3] ^ k1;
        uint32_t n3 = lo0;
        c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
        k0 += W0;
        k1 += W1;
    }
}
// Three N(0, sd^2) draws from one Philox block d by Box-Muller: (sd r1 cos 2 pi u2, sd r1 sin 2 pi u2, sd r2 cos 2 pi u4) with
// r1, r2 = sqrt(-2 log u1), sqrt(-2 log u3), u1, u3 = (d[0] + 1) / 2^32, (d[2] + 1) / 2^32 in (0, 1] (log stays finite) and
// u2, u4 = d[1] / 2^32, d[3] / 2^32 in [0, 1). The Langevin integrator's O step, the Andersen thermostat's resampling and
// random_velocities.
__host__ __device__ __forceinline__ void box_muller3(const uint32_t d[4], double sd, double out[3]) {
    const double two_pi = 6.283185307179586;
    const double u1 = ((double)d[0] + 1.0) * (1.0 / 4294967296.0), u2 = (double)d[1] * (1.0 / 4294967296.0);
    const double u3 = ((double)d[2] + 1.0) * (1.0 / 4294967296.0), u4 = (double)d[3] * (1.0 / 4294967296.0);
    const double r1 = sqrt(-2.0 * log(u1)), r2 = sqrt(-2.0 * log(u3));
    out[0] = sd * r1 * cos(two_pi * u2);
    out[1] = sd * r1 * sin(two_pi * u2);
    out[2] = sd * r2 * cos(two_pi * u4);
}

}  // namespace mb
