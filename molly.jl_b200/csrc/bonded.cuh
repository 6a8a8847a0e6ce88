// bonded.cuh — specific (bonded) interactions on the device: HarmonicBond, HarmonicAngle, PeriodicTorsion.
// SURVEY.md §8(f)-1 / Appendix B.1. One thread per term, forces added to the slot-order force array with atomics
// (the reference's KernelAbstractions kernels do the same, src/kernels.jl:233-342); energies through per-CTA
// partials. Reference formulas: src/interactions/harmonic_bond.jl:13-54, harmonic_angle.jl:45-67,
// periodic_torsion.jl:17-142, dihedral by atan2 (src/spatial.jl:882-894). Displacements are minimum-image.
#pragma once
#include "cells.cuh"

namespace mb {

template <typename T>
struct Vec3 {
    T x, y, z;
};
template <typename T>
__device__ __forceinline__ Vec3<T> v3(T x, T y, T z) { return Vec3<T>{x, y, z}; }
template <typename T>
__device__ __forceinline__ Vec3<T> operator+(Vec3<T> a, Vec3<T> b) { return v3(a.x + b.x, a.y + b.y, a.z + b.z); }
template <typename T>
__device__ __forceinline__ Vec3<T> operator-(Vec3<T> a, Vec3<T> b) { return v3(a.x - b.x, a.y - b.y, a.z - b.z); }
template <typename T>
__device__ __forceinline__ Vec3<T> operator-(Vec3<T> a) { return v3(-a.x, -a.y, -a.z); }
template <typename T>
__device__ __forceinline__ Vec3<T> operator*(T s, Vec3<T> a) { return v3(s * a.x, s * a.y, s * a.z); }
template <typename T>
__device__ __forceinline__ T dot(Vec3<T> a, Vec3<T> b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
template <typename T>
__device__ __forceinline__ Vec3<T> cross(Vec3<T> a, Vec3<T> b) {
    return v3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}

// minimum-image c2 - c1 for positions that may sit in different periodic images
template <typename T>
__device__ __forceinline__ Vec3<T> mic_vec(const typename VT<T>::T4& c1, const typename VT<T>::T4& c2, const T* L, const T* invL) {
    T dx = c2.x - c1.x, dy = c2.y - c1.y, dz = c2.z - c1.z;
    dx -= L[0] * frint(dx * invL[0]);
    dy -= L[1] * frint(dy * invL[1]);
    dz -= L[2] * frint(dz * invL[2]);
    return v3(dx, dy, dz);
}
struct BoxT {
    double L[3];
};
// minimum-image displacement c2 - c1 for the box kind B: BoxT (rectangular) or Tric<T> (TriclinicBoundary's vector,
// src/spatial.jl:528-534)
template <typename T, typename B>
struct Mic;
template <typename T>
struct Mic<T, BoxT> {
    T L[3], invL[3];
    __device__ __forceinline__ explicit Mic(const BoxT& box)
        : L{(T)box.L[0], (T)box.L[1], (T)box.L[2]}, invL{(T)(1.0 / box.L[0]), (T)(1.0 / box.L[1]), (T)(1.0 / box.L[2])} {}
    __device__ __forceinline__ Vec3<T> operator()(const typename VT<T>::T4& c1, const typename VT<T>::T4& c2) const {
        return mic_vec<T>(c1, c2, L, invL);
    }
};
template <typename T>
struct Mic<T, Tric<T>> {
    Tric<T> t;
    __device__ __forceinline__ explicit Mic(const Tric<T>& box) : t(box) {}
    __device__ __forceinline__ Vec3<T> operator()(const typename VT<T>::T4& c1, const typename VT<T>::T4& c2) const {
        T dx = c2.x - c1.x, dy = c2.y - c1.y, dz = c2.z - c1.z;
        tric_vector<T>(t, dx, dy, dz);
        return v3(dx, dy, dz);
    }
};
template <typename T>
__device__ __forceinline__ void add_force(typename VT<T>::T4* f4, int slot, Vec3<T> f) {
    T* p = reinterpret_cast<T*>(&f4[slot]);
    atomicAdd(p, f.x);
    atomicAdd(p + 1, f.y);
    atomicAdd(p + 2, f.z);
}

constexpr int BONDED_THREADS = 128;

// slot_of: original atom index -> slot (inv_orig), or nullptr when positions are in original order
template <typename T, bool ENERGY, typename B>
__device__ __forceinline__ double bond_term(int t, int n, const int* __restrict__ idx, const T* __restrict__ par,
                                            const int* __restrict__ slot_of, const typename VT<T>::T4* __restrict__ pos4,
                                            typename VT<T>::T4* __restrict__ f4, const B& box) {
    double e = 0;
    if (t < n) {
        const Mic<T, B> mic(box);
        int i = idx[2 * t], j = idx[2 * t + 1];
        if (slot_of) { i = slot_of[i]; j = slot_of[j]; }
        const T k = par[2 * t], r0 = par[2 * t + 1];
        Vec3<T> ab = mic(pos4[i], pos4[j]);
        const T r = fsqrt(dot(ab, ab));
        const T c = k * (r - r0);
        Vec3<T> fi = (c / r) * ab;  // f_i = +c ab/|ab|, f_j = -f_i (harmonic_bond.jl:25-33)
        add_force<T>(f4, i, fi);
        add_force<T>(f4, j, -fi);
        if (ENERGY) e = 0.5 * (double)k * (double)(r - r0) * (double)(r - r0);
    }
    return e;
}

template <typename T, bool ENERGY, typename B>
__device__ __forceinline__ double angle_term(int t, int n, const int* __restrict__ idx, const T* __restrict__ par,
                                             const int* __restrict__ slot_of, const typename VT<T>::T4* __restrict__ pos4,
                                             typename VT<T>::T4* __restrict__ f4, const B& box) {
    double e = 0;
    if (t < n) {
        const Mic<T, B> mic(box);
        int i = idx[3 * t], j = idx[3 * t + 1], kk = idx[3 * t + 2];
        if (slot_of) { i = slot_of[i]; j = slot_of[j]; kk = slot_of[kk]; }
        const T k = par[2 * t], th0 = par[2 * t + 1];
        Vec3<T> ba = mic(pos4[j], pos4[i]);
        Vec3<T> bc = mic(pos4[j], pos4[kk]);
        Vec3<T> nrm = cross(ba, bc);
        const T n2 = dot(nrm, nrm);
        if (n2 > (T)0) {
            const T nba = fsqrt(dot(ba, ba)), nbc = fsqrt(dot(bc, bc));
            T cs = dot(ba, bc) / (nba * nbc);
            cs = fmin(fmax(cs, (T)-1), (T)1);
            const T th = acos(cs);
            Vec3<T> pa = cross(ba, nrm), pc = cross(-bc, nrm);
            pa = ((T)1 / fsqrt(dot(pa, pa))) * pa;
            pc = ((T)1 / fsqrt(dot(pc, pc))) * pc;
            const T tq = -k * (th - th0);
            Vec3<T> fa = (tq / nba) * pa, fc = (tq / nbc) * pc;
            add_force<T>(f4, i, fa);
            add_force<T>(f4, kk, fc);
            add_force<T>(f4, j, -(fa + fc));
            if (ENERGY) e = 0.5 * (double)k * (double)(th - th0) * (double)(th - th0);
        }
    }
    return e;
}

// one (periodicity, phase, k) term per entry; a torsion with several terms appears several times
template <typename T, bool ENERGY, typename B>
__device__ __forceinline__ double torsion_term(int t, int n, const int* __restrict__ idx, const T* __restrict__ par,
                                               const int* __restrict__ slot_of, const typename VT<T>::T4* __restrict__ pos4,
                                               typename VT<T>::T4* __restrict__ f4, const B& box) {
    double e = 0;
    if (t < n) {
        const Mic<T, B> mic(box);
        int i = idx[4 * t], j = idx[4 * t + 1], k = idx[4 * t + 2], l = idx[4 * t + 3];
        if (slot_of) { i = slot_of[i]; j = slot_of[j]; k = slot_of[k]; l = slot_of[l]; }
        const T per = par[3 * t], phase = par[3 * t + 1], kk = par[3 * t + 2];
        Vec3<T> ab = mic(pos4[i], pos4[j]);
        Vec3<T> bc = mic(pos4[j], pos4[k]);
        Vec3<T> cd = mic(pos4[k], pos4[l]);
        Vec3<T> m = cross(ab, bc), nn = cross(bc, cd);
        const T nbc = fsqrt(dot(bc, bc));
        const T th = atan2(dot(cross(m, nn), bc) / nbc, dot(m, nn));
        const T ang = per * th - phase;
        const T dedth = -kk * per * sin(ang);
        const T m2 = dot(m, m), n2 = dot(nn, nn);
        if (m2 > (T)0 && n2 > (T)0) {
            Vec3<T> fi = (dedth * nbc / m2) * m;
            Vec3<T> fl = (-dedth * nbc / n2) * nn;
            const T inv_bc2 = (T)1 / (nbc * nbc);
            Vec3<T> v = ((-dot(ab, bc)) * inv_bc2) * fi - ((-dot(cd, bc)) * inv_bc2) * fl;
            add_force<T>(f4, i, fi);
            add_force<T>(f4, j, v - fi);
            add_force<T>(f4, k, -v - fl);
            add_force<T>(f4, l, fl);
            if (ENERGY) e = (double)kk * (1.0 + cos((double)ang));
        }
    }
    return e;
}

// All specific interactions in one launch: CTAs [0, nb0) bonds, [nb0, nb0+nb1) angles, the rest torsions.
struct BondedLists {
    int n[3];
    int nblk[3];
    const int* idx[3];
    const void* par[3];
};
template <typename T, bool ENERGY, typename B>
__global__ void __launch_bounds__(BONDED_THREADS)
    bonded_kernel(BondedLists L, const int* __restrict__ slot_of, const typename VT<T>::T4* __restrict__ pos4,
                  typename VT<T>::T4* __restrict__ f4, B box, double* __restrict__ partial) {
    int blk = blockIdx.x;
    double e = 0;
    if (blk < L.nblk[0]) {
        e = bond_term<T, ENERGY, B>(blk * BONDED_THREADS + threadIdx.x, L.n[0], L.idx[0], static_cast<const T*>(L.par[0]), slot_of, pos4, f4, box);
    } else if (blk < L.nblk[0] + L.nblk[1]) {
        blk -= L.nblk[0];
        e = angle_term<T, ENERGY, B>(blk * BONDED_THREADS + threadIdx.x, L.n[1], L.idx[1], static_cast<const T*>(L.par[1]), slot_of, pos4, f4, box);
    } else {
        blk -= L.nblk[0] + L.nblk[1];
        e = torsion_term<T, ENERGY, B>(blk * BONDED_THREADS + threadIdx.x, L.n[2], L.idx[2], static_cast<const T*>(L.par[2]), slot_of, pos4, f4, box);
    }
    if (ENERGY) {
        e = block_sum<BONDED_THREADS>(e);
        if (threadIdx.x == 0) partial[blockIdx.x] = e;
    }
}

// pe_partial[0..n) summed in index order -> *acc += sum (one CTA of SUM_THREADS)
__global__ void sum_partials_kernel(int n, const double* __restrict__ partial, double* acc) {
    double v[1];
    sum_partials<SUM_THREADS, 1>(partial, n, v);
    if (threadIdx.x == 0) *acc += v[0];
}

template <typename T>
__global__ void add_double_kernel(const double* src, T* dst) { *dst += (T)(*src); }
// general interactions that are plain scalars (LJDispersionCorrection): pe += e; virial diagonal += w (column-major 3x3)
template <typename T>
__global__ void add_scalars_kernel(T* pe, T e, T* vir, T w) {
    if (pe) *pe += e;
    if (vir) { vir[0] += w; vir[4] += w; vir[8] += w; }
}

}  // namespace mb
