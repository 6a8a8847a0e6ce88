// bonded.cuh — specific (bonded) interactions on the device: the ten kinds of SPECIFIC_ATOMS / SPECIFIC_PARAMS below.
// SURVEY.md §8(f)-1 / Appendix B.1. One thread per term, forces added to the slot-order force array with atomics
// (the reference's KernelAbstractions kernels do the same, src/kernels.jl:233-342); energies through per-CTA
// partials. Reference formulas: src/interactions/harmonic_bond.jl:13-54, harmonic_angle.jl:45-67,
// periodic_torsion.jl:17-142, dihedral by atan2 (src/spatial.jl:882-894), and the files named at each term below.
// Displacements are minimum-image.
#pragma once
#include "../../include/mollyb200.h"
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

// The one table of specific interaction kinds (index = MB_SPECIFIC_*): atoms per term and parameters per term. The engine
// sizes its per-kind arrays from it.
constexpr int N_SPECIFIC_KINDS = MB_SPECIFIC_N_KINDS;
constexpr int SPECIFIC_ATOMS[N_SPECIFIC_KINDS] = {2, 3, 4, 1, 2, 2, 3, 3, 4, 4};
constexpr int SPECIFIC_PARAMS[N_SPECIFIC_KINDS] = {2, 2, 3, 4, 3, 4, 2, 4, 2, 4};
static_assert(MB_SPECIFIC_HARMONIC_BOND == 0 && MB_SPECIFIC_HARMONIC_ANGLE == 1 && MB_SPECIFIC_PERIODIC_TORSION == 2 &&
                  MB_SPECIFIC_POSITION_RESTRAINT == 3 && MB_SPECIFIC_MORSE_BOND == 4 && MB_SPECIFIC_FENE_BOND == 5 &&
                  MB_SPECIFIC_COSINE_ANGLE == 6 && MB_SPECIFIC_UREY_BRADLEY == 7 && MB_SPECIFIC_HARMONIC_TORSION == 8 &&
                  MB_SPECIFIC_RB_TORSION == 9 && MB_SPECIFIC_N_KINDS == 10,
              "SPECIFIC_ATOMS / SPECIFIC_PARAMS and bonded_kernel's switch follow the MB_SPECIFIC_* numbering");

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
        const T th = atan2(fsqrt(n2), dot(ba, bc));  // the angle of bond_angle, without acos's loss near 0 and pi
        if (n2 > (T)0) {
            const T nba = fsqrt(dot(ba, ba)), nbc = fsqrt(dot(bc, bc));
            Vec3<T> pa = cross(ba, nrm), pc = cross(-bc, nrm);
            pa = ((T)1 / fsqrt(dot(pa, pa))) * pa;
            pc = ((T)1 / fsqrt(dot(pc, pc))) * pc;
            const T tq = -k * (th - th0);
            Vec3<T> fa = (tq / nba) * pa, fc = (tq / nbc) * pc;
            add_force<T>(f4, i, fa);
            add_force<T>(f4, kk, fc);
            add_force<T>(f4, j, -(fa + fc));
        }
        if (ENERGY) e = 0.5 * (double)k * (double)(th - th0) * (double)(th - th0);  // collinear too (harmonic_angle.jl:64-67)
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
        }
        if (ENERGY) e = (double)kk * (1.0 + cos((double)ang));  // collinear too (periodic_torsion.jl:131-141)
    }
    return e;
}

// HarmonicPositionRestraint (harmonic_position_restraint.jl:18-32): params k, x0, y0, z0. The displacement x0 - x_i is
// minimum-image; the force k (x0 - x_i) is exactly zero at x0.
template <typename T, bool ENERGY, typename B>
__device__ __forceinline__ double restraint_term(int t, int n, const int* __restrict__ idx, const T* __restrict__ par,
                                                 const int* __restrict__ slot_of, const typename VT<T>::T4* __restrict__ pos4,
                                                 typename VT<T>::T4* __restrict__ f4, const B& box) {
    double e = 0;
    if (t < n) {
        const Mic<T, B> mic(box);
        int i = idx[t];
        if (slot_of) i = slot_of[i];
        const T k = par[4 * t];
        Vec3<T> d = mic(pos4[i], make4<T>(par[4 * t + 1], par[4 * t + 2], par[4 * t + 3], (T)0));
        add_force<T>(f4, i, k * d);
        if (ENERGY) e = 0.5 * (double)k * (double)dot(d, d);
    }
    return e;
}

// MorseBond (morse_bond.jl:24-38): params D, a, r0
template <typename T, bool ENERGY, typename B>
__device__ __forceinline__ double morse_term(int t, int n, const int* __restrict__ idx, const T* __restrict__ par,
                                             const int* __restrict__ slot_of, const typename VT<T>::T4* __restrict__ pos4,
                                             typename VT<T>::T4* __restrict__ f4, const B& box) {
    double e = 0;
    if (t < n) {
        const Mic<T, B> mic(box);
        int i = idx[2 * t], j = idx[2 * t + 1];
        if (slot_of) { i = slot_of[i]; j = slot_of[j]; }
        const T D = par[3 * t], a = par[3 * t + 1], r0 = par[3 * t + 2];
        Vec3<T> dr = mic(pos4[i], pos4[j]);
        const T r = fsqrt(dot(dr, dr));
        const T ralp = exp(-a * (r - r0));
        const T c = (T)2 * D * a * ((T)1 - ralp) * ralp;
        Vec3<T> fi = (c / r) * dr;
        add_force<T>(f4, i, fi);
        add_force<T>(f4, j, -fi);
        if (ENERGY) e = (double)D * (1.0 - (double)ralp) * (1.0 - (double)ralp);
    }
    return e;
}

// FENEBond (fene_bond.jl:31-64): params k, r0, sigma, eps. The WCA part acts for r < 2^(1/6) sigma; r >= r0 is not
// clamped (NaN / Inf, as in the reference).
template <typename T, bool ENERGY, typename B>
__device__ __forceinline__ double fene_term(int t, int n, const int* __restrict__ idx, const T* __restrict__ par,
                                            const int* __restrict__ slot_of, const typename VT<T>::T4* __restrict__ pos4,
                                            typename VT<T>::T4* __restrict__ f4, const B& box) {
    double e = 0;
    if (t < n) {
        const Mic<T, B> mic(box);
        int i = idx[2 * t], j = idx[2 * t + 1];
        if (slot_of) { i = slot_of[i]; j = slot_of[j]; }
        const T k = par[4 * t], r0 = par[4 * t + 1], sig = par[4 * t + 2], eps = par[4 * t + 3];
        Vec3<T> dr = mic(pos4[i], pos4[j]);
        const T r2 = dot(dr, dr);
        const T r2inv = (T)1 / r2;
        const T s2 = sig * sig;
        const T sr6 = s2 * s2 * s2 * r2inv * r2inv * r2inv;
        const bool wca = fsqrt(r2) < sig * (T)1.122462048309373;  // 2^(1/6)
        const T fwca = wca ? (T)24 * eps * r2inv * ((T)2 * sr6 * sr6 - sr6) : (T)0;
        const T q = (T)1 - r2 / (r0 * r0);
        Vec3<T> fj = (fwca - k / q) * dr;
        add_force<T>(f4, i, -fj);
        add_force<T>(f4, j, fj);
        if (ENERGY) {
            e = -0.5 * (double)k * (double)r0 * (double)r0 * log((double)q);
            if (wca) e += 4.0 * (double)eps * ((double)sr6 * (double)sr6 - (double)sr6) + (double)eps;
        }
    }
    return e;
}

// bend geometry of atoms i-j-k (j in the middle): ba = x_i - x_j, bc = x_k - x_j, theta = atan2(|ba x bc|, ba . bc), the
// angle of bond_angle (src/spatial.jl:845-853) to a few rounding units at every angle, where acos of the cosine loses
// digits near 0 and pi; exactly collinear atoms give exactly 0 or pi. pa, pc the unit in-plane directions that open the
// angle, set only when not collinear
template <typename T>
struct Bend {
    Vec3<T> ba, bc, pa, pc;
    T nba, nbc, th;
    bool bent;
};
template <typename T, typename B>
__device__ __forceinline__ Bend<T> bend(const Mic<T, B>& mic, const typename VT<T>::T4& xi, const typename VT<T>::T4& xj,
                                        const typename VT<T>::T4& xk) {
    Bend<T> g;
    g.ba = mic(xj, xi);
    g.bc = mic(xj, xk);
    g.nba = fsqrt(dot(g.ba, g.ba));
    g.nbc = fsqrt(dot(g.bc, g.bc));
    Vec3<T> nrm = cross(g.ba, g.bc);
    const T n2 = dot(nrm, nrm);
    g.th = atan2(fsqrt(n2), dot(g.ba, g.bc));
    g.bent = n2 > (T)0;
    if (g.bent) {
        g.pa = cross(g.ba, nrm);
        g.pc = cross(-g.bc, nrm);
        g.pa = ((T)1 / fsqrt(dot(g.pa, g.pa))) * g.pa;
        g.pc = ((T)1 / fsqrt(dot(g.pc, g.pc))) * g.pc;
    }
    return g;
}
// the forces of the torque tq = -dE/dtheta on a bent angle i-j-k
template <typename T>
__device__ __forceinline__ void bend_forces(const Bend<T>& g, T tq, typename VT<T>::T4* f4, int i, int j, int k,
                                            Vec3<T> extra_i = Vec3<T>{0, 0, 0}) {
    Vec3<T> fa = (tq / g.nba) * g.pa, fc = (tq / g.nbc) * g.pc;
    add_force<T>(f4, i, fa + extra_i);
    add_force<T>(f4, k, fc - extra_i);
    add_force<T>(f4, j, -(fa + fc));
}

// CosineAngle (cosine_angle.jl:19-42): params k, theta0; E = k (1 + cos(theta - theta0)), no force when collinear
template <typename T, bool ENERGY, typename B>
__device__ __forceinline__ double cosine_angle_term(int t, int n, const int* __restrict__ idx, const T* __restrict__ par,
                                                    const int* __restrict__ slot_of, const typename VT<T>::T4* __restrict__ pos4,
                                                    typename VT<T>::T4* __restrict__ f4, const B& box) {
    double e = 0;
    if (t < n) {
        const Mic<T, B> mic(box);
        int i = idx[3 * t], j = idx[3 * t + 1], kk = idx[3 * t + 2];
        if (slot_of) { i = slot_of[i]; j = slot_of[j]; kk = slot_of[kk]; }
        const T k = par[2 * t], th0 = par[2 * t + 1];
        const Bend<T> g = bend<T, B>(mic, pos4[i], pos4[j], pos4[kk]);
        if (g.bent) bend_forces<T>(g, k * sin(g.th - th0), f4, i, j, kk);
        if (ENERGY) e = (double)k * (1.0 + cos((double)g.th - (double)th0));
    }
    return e;
}

// UreyBradley (urey_bradley.jl:32-61): params kangle, theta0, kbond, r0. The harmonic angle is zeroed when collinear; the
// harmonic 1-3 bond between i and k always acts.
template <typename T, bool ENERGY, typename B>
__device__ __forceinline__ double urey_bradley_term(int t, int n, const int* __restrict__ idx, const T* __restrict__ par,
                                                    const int* __restrict__ slot_of, const typename VT<T>::T4* __restrict__ pos4,
                                                    typename VT<T>::T4* __restrict__ f4, const B& box) {
    double e = 0;
    if (t < n) {
        const Mic<T, B> mic(box);
        int i = idx[3 * t], j = idx[3 * t + 1], kk = idx[3 * t + 2];
        if (slot_of) { i = slot_of[i]; j = slot_of[j]; kk = slot_of[kk]; }
        const T ka = par[4 * t], th0 = par[4 * t + 1], kb = par[4 * t + 2], r0 = par[4 * t + 3];
        const Bend<T> g = bend<T, B>(mic, pos4[i], pos4[j], pos4[kk]);
        Vec3<T> ik = mic(pos4[i], pos4[kk]);
        const T rik = fsqrt(dot(ik, ik));
        Vec3<T> fb = (kb * (rik - r0) / rik) * ik;
        if (g.bent) {
            bend_forces<T>(g, -ka * (g.th - th0), f4, i, j, kk, fb);
        } else {
            add_force<T>(f4, i, fb);
            add_force<T>(f4, kk, -fb);
        }
        if (ENERGY)
            e = 0.5 * (double)ka * ((double)g.th - (double)th0) * ((double)g.th - (double)th0) +
                0.5 * (double)kb * ((double)rik - (double)r0) * ((double)rik - (double)r0);
    }
    return e;
}

// dihedral geometry of i-j-k-l (torsion_vectors, src/spatial.jl:882-894) and the forces of dE/dtheta, as torsion_term
template <typename T>
struct Dihedral {
    Vec3<T> ab, bc, cd, m, nn;
    T nbc, th;
};
template <typename T, typename B>
__device__ __forceinline__ Dihedral<T> dihedral(const Mic<T, B>& mic, const typename VT<T>::T4& xi, const typename VT<T>::T4& xj,
                                                const typename VT<T>::T4& xk, const typename VT<T>::T4& xl) {
    Dihedral<T> g;
    g.ab = mic(xi, xj);
    g.bc = mic(xj, xk);
    g.cd = mic(xk, xl);
    g.m = cross(g.ab, g.bc);
    g.nn = cross(g.bc, g.cd);
    g.nbc = fsqrt(dot(g.bc, g.bc));
    g.th = atan2(dot(cross(g.m, g.nn), g.bc) / g.nbc, dot(g.m, g.nn));
    return g;
}
template <typename T>
__device__ __forceinline__ void dihedral_forces(const Dihedral<T>& g, T dedth, typename VT<T>::T4* f4, int i, int j, int k, int l) {
    const T m2 = dot(g.m, g.m), n2 = dot(g.nn, g.nn);
    if (m2 > (T)0 && n2 > (T)0) {
        Vec3<T> fi = (dedth * g.nbc / m2) * g.m;
        Vec3<T> fl = (-dedth * g.nbc / n2) * g.nn;
        const T inv_bc2 = (T)1 / (g.nbc * g.nbc);
        Vec3<T> v = ((-dot(g.ab, g.bc)) * inv_bc2) * fi - ((-dot(g.cd, g.bc)) * inv_bc2) * fl;
        add_force<T>(f4, i, fi);
        add_force<T>(f4, j, v - fi);
        add_force<T>(f4, k, -v - fl);
        add_force<T>(f4, l, fl);
    }
}

// HarmonicTorsion (harmonic_torsion.jl:27-44): params k, theta0; E = k (theta - theta0)^2 with theta - theta0 not
// wrapped, as in the reference
template <typename T, bool ENERGY, typename B>
__device__ __forceinline__ double harmonic_torsion_term(int t, int n, const int* __restrict__ idx, const T* __restrict__ par,
                                                        const int* __restrict__ slot_of, const typename VT<T>::T4* __restrict__ pos4,
                                                        typename VT<T>::T4* __restrict__ f4, const B& box) {
    double e = 0;
    if (t < n) {
        const Mic<T, B> mic(box);
        int i = idx[4 * t], j = idx[4 * t + 1], k = idx[4 * t + 2], l = idx[4 * t + 3];
        if (slot_of) { i = slot_of[i]; j = slot_of[j]; k = slot_of[k]; l = slot_of[l]; }
        const T kk = par[2 * t], th0 = par[2 * t + 1];
        const Dihedral<T> g = dihedral<T, B>(mic, pos4[i], pos4[j], pos4[k], pos4[l]);
        dihedral_forces<T>(g, (T)2 * kk * (g.th - th0), f4, i, j, k, l);
        if (ENERGY) e = (double)kk * ((double)g.th - (double)th0) * ((double)g.th - (double)th0);
    }
    return e;
}

// RBTorsion (rb_torsion.jl:19-43): params f1..f4; E = (f1 (1 + cos th) + f2 (1 - cos 2th) + f3 (1 + cos 3th) + f4) / 2.
// The force is -grad E, so dE/dtheta = (-f1 sin th + 2 f2 sin 2th - 3 f3 sin 3th) / 2; rb_torsion.jl:30 has the opposite
// sign (include/mollyb200.h, MB_SPECIFIC_RB_TORSION).
template <typename T, bool ENERGY, typename B>
__device__ __forceinline__ double rb_torsion_term(int t, int n, const int* __restrict__ idx, const T* __restrict__ par,
                                                  const int* __restrict__ slot_of, const typename VT<T>::T4* __restrict__ pos4,
                                                  typename VT<T>::T4* __restrict__ f4, const B& box) {
    double e = 0;
    if (t < n) {
        const Mic<T, B> mic(box);
        int i = idx[4 * t], j = idx[4 * t + 1], k = idx[4 * t + 2], l = idx[4 * t + 3];
        if (slot_of) { i = slot_of[i]; j = slot_of[j]; k = slot_of[k]; l = slot_of[l]; }
        const T f1 = par[4 * t], f2 = par[4 * t + 1], f3 = par[4 * t + 2], f4c = par[4 * t + 3];
        const Dihedral<T> g = dihedral<T, B>(mic, pos4[i], pos4[j], pos4[k], pos4[l]);
        const T dedth = (-f1 * sin(g.th) + (T)2 * f2 * sin((T)2 * g.th) - (T)3 * f3 * sin((T)3 * g.th)) / (T)2;
        dihedral_forces<T>(g, dedth, f4, i, j, k, l);
        if (ENERGY) {
            const double th = g.th;
            e = 0.5 * ((double)f1 * (1.0 + cos(th)) + (double)f2 * (1.0 - cos(2.0 * th)) + (double)f3 * (1.0 + cos(3.0 * th)) + (double)f4c);
        }
    }
    return e;
}

// All specific interactions in one launch. The CTAs of kind k are [blk0[k], blk0[k + 1]); every CTA holds terms of one
// kind only, so the kind is uniform within it.
struct BondedLists {
    int n[N_SPECIFIC_KINDS];
    int blk0[N_SPECIFIC_KINDS + 1];
    const int* idx[N_SPECIFIC_KINDS];
    const void* par[N_SPECIFIC_KINDS];
};
template <typename T, bool ENERGY, typename B>
__global__ void __launch_bounds__(BONDED_THREADS)
    bonded_kernel(BondedLists L, const int* __restrict__ slot_of, const typename VT<T>::T4* __restrict__ pos4,
                  typename VT<T>::T4* __restrict__ f4, B box, double* __restrict__ partial) {
    int kind = 0;
    while ((int)blockIdx.x >= L.blk0[kind + 1]) kind++;
    const int t = ((int)blockIdx.x - L.blk0[kind]) * BONDED_THREADS + threadIdx.x;
    double e = 0;
#define MB_BONDED_CASE(K, FN) \
    case K: e = FN<T, ENERGY, B>(t, L.n[K], L.idx[K], static_cast<const T*>(L.par[K]), slot_of, pos4, f4, box); break;
    switch (kind) {
        MB_BONDED_CASE(MB_SPECIFIC_HARMONIC_BOND, bond_term)
        MB_BONDED_CASE(MB_SPECIFIC_HARMONIC_ANGLE, angle_term)
        MB_BONDED_CASE(MB_SPECIFIC_PERIODIC_TORSION, torsion_term)
        MB_BONDED_CASE(MB_SPECIFIC_POSITION_RESTRAINT, restraint_term)
        MB_BONDED_CASE(MB_SPECIFIC_MORSE_BOND, morse_term)
        MB_BONDED_CASE(MB_SPECIFIC_FENE_BOND, fene_term)
        MB_BONDED_CASE(MB_SPECIFIC_COSINE_ANGLE, cosine_angle_term)
        MB_BONDED_CASE(MB_SPECIFIC_UREY_BRADLEY, urey_bradley_term)
        MB_BONDED_CASE(MB_SPECIFIC_HARMONIC_TORSION, harmonic_torsion_term)
        MB_BONDED_CASE(MB_SPECIFIC_RB_TORSION, rb_torsion_term)
    }
#undef MB_BONDED_CASE
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
