// vrescale.cuh — the velocity-rescaling thermostats (ImmediateThermostat, BerendsenThermostat, VelocityRescaleThermostat;
// src/coupling.jl:82-168, :227-238): the scale factor lambda from the kinetic energy, and the device draws of Bussi's R and S.
// Everything here is __host__ __device__ so that tests/host/thermostat_host.cu can check it against a numpy restatement.
#pragma once
#include "common.cuh"

#include <cfloat>

namespace mb {

enum { VC_NONE = 0, VC_IMMEDIATE = 1, VC_BERENDSEN = 2, VC_VRESCALE = 3 };  // = MB_VC_* of include/mollyb200.h

// one call's coupling, as K2 reads it
struct VCouple {
    int kind;            // VC_*
    int n_steps;         // VC_VRESCALE: couple on steps with step % n_steps == 0
    long long nf;        // degrees of freedom, 3N - 3
    double kT;           // k T0 (kJ/mol)
    double dt, tau;      // time step and coupling constant (ps)
    double total_mass;   // sum m (CM correction of the kinetic energy)
};

// Bussi's draws come from Philox4x32-10 blocks with counter (0xFFFFFFFF - j, step, ctr1_lo, ctr1_hi), key (key_lo, key_hi):
// j = 0 gives R (and the uniform of the shape < 1 boost), j = 1, 2, ... the Marsaglia-Tsang proposals of S. The Andersen
// thermostat uses first words 1..2n (n <= 2e9 atoms), so the two never share a block.
constexpr int VR_MAX_PROPOSALS = 64;  // rejection probability per proposal < 0.05: 64 rejections in a row never happen
__host__ __device__ inline void vrescale_block(uint32_t w[4], uint32_t j, uint32_t step_lo, const uint32_t rng[4]) {
    w[0] = 0xFFFFFFFFu - j; w[1] = step_lo; w[2] = rng[0]; w[3] = rng[1];
    philox4x32_10(w, rng[2], rng[3]);
}
// N(0, 1) from two words by Box-Muller (the transform the Andersen thermostat uses)
__host__ __device__ inline double vrescale_normal(uint32_t a, uint32_t b) {
    const double u1 = ((double)a + 1.0) * (1.0 / 4294967296.0), u2 = (double)b * (1.0 / 4294967296.0);
    return sqrt(-2.0 * log(u1)) * cos(6.283185307179586 * u2);
}
// chi^2 with k degrees of freedom = 2 Gamma(k/2): Marsaglia-Tsang (2000); for shape k/2 < 1 the draw of shape k/2 + 1 is
// multiplied by U^(2/k). k <= 0: 0.
__host__ __device__ inline double vrescale_chi2(long long k, uint32_t step_lo, const uint32_t rng[4]) {
    if (k <= 0) return 0.0;
    const double a = 0.5 * (double)k;
    const bool boost = a < 1.0;
    const double d = (boost ? a + 1.0 : a) - 1.0 / 3.0, c = 1.0 / sqrt(9.0 * d);
    double g = d;  // (mean of the proposal: only reached after VR_MAX_PROPOSALS rejections)
    uint32_t w[4];
    for (int j = 1; j <= VR_MAX_PROPOSALS; j++) {
        vrescale_block(w, (uint32_t)j, step_lo, rng);
        const double x = vrescale_normal(w[0], w[1]);
        const double t = 1.0 + c * x;
        if (t <= 0.0) continue;
        const double v = t * t * t;
        const double u = ((double)w[2] + 1.0) * (1.0 / 4294967296.0);
        if (log(u) < 0.5 * x * x + d - d * v + d * log(v)) {
            g = d * v;
            break;
        }
    }
    if (boost) {
        vrescale_block(w, 0u, step_lo, rng);
        g *= pow(((double)w[2] + 1.0) * (1.0 / 4294967296.0), 1.0 / a);
    }
    return 2.0 * g;
}

// lambda for kinetic energy K (after the step's CM removal) at step `step`; rng = (ctr1_lo, ctr1_hi, key_lo, key_hi).
// K <= 0 or nf <= 0 leaves the velocities as they are (lambda = 1).
__host__ __device__ inline double vcouple_lambda(const VCouple& p, double K, long long step, const uint32_t rng[4]) {
    if (!(K > 0.0) || p.nf <= 0) return 1.0;
    const double nf = (double)p.nf;
    if (p.kind == VC_IMMEDIATE) return sqrt(p.kT / (2.0 * K / nf));                              // sqrt(T0 / T)
    if (p.kind == VC_BERENDSEN) return sqrt(1.0 + (p.dt / p.tau) * (p.kT / (2.0 * K / nf) - 1.0));
    if (p.kind != VC_VRESCALE || step % p.n_steps != 0) return 1.0;
    const double c = exp(-(p.dt * p.n_steps) / p.tau);
    const double A = (nf * p.kT / 2.0) / (nf * K);  // Kbar / (Nf K)
    uint32_t w[4];
    vrescale_block(w, 0u, (uint32_t)step, rng);
    const double R = vrescale_normal(w[0], w[1]);
    const double S = vrescale_chi2(p.nf - 1, (uint32_t)step, rng);
    double lam2 = c + (1.0 - c) * A * (R * R + S) + 2.0 * sqrt(c * (1.0 - c) * A) * R;
    lam2 = fmax(lam2, DBL_EPSILON);
    return sqrt(lam2);
}

}  // namespace mb
