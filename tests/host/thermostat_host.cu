// Test harness (NOT product code): the __host__ __device__ draw and lambda functions of csrc/vrescale.cuh compiled for the
// HOST, so that tests/test_thermostats_host.py can check them against tests/thermostat_oracle.py without a GPU.
// rng = (ctr1_lo, ctr1_hi, key_lo, key_hi), as the device reads them from the control block.
#include "../../molly.jl_b200/csrc/vrescale.cuh"

using namespace mb;

extern "C" {
void thh_block(uint32_t j, uint32_t step, const uint32_t* rng, uint32_t* out4) { vrescale_block(out4, j, step, rng); }
double thh_normal(uint32_t a, uint32_t b) { return vrescale_normal(a, b); }
// chi^2_k draws at steps step0, step0 + 1, ..., step0 + count - 1
void thh_chi2(long long k, long long count, uint32_t step0, const uint32_t* rng, double* out) {
    for (long long i = 0; i < count; i++) out[i] = vrescale_chi2(k, step0 + (uint32_t)i, rng);
}
// lambda at steps step0 .. step0 + count - 1 for the same K
void thh_lambda(int kind, int n_steps, long long nf, double kT, double dt, double tau, double K, long long step0, long long count,
                const uint32_t* rng, double* out) {
    const VCouple p{kind, n_steps, nf, kT, dt, tau, 0.0};
    for (long long i = 0; i < count; i++) out[i] = vcouple_lambda(p, K, step0 + i, rng);
}
}
