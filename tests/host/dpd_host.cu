// Test harness (NOT product code): the DPD pair term and pairwise draw (dpd_pair, dpd_normal of csrc/dpd.cuh) compiled for
// the HOST, so that tests/test_dpd_host.py can check them against tests/dpd_oracle.py without a GPU.
#include "../../molly.jl_b200/csrc/dpd.cuh"

using namespace mb;

template <typename T>
static void pair_all(int n, const double* par, unsigned long long key, const double* r, const double* d, const double* dv,
                     const double* xi, T* fr, T* e) {
    DpdArgs<T> P;
    memset(&P, 0, sizeof(P));
    P.a = (T)par[0];
    P.gamma = (T)par[1];
    P.sigma = (T)par[2];
    P.rc = (T)par[3];
    P.inv_sqrt_dt = (T)(1.0 / std::sqrt(par[4]));
    P.e_pre = (T)(par[0] / 2) * (T)par[3];
    P.key_lo = (uint32_t)key;
    P.key_hi = (uint32_t)(key >> 32);
    for (int k = 0; k < n; k++)
        dpd_pair<T>(P, (T)r[k], (T)d[3 * k], (T)d[3 * k + 1], (T)d[3 * k + 2], (T)dv[3 * k], (T)dv[3 * k + 1], (T)dv[3 * k + 2],
                    (T)xi[k], fr[k], e[k]);
}

extern "C" {
// par = (a, gamma, sigma, r_c, dt); r, xi: n values; d, dv: n x 3 (d = c_i - c_j, dv = v_i - v_j); outputs fr, e: n values
void dh_pair_f64(int n, const double* par, const double* r, const double* d, const double* dv, const double* xi, double* fr,
                 double* e) {
    pair_all<double>(n, par, 0, r, d, dv, xi, fr, e);
}
void dh_pair_f32(int n, const double* par, const double* r, const double* d, const double* dv, const double* xi, float* fr,
                 float* e) {
    pair_all<float>(n, par, 0, r, d, dv, xi, fr, e);
}
// out[k] = xi of pair (i[k], j[k]) (0-based) at step[k] with `key`
void dh_normal(int n, const int* i, const int* j, const long long* step, unsigned long long key, double* out) {
    for (int k = 0; k < n; k++) out[k] = dpd_normal(i[k], j[k], step[k], (uint32_t)key, (uint32_t)(key >> 32));
}
}
