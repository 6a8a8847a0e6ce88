// Test harness (NOT product code): the Nose-Hoover zeta update (nh_zeta_step of csrc/nosehoover.cuh) compiled for the HOST,
// so that tests/test_nosehoover_host.py can check it against tests/nosehoover_oracle.py without a GPU.
#include "../../molly.jl_b200/csrc/nosehoover.cuh"

using namespace mb;

extern "C" {
// zeta after each of `count` steps starting from zeta0, with the kinetic sums of step k at mv2_old[k], mv2_half[k]
void nhh_zeta(double zeta0, long long count, const double* mv2_old, const double* mv2_half, double coef, double nf_kT, double* out) {
    const NhCoef c{coef, nf_kT};
    double z = zeta0;
    for (long long k = 0; k < count; k++) out[k] = z = nh_zeta_step(z, mv2_old[k], mv2_half[k], c);
}
}
