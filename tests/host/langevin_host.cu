// Test harness (NOT product code): the Langevin O step's draws (philox4x32_10 + box_muller3 of csrc/common.cuh) compiled for
// the HOST, so that tests/test_langevin_host.py can check them against tests/langevin_oracle.py without a GPU.
// rng = (ctr1_lo, ctr1_hi, key_lo, key_hi), as the device reads them from the control block.
#include "../../molly.jl_b200/csrc/common.cuh"

using namespace mb;

extern "C" {
// atoms 1..n at `step`: the Philox words (n x 4) and sd * xi (n x 3), counter (i, step, ctr1_lo, ctr1_hi)
void lgh_draws(int n, uint32_t step, const uint32_t* rng, double sd, uint32_t* words, double* out) {
    for (int i = 0; i < n; i++) {
        uint32_t w[4] = {(uint32_t)(i + 1), step, rng[0], rng[1]};
        philox4x32_10(w, rng[2], rng[3]);
        for (int k = 0; k < 4; k++) words[4 * i + k] = w[k];
        box_muller3(w, sd, out + 3 * i);
    }
}
}
