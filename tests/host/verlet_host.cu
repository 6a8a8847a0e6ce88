// Test harness (NOT product code): the per-atom update of Verlet, StormerVerlet and OverdampedLangevin (verlet_update of
// csrc/verlet.cuh) compiled for the HOST, so that tests/test_verlet_host.py can check it against tests/verlet_oracle.py
// without a GPU.
#include "../../molly.jl_b200/csrc/verlet.cuh"

using namespace mb;

template <typename T>
static void update_all(int kind, int n, T* p, T* v, const T* f, const T* inv_m, double dt, double friction, int first,
                       const double* g) {
    const VerletCoef c{dt * dt, friction > 0 ? dt / friction : 0.0, 0.0, 0.0};
    for (int i = 0; i < n; i++) {
        typename VT<T>::T4 pi = make4<T>(p[3 * i], p[3 * i + 1], p[3 * i + 2], (T)0);
        typename VT<T>::T4 vi = make4<T>(v[3 * i], v[3 * i + 1], v[3 * i + 2], inv_m[i]);
        const typename VT<T>::T4 fi = make4<T>(f[3 * i], f[3 * i + 1], f[3 * i + 2], (T)0);
        if (kind == VERLET_LEAPFROG) verlet_update<T, VERLET_LEAPFROG>(pi, vi, fi, (T)dt, c, first != 0, g + 3 * i);
        else if (kind == VERLET_STORMER) verlet_update<T, VERLET_STORMER>(pi, vi, fi, (T)dt, c, first != 0, g + 3 * i);
        else verlet_update<T, VERLET_OVERDAMPED>(pi, vi, fi, (T)dt, c, first != 0, g + 3 * i);
        p[3 * i] = pi.x; p[3 * i + 1] = pi.y; p[3 * i + 2] = pi.z;
        v[3 * i] = vi.x; v[3 * i + 1] = vi.y; v[3 * i + 2] = vi.z;
    }
}

extern "C" {
// one step of `kind` (VERLET_*) for n atoms in place: p, v, f, g are n x 3, inv_m has n entries; g is the overdamped noise
void vh_update_f64(int kind, int n, double* p, double* v, const double* f, const double* inv_m, double dt, double friction,
                   int first, const double* g) {
    update_all<double>(kind, n, p, v, f, inv_m, dt, friction, first, g);
}
void vh_update_f32(int kind, int n, float* p, float* v, const float* f, const float* inv_m, double dt, double friction,
                   int first, const double* g) {
    update_all<float>(kind, n, p, v, f, inv_m, dt, friction, first, g);
}
}
