// engine.cu — host side of libmollyb200: context, parameter digestion, rebuild pipeline driver,
// kernel dispatch and the C ABI declared in include/mollyb200.h.
//
// There is deliberately no CPU code path: every entry point needs a CUDA device.
#include <algorithm>
#include <array>
#include <map>
#include <memory>
#include <tuple>
#include <type_traits>

#include "../../include/mollyb200.h"
#include "bonded.cuh"
#include "cells.cuh"
#include "common.cuh"
#include "force.cuh"
#include "gbsa.cuh"
#include "langevin.cuh"
#include "verlet.cuh"
#include "minimize.cuh"
#include "mts.cuh"
#include "nosehoover.cuh"
#include "pair.cuh"
#include "pme.cuh"
#include "splitting.cuh"
#include "vv.cuh"
static_assert(mb::MTS_MAX_LEVELS == MB_MTS_MAX_LEVELS, "mts.cuh levels = MB_MTS_MAX_LEVELS");
static_assert((int)mb::VC_NONE == (int)MB_VC_NONE && (int)mb::VC_IMMEDIATE == (int)MB_VC_IMMEDIATE &&
                  (int)mb::VC_BERENDSEN == (int)MB_VC_BERENDSEN && (int)mb::VC_VRESCALE == (int)MB_VC_VRESCALE,
              "vrescale.cuh kinds = MB_VC_*");

namespace mb {

static thread_local std::string g_last_error;
static int set_error(int code, const std::string& msg) {
    g_last_error = msg;
    return code;
}

#define MB_CUDA(call)                                                                                  \
    do {                                                                                               \
        cudaError_t err__ = (call);                                                                    \
        if (err__ != cudaSuccess) {                                                                    \
            return set_error(MB_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(err__) + " (" + \
                                              __FILE__ + ":" + std::to_string(__LINE__) + ")");        \
        }                                                                                              \
    } while (0)
#define MB_TRY(expr)                 \
    do {                             \
        int rc__ = (expr);           \
        if (rc__ != MB_OK) return rc__; \
    } while (0)

struct DevBuf {
    void* p = nullptr;
    size_t bytes = 0;
    ~DevBuf() { release(); }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        bytes = 0;
    }
    cudaError_t ensure(size_t nbytes) {
        if (nbytes <= bytes) return cudaSuccess;
        release();
        cudaError_t e = cudaMalloc(&p, nbytes);
        if (e == cudaSuccess) bytes = nbytes;
        return e;
    }
    template <typename U>
    U* as() const {
        return reinterpret_cast<U*>(p);
    }
};

// a caller's array: `dev` is the array itself when it is device memory, or its device staging copy (`staged`)
struct CallerBuf {
    void* user;
    void* dev;
    bool staged;
    template <typename U>
    U* as() const {
        return reinterpret_cast<U*>(dev);
    }
};

static bool is_device_ptr(const void* p) {
    if (!p) return false;
    cudaPointerAttributes a;
    cudaError_t e = cudaPointerGetAttributes(&a, p);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

// Kernel variant selection: calls f(std::integral_constant<..., C>{}) for the first C of the list that equals the run-time
// value v, or for the last one when none does. f is instantiated for exactly the listed constants, so a launch site writes
// its launch once and names the variants that exist, e.g. with_const<true, false>(energy, [&](auto EN) { k<T, EN><<<...>>>(...); }).
template <auto C0, auto... Cs, typename V, typename F>
static auto with_const(V v, F&& f) {
    if constexpr (sizeof...(Cs) == 0) return f(std::integral_constant<decltype(C0), C0>{});
    else return v == C0 ? f(std::integral_constant<decltype(C0), C0>{}) : with_const<Cs...>(v, f);
}

// Optional per-category device timing with CUDA events on the engine's stream (mb_set_profiling).
struct Prof {
    enum { FORCE = 0, VV = 1, REBUILD = 2, NCAT = 3 };
    bool enabled = false;
    cudaStream_t stream = nullptr;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> ev[NCAT];
    size_t used[NCAT] = {0, 0, 0};
    double ms[NCAT] = {0, 0, 0};
    long long count[NCAT] = {0, 0, 0};
    ~Prof() {
        for (int c = 0; c < NCAT; c++)
            for (auto& p : ev[c]) { cudaEventDestroy(p.first); cudaEventDestroy(p.second); }
    }
    void begin(int c) {
        if (!enabled) return;
        if (used[c] == ev[c].size()) {
            if (ev[c].size() >= 8192) { collect(); }
            if (used[c] == ev[c].size()) {
                cudaEvent_t a, b;
                cudaEventCreate(&a);
                cudaEventCreate(&b);
                ev[c].emplace_back(a, b);
            }
        }
        cudaEventRecord(ev[c][used[c]].first, stream);
    }
    void end(int c) {
        if (!enabled) return;
        cudaEventRecord(ev[c][used[c]].second, stream);
        used[c]++;
    }
    void collect() {
        cudaStreamSynchronize(stream);
        for (int c = 0; c < NCAT; c++) {
            for (size_t k = 0; k < used[c]; k++) {
                float t = 0;
                if (cudaEventElapsedTime(&t, ev[c][k].first, ev[c][k].second) == cudaSuccess) { ms[c] += t; count[c]++; }
            }
            used[c] = 0;
        }
    }
    void reset() {
        collect();
        for (int c = 0; c < NCAT; c++) { ms[c] = 0; count[c] = 0; }
    }
};

// ---------------------------------------------------------------------------------------------
// NCCL, bound at run time (dlopen) so that single-GPU users do not need the library. Only what the
// decomposed step uses: point-to-point halo exchange, grouped broadcasts, one tiny all-reduce.
// ---------------------------------------------------------------------------------------------
#include <dlfcn.h>
extern "C" {
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef enum { ncclSuccess = 0 } ncclResult_t;
typedef enum { ncclInt8 = 0, ncclChar = 0, ncclFloat64 = 8, ncclDouble = 8 } ncclDataType_t;
typedef enum { ncclSum = 0 } ncclRedOp_t;
}
struct Nccl {
    void* lib = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    bool load() {
        if (lib) return true;
        lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!lib) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        if (!lib) return false;
#define MB_SYM(field, name) field = reinterpret_cast<decltype(field)>(dlsym(lib, name)); if (!field) return false
        MB_SYM(GetUniqueId, "ncclGetUniqueId");
        MB_SYM(CommInitRank, "ncclCommInitRank");
        MB_SYM(CommDestroy, "ncclCommDestroy");
        MB_SYM(GroupStart, "ncclGroupStart");
        MB_SYM(GroupEnd, "ncclGroupEnd");
        MB_SYM(Send, "ncclSend");
        MB_SYM(Recv, "ncclRecv");
        MB_SYM(Broadcast, "ncclBroadcast");
        MB_SYM(AllReduce, "ncclAllReduce");
        MB_SYM(AllGather, "ncclAllGather");
        MB_SYM(GetErrorString, "ncclGetErrorString");
#undef MB_SYM
        return true;
    }
};
static Nccl g_nccl;

// cuFFT, bound at run time like NCCL (only PME systems need it). Plain library FFT: the spreading, convolution and
// interpolation kernels around it are ours (pme.cuh).
struct Cufft {
    void* lib = nullptr;
    int (*Plan3d)(int*, int, int, int, int) = nullptr;
    int (*SetStream)(int, cudaStream_t) = nullptr;
    int (*ExecC2C)(int, void*, void*, int) = nullptr;
    int (*ExecZ2Z)(int, void*, void*, int) = nullptr;
    int (*Destroy)(int) = nullptr;
    bool load() {
        if (lib) return true;
        lib = dlopen("libcufft.so.11", RTLD_NOW | RTLD_GLOBAL);
        if (!lib) lib = dlopen("libcufft.so", RTLD_NOW | RTLD_GLOBAL);
        if (!lib) return false;
#define MB_SYM(field, name) field = reinterpret_cast<decltype(field)>(dlsym(lib, name)); if (!field) return false
        MB_SYM(Plan3d, "cufftPlan3d");
        MB_SYM(SetStream, "cufftSetStream");
        MB_SYM(ExecC2C, "cufftExecC2C");
        MB_SYM(ExecZ2Z, "cufftExecZ2Z");
        MB_SYM(Destroy, "cufftDestroy");
#undef MB_SYM
        return true;
    }
};
static Cufft g_cufft;
#define MB_NCCL(call)                                                                                       \
    do {                                                                                                    \
        ncclResult_t r__ = (call);                                                                          \
        if (r__ != ncclSuccess)                                                                             \
            return set_error(MB_ERR_CUDA, std::string(#call) + ": " + g_nccl.GetErrorString(r__));          \
    } while (0)

// ---------------------------------------------------------------------------------------------
// Slab decomposition plan (pure host logic, exported as mb_decomp_plan so it can be tested without a GPU):
// rank q owns cell layers [q*ncz/P, (q+1)*ncz/P); it needs the h layers below and above its slab (periodic).
// Segments are contiguous slot ranges [start, start+count) taken from layer_start (ncz + 1 prefix offsets).
// Both ends enumerate the segments of a (sender, receiver) pair in the receiver's order, so the grouped
// ncclSend/ncclRecv calls match up.
// ---------------------------------------------------------------------------------------------
struct DecompSeg { int peer, start, count; };
static inline int decomp_layer_lo(int q, int ncz, int nranks) { return (int)(((long long)q * ncz) / nranks); }
static inline int decomp_layer_owner(int layer, int ncz, int nranks) {
    for (int q = 0; q < nranks; q++)
        if (layer >= decomp_layer_lo(q, ncz, nranks) && layer < decomp_layer_lo(q + 1, ncz, nranks)) return q;
    return nranks - 1;
}
static void decomp_needed(int q, int ncz, int h, int nranks, std::vector<int>& out) {
    out.clear();
    const int lo = decomp_layer_lo(q, ncz, nranks), hi = decomp_layer_lo(q + 1, ncz, nranks);
    std::vector<char> seen(ncz, 0);
    for (int l = lo; l < hi; l++) seen[l] = 1;
    for (int l = lo - h; l < lo; l++) { int w = ((l % ncz) + ncz) % ncz; if (!seen[w]) { seen[w] = 1; out.push_back(w); } }
    for (int l = hi; l < hi + h; l++) { int w = l % ncz; if (!seen[w]) { seen[w] = 1; out.push_back(w); } }
}
static void decomp_plan(int ncz, int h, int nranks, int rank, const int* layer_start, std::vector<DecompSeg>& send,
                        std::vector<DecompSeg>& recv) {
    auto add = [&](std::vector<DecompSeg>& v, int peer, int layer) {
        int st = layer_start[layer], cnt = layer_start[layer + 1] - st;
        if (!v.empty() && v.back().peer == peer && v.back().start + v.back().count == st) v.back().count += cnt;
        else v.push_back({peer, st, cnt});
    };
    send.clear();
    recv.clear();
    std::vector<int> need;
    decomp_needed(rank, ncz, h, nranks, need);
    for (int l : need) add(recv, decomp_layer_owner(l, ncz, nranks), l);
    for (int q = 0; q < nranks; q++) {
        if (q == rank) continue;
        decomp_needed(q, ncz, h, nranks, need);
        for (int l : need)
            if (decomp_layer_owner(l, ncz, nranks) == rank) add(send, q, l);
    }
}

// ---------------------------------------------------------------------------------------------
// PME plan (pure host logic, exported as mb_pme_plan so it is tested on the CPU against oracle/pme.py):
// alpha = sqrt(-ln(2 tol)) / rc (ewald.jl:373), mesh dims = max(6, ceil(2 alpha L / (3 tol^0.2))) (:484-487),
// B-spline moduli (:311-361).
// ---------------------------------------------------------------------------------------------
static void pme_plan_host(const double box[3], double r_cut, double error_tol, int order, double* alpha_out, int K[3],
                          std::vector<double> moduli[3]) {
    const double alpha = std::sqrt(-std::log(2.0 * error_tol)) / r_cut;
    *alpha_out = alpha;
    for (int d = 0; d < 3; d++) K[d] = std::max((int)std::ceil(2.0 * alpha * box[d] / (3.0 * std::pow(error_tol, 0.2))), 6);
    std::vector<double> data(order, 0.0);
    data[0] = 1.0;
    for (int k = 3; k < order; k++) {
        const double d = 1.0 / (k - 1.0);
        data[k - 1] = 0.0;
        for (int l = 1; l <= k - 2; l++) data[k - l - 1] = d * (l * data[k - l - 2] + (k - l) * data[k - l - 1]);
        data[0] *= d;
    }
    {
        const double d = 1.0 / (order - 1.0);
        data[order - 1] = 0.0;
        for (int l = 1; l <= order - 2; l++) data[order - l - 1] = d * (l * data[order - l - 2] + (order - l) * data[order - l - 1]);
        data[0] *= d;
    }
    const double two_pi = 6.283185307179586476925;
    for (int d = 0; d < 3; d++) {
        const int nd = K[d];
        std::vector<double> bs((size_t)std::max(nd, order + 1), 0.0);
        std::vector<double>& mod = moduli[d];
        mod.assign(nd, 0.0);
        for (int i = 0; i < order; i++) bs[i + 1] = data[i];
        for (int i = 0; i < nd; i++) {
            double sc = 0, ss = 0;
            for (int j = 0; j < nd; j++) {
                const double arg = two_pi * i * j / nd;
                sc += bs[j] * std::cos(arg);
                ss += bs[j] * std::sin(arg);
            }
            mod[i] = sc * sc + ss * ss;
        }
        for (int i = 0; i < nd; i++)
            if (mod[i] < 1e-7) mod[i] = 0.5 * (mod[(i - 1 + nd) % nd] + mod[(i + 1) % nd]);
    }
}

// The integrator of one simulate call: VelocityVerlet (vv.cuh), Langevin (langevin.cuh), Nose-Hoover (nosehoover.cuh), the
// multiple-time-step integrators (mts.cuh), LangevinSplitting (splitting.cuh), or Verlet, StormerVerlet and
// OverdampedLangevin (verlet.cuh), or DPDVelocityVerlet (vv.cuh's step with the DPD drift, dpd.cuh). Each mb_simulate_* entry
// point fills one from its own parameters.
enum { INTEG_VV = 0, INTEG_LANGEVIN = 1, INTEG_NH = 2, INTEG_MTS = 3, INTEG_MTS_LANGEVIN = 4, INTEG_SPLIT = 5, INTEG_VERLET = 6,
       INTEG_STORMER = 7, INTEG_OVERDAMPED = 8, INTEG_DPD_VV = 9 };
static_assert(SPLIT_MAX_OPS == MB_SPLIT_MAX_OPS, "splitting length");
static bool is_mts(int kind) { return kind == INTEG_MTS || kind == INTEG_MTS_LANGEVIN; }
struct Integrator {
    int kind = INTEG_VV;  // INTEG_*
    double dt = 0;
    int64_t n_steps = 0, init_step = 0;
    int remove_cm_every = 0;
    uint64_t rng_ctr1 = 0, rng_key = 0;
    double andersen_kT = 0, andersen_prob = 0;  // VelocityVerlet's and Verlet's Andersen thermostat (kT <= 0 or prob <= 0: none)
    double kT = 0, friction = 0, damping = 0;   // Langevin, MTSLangevinIntegrator, LangevinSplitting and OverdampedLangevin:
                                                // kT, friction;
                                                // Nose-Hoover: kT, damping
    int n_levels = 0;                           // the multiple-time-step integrators' ordered fractions (0 levels: none)
    std::array<int, MTS_MAX_LEVELS> fractions = {};
    int n_ops = 0;                              // LangevinSplitting's splitting: the letters 'A', 'B', 'O' (0: none)
    std::array<char, SPLIT_MAX_OPS> ops = {};
    double lambda = 0;                          // DPDVelocityVerlet's velocity prediction parameter
    // What the step graphs bake in (GraphKey): every field but n_steps, init_step and the RNG keys, which are uploaded
    // into Control on every call
    auto graph_fields() const {
        return std::tie(kind, dt, remove_cm_every, andersen_kT, andersen_prob, kT, friction, damping, n_levels, fractions, n_ops,
                        ops, lambda);
    }
};

// LangevinSplitting's step cut into passes at its force evaluations (simulate!'s force_computation_steps, src/simulators.jl:
// 1305-1324). Forces are known at the start of a step unless an A follows the last B; an A makes them unknown and a B
// recomputes them only when they are unknown. A recomputing B is served by an evaluation right after the last A in front of
// it; only O's lie between the two, so the positions are the same. One that has no A in front of it in the step is served by
// an evaluation at the end of the step before (at the first step: the call's F0). Passes never come out empty.
struct SplitPlan {
    int n_pass = 0, n_evals = 0;                // passes and force evaluations per step
    std::array<SplitProg, SPLIT_MAX_OPS> pass;  // (apply_cm, last set; the letters as SPLIT_*)
    std::array<bool, SPLIT_MAX_OPS> eval_after; // a force evaluation follows the pass (the last pass: the end-of-step one)
    int count[3] = {0, 0, 0};                   // letters A, B, O in the splitting
};
static SplitPlan split_plan(const Integrator& ig) {
    SplitPlan sp;
    const int n = ig.n_ops;
    std::array<int, SPLIT_MAX_OPS> op = {};
    int last_b = -1;
    for (int k = 0; k < n; k++) {
        op[k] = ig.ops[k] == 'A' ? SPLIT_A : (ig.ops[k] == 'B' ? SPLIT_B : SPLIT_O);
        sp.count[op[k]]++;
        if (op[k] == SPLIT_B) last_b = k;
    }
    bool a_after_last_b = false;  // the splitting matches ^.*B[^B]*A[^B]*$
    for (int k = last_b + 1; last_b >= 0 && k < n; k++) a_after_last_b |= op[k] == SPLIT_A;
    std::array<bool, SPLIT_MAX_OPS> cut = {};  // an evaluation after letter k
    bool known = !a_after_last_b, end_eval = false;
    int last_a = -1;
    for (int k = 0; k < n; k++) {
        if (op[k] == SPLIT_A) { known = false; last_a = k; }
        if (op[k] == SPLIT_B && !known) {
            known = true;
            if (last_a >= 0) cut[last_a] = true;
            else end_eval = true;
        }
    }
    sp.pass.fill(SplitProg{});
    sp.eval_after.fill(false);
    int j = 0;
    for (int k = 0; k < n; k++) {
        SplitProg& pg = sp.pass[sp.n_pass];
        if (pg.n_ops == 0) pg.o_base = j;
        pg.ops |= (unsigned long long)op[k] << (2 * pg.n_ops);
        pg.n_ops++;
        j += op[k] == SPLIT_O ? 1 : 0;
        pg.has_a |= op[k] == SPLIT_A;
        pg.has_b |= op[k] == SPLIT_B;
        pg.has_o |= op[k] == SPLIT_O;
        if (cut[k] || k == n - 1) {
            sp.eval_after[sp.n_pass] = cut[k] || end_eval;
            sp.n_evals += sp.eval_after[sp.n_pass] ? 1 : 0;
            sp.n_pass++;
        }
    }
    sp.pass[0].apply_cm = 1;  // (every pass reads v)
    sp.pass[sp.n_pass - 1].last = 1;
    return sp;
}

class EngineBase {
   public:
    virtual ~EngineBase() {}
    virtual int set_atoms_aos(int64_t n, const void* aos) = 0;
    virtual int set_atoms_soa(int64_t n, const void* mass, const void* charge, const void* sigma, const void* eps) = 0;
    virtual int set_box(const double side[3]) = 0;
    virtual int set_box_triclinic(const double basis[9]) = 0;
    virtual int set_inters(int n, const mb_inter_t* in) = 0;
    virtual int set_exceptions(int64_t ne, const int32_t* ei, const int32_t* ej, int64_t ns, const int32_t* si,
                               const int32_t* sj) = 0;
    virtual int set_neighbor_policy(double r_list, int rebuild_every) = 0;
    virtual int forces_energy(const void* coords, void* fs, void* pe, void* vir, int64_t step_n, bool with_specific,
                              const void* vels) = 0;
    virtual int simulate(void* coords, void* vels, const Integrator& ig, mb_log_t* log) = 0;
    // simulate's phases, for mb_simulate_group (single-GPU contexts only): sim_begin, then sim_step(k) for k = 1 ..
    // ig.n_steps, then sim_end
    virtual int sim_begin(void* coords, void* vels, const Integrator& ig, mb_log_t* log) = 0;
    virtual int sim_step(int64_t k) = 0;
    virtual int sim_end() = 0;
    virtual bool is_decomposed() const = 0;
    virtual int remove_cm(void* vels) = 0;
    virtual int kinetic_energy(const void* vels, double* out) = 0;
    virtual int rebuild(const void* coords) = 0;
    virtual int stats(mb_stats_t* out) = 0;
    virtual int synchronize() = 0;
    virtual int set_capacity_scale(double s) = 0;
    virtual int set_launch_config(const int32_t bd[3], int32_t lpa) = 0;
    virtual int set_profiling(int enable) = 0;
    virtual int comm_init(const void* uid, int rank, int nranks) = 0;
    virtual int set_specific(int kind, int64_t n, const int32_t* idx, const double* par) = 0;
    virtual int set_specific_levels(int kind, int64_t n, const int32_t* level) = 0;
    virtual int set_pme(double r_cut, double error_tol, int order, double eps_r, int64_t n_pairs, const int32_t* pi, const int32_t* pj) = 0;
    virtual int set_dispersion(double r_cut) = 0;
    virtual int set_implicit_solvent(const mb_gbsa_t* p, const double* or_, const double* sr, const double* alpha, const double* beta,
                                     const double* gamma, const int32_t* cls, const double* d0, const double* m0) = 0;
    virtual int random_velocities(void* vels, double kT, uint64_t ctr1, uint64_t key) = 0;
    virtual int kinetic_tensor(const void* vels, double* out9) = 0;
    virtual int minimize_sd(void* coords, mb_sd_params_t* p) = 0;
    virtual int set_dpd(const mb_dpd_t* p) = 0;
    mb_vcoupling_t vcoupling = {MB_VC_NONE, 0, 0.0, 0.0};  // mb_set_velocity_coupling (validated there)
};

template <typename T>
class Engine : public EngineBase {
    using T4 = typename VT<T>::T4;
    using T2 = typename VT<T>::T2;

   public:
    Engine(int device, cudaStream_t stream) : stream_(stream) {
        cudaDeviceProp prop;
        cudaGetDeviceProperties(&prop, device);
        sm_count_ = prop.multiProcessorCount;
        smem_optin_ = prop.sharedMemPerBlockOptin;
        for (int d = 0; d < 3; d++) box_[d] = 0;
        if (!stream_) {
            // a real (blocking) stream: graph capture is not allowed on the legacy default stream, and a blocking
            // stream keeps the implicit ordering with work the caller issues on the default stream
            if (cudaStreamCreateWithFlags(&stream_, cudaStreamDefault) == cudaSuccess) own_stream_ = true;
            else stream_ = nullptr;
        }
        prof_.stream = stream_;
        const char* ng = getenv("MOLLYB200_NO_GRAPH");
        graph_enabled_ = !(ng && ng[0] == '1');
    }
    ~Engine() override {
        drop_graphs();
        p2p_close();
        if (pme_plan_ >= 0 && g_cufft.Destroy) g_cufft.Destroy(pme_plan_);
        if (own_stream_) cudaStreamDestroy(stream_);
    }

    // ------------------------------------------------------------------------------------------
    int set_atoms_aos(int64_t n, const void* aos) override {
        if (n <= 0 || !aos) return set_error(MB_ERR_INVALID, "mb_set_atoms: n <= 0 or null atoms");
        // Atom{Int32,T,T,T,T,T}: int32 index, int32 atom_type, T mass, T charge, T sigma, T eps, T lambda, int32 role
        const size_t rec = (sizeof(T) == 4) ? 32 : 56;
        std::vector<unsigned char> host((size_t)n * rec);
        MB_CUDA(cudaMemcpy(host.data(), aos, host.size(), cudaMemcpyDefault));
        h_mass_.resize(n); h_charge_.resize(n); h_sigma_.resize(n); h_eps_.resize(n); h_eps_raw_.resize(n);
        for (int64_t i = 0; i < n; i++) {
            const unsigned char* r = host.data() + (size_t)i * rec;
            T vals[5];
            memcpy(vals, r + 8, 5 * sizeof(T));
            h_mass_[i] = vals[0];
            h_charge_[i] = vals[1];
            h_sigma_[i] = vals[2];
            h_eps_[i] = (vals[4] == (T)0) ? (T)0 : vals[3];  // lambda == 0 -> LJ zero shortcut (mixing.jl:7-11)
            h_eps_raw_[i] = vals[3];
        }
        n_ = n;
        dirty_ = true;
        pme_ready_ = disp_ready_ = false;  // the PME self energy and the dispersion factors come from the atoms
        return MB_OK;
    }
    int set_atoms_soa(int64_t n, const void* mass, const void* charge, const void* sigma, const void* eps) override {
        if (n <= 0 || !mass || !charge || !sigma || !eps)
            return set_error(MB_ERR_INVALID, "mb_set_atoms_soa: n <= 0 or null array");
        h_mass_.resize(n); h_charge_.resize(n); h_sigma_.resize(n); h_eps_.resize(n);
        MB_CUDA(cudaMemcpy(h_mass_.data(), mass, n * sizeof(T), cudaMemcpyDefault));
        MB_CUDA(cudaMemcpy(h_charge_.data(), charge, n * sizeof(T), cudaMemcpyDefault));
        MB_CUDA(cudaMemcpy(h_sigma_.data(), sigma, n * sizeof(T), cudaMemcpyDefault));
        MB_CUDA(cudaMemcpy(h_eps_.data(), eps, n * sizeof(T), cudaMemcpyDefault));
        h_eps_raw_ = h_eps_;
        n_ = n;
        dirty_ = true;
        pme_ready_ = disp_ready_ = false;
        return MB_OK;
    }
    int set_box(const double side[3]) override {
        for (int d = 0; d < 3; d++) {
            if (!(side[d] > 0) || std::isinf(side[d]))
                return set_error(MB_ERR_INVALID, "mb_set_box: side lengths must be finite and > 0 (CubicBoundary)");
            box_[d] = side[d];
        }
        memset(&tric_, 0, sizeof(tric_));
        dirty_ = true;
        return MB_OK;
    }
    // TriclinicBoundary(bv1, bv2, bv3) (src/spatial.jl:165-215): lower-triangular basis, positive diagonal. Such systems run
    // on the no-list kernel (minimum image :528-534, wrap :584-600); the cell-list path is for Cubic/Rectangular boxes.
    int set_box_triclinic(const double b[9]) override {
        if (!(b[0] > 0) || b[1] != 0 || b[2] != 0)
            return set_error(MB_ERR_INVALID, "mb_set_box_triclinic: first basis vector must be along the x-axis with a positive x component");
        if (!(b[4] > 0) || b[5] != 0)
            return set_error(MB_ERR_INVALID, "mb_set_box_triclinic: second basis vector must be in the xy plane with a positive y component");
        if (!(b[8] > 0)) return set_error(MB_ERR_INVALID, "mb_set_box_triclinic: third basis vector must have a positive z component");
        for (int k = 0; k < 9; k++)
            if (std::isinf(b[k]) || std::isnan(b[k])) return set_error(MB_ERR_INVALID, "mb_set_box_triclinic: infinite boundaries are not supported");
        Tric<T> t;
        memset(&t, 0, sizeof(t));
        t.on = 1;
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) t.bv[i][j] = (T)b[3 * i + j];
        t.rs[0] = (T)(1.0 / b[0]); t.rs[1] = (T)(1.0 / b[4]); t.rs[2] = (T)(1.0 / b[8]);
        const double by = b[4], bz = b[5], cy = b[7], cz = b[8];
        t.cot_bprojyz_cprojyz = (T)std::fabs((by * cy + bz * cz) / (by * cz - bz * cy));
        t.cprojxy_x_over_z = (T)(b[6] / std::fabs(b[8]));
        t.cprojxy_y_over_z = (T)(b[7] / std::fabs(b[8]));
        t.cot_a_b = (T)(b[3] / b[4]);
        tric_ = t;
        box_[0] = b[0]; box_[1] = b[4]; box_[2] = b[8];  // heights: volume = their product
        dirty_ = true;
        return MB_OK;
    }
    int set_inters(int n, const mb_inter_t* in) override {
        if (n < 0 || (n > 0 && !in)) return set_error(MB_ERR_INVALID, "mb_set_inters: bad arguments");
        int n_lj = 0, n_c = 0;
        for (int k = 0; k < n; k++) {
            if (in[k].kind == MB_LJ) n_lj++;
            else if (in[k].kind == MB_COULOMB || in[k].kind == MB_CRF || in[k].kind == MB_EWALD_REAL) n_c++;
            else return set_error(MB_ERR_INVALID, "mb_set_inters: unknown interaction kind");
            if (in[k].cutoff_kind < MB_CUT_NONE || in[k].cutoff_kind > MB_CUT_POLYNOMIAL)
                return set_error(MB_ERR_INVALID, "mb_set_inters: unsupported cutoff kind");
            if (in[k].cutoff_kind >= MB_CUT_CUBIC_SPLINE) {
                // CubicSplineCutoff / PolynomialCutoff constructors, src/cutoffs.jl:181-187, :239-245
                if (in[k].kind != MB_LJ && in[k].kind != MB_COULOMB)
                    return set_error(MB_ERR_INVALID, "mb_set_inters: two-point cutoffs apply to LennardJones and Coulomb only");
                if (!(in[k].r_act > 0) || !(in[k].r_cut > in[k].r_act))
                    return set_error(MB_ERR_INVALID, "mb_set_inters: the cutoff radius must be larger than the activation radius");
            }
            if (in[k].kind == MB_LJ && in[k].eps_mix != MB_MIX_GEOMETRIC)
                return set_error(MB_ERR_INVALID, "mb_set_inters: only geometric epsilon mixing is supported");
        }
        if (n_lj > 1 || n_c > 1)
            return set_error(MB_ERR_INVALID, "mb_set_inters: at most one LJ and one Coulomb-family interaction");
        inters_.assign(in, in + n);
        dirty_ = true;
        return MB_OK;
    }
    int set_exceptions(int64_t ne, const int32_t* ei, const int32_t* ej, int64_t ns, const int32_t* si,
                       const int32_t* sj) override {
        if (n_ <= 0) return set_error(MB_ERR_STATE, "mb_set_exceptions: set atoms first");
        auto build = [&](int64_t m, const int32_t* a, const int32_t* b, std::vector<int>& ptr, std::vector<int>& idx,
                         const std::vector<int>* skip_ptr, const std::vector<int>* skip_idx) -> int {
            std::vector<std::pair<int, int>> pr;
            pr.reserve(2 * m);
            for (int64_t k = 0; k < m; k++) {
                int i = a[k] - 1, j = b[k] - 1;  // 1-based in, 0-based inside
                if (i < 0 || j < 0 || i >= n_ || j >= n_)
                    return set_error(MB_ERR_INVALID, "mb_set_exceptions: index out of bounds");
                if (i == j) continue;
                if (skip_ptr && !skip_ptr->empty()) {
                    bool ex = false;
                    for (int q = (*skip_ptr)[i]; q < (*skip_ptr)[i + 1]; q++) ex |= ((*skip_idx)[q] == j);
                    if (ex) continue;  // excluded wins over special
                }
                pr.emplace_back(i, j);
                pr.emplace_back(j, i);
            }
            std::sort(pr.begin(), pr.end());
            pr.erase(std::unique(pr.begin(), pr.end()), pr.end());
            ptr.assign(n_ + 1, 0);
            idx.resize(pr.size());
            for (auto& p : pr) ptr[p.first + 1]++;
            for (int64_t i = 0; i < n_; i++) ptr[i + 1] += ptr[i];
            for (size_t k = 0; k < pr.size(); k++) idx[k] = pr[k].second;
            return MB_OK;
        };
        MB_TRY(build(ne, ei, ej, ex_ptr_, ex_idx_, nullptr, nullptr));
        MB_TRY(build(ns, si, sj, sp_ptr_, sp_idx_, &ex_ptr_, &ex_idx_));
        if (ex_idx_.empty()) ex_ptr_.clear();
        if (sp_idx_.empty()) sp_ptr_.clear();
        dirty_ = true;
        return MB_OK;
    }
    int set_neighbor_policy(double r_list, int rebuild_every) override {
        if (r_list < 0 || rebuild_every < 0) return set_error(MB_ERR_INVALID, "mb_set_neighbor_policy: negative value");
        r_list_ = r_list;
        rebuild_every_ = rebuild_every;
        dirty_ = true;
        return MB_OK;
    }
    int set_capacity_scale(double s) override {
        if (!(s >= 1.0)) return set_error(MB_ERR_INVALID, "capacity scale must be >= 1");
        cap_scale_ = s;
        have_list_ = false;
        return MB_OK;
    }
    int set_launch_config(const int32_t bd[3], int32_t lpa) override {
        for (int d = 0; d < 3; d++) {
            if (bd[d] < 0 || bd[d] > 8) return set_error(MB_ERR_INVALID, "brick dims must be in 0..8");
            user_b_[d] = bd[d];
        }
        if (!(lpa == 0 || lpa == 8))
            return set_error(MB_ERR_INVALID, "lanes_per_atom must be 0 (default) or 8: the 4- and 16-lane variants were measured slower and removed");
        have_list_ = false;
        dirty_ = true;
        return MB_OK;
    }
    int set_profiling(int enable) override {
        prof_.reset();
        prof_.enabled = enable != 0;
        return MB_OK;
    }
    int synchronize() override {
        MB_CUDA(cudaStreamSynchronize(stream_));
        return MB_OK;
    }

    // ------------------------------------------------------------------------------------------
    // digest parameters -> kernel constants, allocate per-atom state
    int prepare() {
        if (!dirty_) return MB_OK;
        drop_graphs();  // they bake in what is digested here (Graph)
        if (n_ <= 0) return set_error(MB_ERR_STATE, "atoms not set");
        if (!(box_[0] > 0)) return set_error(MB_ERR_STATE, "box not set");
        if (n_ > 2000000000LL) return set_error(MB_ERR_INVALID, "too many atoms");
        // mb_set_pme checked its pairs against the atom count of that time; mb_set_atoms may have lowered it since. This
        // runs before any kernel of the evaluation writes into the forces.
        if (pme_on_)
            for (int a : pme_pairs_)
                if (a >= n_) return set_error(MB_ERR_STATE, "PME: an exclusion pair indexes past the atom count set by mb_set_atoms; call mb_set_pme again");
        memset(&P_, 0, sizeof(P_));
        MB_TRY(check_dpd());
        const double inf = std::numeric_limits<double>::infinity();
        bool all_nl = dpd_on_ ? dpd_.use_neighbors != 0 : !inters_.empty();  // (a DPD context has no mb_inter_t: check_dpd)
        double max_rc = dpd_on_ ? dpd_.r_c : 0;
        bool any_nocut_nl = false;
        for (auto& in : inters_) {
            if (!in.use_neighbors) all_nl = false;
            if (in.cutoff_kind != MB_CUT_NONE || in.kind == MB_CRF || in.kind == MB_EWALD_REAL)
                max_rc = std::max(max_rc, in.r_cut);
            else if (in.use_neighbors)
                any_nocut_nl = true;
        }
        const double min_box = std::min(box_[0], std::min(box_[1], box_[2]));
        path_ = (all_nl && r_list_ > 0 && min_box >= 2.5 * r_list_ && n_ >= 64 && !tric_.on) ? 1 : 0;
        if (tric_.on && pme_on_) return set_error(MB_ERR_INVALID, "TriclinicBoundary: PME is not supported by this engine");
        if (tric_.on && has_lists() && all_nl && r_list_ > 0 && n_ >= 64) {
            // A system this large would take the cell-list path in a rectangular box; the cell-list path does not handle
            // triclinic boxes, so its pairs would run on the O(N^2) no-list kernel. Bonded terms in a triclinic box are served
            // only where the no-list kernel is the intended path (box heights below 2.5 r_list).
            const double ax = tric_.bv[0][0], bx = tric_.bv[1][0], by = tric_.bv[1][1];
            const double cx = tric_.bv[2][0], cy = tric_.bv[2][1], cz = tric_.bv[2][2];
            const double vol = ax * by * cz;
            const double h0 = vol / std::sqrt(by * cz * by * cz + bx * cz * bx * cz + (bx * cy - by * cx) * (bx * cy - by * cx));
            const double h1 = vol / (ax * std::sqrt(cz * cz + cy * cy));
            if (std::min(h0, std::min(h1, cz)) >= 2.5 * r_list_)
                return set_error(MB_ERR_INVALID, "TriclinicBoundary: specific interaction lists in a box this large need the cell-list "
                                                 "path, which does not support triclinic boxes yet");
        }
        if (tric_.on && decomposed()) return set_error(MB_ERR_INVALID, "TriclinicBoundary: not available in decomposed (multi-GPU) runs");
        if (path_ == 1 && max_rc > r_list_)
            return set_error(MB_ERR_INVALID, "neighbour list radius is smaller than an interaction cutoff");
        skin_ = (path_ == 1) ? (any_nocut_nl ? 0.0 : r_list_ - max_rc) : 0.0;
        P_.has_lj = 0;
        P_.coul_kind = COUL_NONE;
        P_.lj_rc2 = (T)0;
        P_.c_rc2 = (T)0;
        cutm_ = CUTM_PLAIN;
        bool geo_sigma = false;
        for (auto& in : inters_) {
            // effective cutoff: NoCutoff with a neighbour list -> the finder radius (ext/MollyCUDAExt.jl:1691)
            double rc = inf;
            int ck = in.cutoff_kind;
            if (in.kind == MB_CRF || in.kind == MB_EWALD_REAL) {
                rc = in.r_cut;
                ck = MB_CUT_DISTANCE;
            } else if (ck != MB_CUT_NONE) {
                rc = in.r_cut;
            } else if (in.use_neighbors && r_list_ > 0) {
                rc = r_list_;
            }
            if (ck >= MB_CUT_CUBIC_SPLINE) cutm_ = CUTM_TWO_POINT;
            else if (ck >= MB_CUT_SHIFTED_POTENTIAL && cutm_ == CUTM_PLAIN) cutm_ = CUTM_SHIFTED;
            if (in.kind == MB_LJ) {
                P_.has_lj = 1;
                P_.lj_cut_kind = ck;
                P_.lj_rc = (T)rc; P_.lj_rc2 = (T)(rc * rc); P_.lj_inv_rc = (T)(1.0 / rc); P_.lj_inv_rc2 = (T)(1.0 / (rc * rc));
                P_.lj_ra = (T)in.r_act; P_.lj_inv_ra2 = (in.r_act > 0) ? (T)(1.0 / (in.r_act * in.r_act)) : (T)0;
                P_.lj_w14 = (T)in.weight_special;
                P_.lj_nl = in.use_neighbors ? 1 : 0;
                geo_sigma = (in.sigma_mix == MB_MIX_GEOMETRIC);
            } else {
                P_.coul_kind = (in.kind == MB_COULOMB) ? COUL_PLAIN : (in.kind == MB_CRF ? COUL_CRF : COUL_EWALD);
                P_.coul_cut_kind = ck;
                P_.c_rc = (T)rc; P_.c_rc2 = (T)(rc * rc); P_.c_inv_rc = (T)(1.0 / rc); P_.c_inv_rc2 = (T)(1.0 / (rc * rc));
                P_.ke = (T)in.coulomb_const;
                P_.c_w14 = (T)in.weight_special;
                P_.c_nl = in.use_neighbors ? 1 : 0;
                P_.alpha = (T)in.ewald_alpha;
                P_.c_ra = (T)in.r_act;
                P_.approx_erfc = (in.kind == MB_EWALD_REAL && in.approx_erfc) ? 1 : 0;
                if (in.kind == MB_CRF) {
                    double e = in.solvent_dielectric;
                    double krf, crf;
                    if (std::isinf(e)) { krf = 1.0 / (2.0 * rc * rc * rc); crf = 3.0 / (2.0 * rc); }
                    else { krf = (1.0 / (rc * rc * rc)) * (e - 1.0) / (2.0 * e + 1.0); crf = (1.0 / rc) * (3.0 * e) / (2.0 * e + 1.0); }
                    P_.krf = (T)krf;
                    P_.crf = (T)crf;
                }
            }
        }
        P_.geo_sigma = geo_sigma ? 1 : 0;
        // per-atom LJ parts (zero shortcut folded into a zero eps part)
        std::vector<T2> ljp(n_);
        bool uniform = true;
        for (int64_t i = 0; i < n_; i++) {
            T s = h_sigma_[i], e = h_eps_[i];
            bool zero = (!P_.has_lj) || s == (T)0 || e == (T)0;
            ljp[i].x = zero ? (T)0 : (geo_sigma ? (T)std::sqrt((double)s) : s / (T)2);
            ljp[i].y = zero ? (T)0 : (T)std::sqrt((double)e);
            if (h_sigma_[i] != h_sigma_[0] || h_eps_[i] != h_eps_[0]) uniform = false;
        }
        if (!P_.has_lj || h_sigma_[0] == (T)0 || h_eps_[0] == (T)0) uniform = uniform && !P_.has_lj;
        P_.uniform_lj = ((uniform || dpd_on_) && P_.coul_kind == COUL_NONE) ? 1 : 0;  // (DPD stages positions only)
        if (P_.uniform_lj) {
            P_.uni_sig2 = P_.has_lj ? h_sigma_[0] * h_sigma_[0] : (T)0;
            P_.uni_eps = P_.has_lj ? h_eps_[0] : (T)0;
            const double s6 = std::pow((double)h_sigma_[0], 6.0), e0 = P_.has_lj ? (double)h_eps_[0] : 0.0;
            P_.uni_A = (T)(48.0 * e0 * s6 * s6);
            P_.uni_B = (T)(24.0 * e0 * s6);
        }
        total_mass_ = 0;
        for (int64_t i = 0; i < n_; i++) total_mass_ += (double)h_mass_[i];

        // per-atom device arrays (original order)
        const size_t np = (size_t)n_ + 16;
        MB_CUDA(d_mass_in_.ensure(np * sizeof(T)));
        MB_CUDA(d_charge_in_.ensure(np * sizeof(T)));
        MB_CUDA(d_ljp_in_.ensure(np * sizeof(T2)));
        MB_CUDA(cudaMemcpyAsync(d_mass_in_.p, h_mass_.data(), n_ * sizeof(T), cudaMemcpyHostToDevice, stream_));
        // a DPD context's position records carry the original index (exact up to 2^24 in f32: check_dpd) in place of the charge
        std::vector<T> index_w;
        if (dpd_on_) {
            index_w.resize(n_);
            for (int64_t i = 0; i < n_; i++) index_w[i] = (T)i;
        }
        MB_CUDA(cudaMemcpyAsync(d_charge_in_.p, dpd_on_ ? index_w.data() : h_charge_.data(), n_ * sizeof(T), cudaMemcpyHostToDevice, stream_));
        MB_CUDA(cudaMemcpyAsync(d_ljp_in_.p, ljp.data(), n_ * sizeof(T2), cudaMemcpyHostToDevice, stream_));
        MB_CUDA(cudaStreamSynchronize(stream_));  // ljp and index_w are locals
        // slot-order state
        MB_CUDA(d_pos4_.ensure(np * sizeof(T4)));
        MB_CUDA(d_vel4_.ensure(np * sizeof(T4)));
        MB_CUDA(d_f4_.ensure(np * sizeof(T4)));
        MB_CUDA(d_xref4_.ensure(np * sizeof(T4)));
        MB_CUDA(d_lj2_.ensure(np * sizeof(T2)));
        MB_CUDA(d_orig_.ensure(np * sizeof(int)));
        MB_CUDA(d_inv_orig_.ensure(np * sizeof(int)));
        MB_CUDA(d_mass_.ensure(np * sizeof(T)));
        MB_CUDA(cudaMemsetAsync(d_f4_.p, 0, np * sizeof(T4), stream_));
        MB_CUDA(cudaMemsetAsync(d_lj2_.p, 0, np * sizeof(T2), stream_));
        MB_CUDA(cudaMemsetAsync(d_pos4_.p, 0, np * sizeof(T4), stream_));
        MB_CUDA(d_ctl_.ensure(sizeof(Control)));
        MB_CUDA(cudaMemsetAsync(d_ctl_.p, 0, sizeof(Control), stream_));
        MB_CUDA(d_cm_.ensure(sizeof(CmState<T>)));
        MB_CUDA(cudaMemsetAsync(d_cm_.p, 0, sizeof(CmState<T>), stream_));
        MB_CUDA(d_nh_.ensure(sizeof(NhState)));
        MB_CUDA(d_stage_a_.ensure(3 * np * sizeof(T)));
        MB_CUDA(d_stage_b_.ensure(3 * np * sizeof(T)));
        MB_CUDA(d_stage_c_.ensure(3 * np * sizeof(T)));
        MB_CUDA(d_scalars_.ensure(10 * sizeof(T)));  // [pe, vir(9)] of forces_energy
        if (dpd_on_) {
            MB_CUDA(d_vpred4_.ensure(np * sizeof(T4)));
            MB_CUDA(cudaMemsetAsync(d_vpred4_.p, 0, np * sizeof(T4), stream_));
            const DpdArgs<T> da = dpd_args();  // (the buffers it points at are allocated above)
            MB_CUDA(d_dpd_args_.ensure(sizeof(da)));
            MB_CUDA(cudaMemcpy(d_dpd_args_.p, &da, sizeof(da), cudaMemcpyHostToDevice));
        }
        // exclusion CSR
        auto up = [&](DevBuf& b, const std::vector<int>& v) -> cudaError_t {
            if (v.empty()) return cudaSuccess;
            cudaError_t e = b.ensure(v.size() * sizeof(int));
            if (e != cudaSuccess) return e;
            return cudaMemcpy(b.p, v.data(), v.size() * sizeof(int), cudaMemcpyHostToDevice);
        };
        MB_CUDA(up(d_ex_ptr_, ex_ptr_)); MB_CUDA(up(d_ex_idx_, ex_idx_));
        MB_CUDA(up(d_sp_ptr_, sp_ptr_)); MB_CUDA(up(d_sp_idx_, sp_idx_));
        max_special_host_ = 0;
        for (size_t i = 0; i + 1 < sp_ptr_.size(); i++) max_special_host_ = std::max(max_special_host_, sp_ptr_[i + 1] - sp_ptr_[i]);
        const int vvb = (int)((n_ + VV_THREADS - 1) / VV_THREADS);
        MB_CUDA(d_partial_.ensure((size_t)std::max(vvb, 2048) * 8 * sizeof(double)));
        // geometry of the all-pairs path: the box only (no cells, no skin)
        memset(&g_ap_, 0, sizeof(g_ap_));
        for (int d = 0; d < 3; d++) { g_ap_.L[d] = (T)box_[d]; g_ap_.invL[d] = (T)(1.0 / box_[d]); }
        g_ap_.skin_half2 = std::numeric_limits<T>::infinity();
        g_ap_.tric = tric_;
        floor_ = CapFloor();
        have_list_ = false;
        dirty_ = false;
        return MB_OK;
    }

    const int* ex_ptr_dev() const { return ex_ptr_.empty() ? nullptr : d_ex_ptr_.as<int>(); }
    const int* ex_idx_dev() const { return ex_idx_.empty() ? nullptr : d_ex_idx_.as<int>(); }
    const int* sp_ptr_dev() const { return sp_ptr_.empty() ? nullptr : d_sp_ptr_.as<int>(); }
    const int* sp_idx_dev() const { return sp_idx_.empty() ? nullptr : d_sp_idx_.as<int>(); }

    // ------------------------------------------------------------------------------------------
    // geometry / capacity selection for the brick path
    int choose_geometry() {
        Geom<T>& g = g_;
        memset(&g, 0, sizeof(g));
        g.n = (int)n_;
        g.h = 2;
        g.align = 16 / (int)sizeof(T2);
        double vol = 1;
        for (int d = 0; d < 3; d++) {
            g.L[d] = (T)box_[d];
            g.invL[d] = (T)(1.0 / box_[d]);
            g.Ld[d] = box_[d];
            int nc = (int)std::floor(2.0 * box_[d] / r_list_);
            nc = std::max(nc, 5);
            while (nc > 5 && box_[d] / nc < 0.5 * r_list_ * (1.0 + 1e-6)) nc--;
            g.nc[d] = nc;
            g.celld[d] = box_[d] / nc;
            g.inv_cell[d] = (T)(nc / box_[d]);
            vol *= box_[d];
        }
        if ((double)g.nc[0] * g.nc[1] * g.nc[2] > 2.0e8) return set_error(MB_ERR_INVALID, "cell grid too large");
        if (nranks_ > g.nc[2]) return set_error(MB_ERR_INVALID, "more ranks than cell layers along z");
        g.ncells = g.nc[0] * g.nc[1] * g.nc[2];
        g.rlist2 = (T)(r_list_ * r_list_);
        g.skin_half2 = (T)(0.25 * skin_ * skin_);
        const double rho_c = (double)n_ / g.ncells;
        const double bytes_per_atom = sizeof(T4) + (P_.uniform_lj ? 0 : sizeof(T2));
        const double smem_budget = (double)smem_optin_ - 4096;
        int best[3] = {1, 1, 1};
        if (user_b_[0] > 0 && user_b_[1] > 0 && user_b_[2] > 0) {
            for (int d = 0; d < 3; d++) best[d] = std::min(user_b_[d], g.nc[d]);
            if (nranks_ > 1) best[2] = 1;
        } else {
            // Cost model in pair-evaluation units. The persistent force kernel keeps two CTAs per SM busy through a ring of
            // stages (one stage = one brick's halo), so a brick costs its pair work plus a staging share per halo atom and a
            // fixed hand-over cost; smaller bricks balance better across the 2 x n_sm CTAs (dynamic tickets), larger ones
            // stage fewer halo atoms per owned atom. The stage must leave room for at least two of them per CTA.
            const double nbrs = 4.18879 * r_list_ * r_list_ * r_list_ * (double)n_ / vol;
            const double cta_budget = ((double)smem_optin_ + 1024.0) / 2.0 - 3072.0;  // two CTAs share an SM's 228 KB
            const double slots = 2.0 * sm_count_;
            double best_t = 1e300;
            for (int bx = 1; bx <= 8; bx++)
                for (int by = 1; by <= bx; by++)
                    for (int bz = 1; bz <= by; bz++) {
                        if (bx > g.nc[0] || by > g.nc[1] || bz > g.nc[2]) continue;
                        if (nranks_ > 1 && bz != 1) continue;  // slabs are whole cell layers
                        double halo = (bx + 4.0) * (by + 4.0) * (bz + 4.0) * rho_c * 1.25 + 64;
                        double owned = (double)bx * by * bz * rho_c;
                        double smem = halo * bytes_per_atom + owned * 1.3 * 8.0 + 256;
                        if (smem > smem_budget || halo * 1.1 + 96 > LIST_MAX_HALO) continue;
                        const int stages2 = (int)std::floor(cta_budget / smem);  // ring depth with two CTAs per SM
                        double eff = stages2 >= 2 ? 1.0 : (stages2 == 1 ? 0.8 : 0.5);
                        // a stage hands out owned/4 quads to 15 consumer warps: with fewer than ~15 quads in flight over the
                        // ring the warps wait for the producer
                        eff *= std::min(1.0, std::max(1, std::min(stages2, 3)) * (owned / 4.0) / 15.0);
                        double cost_b = owned * nbrs + 6.0 * halo + 2000.0;
                        double nbr = std::ceil((double)g.nc[0] / bx) * std::ceil((double)g.nc[1] / by) * std::ceil((double)g.nc[2] / bz);
                        double t = (std::max(nbr / slots, 1.0) + 1.5) * cost_b / eff;  // + start-up and tail: about a brick and a half
                        if (t < best_t * 0.999) { best_t = t; best[0] = bx; best[1] = by; best[2] = bz; }
                    }
        }
        for (int d = 0; d < 3; d++) {
            g.b[d] = best[d];
            g.nb[d] = (g.nc[d] + g.b[d] - 1) / g.b[d];
            g.H[d] = g.b[d] + 2 * g.h;
        }
        g.nbricks = g.nb[0] * g.nb[1] * g.nb[2];
        for (int d = 0; d < 3; d++) g.nce[d] = g.nc[d] + 2 * g.h;
        g.necells = g.nce[0] * g.nce[1] * g.nce[2];
        g.nerows = g.nce[1] * g.nce[2];
        g.max_runs = g.H[1] * g.H[2];
        g.hcells = g.H[0] * g.H[1] * g.H[2];
        g.n_irows = g.b[1] * g.b[2];
        return MB_OK;
    }

    // geometry of the current path (wrap, ingest, log and export kernels)
    const Geom<T>& geom() const { return path_ == 1 ? g_ : g_ap_; }

    ExtMap<T> ext_map() const {
        ExtMap<T> m;
        m.ext_of = d_ext_of_.as<int>();
        m.gptr = d_gptr_.as<unsigned int>();
        m.ghosts = d_ghosts_.as<int2>();
        m.pos4e = (path_ == 1) ? d_pos4e_.as<T4>() : nullptr;
        for (int d = 0; d < 3; d++) m.Ld[d] = box_[d];
        return m;
    }
    // pos4e <- pos4 for slots [s0, s0 + n) (positions changed outside K1 and outside a rebuild)
    int ext_fill(int s0, int n) {
        if (n <= 0) return MB_OK;
        ext_fill_kernel<T><<<(n + 255) / 256, 256, 0, stream_>>>(ext_map(), s0, n, d_pos4_.as<T4>());
        launches_++;
        MB_CUDA(cudaGetLastError());
        return MB_OK;
    }
    size_t force_stage() const { return force_stage_bytes<T>(g_.halo_cap, g_.task_cap, P_.uniform_lj != 0); }
    // launch shape of the persistent force kernel: ring depth and CTAs per SM from the stage size. Two CTAs per SM when at
    // least one stage each fits (the f64 variants hold 128 registers per thread: one CTA), up to FORCE_MAX_STAGES stages.
    void force_shape(int& nbuf, int& ctas_per_sm) const {
        const size_t stage = force_stage();
        const size_t sm_total = smem_optin_ + 1024;  // 228 KB per SM, 1 KB reserved per resident CTA
        const size_t static_bytes = 1024;
        ctas_per_sm = (sizeof(T) == 8 || dpd_on_) ? 1 : FORCE_CTAS_F32;  // (the DPD variants are compiled for one CTA per SM)
        while (ctas_per_sm > 1 && (sm_total / ctas_per_sm - 1024 - static_bytes) / stage < 1) ctas_per_sm--;
        const size_t budget = (ctas_per_sm > 1) ? sm_total / ctas_per_sm - 1024 - static_bytes : smem_optin_ - static_bytes;
        nbuf = (int)std::min<size_t>(FORCE_MAX_STAGES, std::max<size_t>(1, budget / stage));
    }
    static size_t build_smem_bytes(int halo_cap, int hcells, int n_irows) {
        return (size_t)halo_cap * (sizeof(T4) + sizeof(int)) + (size_t)((hcells + 3) & ~3) * sizeof(ushort2) +
               (size_t)n_irows * sizeof(IRow);
    }
    size_t build_smem_bytes() const { return build_smem_bytes(g_.halo_cap, g_.hcells, g_.n_irows); }
    // shared memory the force kernel (one stage) and the list builder need for bricks of b cells with these capacities
    size_t brick_smem_need(int halo_cap, int task_cap, const int b[3]) const {
        const int hc = (b[0] + 2 * g_.h) * (b[1] + 2 * g_.h) * (b[2] + 2 * g_.h);
        return std::max(force_stage_bytes<T>(halo_cap, task_cap, P_.uniform_lj != 0) + 2048,
                        build_smem_bytes(halo_cap, hc, b[1] * b[2]) + 1024);
    }

    int alloc_brick_tables() {
        const Geom<T>& g = g_;
        MB_CUDA(d_cid_.ensure((size_t)(n_ + 16) * sizeof(int)));
        MB_CUDA(d_perm_.ensure((size_t)(n_ + 16) * sizeof(int)));
        MB_CUDA(d_cell_count_.ensure((size_t)(g.ncells + 2) * sizeof(int)));
        MB_CUDA(d_cell_start_.ensure((size_t)(g.ncells + 2) * sizeof(int)));
        MB_CUDA(d_cell_fill_.ensure((size_t)(g.ncells + 2) * sizeof(int)));
        MB_CUDA(cudaMemsetAsync(d_cell_count_.p, 0, (size_t)(g.ncells + 2) * sizeof(int), stream_));
        MB_CUDA(d_erow_total_.ensure((size_t)(g.nerows + 2) * sizeof(int)));
        MB_CUDA(d_erow_start_.ensure((size_t)(g.nerows + 2) * sizeof(int)));
        MB_CUDA(d_erow_fill_.ensure((size_t)(g.nerows + 2) * sizeof(int)));
        MB_CUDA(d_ecell_start_.ensure((size_t)(g.necells + 2) * sizeof(int)));
        MB_CUDA(d_ext_of_.ensure((size_t)(n_ + 16) * sizeof(int)));
        MB_CUDA(d_gptr_.ensure((size_t)(n_ + 16) * sizeof(unsigned int)));
        MB_CUDA(d_hdrs_.ensure((size_t)g.nbricks * sizeof(BrickHdr)));
        MB_CUDA(d_runs_.ensure((size_t)g.nbricks * g.max_runs * sizeof(Run)));
        MB_CUDA(d_irows_.ensure((size_t)g.nbricks * g.n_irows * sizeof(IRow)));
        MB_CUDA(d_hcs_.ensure((size_t)g.nbricks * g.hcells * sizeof(ushort2)));
        MB_CUDA(d_counts_.ensure((size_t)(n_ + 16) * sizeof(ushort2)));
        const size_t np = (size_t)n_ + 16;
        MB_CUDA(d_pos4_t_.ensure(np * sizeof(T4)));
        MB_CUDA(d_vel4_t_.ensure(np * sizeof(T4)));
        MB_CUDA(d_lj2_t_.ensure(np * sizeof(T2)));
        MB_CUDA(d_orig_t_.ensure(np * sizeof(int)));
        MB_CUDA(d_mass_t_.ensure(np * sizeof(T)));
        MB_CUDA(d_pe_partial_.ensure((size_t)std::max(std::max(g.nbricks, 4 * sm_count_), 1) * 7 * sizeof(double)));
        if (!d_sched_.p) {
            MB_CUDA(d_sched_.ensure(4 * sizeof(unsigned int)));
            MB_CUDA(cudaMemsetAsync(d_sched_.p, 0, 4 * sizeof(unsigned int), stream_));
        }
        return MB_OK;
    }

    // ---- specific (bonded) interaction lists: kind MB_SPECIFIC_*, SPECIFIC_ATOMS / SPECIFIC_PARAMS per term (bonded.cuh)
    int set_specific(int kind, int64_t n, const int32_t* idx, const double* par) override {
        if (kind < 0 || kind >= N_SPECIFIC_KINDS || n < 0 || (n > 0 && (!idx || !par)))
            return set_error(MB_ERR_INVALID, "mb_set_specific: bad arguments");
        if (n_ <= 0) return set_error(MB_ERR_STATE, "mb_set_specific: set atoms first");
        const int na = SPECIFIC_ATOMS[kind], np_ = SPECIFIC_PARAMS[kind];
        std::vector<int> hidx((size_t)n * na);
        std::vector<T> hpar((size_t)n * np_);
        for (int64_t t = 0; t < n * na; t++) {
            int a = idx[t] - 1;  // 1-based in, like InteractionList{1,2,3,4}Atoms (src/types.jl:89-157)
            if (a < 0 || a >= n_) return set_error(MB_ERR_INVALID, "mb_set_specific: atom index out of bounds");
            hidx[t] = a;
        }
        for (int64_t t = 0; t < n * np_; t++) hpar[t] = (T)par[t];
        sp_n_[kind] = n;
        if (n > 0) {
            MB_CUDA(d_sp_idx_k_[kind].ensure(hidx.size() * sizeof(int)));
            MB_CUDA(d_sp_par_k_[kind].ensure(hpar.size() * sizeof(T)));
            MB_CUDA(cudaMemcpy(d_sp_idx_k_[kind].p, hidx.data(), hidx.size() * sizeof(int), cudaMemcpyHostToDevice));
            MB_CUDA(cudaMemcpy(d_sp_par_k_[kind].p, hpar.data(), hpar.size() * sizeof(T), cudaMemcpyHostToDevice));
        }
        h_sp_idx_[kind] = std::move(hidx);  // (kept in the caller's order: mb_set_specific_levels regroups them)
        h_sp_par_[kind] = std::move(hpar);
        h_sp_level_[kind].assign(n, 0);
        for (int l = 0; l <= MTS_MAX_LEVELS; l++) sp_lvl_off_[kind][l] = (l == 0) ? 0 : n;
        int64_t blocks = 0;  // one energy partial per CTA of the bonded launch
        for (int k = 0; k < N_SPECIFIC_KINDS; k++) blocks += (sp_n_[k] + BONDED_THREADS - 1) / BONDED_THREADS;
        MB_CUDA(d_sp_partial_.ensure((size_t)(blocks + 8) * sizeof(double)));
        drop_graphs();  // the graphs bake the term counts in
        return MB_OK;
    }
    // multiple-time-step levels: the device arrays of a kind hold its terms grouped by level (stable), level l in
    // [sp_lvl_off_[kind][l], sp_lvl_off_[kind][l + 1])
    int set_specific_levels(int kind, int64_t n, const int32_t* level) override {
        if (kind < 0 || kind >= N_SPECIFIC_KINDS || n < 0 || (n > 0 && !level))
            return set_error(MB_ERR_INVALID, "mb_set_specific_levels: bad arguments");
        if (n != sp_n_[kind])
            return set_error(MB_ERR_INVALID, "mb_set_specific_levels: " + std::to_string(n) + " levels for " + std::to_string(sp_n_[kind]) +
                                                 " terms of kind " + std::to_string(kind) + " (mb_set_specific)");
        for (int64_t t = 0; t < n; t++)
            if (level[t] < 0 || level[t] >= MTS_MAX_LEVELS)
                return set_error(MB_ERR_INVALID, "mb_set_specific_levels: a level outside 0 .. MB_MTS_MAX_LEVELS - 1");
        if (std::equal(level, level + n, h_sp_level_[kind].begin())) return MB_OK;  // (the captured graphs stay valid)
        const int na = SPECIFIC_ATOMS[kind], np_ = SPECIFIC_PARAMS[kind];
        std::vector<int64_t> order(n);
        for (int64_t t = 0; t < n; t++) order[t] = t;
        std::stable_sort(order.begin(), order.end(), [&](int64_t a, int64_t b) { return level[a] < level[b]; });
        std::vector<int> hidx((size_t)n * na);
        std::vector<T> hpar((size_t)n * np_);
        for (int64_t k = 0; k < n; k++) {
            std::copy_n(&h_sp_idx_[kind][(size_t)order[k] * na], na, &hidx[(size_t)k * na]);
            std::copy_n(&h_sp_par_[kind][(size_t)order[k] * np_], np_, &hpar[(size_t)k * np_]);
        }
        MB_CUDA(cudaMemcpy(d_sp_idx_k_[kind].p, hidx.data(), hidx.size() * sizeof(int), cudaMemcpyHostToDevice));
        MB_CUDA(cudaMemcpy(d_sp_par_k_[kind].p, hpar.data(), hpar.size() * sizeof(T), cudaMemcpyHostToDevice));
        h_sp_level_[kind].assign(level, level + n);
        for (int l = 0; l <= MTS_MAX_LEVELS; l++)
            sp_lvl_off_[kind][l] = std::count_if(level, level + n, [l](int32_t v) { return v < l; });
        drop_graphs();  // the graphs bake the level ranges in
        return MB_OK;
    }
    // the deepest level any term sits at
    int max_specific_level() const {
        int m = 0;
        for (int kind = 0; kind < N_SPECIFIC_KINDS; kind++)
            for (int32_t v : h_sp_level_[kind]) m = std::max(m, (int)v);
        return m;
    }
    bool has_lists() const { return std::any_of(sp_n_, sp_n_ + N_SPECIFIC_KINDS, [](int64_t v) { return v > 0; }); }
    bool has_specific() const { return has_lists() || pme_on_ || gb_on_; }  // everything that is added after the pair kernel
    // the slot of every atom for kernels that index atoms in original order (null: the all-pairs path keeps that order)
    const int* slot_of() const { return path_ == 1 ? d_inv_orig_.as<int>() : nullptr; }
    // add the bonded forces to f4 (slot order on the brick path, original order on the all-pairs path; default d_f4_);
    // with energy: per-kernel partials are summed into d_sp_energy_ (double, device). level: the terms of one
    // multiple-time-step level (PME and GB belong to level 0), or -1 for all of them
    int launch_bonded(bool energy, T4* f4 = nullptr, int level = -1) {
        if (!f4) f4 = d_f4_.as<T4>();
        if (!has_specific() || (level > 0 && !has_lists())) return MB_OK;
        MB_CUDA(d_sp_partial_.ensure(64 * sizeof(double)));  // (set_specific sizes it for the lists; PME alone needs it to exist)
        BoxT bx;
        for (int d = 0; d < 3; d++) bx.L[d] = box_[d];
        if (energy) {
            MB_CUDA(d_sp_energy_.ensure(sizeof(double)));
            MB_CUDA(cudaMemsetAsync(d_sp_energy_.p, 0, sizeof(double), stream_));
        }
        double* part = d_sp_partial_.as<double>();
        BondedLists L;
        L.blk0[0] = 0;
        for (int kind = 0; kind < N_SPECIFIC_KINDS; kind++) {
            const int64_t lo = level < 0 ? 0 : sp_lvl_off_[kind][level], hi = level < 0 ? sp_n_[kind] : sp_lvl_off_[kind][level + 1];
            L.n[kind] = (int)(hi - lo);
            L.blk0[kind + 1] = L.blk0[kind] + (L.n[kind] + BONDED_THREADS - 1) / BONDED_THREADS;
            L.idx[kind] = d_sp_idx_k_[kind].as<int>() + lo * SPECIFIC_ATOMS[kind];
            L.par[kind] = d_sp_par_k_[kind].as<T>() + lo * SPECIFIC_PARAMS[kind];
        }
        const int total_blk = L.blk0[N_SPECIFIC_KINDS];
        if (total_blk > 0) {
            auto go = [&](auto box) {
                with_const<true, false>(energy, [&](auto EN) {
                    bonded_kernel<T, EN, decltype(box)><<<total_blk, BONDED_THREADS, 0, stream_>>>(L, slot_of(), d_pos4_.as<T4>(), f4, box, part);
                });
            };
            if (tric_.on) go(tric_);
            else go(bx);
            launches_++;
            if (energy) {
                sum_partials_kernel<<<1, SUM_THREADS, 0, stream_>>>(total_blk, part, d_sp_energy_.as<double>());
                launches_++;
            }
        }
        MB_CUDA(cudaGetLastError());
        if (pme_on_ && level <= 0) MB_TRY(launch_pme(energy, f4));
        if (gb_on_ && level <= 0) MB_TRY(launch_gb(energy, f4));
        return MB_OK;
    }

    // ---- generalized-Born implicit solvent (gbsa.cuh) -------------------------------------------------------------------
    int set_implicit_solvent(const mb_gbsa_t* p, const double* or_, const double* sr, const double* alpha, const double* beta,
                             const double* gamma, const int32_t* cls, const double* d0, const double* m0) override {
        const std::string who = "mb_set_implicit_solvent: ";
        if (!p) {
            if (gb_on_) drop_graphs();
            gb_on_ = false;
            return MB_OK;
        }
        if (n_ <= 0) return set_error(MB_ERR_STATE, who + "set atoms first");
        if (decomposed()) return set_error(MB_ERR_INVALID, who + "not available in decomposed (multi-GPU) runs");
        const int nc = p->n_neck_classes;
        if (nc < 0 || nc > GB_MAX_CLASSES) return set_error(MB_ERR_INVALID, who + "n_neck_classes outside 0 .. MB_GB_MAX_NECK_CLASSES");
        if (!or_ || !sr || !alpha || !beta || !gamma || (nc > 0 && (!cls || !d0 || !m0))) return set_error(MB_ERR_INVALID, who + "null array");
        const double sc[9] = {p->dist_cutoff, p->offset, p->probe_radius, p->sa_factor, p->factor_solute, p->factor_solvent,
                              p->kappa, p->neck_scale, p->neck_cut};
        for (double v : sc)
            if (!std::isfinite(v)) return set_error(MB_ERR_INVALID, who + "non-finite parameter");
        if (p->dist_cutoff < 0) return set_error(MB_ERR_INVALID, who + "negative dist_cutoff");
        if (p->offset < 0) return set_error(MB_ERR_INVALID, who + "negative offset");
        const int64_t n = n_;
        std::vector<T4> par(n), abg(n);
        for (int64_t i = 0; i < n; i++) {
            const double v[5] = {or_[i], sr[i], alpha[i], beta[i], gamma[i]};
            for (double x : v)
                if (!std::isfinite(x)) return set_error(MB_ERR_INVALID, who + "non-finite per-atom value");
            if (!(or_[i] > 0)) return set_error(MB_ERR_INVALID, who + "an offset radius <= 0");
            const int c = nc > 0 ? cls[i] : 0;
            if (nc > 0 && (c < 0 || c >= nc)) return set_error(MB_ERR_INVALID, who + "a neck class out of range");
            const T o = (T)or_[i];
            par[i] = make4<T>(o, (T)sr[i], o + (T)p->offset, (T)c);  // radius = offset radius + offset, in T as the reference
            abg[i] = make4<T>((T)alpha[i], (T)beta[i], (T)gamma[i], (T)0);
        }
        std::vector<T> tab(2 * (size_t)std::max(nc * nc, 1), (T)0);
        for (int k = 0; k < nc * nc; k++) {
            if (!std::isfinite(d0[k]) || !std::isfinite(m0[k])) return set_error(MB_ERR_INVALID, who + "non-finite d0 / m0");
            tab[k] = (T)d0[k];
            tab[(size_t)nc * nc + k] = (T)m0[k];
        }
        const int nib = (int)((n + GB_THREADS - 1) / GB_THREADS);
        const int tiles = (int)((n + GB_CHUNK - 1) / GB_CHUNK);
        // split j so that the grid holds about four CTAs per SM (1170 atoms: 10 atom blocks alone fill 10 SMs)
        int ns = std::min(tiles, std::max(1, (4 * sm_count_ + nib - 1) / nib));
        gb_chunk_ = ((tiles + ns - 1) / ns) * GB_CHUNK;
        gb_nsplit_ = (int)((n + gb_chunk_ - 1) / gb_chunk_);
        const size_t np = (size_t)n + 16;
        MB_CUDA(d_gb_par_.ensure(np * sizeof(T4)));
        MB_CUDA(d_gb_abg_.ensure(np * sizeof(T4)));
        MB_CUDA(d_gb_tab_.ensure(tab.size() * sizeof(T)));
        MB_CUDA(d_gb_B_.ensure(np * sizeof(T)));
        MB_CUDA(d_gb_b_.ensure(np * sizeof(T)));
        MB_CUDA(d_gb_st_.ensure(np * sizeof(dbl4)));
        MB_CUDA(d_gb_pd_.ensure((size_t)gb_nsplit_ * n * sizeof(double)));
        MB_CUDA(d_gb_pf_.ensure((size_t)gb_nsplit_ * n * sizeof(T4)));
        MB_CUDA(d_gb_pe_.ensure(((size_t)nib * gb_nsplit_ + nib) * sizeof(double)));
        MB_CUDA(d_gb_tk_.ensure(((size_t)nib + 1) * sizeof(unsigned int)));
        MB_CUDA(cudaMemcpy(d_gb_par_.p, par.data(), n * sizeof(T4), cudaMemcpyHostToDevice));
        MB_CUDA(cudaMemcpy(d_gb_abg_.p, abg.data(), n * sizeof(T4), cudaMemcpyHostToDevice));
        MB_CUDA(cudaMemcpy(d_gb_tab_.p, tab.data(), tab.size() * sizeof(T), cudaMemcpyHostToDevice));
        MB_CUDA(cudaMemset(d_gb_tk_.p, 0, ((size_t)nib + 1) * sizeof(unsigned int)));
        GbParams<T>& P = gb_p_;
        memset(&P, 0, sizeof(P));
        P.n = (int)n;
        P.n_cls = nc;
        P.chunk = gb_chunk_;
        P.use_ace = p->use_ace ? 1 : 0;
        P.rc = (T)p->dist_cutoff;
        P.rc2 = (T)(p->dist_cutoff * p->dist_cutoff);
        P.offset = (T)p->offset;
        P.neck_scale = (T)p->neck_scale;
        P.neck_cut = (T)p->neck_cut;
        P.kappa = (T)p->kappa;
        P.f_solute = (T)p->factor_solute;
        P.f_solvent = (T)p->factor_solvent;
        P.offset_d = (double)(T)p->offset;
        P.probe = (double)(T)p->probe_radius;
        P.sa_factor = (double)(T)p->sa_factor;
        gb_n_ = n;
        gb_on_ = true;
        drop_graphs();  // the graphs bake the GB parameters and buffers in
        return MB_OK;
    }
    // the three GB passes into f4 (slot order), with energy added to d_sp_energy_
    int launch_gb(bool energy, T4* f4) {
        if (gb_n_ != n_) return set_error(MB_ERR_STATE, "implicit solvent: the atom count changed since mb_set_implicit_solvent");
        if (decomposed()) return set_error(MB_ERR_INVALID, "implicit solvent: not available in decomposed (multi-GPU) runs");
        GbArgs<T> a;
        a.par = d_gb_par_.as<T4>();
        a.abg = d_gb_abg_.as<T4>();
        a.d0 = d_gb_tab_.as<T>();
        a.m0 = d_gb_tab_.as<T>() + (size_t)gb_p_.n_cls * gb_p_.n_cls;
        a.orig = d_orig_.as<int>();  // (the identity on the all-pairs path)
        a.pos4 = d_pos4_.as<T4>();
        a.f4 = f4;
        a.B = d_gb_B_.as<T>();
        a.b = d_gb_b_.as<T>();
        a.st = d_gb_st_.as<dbl4>();
        a.pd = d_gb_pd_.as<double>();
        a.pf = d_gb_pf_.as<T4>();
        a.pe = d_gb_pe_.as<double>();
        a.tk = d_gb_tk_.as<unsigned int>();
        a.acc = energy ? d_sp_energy_.as<double>() : nullptr;
        const dim3 grid((unsigned)((n_ + GB_THREADS - 1) / GB_THREADS), (unsigned)gb_nsplit_);
        auto go = [&](auto box) {
            using B = decltype(box);
            gb_born_kernel<T, B><<<grid, GB_THREADS, 0, stream_>>>(gb_p_, a, box);
            with_const<true, false>(energy, [&](auto EN) { gb_pair_kernel<T, EN, B><<<grid, GB_THREADS, 0, stream_>>>(gb_p_, a, box); });
            gb_chain_kernel<T, B><<<grid, GB_THREADS, 0, stream_>>>(gb_p_, a, box);
        };
        if (tric_.on) {
            go(tric_);
        } else {
            BoxT bx;
            for (int d = 0; d < 3; d++) bx.L[d] = box_[d];
            go(bx);
        }
        launches_ += 3;
        MB_CUDA(cudaGetLastError());
        return MB_OK;
    }

    // ---- PME reciprocal space + Ewald exclusions (pme.cuh; SURVEY.md §8(f)-3) -------------------------------
    int set_pme(double r_cut, double error_tol, int order, double eps_r, int64_t n_pairs, const int32_t* pi, const int32_t* pj) override {
        if (order == 0) { pme_on_ = false; return MB_OK; }
        if (order != PME_ORDER) return set_error(MB_ERR_INVALID, "mb_set_pme: only B-spline order 5 is implemented (the reference's default)");
        if (!(r_cut > 0) || !(error_tol > 0 && error_tol < 0.5) || !(eps_r > 0) || n_pairs < 0 || (n_pairs > 0 && (!pi || !pj)))
            return set_error(MB_ERR_INVALID, "mb_set_pme: bad arguments");
        if (n_ <= 0) return set_error(MB_ERR_STATE, "mb_set_pme: set atoms first");
        if (!g_cufft.load()) return set_error(MB_ERR_INVALID, "mb_set_pme: libcufft could not be loaded");
        pme_pairs_.resize((size_t)2 * n_pairs);
        for (int64_t k = 0; k < n_pairs; k++) {
            const int a = pi[k] - 1, b = pj[k] - 1;  // 1-based in
            if (a < 0 || b < 0 || a >= n_ || b >= n_) return set_error(MB_ERR_INVALID, "mb_set_pme: pair index out of bounds");
            pme_pairs_[2 * k] = a;
            pme_pairs_[2 * k + 1] = b;
        }
        pme_rc_ = r_cut; pme_tol_ = error_tol; pme_epsr_ = eps_r;
        pme_on_ = true;
        pme_ready_ = false;
        drop_graphs();  // the captured graphs do not contain the PME launches
        return MB_OK;
    }
    // ---- LJDispersionCorrection (general interaction; lennard_jones.jl:163-275) -----------------------------------
    int set_dispersion(double r_cut) override {
        if (r_cut < 0) return set_error(MB_ERR_INVALID, "mb_set_lj_dispersion_correction: negative cutoff");
        disp_rc_ = r_cut;
        disp_ready_ = false;
        return MB_OK;
    }
    // ---- DPDInteraction (dpd.cuh): replaces the pairwise interactions; prepare() digests it and picks the path -------------
    int set_dpd(const mb_dpd_t* p) override {
        const std::string who = "mb_set_dpd: ";
        if (p) {
            if (!(std::isfinite(p->r_c) && p->r_c > 0)) return set_error(MB_ERR_INVALID, who + "r_c must be finite and > 0");
            if (!(std::isfinite(p->dt) && p->dt > 0)) return set_error(MB_ERR_INVALID, who + "dt must be finite and > 0");
            if (!(std::isfinite(p->gamma) && p->gamma >= 0)) return set_error(MB_ERR_INVALID, who + "gamma must be finite and >= 0");
            if (!(std::isfinite(p->sigma) && p->sigma >= 0)) return set_error(MB_ERR_INVALID, who + "sigma must be finite and >= 0");
            if (!std::isfinite(p->a)) return set_error(MB_ERR_INVALID, who + "a must be finite");
            dpd_ = *p;
        }
        if (dpd_on_ || p) dirty_ = true;  // (prepare drops the graphs: they bake the DPD constants in)
        dpd_on_ = p != nullptr;
        return MB_OK;
    }
    // What a DPD context cannot be combined with; checked before every evaluation and simulate call
    int check_dpd() const {
        if (!dpd_on_) return MB_OK;
        const std::string who = "DPDInteraction (mb_set_dpd): ";
        if (!inters_.empty()) return set_error(MB_ERR_INVALID, who + "cannot be combined with other pairwise interactions (mb_set_inters)");
        if (pme_on_ || disp_rc_ > 0 || gb_on_)
            return set_error(MB_ERR_INVALID, who + "cannot be combined with PME, LJDispersionCorrection or implicit solvent");
        if (decomposed()) return set_error(MB_ERR_INVALID, who + "not available in decomposed (multi-GPU) runs");
        if (sizeof(T) == 4 && n_ > (1 << 24))
            return set_error(MB_ERR_INVALID, who + "an f32 context holds at most 2^24 atoms (the position records carry the atom index as a float)");
        return MB_OK;
    }
    // The brick kernel's DPD variant takes the address of its DpdArgs (uploaded by prepare) in place of the LJ parameters it
    // does not stage; dpd_args_of reads it back. Only launch_dpd_pairs passes it.
    const T2* dpd_args_as_lj2e() const { return reinterpret_cast<const T2*>(d_dpd_args_.p); }
    DpdArgs<T> dpd_args() const {
        DpdArgs<T> a;
        memset(&a, 0, sizeof(a));
        if (!dpd_on_) return a;
        a.a = (T)dpd_.a;
        a.gamma = (T)dpd_.gamma;
        a.sigma = (T)dpd_.sigma;
        a.rc = (T)dpd_.r_c;
        a.inv_sqrt_dt = (T)(1.0 / std::sqrt(dpd_.dt));
        a.e_pre = (T)(dpd_.a / 2) * (T)dpd_.r_c;
        a.key_lo = (uint32_t)dpd_.key;
        a.key_hi = (uint32_t)(dpd_.key >> 32);
        a.nl = dpd_.use_neighbors ? 1 : 0;
        a.dissipative = (dpd_.gamma != 0 || dpd_.sigma != 0) ? 1 : 0;
        a.vpred = d_vpred4_.as<T4>();
        a.step = &d_ctl_.as<Control>()->step;
        return a;
    }
    // factor_6 / factor_12 of the constructor (:170-226): means over all i <= j pairs, N (N + 1) / 2 terms, Lorentz sigma
    // and geometric epsilon without the zero shortcut; accumulated in double, grouped by distinct (sigma, eps)
    int dispersion_prepare() {
        if (disp_ready_ || disp_rc_ <= 0) return MB_OK;
        if (n_ <= 0) return set_error(MB_ERR_STATE, "LJ dispersion correction: atoms not set");
        std::map<std::pair<double, double>, double> types;
        for (int64_t i = 0; i < n_; i++) types[{(double)h_sigma_[i], (double)h_eps_raw_[i]}] += 1.0;
        std::vector<std::pair<std::pair<double, double>, double>> tv(types.begin(), types.end());
        double s6 = 0, s12 = 0;
        for (size_t a = 0; a < tv.size(); a++)
            for (size_t b = a; b < tv.size(); b++) {
                const double np = (a == b) ? tv[a].second * (tv[a].second + 1.0) / 2.0 : tv[a].second * tv[b].second;
                const double sig = (tv[a].first.first + tv[b].first.first) / 2.0;
                const double e = std::sqrt(tv[a].first.second * tv[b].first.second);
                const double sg6 = sig * sig * sig * sig * sig * sig;
                s6 += np * e * sg6;
                s12 += np * e * sg6 * sg6;
            }
        const double nd = (double)n_, n_pairs = nd * (nd + 1.0) / 2.0, pi_ = 3.14159265358979323846;
        const double rc3 = disp_rc_ * disp_rc_ * disp_rc_;
        disp_f6_ = 8.0 * pi_ * nd * nd * (-(s6 / n_pairs) / (3.0 * rc3));
        disp_f12_ = 8.0 * pi_ * nd * nd * ((s12 / n_pairs) / (9.0 * rc3 * rc3 * rc3));
        disp_ready_ = true;
        return MB_OK;
    }
    // grid dimensions, B-spline moduli, plan, self energy: ewald.jl:363-421 (constructor) and :947-956
    int pme_prepare() {
        bool same_box = pme_ready_;
        for (int d = 0; d < 3; d++) same_box = same_box && (pme_g_.L[d] == box_[d]);
        if (same_box) return MB_OK;
        std::vector<double> moduli[3];
        pme_plan_host(box_, pme_rc_, pme_tol_, PME_ORDER, &pme_alpha_, pme_g_.K, moduli);
        for (int d = 0; d < 3; d++) {
            pme_g_.L[d] = box_[d];
            MB_CUDA(d_pme_bsm_[d].ensure(moduli[d].size() * sizeof(double)));
            MB_CUDA(cudaMemcpy(d_pme_bsm_[d].p, moduli[d].data(), moduli[d].size() * sizeof(double), cudaMemcpyHostToDevice));
        }
        const size_t total = (size_t)pme_g_.K[0] * pme_g_.K[1] * pme_g_.K[2];
        MB_CUDA(d_pme_grid_.ensure(total * sizeof(T2)));
        const int conv_blk = (int)((total + PME_THREADS - 1) / PME_THREADS);
        const int ex_blk = (int)((pme_pairs_.size() / 2 + PME_THREADS - 1) / PME_THREADS);
        MB_CUDA(d_pme_partial_.ensure((size_t)(conv_blk + ex_blk + 8) * sizeof(double)));
        if (!pme_pairs_.empty()) {
            MB_CUDA(d_pme_pairs_.ensure(pme_pairs_.size() * sizeof(int)));
            MB_CUDA(cudaMemcpy(d_pme_pairs_.p, pme_pairs_.data(), pme_pairs_.size() * sizeof(int), cudaMemcpyHostToDevice));
        }
        if (pme_plan_ >= 0) { g_cufft.Destroy(pme_plan_); pme_plan_ = -1; }
        const int type = (sizeof(T) == 4) ? 0x29 /* CUFFT_C2C */ : 0x69 /* CUFFT_Z2Z */;
        if (g_cufft.Plan3d(&pme_plan_, pme_g_.K[0], pme_g_.K[1], pme_g_.K[2], type) != 0) {
            pme_plan_ = -1;
            return set_error(MB_ERR_CUDA, "cufftPlan3d failed");
        }
        if (g_cufft.SetStream(pme_plan_, stream_) != 0) return set_error(MB_ERR_CUDA, "cufftSetStream failed");
        // self and neutralising-background energy (ewald.jl:947-956)
        double qs = 0, q2 = 0;
        for (int64_t i = 0; i < n_; i++) { qs += (double)h_charge_[i]; q2 += (double)h_charge_[i] * (double)h_charge_[i]; }
        const double f_div = pme_ke_ / pme_epsr_;
        const double V = box_[0] * box_[1] * box_[2];
        const double pi_ = 3.14159265358979323846;
        pme_self_e_ = -f_div * q2 * pme_alpha_ / std::sqrt(pi_) - f_div * pi_ * qs * qs / (2.0 * V * pme_alpha_ * pme_alpha_);
        pme_ready_ = true;
        return MB_OK;
    }
    int launch_pme(bool energy, T4* f4) {
        MB_TRY(pme_prepare());
        const int nb = (int)((n_ + PME_THREADS - 1) / PME_THREADS);
        const size_t total = (size_t)pme_g_.K[0] * pme_g_.K[1] * pme_g_.K[2];
        const int conv_blk = (int)((total + PME_THREADS - 1) / PME_THREADS);
        const int n_ex = (int)(pme_pairs_.size() / 2);
        const int ex_blk = (n_ex + PME_THREADS - 1) / PME_THREADS;
        const double f_div = pme_ke_ / pme_epsr_;
        const double pi_ = 3.14159265358979323846;
        const double factor = pi_ * pi_ / (pme_alpha_ * pme_alpha_);
        const double boxfactor = pi_ * box_[0] * box_[1] * box_[2];
        double* part = d_pme_partial_.as<double>();
        T2* grid = d_pme_grid_.as<T2>();
        MB_CUDA(cudaMemsetAsync(grid, 0, total * sizeof(T2), stream_));
        pme_spread_kernel<T><<<nb, PME_THREADS, 0, stream_>>>((int)n_, pme_g_, d_pos4_.as<T4>(), grid);
        auto fft = [&](int dir) -> int {
            const int rc = (sizeof(T) == 4) ? g_cufft.ExecC2C(pme_plan_, grid, grid, dir) : g_cufft.ExecZ2Z(pme_plan_, grid, grid, dir);
            return rc == 0 ? MB_OK : set_error(MB_ERR_CUDA, "cufftExec failed");
        };
        MB_TRY(fft(-1));
        with_const<true, false>(energy, [&](auto EN) {
            pme_conv_kernel<T, EN><<<conv_blk, PME_THREADS, 0, stream_>>>(pme_g_, f_div, factor, boxfactor, d_pme_bsm_[0].as<double>(),
                                                                         d_pme_bsm_[1].as<double>(), d_pme_bsm_[2].as<double>(), grid, part);
        });
        MB_TRY(fft(1));
        pme_interp_kernel<T><<<nb, PME_THREADS, 0, stream_>>>((int)n_, pme_g_, d_pos4_.as<T4>(), grid, f4);
        launches_ += 3;
        if (n_ex > 0) {
            with_const<true, false>(energy, [&](auto EN) {
                ewald_exclusion_kernel<T, EN><<<ex_blk, PME_THREADS, 0, stream_>>>(n_ex, d_pme_pairs_.as<int>(), slot_of(), d_pos4_.as<T4>(), f4,
                                                                                  pme_g_, pme_alpha_, f_div, part + conv_blk);
            });
            launches_++;
        }
        if (energy) {
            sum_partials_kernel<<<1, SUM_THREADS, 0, stream_>>>(conv_blk + (n_ex > 0 ? ex_blk : 0), part, d_sp_energy_.as<double>());
            add_const_kernel<<<1, 1, 0, stream_>>>(d_sp_energy_.as<double>(), pme_self_e_);
            launches_ += 2;
        }
        MB_CUDA(cudaGetLastError());
        return MB_OK;
    }

    // ---- decomposition helpers --------------------------------------------------------------------------
    bool decomposed() const { return nranks_ > 1; }
    int own_brick0() const { return build_nb_ < 0 ? 0 : build_b0_; }
    int own_nbricks() const { return build_nb_ < 0 ? g_.nbricks : build_nb_; }
    int layer_lo(int q) const { return decomp_layer_lo(q, g_.nc[2], nranks_); }
    // slot ranges and halo segments follow from the cell layer offsets of the current sort (host copy)
    int decomposed_interval() const { return rebuild_every_ > 0 ? rebuild_every_ : auto_every_; }
    int update_ownership() {
        own_valid_ = true;
        const int ncz = g_.nc[2], per_layer = g_.nc[0] * g_.nc[1];
        layer_start_.resize(ncz + 1);
        MB_CUDA(d_layer_start_.ensure((size_t)(ncz + 1) * sizeof(int)));
        MB_CUDA(cudaMemcpy2DAsync(d_layer_start_.p, sizeof(int), d_cell_start_.p, (size_t)per_layer * sizeof(int), sizeof(int),
                                  (size_t)ncz + 1, cudaMemcpyDeviceToDevice, stream_));
        MB_CUDA(cudaMemcpyAsync(layer_start_.data(), d_layer_start_.p, (size_t)(ncz + 1) * sizeof(int), cudaMemcpyDeviceToHost, stream_));
        MB_CUDA(cudaStreamSynchronize(stream_));
        const int nbxy = g_.nb[0] * g_.nb[1];
        own_b0_ = layer_lo(rank_) * nbxy;
        own_nb_ = (layer_lo(rank_ + 1) - layer_lo(rank_)) * nbxy;
        own_s0_ = layer_start_[layer_lo(rank_)];
        own_n_ = layer_start_[layer_lo(rank_ + 1)] - own_s0_;
        decomp_plan(ncz, g_.h, nranks_, rank_, layer_start_.data(), halo_send_, halo_recv_);
        // The peer-memory transport carries at most MB_MAX_SEG segments / peers per rank. Whether the plan fits must be
        // the same answer on every rank and every step, so it is evaluated for all ranks on unit-sized layers
        // (the segment structure depends only on ncz, h and the rank count).
        if (plan_key_[0] != ncz || plan_key_[1] != g_.h || plan_key_[2] != nranks_) {
            plan_key_[0] = ncz; plan_key_[1] = g_.h; plan_key_[2] = nranks_;
            std::vector<int> unit(ncz + 1);
            for (int l = 0; l <= ncz; l++) unit[l] = l;
            plan_fits_ = nranks_ <= MB_MAX_RANKS;
            std::vector<DecompSeg> sd, rv;
            std::vector<int> a, b;
            for (int q = 0; q < nranks_ && plan_fits_; q++) {
                decomp_plan(ncz, g_.h, nranks_, q, unit.data(), sd, rv);
                distinct_peers(sd, a);
                distinct_peers(rv, b);
                if ((int)sd.size() > MB_MAX_SEG || (int)a.size() > MB_MAX_SEG || (int)b.size() > MB_MAX_SEG) plan_fits_ = false;
            }
        }
        return MB_OK;
    }
    bool p2p_active() const { return p2p_ && plan_fits_; }
    // Decomposed runs rebuild at a fixed interval (every rank must take the same branch without a host round trip).
    // The interval for the NEXT call is derived from the largest displacement any interval of this call reached:
    // n_next = 0.8 * n * (skin/2) / d_max, agreed between ranks with one max-all-reduce. Violations are still counted.
    int adapt_interval() {
        // largest displacement any rebuild interval of this call reached (device) -> max over ranks -> host; the only host
        // wait is the one the end of the call has anyway
        float* dbuf = reinterpret_cast<float*>(d_mom_.as<double>() + 7);
        max_disp_kernel<<<1, 1, 0, stream_>>>(d_ctl_.as<Control>(), dbuf);
        launches_++;
        MB_NCCL(g_nccl.AllReduce(dbuf, dbuf, 1, (ncclDataType_t)7 /* ncclFloat32 */, (ncclRedOp_t)2 /* ncclMax */, comm_, stream_));
        float d2 = 0.f;
        MB_CUDA(cudaMemcpyAsync(&d2, dbuf, sizeof(float), cudaMemcpyDeviceToHost, stream_));
        MB_CUDA(cudaStreamSynchronize(stream_));
        if (d2 > 0.f && skin_ > 0) {
            // d2 was reached within adapt_span_ steps of a rebuild; displacements grow at most linearly in time
            double n_next = 0.8 * std::max(adapt_span_, 1) * (0.5 * skin_) / std::sqrt((double)d2);
            auto_every_ = (int)std::min(400.0, std::max(5.0, std::floor(n_next)));
        }
        return MB_OK;
    }
    // forward halo exchange of positions (x, y, z, q as 16/32-byte records): grouped NCCL send/recv between slabs
    int halo_exchange() {
        MB_NCCL(g_nccl.GroupStart());
        for (auto& sg : halo_send_)
            if (sg.count > 0) MB_NCCL(g_nccl.Send(d_pos4_.as<T4>() + sg.start, (size_t)sg.count * sizeof(T4), ncclChar, sg.peer, comm_, stream_));
        for (auto& sg : halo_recv_)
            if (sg.count > 0) MB_NCCL(g_nccl.Recv(d_pos4_.as<T4>() + sg.start, (size_t)sg.count * sizeof(T4), ncclChar, sg.peer, comm_, stream_));
        MB_NCCL(g_nccl.GroupEnd());
        for (auto& sg : halo_recv_) MB_TRY(ext_fill(sg.start, sg.count));  // received slots -> extended array (+ ghost copies)
        return MB_OK;
    }
    // replicate the owned segments of positions and velocities on every rank (rebuild / export)
    int allgather_state() {
        MB_NCCL(g_nccl.GroupStart());
        for (int q = 0; q < nranks_; q++) {
            const int st = layer_start_[layer_lo(q)], cnt = layer_start_[layer_lo(q + 1)] - st;
            if (cnt <= 0) continue;
            MB_NCCL(g_nccl.Broadcast(d_pos4_.as<T4>() + st, d_pos4_.as<T4>() + st, (size_t)cnt * sizeof(T4), ncclChar, q, comm_, stream_));
            MB_NCCL(g_nccl.Broadcast(d_vel4_.as<T4>() + st, d_vel4_.as<T4>() + st, (size_t)cnt * sizeof(T4), ncclChar, q, comm_, stream_));
        }
        MB_NCCL(g_nccl.GroupEnd());
        return MB_OK;
    }
    // ---- peer-memory transport (peer.cuh) -------------------------------------------------------------------
    void p2p_close() {
        for (int r = 0; r < (int)peer_pos_.size(); r++) {
            if (r == rank_) continue;
            if (peer_pos_[r]) cudaIpcCloseMemHandle(peer_pos_[r]);
            if (peer_comm_[r]) cudaIpcCloseMemHandle(peer_comm_[r]);
        }
        peer_pos_.clear();
        peer_comm_.clear();
        p2p_ = false;
        p2p_pos_base_ = nullptr;
    }
    // Collective: every rank exports its position array and its PeerComm block as CUDA IPC handles, the handles travel
    // by one ncclAllGather, and every rank maps the others'. Any failure on any rank (no peer access, IPC not permitted
    // in this container, too many ranks) leaves ALL ranks on the NCCL transport.
    int p2p_setup() {
        if (p2p_pos_base_ == d_pos4e_.p && !peer_pos_.empty()) return MB_OK;  // mapping is current
        p2p_close();
        p2p_pos_base_ = d_pos4e_.p;
        peer_pos_.assign(nranks_, nullptr);
        peer_comm_.assign(nranks_, nullptr);
        const char* env = getenv("MOLLYB200_P2P");
        int ok = !(env && env[0] == '0') && nranks_ <= MB_MAX_RANKS;
        struct Rec { cudaIpcMemHandle_t pos, comm; };
        static_assert(sizeof(Rec) == 128, "two 64-byte IPC handles");
        // 2 MiB so the block is an allocation of its own; zeroed before any peer can learn its address
        MB_CUDA(d_comm_.ensure(2u << 20));
        MB_CUDA(cudaMemsetAsync(d_comm_.p, 0, sizeof(PeerComm), stream_));
        const unsigned long long magic = 0x6d62323030ull + (unsigned long long)rank_;
        MB_CUDA(cudaMemcpyAsync(reinterpret_cast<char*>(d_comm_.p) + offsetof(PeerComm, magic), &magic, sizeof(magic),
                                cudaMemcpyHostToDevice, stream_));
        Rec mine;
        memset(&mine, 0, sizeof(mine));
        if (ok && cudaIpcGetMemHandle(&mine.pos, d_pos4e_.p) != cudaSuccess) { ok = 0; cudaGetLastError(); }
        if (ok && cudaIpcGetMemHandle(&mine.comm, d_comm_.p) != cudaSuccess) { ok = 0; cudaGetLastError(); }
        MB_CUDA(d_ipc_.ensure((size_t)(nranks_ + 1) * sizeof(Rec) + 16));
        Rec* d_all = d_ipc_.as<Rec>();
        MB_CUDA(cudaMemcpyAsync(d_all + nranks_, &mine, sizeof(Rec), cudaMemcpyHostToDevice, stream_));
        MB_NCCL(g_nccl.AllGather(d_all + nranks_, d_all, sizeof(Rec), ncclChar, comm_, stream_));
        std::vector<Rec> all(nranks_);
        MB_CUDA(cudaMemcpyAsync(all.data(), d_all, (size_t)nranks_ * sizeof(Rec), cudaMemcpyDeviceToHost, stream_));
        MB_CUDA(cudaStreamSynchronize(stream_));
        for (int r = 0; r < nranks_ && ok; r++) {
            if (r == rank_) { peer_pos_[r] = d_pos4e_.p; peer_comm_[r] = d_comm_.p; continue; }
            if (cudaIpcOpenMemHandle(&peer_pos_[r], all[r].pos, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess ||
                cudaIpcOpenMemHandle(&peer_comm_[r], all[r].comm, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
                ok = 0;
                cudaGetLastError();
                break;
            }
            unsigned long long got = 0;  // the mapping must show the owner's tag
            if (cudaMemcpy(&got, reinterpret_cast<char*>(peer_comm_[r]) + offsetof(PeerComm, magic), sizeof(got),
                           cudaMemcpyDeviceToHost) != cudaSuccess || got != 0x6d62323030ull + (unsigned long long)r) {
                ok = 0;
                cudaGetLastError();
            }
        }
        // agree: min over ranks
        float okf = (float)ok;
        float* dbuf = reinterpret_cast<float*>(reinterpret_cast<char*>(d_ipc_.p) + (size_t)(nranks_ + 1) * sizeof(Rec));
        MB_CUDA(cudaMemcpyAsync(dbuf, &okf, sizeof(float), cudaMemcpyHostToDevice, stream_));
        MB_NCCL(g_nccl.AllReduce(dbuf, dbuf, 1, (ncclDataType_t)7 /* ncclFloat32 */, (ncclRedOp_t)3 /* ncclMin */, comm_, stream_));
        MB_CUDA(cudaMemcpyAsync(&okf, dbuf, sizeof(float), cudaMemcpyDeviceToHost, stream_));
        MB_CUDA(cudaStreamSynchronize(stream_));
        if (okf < 0.5f) {
            void* keep = p2p_pos_base_;
            p2p_close();
            p2p_pos_base_ = keep;            // do not retry on every call
            peer_pos_.assign(nranks_, nullptr);
            return MB_OK;
        }
        p2p_ = true;
        return MB_OK;
    }
    PeerComm* comm_of(int r) const { return reinterpret_cast<PeerComm*>(peer_comm_[r]); }
    // distinct peers of a segment list, in first-appearance order
    static void distinct_peers(const std::vector<DecompSeg>& v, std::vector<int>& out) {
        out.clear();
        for (auto& sg : v)
            if (sg.count > 0 && std::find(out.begin(), out.end(), sg.peer) == out.end()) out.push_back(sg.peer);
    }
    PeerPush<T> make_push(unsigned long long epoch, bool with_data) const {
        PeerPush<T> ps;
        memset(&ps, 0, sizeof(ps));
        ps.epoch = epoch;
        std::vector<int> peers;
        distinct_peers(halo_send_, peers);
        if (with_data)
            for (auto& sg : halo_send_) {
                if (sg.count <= 0) continue;
                ps.start[ps.n_seg] = sg.start;
                ps.count[ps.n_seg] = sg.count;
                ps.dst[ps.n_seg] = reinterpret_cast<T4*>(peer_pos_[sg.peer]);
                ps.n_seg++;
            }
        for (int q : peers) {
            ps.wait_flag[ps.n_peer] = &comm_of(rank_)->read_epoch[q];
            ps.signal_flag[ps.n_peer] = &comm_of(q)->halo_epoch[rank_];
            ps.n_peer++;
        }
        return ps;
    }
    PeerWait make_wait(unsigned long long epoch) const {
        PeerWait w;
        memset(&w, 0, sizeof(w));
        w.epoch = epoch;
        std::vector<int> peers;
        distinct_peers(halo_recv_, peers);
        for (int q : peers) w.flag[w.n++] = &comm_of(rank_)->halo_epoch[q];
        return w;
    }
    PeerSignal make_signal(unsigned long long epoch, bool with_mom) const {
        PeerSignal sg;
        memset(&sg, 0, sizeof(sg));
        sg.epoch = epoch;
        std::vector<int> peers;
        distinct_peers(halo_recv_, peers);
        for (int q : peers) sg.read_flag[sg.n_peer++] = &comm_of(q)->read_epoch[rank_];
        if (with_mom) {
            const int par = (int)(epoch & 1ull);
            sg.n_mom = nranks_;
            for (int r = 0; r < nranks_; r++) {
                sg.mom_dst[r] = comm_of(r)->mom[par][rank_];
                sg.mom_flag[r] = &comm_of(r)->mom_epoch[par][rank_];
            }
        }
        return sg;
    }

    int comm_init(const void* uid, int rank, int nranks) override {
        if (nranks < 1 || rank < 0 || rank >= nranks || !uid) return set_error(MB_ERR_INVALID, "mb_comm_init: bad arguments");
        if (!g_nccl.load()) return set_error(MB_ERR_INVALID, "mb_comm_init: libnccl.so.2 could not be loaded");
        p2p_close();
        if (comm_) { g_nccl.CommDestroy(comm_); comm_ = nullptr; }
        rank_ = rank;
        nranks_ = nranks;
        if (nranks > 1) {
            ncclUniqueId id;
            memcpy(&id, uid, sizeof(id));
            MB_NCCL(g_nccl.CommInitRank(&comm_, nranks, id, rank));
            MB_CUDA(d_mom_.ensure(8 * sizeof(double)));
        }
        have_list_ = false;
        dirty_ = true;
        return MB_OK;
    }

    // launch the list builder (count-only or real; with or without exclusion handling)
    int launch_build(bool count_only) {
        const size_t smem = build_smem_bytes();
        const bool has_ex = !ex_ptr_.empty() || !sp_ptr_.empty();
        MB_TRY((with_const<true, false>(count_only, [&](auto CO) { return with_const<true, false>(has_ex, [&](auto EX) -> int {
            auto kern = build_lists_kernel<T, CO, EX>;
            MB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            // few bricks (small systems, narrow slabs): several CTAs share a brick's atoms so that the SMs are filled
            const int split = std::max(1, std::min(4, (4 * sm_count_ + own_nbricks() - 1) / std::max(own_nbricks(), 1)));
            kern<<<own_nbricks() * split, 256, smem, stream_>>>(d_ctl_.as<Control>(), g_, d_hdrs_.as<BrickHdr>(), d_runs_.as<Run>(),
                                                     d_irows_.as<IRow>(), d_hcs_.as<ushort2>(), d_pos4e_.as<T4>(), d_orig_e_.as<int>(),
                                                     ex_ptr_dev(), ex_idx_dev(), sp_ptr_dev(), sp_idx_dev(),
                                                     count_only ? nullptr : d_list_.as<unsigned short>(),
                                                     count_only ? nullptr : d_slist_.as<unsigned short>(),
                                                     count_only ? nullptr : d_counts_.as<ushort2>(),
                                                     count_only ? nullptr : d_task_tab_.as<int2>(), own_brick0(), split);
            return MB_OK;
        }); })));
        launches_++;
        MB_CUDA(cudaGetLastError());
        return MB_OK;
    }

    // enqueue the gated rebuild sequence. count_only: first pass of the capacity derivation.
    int enqueue_rebuild(bool lists, bool count_only) {
        const Geom<T>& g = g_;
        Control* ctl = d_ctl_.as<Control>();
        const int nb = (int)((n_ + 255) / 256);
        prof_.begin(Prof::REBUILD);
        rebuild_begin_kernel<<<1, 32, 0, stream_>>>(ctl);
        bin_count_kernel<T><<<nb, 256, 0, stream_>>>(ctl, g, d_pos4_.as<T4>(), d_cid_.as<int>(), d_cell_count_.as<int>());
        cell_scan_kernel<<<1, 1024, 0, stream_>>>(ctl, g.ncells, g.n, d_cell_count_.as<int>(), d_cell_start_.as<int>(),
                                                  d_cell_fill_.as<int>());
        cell_scatter_kernel<<<nb, 256, 0, stream_>>>(ctl, g.n, d_cid_.as<int>(), d_cell_start_.as<int>(),
                                                     d_cell_fill_.as<int>(), d_perm_.as<int>());
        cell_sort_kernel<<<(g.ncells + 127) / 128, 128, 0, stream_>>>(ctl, g.ncells, d_cell_start_.as<int>(),
                                                                     d_perm_.as<int>(), d_cell_count_.as<int>());
        permute_gather_kernel<T><<<nb, 256, 0, stream_>>>(ctl, g.n, d_perm_.as<int>(), d_pos4_.as<T4>(), d_vel4_.as<T4>(),
                                                         d_lj2_.as<T2>(), d_orig_.as<int>(), d_mass_.as<T>(),
                                                         d_pos4_t_.as<T4>(), d_vel4_t_.as<T4>(), d_lj2_t_.as<T2>(),
                                                         d_orig_t_.as<int>(), d_mass_t_.as<T>());
        permute_commit_kernel<T><<<nb, 256, 0, stream_>>>(ctl, g.n, d_pos4_t_.as<T4>(), d_vel4_t_.as<T4>(), d_lj2_t_.as<T2>(),
                                                         d_orig_t_.as<int>(), d_mass_t_.as<T>(), d_pos4_.as<T4>(),
                                                         d_vel4_.as<T4>(), d_lj2_.as<T2>(), d_orig_.as<int>(), d_mass_.as<T>(),
                                                         d_xref4_.as<T4>(), d_inv_orig_.as<int>());
        // extended (ghost-padded) grid: row totals -> row starts (scan) -> cell starts -> per-atom map + ghost copies
        ext_row_totals_kernel<T><<<(g.nerows + 255) / 256, 256, 0, stream_>>>(ctl, g, d_cell_start_.as<int>(), d_erow_total_.as<int>());
        cell_scan_kernel<<<1, 1024, 0, stream_>>>(ctl, g.nerows, -1, d_erow_total_.as<int>(), d_erow_start_.as<int>(),
                                                  d_erow_fill_.as<int>());
        ext_cells_kernel<T><<<(g.necells + 1 + 255) / 256, 256, 0, stream_>>>(ctl, g, d_cell_start_.as<int>(), d_erow_start_.as<int>(),
                                                                            d_ecell_start_.as<int>());
        ext_atoms_kernel<T><<<nb, 256, 0, stream_>>>(ctl, g, d_cell_start_.as<int>(), d_ecell_start_.as<int>(), d_pos4_.as<T4>(),
                                                     P_.uniform_lj ? nullptr : d_lj2_.as<T2>(), d_ext_of_.as<int>(),
                                                     d_gptr_.as<unsigned int>(), d_ghosts_.as<int2>(), d_pos4e_.as<T4>(),
                                                     P_.uniform_lj ? nullptr : d_lj2e_.as<T2>(), d_orig_.as<int>(),
                                                     (ex_ptr_.empty() && sp_ptr_.empty()) ? nullptr : d_orig_e_.as<int>());
        brick_tables_kernel<T><<<g.nbricks, 128, 2 * g.max_runs * sizeof(int), stream_>>>(
            ctl, g, d_cell_start_.as<int>(), d_ecell_start_.as<int>(), d_hdrs_.as<BrickHdr>(), d_runs_.as<Run>(), d_irows_.as<IRow>(),
            d_hcs_.as<ushort2>(), g.task_cap > 0 ? d_task_tab_.as<int2>() : nullptr, P_.uniform_lj);
        launches_ += 12;
        if (lists) MB_TRY(launch_build(count_only));
        if (!count_only) {
            rebuild_finish_kernel<<<1, 32, 0, stream_>>>(ctl);
            launches_ += 1;
        }
        prof_.end(Prof::REBUILD);
        MB_CUDA(cudaGetLastError());
        return MB_OK;
    }

    int read_ctl(Control& c) {
        MB_CUDA(cudaMemcpyAsync(&c, d_ctl_.p, sizeof(Control), cudaMemcpyDeviceToHost, stream_));
        MB_CUDA(cudaStreamSynchronize(stream_));
        return MB_OK;
    }
    int set_flag_rebuild() {
        static const int one = 1;
        MB_CUDA(cudaMemcpyAsync(&d_ctl_.as<Control>()->rebuild, &one, sizeof(int), cudaMemcpyHostToDevice, stream_));
        return MB_OK;
    }

    // slot-order state from coords_dev (n x 3 device array) in original order, with identity slots
    void init_slots(const T* coords_dev) {
        init_slots_kernel<T><<<(int)((n_ + 255) / 256), 256, 0, stream_>>>((int)n_, coords_dev, d_charge_in_.as<T>(), d_ljp_in_.as<T2>(),
                                                                           d_mass_in_.as<T>(), d_pos4_.as<T4>(), d_vel4_.as<T4>(),
                                                                           d_lj2_.as<T2>(), d_orig_.as<int>(), d_inv_orig_.as<int>(),
                                                                           d_mass_.as<T>(), d_xref4_.as<T4>());
        launches_++;
    }
    // Synchronous first build: derives halo capacity and list stride from the actual configuration.
    // coords_dev: n x 3 device array in original order.
    int first_build(const T* coords_dev) {
        build_nb_ = -1;  // lists for every brick (capacities are global; mb_forces evaluates the whole box)
        own_valid_ = false;
        init_slots(coords_dev);
        static const int zeros[5] = {0, 0, 0, 0, 0};  // peak_ghost .. peak_neighbors
        MB_CUDA(cudaMemcpyAsync(&d_ctl_.as<Control>()->peak_ghost, zeros, sizeof(zeros), cudaMemcpyHostToDevice, stream_));
        for (;;) {  // ends: every retry makes the brick smaller, and a single cell that does not fit is refused
            MB_TRY(choose_geometry());
            drop_graphs();  // they bake in the geometry and the list buffers sized for it
            MB_TRY(alloc_brick_tables());
            // pass A: sort + tables with unlimited halo capacity to measure
            g_.halo_cap = 65535;
            g_.stride = 0;
            g_.sstride = 0;
            g_.task_cap = 0;
            g_.ext_cap = 0;
            g_.ghost_cap = 0;
            MB_TRY(set_flag_rebuild());
            MB_TRY(enqueue_rebuild(false, true));
            Control c;
            MB_TRY(read_ctl(c));
            // measured sizes, but at least those of a rebuild that overflowed the previous capacities (floor_)
            const int hvol = g_.hcells, bvol = g_.b[0] * g_.b[1] * g_.b[2];
            const double max_halo = std::max((double)c.max_halo, std::ceil(floor_.halo_per_hcell * hvol));
            const double max_icount = std::max((double)c.max_icount, std::ceil(floor_.icount_per_cell * bvol));
            int cap = (int)(max_halo * (1.0 + 0.08 * cap_scale_)) + 32;  // temporal drift of the fullest brick's halo
            cap = (cap + 63) & ~63;
            g_.halo_cap = std::min(cap, LIST_MAX_HALO);
            g_.task_cap = (((int)(max_icount * (1.0 + 0.08 * cap_scale_)) + 8) + 1) & ~1;  // even: 16-byte rows for the bulk copy
            if (cap > LIST_MAX_HALO || brick_smem_need(g_.halo_cap, g_.task_cap, g_.b) > smem_optin_) {
                // List entries are 16-bit byte offsets of float4 records, and a stage must fit in shared memory. Pick the
                // next brick from the measurement: the fullest halo's atoms per halo cell (and the fullest brick's owned
                // atoms per cell) times the cells of a smaller brick, shrinking its largest dimension until that fits.
                if (g_.b[0] == 1 && g_.b[1] == 1 && g_.b[2] == 1)
                    return set_error(MB_ERR_CAPACITY, "halo of a single cell does not fit in shared memory (density too high for r_list)");
                const double per_hcell = (double)cap / hvol, per_cell = (double)g_.task_cap / bvol;
                int cur[3] = {g_.b[0], g_.b[1], g_.b[2]};
                for (;;) {
                    int dmax = 0;
                    for (int d = 1; d < 3; d++) if (cur[d] > cur[dmax]) dmax = d;
                    cur[dmax]--;
                    if (cur[0] == 1 && cur[1] == 1 && cur[2] == 1) break;
                    const int hc = (cur[0] + 2 * g_.h) * (cur[1] + 2 * g_.h) * (cur[2] + 2 * g_.h);
                    const int est_cap = ((int)std::ceil(per_hcell * hc) + 63) & ~63;
                    const int est_task = ((int)std::ceil(per_cell * cur[0] * cur[1] * cur[2]) + 1) & ~1;
                    if (est_cap <= LIST_MAX_HALO && brick_smem_need(est_cap, est_task, cur) <= smem_optin_) break;
                }
                for (int d = 0; d < 3; d++) user_b_[d] = cur[d];
                continue;
            }
            MB_CUDA(d_task_tab_.ensure((size_t)g_.nbricks * g_.task_cap * sizeof(int2)));
            // extended array / ghost table: measured sizes plus room for the boundary cells' population to drift
            const double n_ext = std::max((double)c.n_ext, (double)floor_.ext);
            const double n_ghost = std::max((double)c.n_ghost, (double)floor_.ghost);
            g_.ext_cap = (int)std::min<double>(2.0e9, n_ext + (n_ext - (double)n_) * 0.10 * cap_scale_ + 1024);
            g_.ghost_cap = (int)std::min<double>(2.6e8, n_ghost * (1.0 + 0.10 * cap_scale_) + 1024);
            MB_CUDA(d_pos4e_.ensure(((size_t)g_.ext_cap + 64) * sizeof(T4)));
            MB_CUDA(cudaMemsetAsync(d_pos4e_.p, 0, ((size_t)g_.ext_cap + 64) * sizeof(T4), stream_));
            if (!P_.uniform_lj) {
                MB_CUDA(d_lj2e_.ensure(((size_t)g_.ext_cap + 64) * sizeof(T2)));
                MB_CUDA(cudaMemsetAsync(d_lj2e_.p, 0, ((size_t)g_.ext_cap + 64) * sizeof(T2), stream_));
            }
            if (!(ex_ptr_.empty() && sp_ptr_.empty())) MB_CUDA(d_orig_e_.ensure(((size_t)g_.ext_cap + 64) * sizeof(int)));
            MB_CUDA(d_ghosts_.ensure(((size_t)g_.ghost_cap + 64) * sizeof(int2)));
            // pass B: the pipeline again (idempotent: the positions are sorted) now that the extended array exists, with the
            // list builder only counting neighbours (the rebuild flag is still set because finish did not run)
            MB_TRY(enqueue_rebuild(true, true));
            MB_TRY(read_ctl(c));
            int stride = (int)(std::max(c.max_neighbors, floor_.neighbors) * (1.0 + 0.10 * cap_scale_)) + 16;
            stride = (stride + 31) & ~31;
            g_.stride = std::max(stride, 32);
            g_.sstride = std::max(8, (std::max(c.max_special, max_special_host_) + 7) & ~7);
            if (g_.stride > TASK_MAX_MAIN || g_.sstride > TASK_MAX_SPECIAL)
                return set_error(MB_ERR_CAPACITY, "neighbour rows longer than 4095 entries (or more than 255 special partners) are not supported");
            MB_CUDA(d_list_.ensure((size_t)(n_ + 16) * g_.stride * sizeof(unsigned short)));
            MB_CUDA(d_slist_.ensure((size_t)(n_ + 16) * g_.sstride * sizeof(unsigned short)));
            // pass C: the real build. The positions are already sorted; the pipeline is idempotent.
            MB_TRY(enqueue_rebuild(true, false));
            MB_TRY(read_ctl(c));
            if (c.overflow) return set_error(MB_ERR_CAPACITY, "neighbour capacity overflow during first build");
            have_list_ = true;
            if (decomposed()) {
                MB_TRY(update_ownership());
                since_rebuild_ = 0;
            }
            return MB_OK;
        }
    }

    // ------------------------------------------------------------------------------------------
    // energy/virial partials of a pair-force launch: pe[n], vir[6 n] (read by reduce_partials_kernel and log_kernel)
    struct Partials { const double *pe, *vir; int n; };
    // Pair forces of the current path (all-pairs or brick kernel) into f4, with energy and virial partials when `energy`
    // (returned through `parts`). owned_only: in a decomposed run the step loop evaluates only this rank's slab of bricks.
    int launch_pairs(bool energy, T4* f4, bool owned_only = false, Partials* parts = nullptr) {
        ForceOut<T> out = {};
        int grid, vir_at, nbuf = 0, per_sm, nbr = 0, b0 = 0;
        size_t smem = 0;
        if (path_ == 0) {
            grid = vir_at = (int)((n_ + AP_THREADS - 1) / AP_THREADS);
            MB_CUDA(d_pe_partial_.ensure((size_t)grid * 7 * sizeof(double)));
        } else {
            b0 = owned_only ? own_b0_ : 0;
            nbr = owned_only ? own_nb_ : g_.nbricks;
            force_shape(nbuf, per_sm);
            smem = (size_t)nbuf * force_stage();
            grid = std::max(1, std::min(nbr, per_sm * sm_count_));
            vir_at = std::max(g_.nbricks, 4 * sm_count_);  // (alloc_brick_tables sizes the partials for any grid)
            out.f4 = f4;
            out.gate = gate_;  // one-shot: set by the decomposed step in front of this launch
            memset(&gate_, 0, sizeof(gate_));
        }
        out.pe_partial = d_pe_partial_.as<double>();
        out.vir_partial = out.pe_partial + vir_at;
        if (dpd_on_) {
            MB_TRY(launch_dpd_pairs(energy, f4, out, grid, smem, nbuf, b0, nbr));
        } else {
        MB_TRY((with_const<COUL_NONE, COUL_PLAIN, COUL_CRF, COUL_EWALD>(P_.coul_kind, [&](auto COUL) {
            return with_const<CUTM_TWO_POINT, CUTM_SHIFTED, CUTM_PLAIN>(cutm_, [&](auto CUTM) {
                return with_const<true, false>(energy, [&](auto EN) -> int {
                    if (path_ == 0) {
                        prof_.begin(Prof::FORCE);
                        allpairs_force_kernel<T, COUL, CUTM, EN><<<grid, AP_THREADS, 0, stream_>>>(
                            (int)n_, P_, (T)box_[0], (T)box_[1], (T)box_[2], tric_, d_pos4_.as<T4>(), d_lj2_.as<T2>(), ex_ptr_dev(),
                            ex_idx_dev(), sp_ptr_dev(), sp_idx_dev(), f4, out.pe_partial, out.vir_partial, DpdArgs<T>{});
                        prof_.end(Prof::FORCE);
                        return MB_OK;
                    }
                    // the uniform-LJ variants exist only without Coulomb (prepare sets uniform_lj only then)
                    return with_const<COUL == COUL_NONE, false>(P_.uniform_lj != 0, [&](auto UNI) -> int {
                        auto kern = brick_force_kernel<T, COUL, UNI, CUTM, EN>;
                        MB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                        prof_.begin(Prof::FORCE);
                        kern<<<grid, FORCE_THREADS, smem, stream_>>>(g_, P_, d_hdrs_.as<BrickHdr>(), d_runs_.as<Run>(), d_task_tab_.as<int2>(),
                                                                     d_pos4e_.as<T4>(), d_lj2e_.as<T2>(), d_list_.as<unsigned short>(),
                                                                     d_slist_.as<unsigned short>(), out, b0, nbr, nbuf,
                                                                     d_sched_.as<unsigned int>());
                        prof_.end(Prof::FORCE);
                        return MB_OK;
                    });
                });
            });
        })));
        }
        launches_++;
        n_force_evals_++;
        MB_CUDA(cudaGetLastError());
        if (parts) *parts = Partials{out.pe_partial, out.vir_partial, grid};
        return MB_OK;
    }

    // The DPDInteraction variants of the two pair kernels (the launch shape of launch_pairs)
    int launch_dpd_pairs(bool energy, T4* f4, const ForceOut<T>& out, int grid, size_t smem, int nbuf, int b0, int nbr) {
        const DpdArgs<T> da = dpd_args();
        return with_const<true, false>(energy, [&](auto EN) -> int {
            prof_.begin(Prof::FORCE);
            if (path_ == 0) {
                allpairs_force_kernel<T, COUL_NONE, CUTM_PLAIN, EN, true><<<grid, AP_THREADS, 0, stream_>>>(
                    (int)n_, P_, (T)box_[0], (T)box_[1], (T)box_[2], tric_, d_pos4_.as<T4>(), d_lj2_.as<T2>(), ex_ptr_dev(),
                    ex_idx_dev(), sp_ptr_dev(), sp_idx_dev(), f4, out.pe_partial, out.vir_partial, da);
            } else {
                // (the kernel reads its DpdArgs through the LJ-parameter pointer: dpd_args_of, uploaded by prepare)
                auto kern = brick_force_kernel<T, COUL_NONE, true, CUTM_PLAIN, EN, true>;
                MB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                kern<<<grid, FORCE_THREADS, smem, stream_>>>(g_, P_, d_hdrs_.as<BrickHdr>(), d_runs_.as<Run>(), d_task_tab_.as<int2>(),
                                                             d_pos4e_.as<T4>(), dpd_args_as_lj2e(), d_list_.as<unsigned short>(),
                                                             d_slist_.as<unsigned short>(), out, b0, nbr, nbuf, d_sched_.as<unsigned int>());
            }
            prof_.end(Prof::FORCE);
            return MB_OK;
        });
    }

    // A caller's array in host or device memory, as the kernels see it (CallerBuf): for a host array the staging buffer
    // `stage` (from byte `stage_off`), filled from the array when `upload` (inputs, and outputs with ADD semantics).
    // copy_back hands a host array its result.
    int caller_buf(const void* user, size_t bytes, DevBuf& stage, bool upload, CallerBuf& b, size_t stage_off = 0) {
        b.user = b.dev = const_cast<void*>(user);
        b.staged = user && !is_device_ptr(user);
        if (!b.staged) return MB_OK;
        MB_CUDA(stage.ensure(stage_off + bytes));
        b.dev = reinterpret_cast<char*>(stage.p) + stage_off;
        if (upload) MB_CUDA(cudaMemcpyAsync(b.dev, user, bytes, cudaMemcpyHostToDevice, stream_));
        return MB_OK;
    }
    // `bytes` of the staged result into a host array at byte `user_off` (stream-ordered: the caller synchronises)
    int copy_back(const CallerBuf& b, size_t bytes, size_t user_off = 0) {
        if (b.staged) MB_CUDA(cudaMemcpyAsync(reinterpret_cast<char*>(b.user) + user_off, b.dev, bytes, cudaMemcpyDeviceToHost, stream_));
        return MB_OK;
    }
    // a caller's n x 3 array of T
    int caller_xyz(const void* user, DevBuf& stage, bool upload, CallerBuf& b) { return caller_buf(user, 3 * (size_t)n_ * sizeof(T), stage, upload, b); }
    int copy_back_xyz(const CallerBuf& b) { return copy_back(b, 3 * (size_t)n_ * sizeof(T)); }

    // ------------------------------------------------------------------------------------------
    // make the slot-order state reflect `coords` (and vels), rebuilding the list when required
    int sync_state_from(const T* coords_dev, const T* vels_dev) {
        const int nb = (int)((n_ + 255) / 256);
        if (!have_list_) {
            MB_TRY(first_build(coords_dev));
            if (vels_dev) {
                ingest_kernel<T><<<nb, 256, 0, stream_>>>((int)n_, g_, coords_dev, vels_dev, d_orig_.as<int>(), d_xref4_.as<T4>(),
                                                          d_pos4_.as<T4>(), d_vel4_.as<T4>(), &d_ctl_.as<Control>()->disp);
                launches_++;
                MB_TRY(ext_fill(0, (int)n_));
            }
            return MB_OK;
        }
        ingest_kernel<T><<<nb, 256, 0, stream_>>>((int)n_, g_, coords_dev, vels_dev, d_orig_.as<int>(), d_xref4_.as<T4>(),
                                                  d_pos4_.as<T4>(), d_vel4_.as<T4>(), &d_ctl_.as<Control>()->rebuild);
        launches_++;
        if (decomposed()) {
            // Every rank holds the full state here. The lists of the previous call stay valid until an atom has moved more
            // than skin/2 from its position at the last rebuild (ingest_kernel just checked that on identical data on every
            // rank) or the rebuild interval has run out; the host needs the answer because ownership follows from the sort.
            int flag = 0;
            MB_CUDA(cudaMemcpyAsync(&flag, &d_ctl_.as<Control>()->rebuild, sizeof(int), cudaMemcpyDeviceToHost, stream_));
            MB_CUDA(cudaStreamSynchronize(stream_));
            if (flag || !own_valid_ || since_rebuild_ >= decomposed_interval()) {
                if (own_valid_) { build_b0_ = own_b0_; build_nb_ = own_nb_; }  // lists only for the owned slab
                MB_TRY(set_flag_rebuild());
                MB_TRY(enqueue_rebuild(true, false));
                MB_TRY(update_ownership());
                since_rebuild_ = 0;
            } else {
                MB_TRY(ext_fill(0, (int)n_));
            }
            return MB_OK;
        }
        MB_TRY(enqueue_rebuild(true, false));
        MB_TRY(ext_fill(0, (int)n_));  // (a rebuild refilled pos4e itself; without one the ingested positions go in here)
        return MB_OK;
    }

    int check_overflow_sync() {
        Control c;
        MB_TRY(read_ctl(c));
        if (c.overflow) {
            have_list_ = false;  // next call re-derives capacities, with room for what overflowed
            // The next first build measures the configuration it is given, which for a retry of mb_simulate_vv is the
            // start of the run that overflowed. The peaks of that run become floors, the halo and owned-atom counts
            // per cell so that they also apply when the next build picks a different brick.
            floor_.ghost = std::max(floor_.ghost, c.peak_ghost);
            floor_.ext = std::max(floor_.ext, c.peak_ext);
            floor_.neighbors = std::max(floor_.neighbors, c.peak_neighbors);
            floor_.halo_per_hcell = std::max(floor_.halo_per_hcell, (double)c.peak_halo / g_.hcells);
            floor_.icount_per_cell = std::max(floor_.icount_per_cell, (double)c.peak_icount / (g_.b[0] * g_.b[1] * g_.b[2]));
            static const int zero = 0;
            cudaMemcpyAsync(&d_ctl_.as<Control>()->overflow, &zero, sizeof(int), cudaMemcpyHostToDevice, stream_);
            return set_error(MB_ERR_CAPACITY, "neighbour/halo capacity overflow; results of this call are invalid, retry");
        }
        return MB_OK;
    }

    // ------------------------------------------------------------------------------------------
    // vels: the velocities a velocity-dependent pair term (DPD) is evaluated with (mb_forces_energy_vel); null elsewhere
    int forces_energy(const void* coords, void* fs, void* pe, void* vir, int64_t step_n, bool with_specific,
                      const void* vels) override {
        MB_TRY(prepare());
        MB_TRY(check_dpd());
        if (!coords) return set_error(MB_ERR_INVALID, "coords is null");
        if (dpd_on_ && fs && !vels)
            return set_error(MB_ERR_INVALID, "the DPDInteraction forces depend on the velocities: use mb_forces_energy_vel");
        if (dpd_on_ && vir) return set_error(MB_ERR_INVALID, "a DPDInteraction has no virial: the virial output must be null");
        if (!dpd_on_ && vels) return set_error(MB_ERR_INVALID, "mb_forces_energy_vel: no velocity-dependent interaction is set (mb_set_dpd)");
        CallerBuf xb;
        MB_TRY(caller_xyz(coords, d_stage_a_, true, xb));
        const bool energy = (pe != nullptr) || (vir != nullptr);
        if (path_ == 0) {
            init_slots(xb.as<T>());  // original order; posq packed into pos4
        } else {
            if (decomposed()) have_list_ = false;  // forces()/potential_energy() evaluate the whole box on every rank
            MB_TRY(sync_state_from(xb.as<T>(), nullptr));
        }
        if (dpd_on_) {  // the draws of step step_n (the Control step counter, rewritten by every simulate call) and v_pred = vels
            const long long st = step_n;
            MB_CUDA(cudaMemcpyAsync(&d_ctl_.as<Control>()->step, &st, sizeof(st), cudaMemcpyHostToDevice, stream_));
            if (vels) {
                CallerBuf vb;
                MB_TRY(caller_xyz(vels, d_stage_c_, true, vb));
                dpd_vpred_from_kernel<T><<<(int)((n_ + 255) / 256), 256, 0, stream_>>>((int)n_, vb.as<T>(), d_vpred4_.as<T4>());
                launches_++;
            }
        }
        Partials parts;
        MB_TRY(launch_pairs(energy, d_f4_.as<T4>(), false, &parts));
        if (with_specific) MB_TRY(launch_bonded(pe != nullptr));
        // outputs (ADD semantics)
        if (fs) {
            CallerBuf fb;
            MB_TRY(caller_xyz(fs, d_stage_b_, true, fb));
            scatter_forces_kernel<T><<<(int)((n_ + 255) / 256), 256, 0, stream_>>>((int)n_, d_f4_.as<T4>(), path_ == 1 ? d_orig_.as<int>() : nullptr,
                                                                                 fb.as<T>());
            launches_++;
            MB_TRY(copy_back_xyz(fb));
        }
        if (energy) {
            // pe and vir of a host caller share one staging block [pe, vir(9)]: one upload, one download
            T sc[10] = {0};
            CallerBuf peb, virb;
            MB_TRY(caller_buf(pe, sizeof(T), d_scalars_, false, peb));
            MB_TRY(caller_buf(vir, 9 * sizeof(T), d_scalars_, false, virb, sizeof(T)));
            const bool staged = peb.staged || virb.staged;
            if (peb.staged) sc[0] = *reinterpret_cast<T*>(pe);
            if (virb.staged) memcpy(sc + 1, vir, 9 * sizeof(T));
            if (staged) MB_CUDA(cudaMemcpyAsync(d_scalars_.p, sc, sizeof(sc), cudaMemcpyHostToDevice, stream_));
            reduce_partials_kernel<T><<<1, SUM_THREADS, 0, stream_>>>(parts.n, parts.pe, parts.vir, peb.as<T>(), virb.as<T>());
            launches_++;
            if (with_specific && has_specific() && pe) {
                add_double_kernel<T><<<1, 1, 0, stream_>>>(d_sp_energy_.as<double>(), peb.as<T>());
                launches_++;
            }
            if (with_specific && disp_rc_ > 0) {  // LJDispersionCorrection: E = (f6 + f12) / V; virial 2 U6 + 4 U12 on the diagonal
                MB_TRY(dispersion_prepare());
                const double vol = box_[0] * box_[1] * box_[2];
                const double u6 = disp_f6_ / vol, u12 = disp_f12_ / vol;
                add_scalars_kernel<T><<<1, 1, 0, stream_>>>(peb.as<T>(), (T)(u6 + u12), virb.as<T>(), (T)(2.0 * u6 + 4.0 * u12));
                launches_++;
            }
            if (staged) {
                MB_CUDA(cudaMemcpyAsync(sc, d_scalars_.p, sizeof(sc), cudaMemcpyDeviceToHost, stream_));
                MB_CUDA(cudaStreamSynchronize(stream_));
                if (peb.staged) *reinterpret_cast<T*>(pe) = sc[0];
                if (virb.staged) memcpy(vir, sc + 1, 9 * sizeof(T));
            }
        }
        MB_CUDA(cudaGetLastError());
        if (path_ == 1) MB_TRY(check_overflow_sync());
        else MB_CUDA(cudaStreamSynchronize(stream_));
        return MB_OK;
    }

    // ------------------------------------------------------------------------------------------
    // One MD step enqueued on the stream. In capture mode the neighbour rebuild becomes the body of a CUDA-graph
    // conditional node driven by decide_kernel, otherwise the gated pipeline is enqueued when it may be needed.
    struct StepCfg {
        Integrator ig;    // the call's integrator
        T dt, dt_half, skin_half2, kT;
        double inv_mass;
        int do_cm;        // 0/1 constant, or -1: caller decides per step (stream path only)
        bool thermostat;
        int* flag_ptr;
        VCouple vc;       // velocity-rescaling thermostat (kind VC_NONE: none)
        LangevinCoef lc;  // Langevin's (or MTSLangevinIntegrator's) c, sqrt(1 - c^2) and kT
        NhCoef nc;        // Nose-Hoover's dt / (2 Q^2) and Nf k T0
        SplitCoef<T> sc;  // LangevinSplitting's dt_A, dt_B, -friction dt_O and kT
        SplitPlan sp;     // LangevinSplitting's passes and evaluations
        VerletCoef vt;    // StormerVerlet's dt^2; OverdampedLangevin's dt / gamma, sqrt(2 dt / gamma) and kT
        T lam_dt;         // DPDVelocityVerlet's (lambda - 1/2) dt
    };
    // Langevin's c = exp(-dt friction), sqrt(1 - c^2) and kT (src/simulators.jl:1092-1097), in double. MTSLangevinIntegrator
    // runs its O step at the innermost substep, with f the innermost fraction: c = exp(-dt friction / f) (:1736-1738);
    // Langevin passes f = 1, which divides exactly.
    static LangevinCoef langevin_coef(const Integrator& ig, int f) {
        const double c = exp(-ig.dt * ig.friction / f);
        return LangevinCoef{c, sqrt(1.0 - c * c), ig.kT};
    }
    StepCfg step_cfg(const Integrator& ig) const {  // (skin_half2 and flag_ptr follow from the path: simulate sets them)
        StepCfg c;
        c.ig = ig;
        c.dt = (T)ig.dt;
        c.dt_half = (T)ig.dt / (T)2;
        c.inv_mass = (total_mass_ > 0) ? 1.0 / total_mass_ : 0.0;
        c.thermostat = ig.andersen_kT > 0 && ig.andersen_prob > 0;
        c.kT = (T)ig.andersen_kT;
        c.do_cm = (ig.remove_cm_every == 0) ? 0 : (ig.remove_cm_every == 1 ? 1 : -1);
        c.vc = VCouple{vcoupling.kind, vcoupling.n_steps, 3 * (long long)n_ - 3, vcoupling.kT, ig.dt, vcoupling.tau, total_mass_};
        c.lc = LangevinCoef{1.0, 0.0, 0.0};
        if (ig.kind == INTEG_LANGEVIN) c.lc = langevin_coef(ig, 1);
        if (ig.kind == INTEG_MTS_LANGEVIN) c.lc = langevin_coef(ig, ig.fractions[ig.n_levels - 1]);
        c.nc = NhCoef{0.0, 1.0};
        if (ig.kind == INTEG_NH)  // NoseHoover(dt, temperature, damping): dt / (2 damping^2) and Nf k T0 (src/simulators.jl:1575-1579), in double
            c.nc = NhCoef{ig.dt / (2.0 * ig.damping * ig.damping), (double)(3 * (long long)n_ - 3) * ig.kT};
        c.sc = SplitCoef<T>{};
        if (ig.kind == INTEG_SPLIT) {  // effective steps dt / count(letter); the O rate -friction dt / n_O as the reference forms it
            c.sp = split_plan(ig);
            const int* k = c.sp.count;
            c.sc = SplitCoef<T>{k[SPLIT_A] ? (T)(ig.dt / k[SPLIT_A]) : (T)0, k[SPLIT_B] ? (T)(ig.dt / k[SPLIT_B]) : (T)0,
                                k[SPLIT_O] ? -ig.friction * ig.dt / k[SPLIT_O] : 0.0, ig.kT};
        }
        // OverdampedLangevin's noise_prefac = sqrt((2 / friction) dt) (src/simulators.jl:1451), in double
        c.vt = VerletCoef{ig.dt * ig.dt, 0.0, 0.0, 0.0};
        if (ig.kind == INTEG_OVERDAMPED) c.vt = VerletCoef{0.0, ig.dt / ig.friction, sqrt(2.0 / ig.friction * ig.dt), ig.kT};
        c.lam_dt = (T)((ig.lambda - 0.5) * ig.dt);
        return c;
    }
    // what one step does beyond the plain VelocityVerlet step
    struct StepOpts {
        int do_cm = 0;                   // remove_CM_motion after this step's kick
        bool clear_cm_after_k1 = false;  // K1 consumed the pending v_cm and nothing overwrites it this step
        bool rebuild_hint = false;       // a fixed-interval rebuild is due (stream path)
        int log_mask = 0;                // LOG_* records after the step
    };
    // capture mode (capture_graph): the handle of the WHILE loop (if any) and, on the cell-list path, one (handle, body) per
    // conditional rebuild node: CUDA ties a handle to one conditional node, and a graph with a handle that no node reads does
    // not instantiate. So each handle is created when the kernel that publishes its decision is enqueued (rebuild_handle),
    // and a step with several rebuild points (LangevinSplitting) gets one per point.
    struct Capture {
        cudaGraphConditionalHandle loop = 0;
        cudaGraph_t graph = nullptr;                       // the graph the handles belong to
        std::vector<cudaGraphConditionalHandle> rebuild;  // rebuild[i]: the handle of the i-th rebuild node
        std::vector<cudaGraph_t> body;                     // the bodies splice_rebuild has added, in order
    };
    // the handle the next rebuild node will read (0 on the all-pairs path), for the kernel that publishes its decision
    cudaGraphConditionalHandle rebuild_handle(Capture* cap) {
        if (!cap || path_ != 1) return 0;
        if (cap->rebuild.size() <= cap->body.size()) {
            cudaGraphConditionalHandle h = 0;
            if (cudaGraphConditionalHandleCreate(&h, cap->graph, 0, cudaGraphCondAssignDefault) != cudaSuccess) return 0;
            cap->rebuild.push_back(h);  // (a failure leaves one handle short, which splice_rebuild reports)
        }
        return cap->rebuild[cap->body.size()];
    }
    // a conditional IF node on the next rebuild handle in place of the gated rebuild; capture_graph fills its body
    int splice_rebuild(Capture& cap) {
        if (cap.rebuild.size() <= cap.body.size()) return set_error(MB_ERR_CUDA, "no conditional handle for a rebuild node");
        cudaStreamCaptureStatus status;
        const cudaGraphNode_t* deps = nullptr;
        size_t ndeps = 0;
        cudaGraph_t gcap = nullptr;
        MB_CUDA(cudaStreamGetCaptureInfo_v2(stream_, &status, nullptr, &gcap, &deps, &ndeps));
        cudaGraphNodeParams cp = {cudaGraphNodeTypeConditional};
        cp.conditional.handle = cap.rebuild[cap.body.size()];
        cp.conditional.type = cudaGraphCondTypeIf;
        cp.conditional.size = 1;
        cudaGraphNode_t cnode;
        MB_CUDA(cudaGraphAddNode(&cnode, gcap, deps, ndeps, &cp));
        cap.body.push_back(cp.conditional.phGraph_out[0]);
        MB_CUDA(cudaStreamUpdateCaptureDependencies(stream_, &cnode, 1, cudaStreamSetCaptureDependencies));
        return MB_OK;
    }
    // What follows a drift (single GPU): the all-pairs path wraps; the cell-list path splices the conditional rebuild node
    // (capture) or enqueues the gated rebuild when it may be needed (no fixed interval, or `due`: the interval's rebuild)
    int after_drift(Capture* cap, bool due) {
        if (path_ == 0) {
            wrap_kernel<T><<<(int)((n_ + 255) / 256), 256, 0, stream_>>>((int)n_, geom(), d_pos4_.as<T4>());
            launches_++;
        } else if (cap) {
            MB_TRY(splice_rebuild(*cap));
        } else if (rebuild_every_ == 0 || due) {
            MB_TRY(enqueue_rebuild(true, false));
        }
        return MB_OK;
    }
    // The grid of an integration pass (K1, K2, the Langevin step, NH1, NH2) over n atoms: CTAs of VV_THREADS threads with
    // per_thread atoms each, at most per_sm CTAs per SM. The grid decides how grid_sum groups the sums, so a pass keeps its
    // grid from one release to the next. Each CTA writes `width` doubles to d_partial_, which is checked to hold them.
    int integ_grid(int& grid, int n, int per_thread, int per_sm, int width) {
        const int per_cta = per_thread * VV_THREADS;
        grid = std::max(1, std::min((n + per_cta - 1) / per_cta, per_sm * sm_count_));
        if ((size_t)grid * width * sizeof(double) > d_partial_.bytes)
            return set_error(MB_ERR_STATE, "integration pass of " + std::to_string(grid) + " CTAs x " + std::to_string(width) +
                                               " doubles overruns the partial-sum buffer");
        return MB_OK;
    }
    // One step of the call's integrator (single GPU; a decomposed run steps with enqueue_decomposed_step)
    int enqueue_step(const StepCfg& c, const StepOpts& o, Capture* cap = nullptr) {
        switch (c.ig.kind) {
            case INTEG_LANGEVIN: return enqueue_langevin_step(c, o, cap);
            case INTEG_NH: return enqueue_nh_step(c, o, cap);
            case INTEG_MTS:
            case INTEG_MTS_LANGEVIN: return enqueue_mts_step(c, o, cap);
            case INTEG_SPLIT: return enqueue_split_step(c, o, cap);
            case INTEG_VERLET:
            case INTEG_STORMER:
            case INTEG_OVERDAMPED: return enqueue_verlet_step(c, o, cap);
            default: return enqueue_vv_step(c, o, cap);
        }
    }
    // One VelocityVerlet step: K1 (with the previous step's thermostat, thermo_in_k1), [rebuild], forces, K2, [standalone
    // Andersen kernel], [log records]
    int enqueue_vv_step(const StepCfg& c, const StepOpts& o, Capture* cap) {
        const int n = (int)n_;
        Control* ctl = d_ctl_.as<Control>();
        CmState<T>* cm = d_cm_.as<CmState<T>>();
        prof_.begin(Prof::VV);
        int grid;
        const Thermo<T> th = thermo_in_k1(c);
        // (DPDVelocityVerlet on a context without DPD is the VelocityVerlet step)
        const bool dpd = c.ig.kind == INTEG_DPD_VV && dpd_on_;
        const int thk = dpd ? TH_DPD : (th.on ? TH_ANDERSEN : (c.vc.kind != VC_NONE ? TH_SCALE : TH_NONE));
        const DpdDrift<T> dd = {dpd ? d_vpred4_.as<T4>() : nullptr, c.lam_dt};
        MB_TRY(integ_grid(grid, n, 2, 5, 0));  // two atoms per thread, one wave (48 registers: 5 CTAs per SM)
        with_const<TH_NONE, TH_ANDERSEN, TH_SCALE, TH_DPD>(thk, [&](auto TH) {
            vv_kick_drift_kernel<T, TH><<<grid, VV_THREADS, 0, stream_>>>(
                0, n, c.dt, c.dt_half, c.skin_half2, cm, d_f4_.as<T4>(), d_xref4_.as<T4>(), d_pos4_.as<T4>(), d_vel4_.as<T4>(),
                c.flag_ptr, ctl, rebuild_handle(cap), cap && path_ == 1 ? 1 : 0, PeerPush<T>{}, ext_map(), th, dd);
        });
        prof_.end(Prof::VV);
        launches_++;
        if (o.clear_cm_after_k1) {
            clear_cm_kernel<T><<<1, 1, 0, stream_>>>(cm);
            launches_++;
        }
        MB_TRY(after_drift(cap, o.rebuild_hint));
        MB_TRY(launch_pairs(false, d_f4_.as<T4>()));
        MB_TRY(launch_bonded(false));
        MB_TRY(integ_grid(grid, n, 2, 8, c.vc.kind != VC_NONE ? 4 : 3));
        prof_.begin(Prof::VV);
        with_const<true, false>(c.vc.kind != VC_NONE, [&](auto CP) {
            vv_kick2_kernel<T, CP><<<grid, VV_THREADS, 0, stream_>>>(0, n, c.dt_half, o.do_cm, c.inv_mass, d_f4_.as<T4>(), d_mass_.as<T>(),
                                                                     d_vel4_.as<T4>(), d_partial_.as<double>(), ctl, cm, nullptr,
                                                                     PeerSignal{}, c.vc);
        });
        prof_.end(Prof::VV);
        launches_++;
        if (c.thermostat && !th.on) {
            andersen_kernel<T><<<std::max(1, (n + 255) / 256), 256, 0, stream_>>>(0, n, n, c.kT, c.ig.andersen_prob, d_orig_.as<int>(), d_mass_.as<T>(), d_vel4_.as<T4>(), cm, ctl);
            launches_++;
        }
        if (o.log_mask) MB_TRY(enqueue_log(c, o.log_mask));
        MB_CUDA(cudaGetLastError());
        return MB_OK;
    }
    // One Langevin step (langevin.cuh): the fused step kernel, [rebuild], forces, [log records]. The forces are the next
    // step's kick, and the step kernel clears a consumed v_cm itself.
    int enqueue_langevin_step(const StepCfg& c, const StepOpts& o, Capture* cap) {
        const int n = (int)n_;
        prof_.begin(Prof::VV);
        int grid;
        MB_TRY(integ_grid(grid, n, 1, 8, 3));
        langevin_step_kernel<T><<<grid, VV_THREADS, 0, stream_>>>(
            n, c.dt, c.dt_half, c.skin_half2, c.lc, o.do_cm, c.inv_mass, d_cm_.as<CmState<T>>(), d_f4_.as<T4>(), d_xref4_.as<T4>(),
            d_pos4_.as<T4>(), d_vel4_.as<T4>(), d_orig_.as<int>(), d_mass_.as<T>(), d_partial_.as<double>(), c.flag_ptr,
            d_ctl_.as<Control>(), rebuild_handle(cap), cap && path_ == 1 ? 1 : 0, ext_map());
        prof_.end(Prof::VV);
        launches_++;
        MB_TRY(after_drift(cap, o.rebuild_hint));
        MB_TRY(launch_pairs(false, d_f4_.as<T4>()));
        MB_TRY(launch_bonded(false));
        if (o.log_mask) MB_TRY(enqueue_log(c, o.log_mask));
        MB_CUDA(cudaGetLastError());
        return MB_OK;
    }
    // One Verlet, StormerVerlet or OverdampedLangevin step (verlet.cuh): the step kernel, [rebuild], forces, [Verlet's
    // Andersen thermostat], [log records]. The forces are the next step's; the step kernel clears a consumed v_cm itself,
    // and the thermostat applies the v_cm this step publishes before it resamples.
    int enqueue_verlet_step(const StepCfg& c, const StepOpts& o, Capture* cap) {
        const int n = (int)n_;
        Control* ctl = d_ctl_.as<Control>();
        CmState<T>* cm = d_cm_.as<CmState<T>>();
        const int kind = c.ig.kind == INTEG_VERLET ? VERLET_LEAPFROG : c.ig.kind == INTEG_STORMER ? VERLET_STORMER : VERLET_OVERDAMPED;
        prof_.begin(Prof::VV);
        int grid;
        MB_TRY(integ_grid(grid, n, 1, 8, 3));
        with_const<VERLET_LEAPFROG, VERLET_STORMER, VERLET_OVERDAMPED>(kind, [&](auto K) {
            verlet_step_kernel<T, K><<<grid, VV_THREADS, 0, stream_>>>(
                n, c.dt, c.skin_half2, c.vt, o.do_cm, c.inv_mass, cm, d_f4_.as<T4>(), d_xref4_.as<T4>(), d_pos4_.as<T4>(),
                d_vel4_.as<T4>(), d_orig_.as<int>(), d_mass_.as<T>(), d_partial_.as<double>(), c.flag_ptr, ctl,
                rebuild_handle(cap), cap && path_ == 1 ? 1 : 0, ext_map());
        });
        prof_.end(Prof::VV);
        launches_++;
        MB_TRY(after_drift(cap, o.rebuild_hint));
        MB_TRY(launch_pairs(false, d_f4_.as<T4>()));
        MB_TRY(launch_bonded(false));
        if (c.thermostat) {
            andersen_kernel<T><<<std::max(1, (n + 255) / 256), 256, 0, stream_>>>(0, n, n, c.kT, c.ig.andersen_prob, d_orig_.as<int>(), d_mass_.as<T>(), d_vel4_.as<T4>(), cm, ctl);
            launches_++;
        }
        if (o.log_mask) MB_TRY(enqueue_log(c, o.log_mask));
        MB_CUDA(cudaGetLastError());
        return MB_OK;
    }
    // One Nose-Hoover step (nosehoover.cuh): NH1, [rebuild], forces, NH2, [log records]. NH2 clears a consumed v_cm itself.
    int enqueue_nh_step(const StepCfg& c, const StepOpts& o, Capture* cap) {
        const int n = (int)n_;
        Control* ctl = d_ctl_.as<Control>();
        CmState<T>* cm = d_cm_.as<CmState<T>>();
        prof_.begin(Prof::VV);
        int grid;
        MB_TRY(integ_grid(grid, n, 1, 8, 2));
        nh_kick_drift_kernel<T><<<grid, VV_THREADS, 0, stream_>>>(
            n, c.dt, c.dt_half, c.skin_half2, c.nc, d_nh_.as<NhState>(), cm, d_f4_.as<T4>(), d_xref4_.as<T4>(),
            d_pos4_.as<T4>(), d_vel4_.as<T4>(), d_mass_.as<T>(), d_partial_.as<double>(), c.flag_ptr, ctl,
            rebuild_handle(cap), cap && path_ == 1 ? 1 : 0, ext_map());
        prof_.end(Prof::VV);
        launches_++;
        MB_TRY(after_drift(cap, o.rebuild_hint));
        MB_TRY(launch_pairs(false, d_f4_.as<T4>()));
        MB_TRY(launch_bonded(false));
        MB_TRY(integ_grid(grid, n, 1, 8, 3));
        prof_.begin(Prof::VV);
        nh_kick2_kernel<T><<<grid, VV_THREADS, 0, stream_>>>(n, c.dt_half, o.do_cm, c.inv_mass, d_nh_.as<NhState>(),
                                                             d_f4_.as<T4>(), d_mass_.as<T>(), d_vel4_.as<T4>(),
                                                             d_partial_.as<double>(), ctl, cm);
        prof_.end(Prof::VV);
        launches_++;
        if (o.log_mask) MB_TRY(enqueue_log(c, o.log_mask));
        MB_CUDA(cudaGetLastError());
        return MB_OK;
    }
    // One outer step of the multiple-time-step integrators (mts.cuh): mts_substeps! from level 0, unrolled on the host.
    // Level 0's forces stay in d_f4_ from one outer step to the next (pairs, its bonded ranges and PME); the inner levels
    // share d_f4_mts_, which a level recomputes on entry and after each of its substeps, as the reference's one force
    // buffer. The neighbour rebuild (cell-list path) or the wrap (all-pairs path) follows the last innermost drift, so the
    // slot order only changes in front of a pair evaluation.
    struct MtsWalk {
        int substep = 0;        // innermost substeps issued in this outer step
        bool cm_taken = false;  // the first kick (which applies the pending v_cm) has been issued
    };
    // F of one level: level 0 into d_f4_ (pairs, its bonded terms, PME), level l > 0 into d_f4_mts_ (its bonded terms)
    int mts_forces(int level) {
        if (level == 0) {
            MB_TRY(launch_pairs(false, d_f4_.as<T4>()));
            return launch_bonded(false, nullptr, 0);
        }
        MB_CUDA(cudaMemsetAsync(d_f4_mts_.p, 0, (size_t)n_ * sizeof(T4), stream_));
        return launch_bonded(false, d_f4_mts_.as<T4>(), level);
    }
    int enqueue_mts_level(const StepCfg& c, const StepOpts& o, Capture* cap, int l, bool recompute, MtsWalk& w) {
        const int n = (int)n_, n_inner = c.ig.fractions[c.ig.n_levels - 1];
        const double dt_x = (double)c.dt / c.ig.fractions[l];
        const T dt_v = (T)(dt_x / 2);
        T4* f = (l == 0) ? d_f4_.as<T4>() : d_f4_mts_.as<T4>();
        Control* ctl = d_ctl_.as<Control>();
        CmState<T>* cm = d_cm_.as<CmState<T>>();
        int grid;
        MB_TRY(integ_grid(grid, n, 1, 8, 0));
        // after the first kick of the outer step, which applied the pending v_cm: clear it where nothing overwrites it
        auto first_kick_done = [&]() {
            if (w.cm_taken) return;
            w.cm_taken = true;
            if (o.clear_cm_after_k1) {
                clear_cm_kernel<T><<<1, 1, 0, stream_>>>(cm);
                launches_++;
            }
        };
        const int reps = c.ig.fractions[l] / (l == 0 ? 1 : c.ig.fractions[l - 1]);
        for (int r = 0; r < reps; r++) {
            if (recompute) MB_TRY(mts_forces(l));
            const int apply_cm = w.cm_taken ? 0 : 1;
            if (l == c.ig.n_levels - 1) {
                const int last = (w.substep == n_inner - 1) ? 1 : 0;
                prof_.begin(Prof::VV);
                with_const<true, false>(c.ig.kind == INTEG_MTS_LANGEVIN, [&](auto LG) {
                    mts_kick_drift_kernel<T, LG><<<grid, VV_THREADS, 0, stream_>>>(
                        n, dt_v, (T)dt_x, (T)(dt_x / 2), c.skin_half2, c.lc, w.substep, apply_cm, last, cm, f, d_xref4_.as<T4>(),
                        d_pos4_.as<T4>(), d_vel4_.as<T4>(), d_orig_.as<int>(), c.flag_ptr, ctl, rebuild_handle(cap),
                        cap && path_ == 1 ? 1 : 0, ext_map());
                });
                prof_.end(Prof::VV);
                launches_++;
                first_kick_done();
                w.substep++;
                if (last) MB_TRY(after_drift(cap, o.rebuild_hint));
            } else {
                prof_.begin(Prof::VV);
                mts_kick_kernel<T><<<grid, VV_THREADS, 0, stream_>>>(n, dt_v, apply_cm, cm, f, d_vel4_.as<T4>());
                prof_.end(Prof::VV);
                launches_++;
                first_kick_done();
                MB_TRY(enqueue_mts_level(c, o, cap, l + 1, true, w));
            }
            MB_TRY(mts_forces(l));
            prof_.begin(Prof::VV);
            if (l == 0) {  // K2: the closing kick of the outer step, with sum(m v) and v_cm
                MB_TRY(integ_grid(grid, n, 2, 8, 3));
                vv_kick2_kernel<T, false><<<grid, VV_THREADS, 0, stream_>>>(0, n, dt_v, o.do_cm, c.inv_mass, d_f4_.as<T4>(), d_mass_.as<T>(),
                                                                            d_vel4_.as<T4>(), d_partial_.as<double>(), ctl, cm, nullptr,
                                                                            PeerSignal{}, VCouple{});
            } else {
                mts_kick_kernel<T><<<grid, VV_THREADS, 0, stream_>>>(n, dt_v, 0, cm, f, d_vel4_.as<T4>());
            }
            prof_.end(Prof::VV);
            launches_++;
            recompute = false;
        }
        MB_CUDA(cudaGetLastError());
        return MB_OK;
    }
    int enqueue_mts_step(const StepCfg& c, const StepOpts& o, Capture* cap) {
        MtsWalk w;
        MB_TRY(enqueue_mts_level(c, o, cap, 0, false, w));
        if (o.log_mask) MB_TRY(enqueue_log(c, o.log_mask));
        MB_CUDA(cudaGetLastError());
        return MB_OK;
    }
    // One LangevinSplitting step (splitting.cuh): its passes in order (SplitPlan). A pass that moves the atoms is followed by
    // the rebuild node (capture), the gated rebuild (stream: always enqueued, the device flag decides) or the wrap (all-pairs
    // path); a force evaluation into d_f4_ follows where the plan puts one. Graph and stream issue the same kernels.
    int enqueue_split_step(const StepCfg& c, const StepOpts& o, Capture* cap) {
        const int n = (int)n_;
        Control* ctl = d_ctl_.as<Control>();
        for (int p = 0; p < c.sp.n_pass; p++) {
            const SplitProg& pg = c.sp.pass[p];
            int grid;
            MB_TRY(integ_grid(grid, n, 1, 8, 3));
            prof_.begin(Prof::VV);
            split_pass_kernel<T><<<grid, VV_THREADS, 0, stream_>>>(
                n, pg, c.sc, c.skin_half2, o.do_cm, c.inv_mass, d_cm_.as<CmState<T>>(), d_f4_.as<T4>(), d_xref4_.as<T4>(),
                d_pos4_.as<T4>(), d_vel4_.as<T4>(), d_orig_.as<int>(), d_mass_.as<T>(), d_partial_.as<double>(), c.flag_ptr, ctl,
                pg.has_a ? rebuild_handle(cap) : 0, cap && path_ == 1 ? 1 : 0, ext_map());
            prof_.end(Prof::VV);
            launches_++;
            if (pg.has_a) MB_TRY(after_drift(cap, true));
            if (c.sp.eval_after[p]) {
                MB_TRY(launch_pairs(false, d_f4_.as<T4>()));
                MB_TRY(launch_bonded(false));
            }
        }
        if (o.log_mask) MB_TRY(enqueue_log(c, o.log_mask));
        MB_CUDA(cudaGetLastError());
        return MB_OK;
    }
    // Record the state after the current step (LOG_* mask; single-GPU runs). The energy is a second evaluation at the same
    // positions by the ENERGY variants into a scratch force buffer: the trajectory keeps the forces of the plain kernels,
    // so logging does not change it.
    int enqueue_log(const StepCfg& c, int mask) {
        Partials parts = {d_pe_partial_.as<double>(), nullptr, 0};
        if (mask & LOG_ENERGY) {
            T4* scratch = d_f4_log_.as<T4>();
            MB_TRY(launch_pairs(true, scratch, false, &parts));
            MB_TRY(launch_bonded(true, scratch));
        }
        const int nb = (int)((n_ + LOG_THREADS - 1) / LOG_THREADS);
        log_kernel<T><<<nb, LOG_THREADS, 0, stream_>>>((int)n_, mask, geom(), d_pos4_.as<T4>(), d_vel4_.as<T4>(),
                                                       d_orig_.as<int>(), d_mass_.as<T>(), d_cm_.as<CmState<T>>(), d_ctl_.as<Control>(),
                                                       thermo_in_k1(c), parts.pe, parts.n,
                                                       has_specific() ? d_sp_energy_.as<double>() : nullptr,
                                                       d_log_desc_.as<LogDesc<T>>(), d_log_part_.as<double>());
        launches_++;
        MB_CUDA(cudaGetLastError());
        return MB_OK;
    }
    // single-GPU step loop: the thermostat of step n runs at the top of step n+1's drift kernel; the last step of a call is
    // closed by the standalone kernel (simulate). The test is the rank count, not simulate's `dec`, so that a multi-rank
    // context applies the thermostat the same way on both paths: on the all-pairs path it takes the single-GPU step loop, but
    // runs the standalone kernel after every K2 (enqueue_vv_step) as the decomposed step does.
    Thermo<T> thermo_in_k1(const StepCfg& c) const {
        Thermo<T> th;
        memset(&th, 0, sizeof(th));
        if (c.thermostat && c.ig.kind == INTEG_VV && !decomposed()) {  // (Verlet runs the standalone kernel: enqueue_verlet_step)
            th.on = 1;
            th.n = (int)n_;
            th.kT = c.kT;
            th.prob = c.ig.andersen_prob;
            th.orig = d_orig_.as<int>();
            th.mass = d_mass_.as<T>();
        }
        return th;
    }

    // What a simulate call chooses that its step graphs bake in: the integrator's fields (Integrator::graph_fields), the
    // velocity-rescaling thermostat (K2's arguments) and the log mask, the LOG_* records the graph ends with (0: a plain
    // step). The logging kernel's destinations are read from the device descriptor (d_log_desc_), so they are not part of it.
    struct GraphKey {
        Integrator ig;
        mb_vcoupling_t vc;
        int log_mask;
        auto fields() const { return std::tuple_cat(ig.graph_fields(), std::tie(vc.kind, vc.n_steps, vc.kT, vc.tau, log_mask)); }
        bool operator==(const GraphKey& o) const { return fields() == o.fields(); }
    };
    // A captured graph: a step graph (one per log mask; the host loop picks one per step) or the minimiser's loop.
    // Invalidation rule: captured kernel nodes keep their arguments by value (pair parameters, box, masses, term counts,
    // geometry, buffer addresses), so every graph is dropped wherever context state they bake in changes: in prepare(),
    // which every setter of atoms, box, interactions, exceptions, neighbour policy or launch config reaches through dirty_;
    // in first_build(), which picks the geometry and sizes the list buffers; in set_specific() and set_pme(). The key then
    // holds only what a simulate call chooses; the minimiser's graph needs none.
    struct Graph {
        cudaGraph_t graph = nullptr;
        cudaGraphExec_t exec = nullptr;
        int64_t launches = 0;  // kernels per launch outside the rebuild body
        int64_t evals = 0;     // force evaluations (pair-force launches) per launch
        GraphKey key = {};
        void drop() {
            if (exec) cudaGraphExecDestroy(exec);
            if (graph) cudaGraphDestroy(graph);
            exec = nullptr;
            graph = nullptr;
        }
    };
    void drop_graphs() {
        for (Graph& g : graphs_) g.drop();
        sd_graph_.drop();
    }
    // what both graph paths need: graphs enabled, no failed capture, no stage timers, no PME (its cuFFT launches stay
    // outside the captured graphs)
    bool graphs_usable() const { return graph_enabled_ && !graph_failed_ && !prof_.enabled && !pme_on_; }
    // Capture enqueue(cap) into g. On the cell-list path enqueue splices the conditional rebuild node (splice_rebuild) and
    // the rebuild pipeline is captured into its body. loop: enqueue is captured as the body of a WHILE node on cap.loop.
    // launches_ is restored (g.launches counts the captured kernels per launch); a failure ends the capture, clears the
    // error and restores n_force_evals_ too.
    template <typename Enqueue>
    int capture_graph(Graph& g, bool loop, Enqueue enqueue) {
        g.drop();
        const int64_t launches_before = launches_, evals_before = n_force_evals_;
        auto fail = [&]() {
            cudaStreamCaptureStatus st;
            if (cudaStreamIsCapturing(stream_, &st) == cudaSuccess && st != cudaStreamCaptureStatusNone) {
                cudaGraph_t junk = nullptr;
                cudaStreamEndCapture(stream_, &junk);
            }
            cudaGetLastError();
            g.drop();
            launches_ = launches_before;
            n_force_evals_ = evals_before;
            return MB_ERR_CUDA;
        };
        if (cudaGraphCreate(&g.graph, 0) != cudaSuccess) return fail();
        Capture cap;
        cudaGraph_t into = g.graph;
        if (loop) {
            if (cudaGraphConditionalHandleCreate(&cap.loop, g.graph, 1, cudaGraphCondAssignDefault) != cudaSuccess) return fail();
            cudaGraphNodeParams cp = {cudaGraphNodeTypeConditional};
            cp.conditional.handle = cap.loop;
            cp.conditional.type = cudaGraphCondTypeWhile;
            cp.conditional.size = 1;
            cudaGraphNode_t wnode;
            if (cudaGraphAddNode(&wnode, g.graph, nullptr, 0, &cp) != cudaSuccess) return fail();
            into = cp.conditional.phGraph_out[0];
        }
        cap.graph = g.graph;  // (the rebuild handles are created as the step reaches its rebuild points: rebuild_handle)
        auto capture_into = [&](cudaGraph_t graph, auto body) {
            cudaGraph_t out = nullptr;
            return cudaStreamBeginCaptureToGraph(stream_, graph, nullptr, nullptr, 0, cudaStreamCaptureModeRelaxed) == cudaSuccess &&
                   body() == MB_OK && cudaStreamEndCapture(stream_, &out) == cudaSuccess;
        };
        if (!capture_into(into, [&] { return enqueue(cap); })) return fail();
        g.launches = launches_ - launches_before;
        g.evals = n_force_evals_ - evals_before;
        // (a LangevinSplitting step whose splitting has no A moves no atom and has no rebuild node)
        for (cudaGraph_t body : cap.body)
            if (!capture_into(body, [&] { return enqueue_rebuild(true, false); })) return fail();
        if (cudaGraphInstantiate(&g.exec, g.graph, 0) != cudaSuccess) return fail();
        launches_ = launches_before;
        return MB_OK;
    }
    // One MD step (K1, [IF rebuild], force, K2, [thermostat], [log records]; Langevin: L, [IF rebuild], force,
    // [log records]; Nose-Hoover: NH1, [IF rebuild], force, NH2, [log records]; multiple time steps: the unrolled substeps
    // of enqueue_mts_step, [log records]; LangevinSplitting: the passes of enqueue_split_step, [log records]) as an
    // executable graph.
    int build_step_graph(const StepCfg& c, const GraphKey& key) {
        StepOpts o;
        o.do_cm = c.do_cm;
        o.log_mask = key.log_mask;
        Graph& g = graphs_[key.log_mask];
        MB_TRY(capture_graph(g, false, [&](Capture& cap) { return enqueue_step(c, o, &cap); }));
        g.key = key;
        return MB_OK;
    }

    // records of one interval in a call: steps s in (init_step, init_step + n_steps] with s % every == 0, and init_step
    // itself when `initial` (GeneralObservableLogger's rule, src/loggers.jl:96-102)
    static int64_t log_count(int64_t every, int64_t init_step, int64_t n_steps, bool initial) {
        if (every <= 0) return 0;
        auto fdiv = [every](int64_t a) { return a >= 0 ? a / every : -((-a + every - 1) / every); };
        return fdiv(init_step + n_steps) - fdiv(init_step) + ((initial && init_step % every == 0) ? 1 : 0);
    }
    static int log_mask_at(const mb_log_t* L, int64_t step) {
        if (!L) return 0;
        int m = 0;
        if (L->energy_every > 0 && step % L->energy_every == 0) m |= LOG_ENERGY;
        if (L->coords_every > 0 && step % L->coords_every == 0) m |= LOG_COORDS;
        if (L->vels_every > 0 && step % L->vels_every == 0) m |= LOG_VELS;
        return m;
    }

    // The device-side loggers of one simulate call. Device outputs are written in place; host outputs go through device
    // staging: all energy records, copied at the end, and a bounded ring of frames per kind, copied out whenever it is full.
    struct LogRun {
        mb_log_t* log = nullptr;
        int64_t n[3] = {0, 0, 0};  // energy records, coordinate frames, velocity frames this call writes
        CallerBuf out[3] = {};
        int64_t ring[2] = {0, 0}, framed[2] = {0, 0};
        size_t frame_bytes = 0;
    };
    // validate the request, plan the destinations and upload the logging kernel's descriptor (read by log_kernel only)
    int log_begin(mb_log_t* log, const Integrator& ig, LogRun& lr) {
        lr.log = log;
        if (!log) return MB_OK;
        if (decomposed()) return set_error(MB_ERR_INVALID, "mb_simulate_vv_log: logging is not available in decomposed (multi-GPU) runs");
        const int64_t every[3] = {log->energy_every, log->coords_every, log->vels_every};
        const int64_t cap[3] = {log->energy_capacity, log->coords_capacity, log->vels_capacity};
        void* const outs[3] = {log->energies, log->coords, log->vels};
        for (int k = 0; k < 3; k++) {
            if (every[k] < 0 || cap[k] < 0) return set_error(MB_ERR_INVALID, "mb_simulate_vv_log: negative interval or capacity");
            if (every[k] > 0 && !outs[k]) return set_error(MB_ERR_INVALID, "mb_simulate_vv_log: null output for a non-zero interval");
            lr.n[k] = log_count(every[k], ig.init_step, ig.n_steps, log->log_initial != 0);
            if (lr.n[k] > cap[k])
                return set_error(MB_ERR_INVALID, "mb_simulate_vv_log: capacity too small: this call writes " + std::to_string(lr.n[k]) +
                                                     (k == 0 ? " energy records" : k == 1 ? " coordinate frames" : " velocity frames"));
        }
        log->n_energies = log->n_coords = log->n_vels = 0;
        lr.frame_bytes = 3 * (size_t)n_ * sizeof(T);
        LogDesc<T> desc;
        memset(&desc, 0, sizeof(desc));
        if (lr.n[0] > 0) {
            MB_TRY(caller_buf(outs[0], (size_t)lr.n[0] * 3 * sizeof(double), d_log_rec_, false, lr.out[0]));
            desc.rec = static_cast<double*>(lr.out[0].dev);
            MB_CUDA(d_f4_log_.ensure(((size_t)n_ + 16) * sizeof(T4)));
            MB_CUDA(d_sp_energy_.ensure(sizeof(double)));
            if (disp_rc_ > 0) {
                MB_TRY(dispersion_prepare());
                desc.pe_const = (disp_f6_ + disp_f12_) / (box_[0] * box_[1] * box_[2]);
            }
        }
        for (int k = 0; k < 2; k++) {
            if (lr.n[k + 1] == 0) continue;
            const int64_t ring = std::min<int64_t>(lr.n[k + 1], std::max<int64_t>(1, (int64_t)(64u << 20) / (int64_t)lr.frame_bytes));
            MB_TRY(caller_buf(outs[k + 1], (size_t)ring * lr.frame_bytes, d_log_frames_[k], false, lr.out[k + 1]));
            lr.ring[k] = lr.out[k + 1].staged ? ring : lr.n[k + 1];
            desc.frames[k] = static_cast<T*>(lr.out[k + 1].dev);
            desc.ring[k] = lr.ring[k];
        }
        MB_CUDA(d_log_desc_.ensure(sizeof(desc)));
        MB_CUDA(d_log_part_.ensure((size_t)((n_ + LOG_THREADS - 1) / LOG_THREADS) * sizeof(double)));
        MB_CUDA(cudaMemcpyAsync(d_log_desc_.p, &desc, sizeof(desc), cudaMemcpyHostToDevice, stream_));
        return MB_OK;
    }
    // after a step that recorded `mask`: a full host frame ring is copied out
    int log_step(LogRun& lr, int mask) {
        for (int k = 0; k < 2; k++) {
            if (!(mask & (LOG_COORDS << k))) continue;
            lr.framed[k]++;
            if (lr.framed[k] % lr.ring[k] == 0)
                MB_TRY(copy_back(lr.out[k + 1], (size_t)lr.ring[k] * lr.frame_bytes, (size_t)(lr.framed[k] - lr.ring[k]) * lr.frame_bytes));
        }
        return MB_OK;
    }
    // end of the call: the staged energy records and the rest of the frame rings, and the counts
    int log_end(LogRun& lr) {
        if (!lr.log) return MB_OK;
        if (lr.n[0] > 0) MB_TRY(copy_back(lr.out[0], (size_t)lr.n[0] * 3 * sizeof(double)));
        for (int k = 0; k < 2; k++) {
            const int64_t rest = lr.ring[k] > 0 ? lr.framed[k] % lr.ring[k] : 0;
            if (rest > 0) MB_TRY(copy_back(lr.out[k + 1], (size_t)rest * lr.frame_bytes, (size_t)(lr.framed[k] - rest) * lr.frame_bytes));
        }
        // (after MB_ERR_CAPACITY in simulate these records are as invalid as the coordinates)
        lr.log->n_energies = lr.n[0];
        lr.log->n_coords = lr.framed[0];
        lr.log->n_vels = lr.framed[1];
        return MB_OK;
    }

    // One decomposed VelocityVerlet step (cell-list path) over the owned slab. The thermostat runs after K2 (thermo_in_k1),
    // and velocity couplings are refused (check_simulate). defer_cm: another step of this call follows.
    int enqueue_decomposed_step(const StepCfg& c, const StepOpts& o, bool defer_cm) {
        Control* ctl = d_ctl_.as<Control>();
        CmState<T>* cm = d_cm_.as<CmState<T>>();
        // decomposed run over peer memory (peer.cuh): K1 mirrors the boundary slots into the neighbours while it drifts
        const unsigned long long epoch = ++epoch_;
        const bool p2p_halo = p2p_active() && !o.rebuild_hint;  // rebuild steps all-gather the state instead
        PeerPush<T> push;
        memset(&push, 0, sizeof(push));
        if (p2p_halo) push = make_push(epoch, true);
        if (cm_deferred_epoch_) {  // the previous step left v_cm in the momentum all-to-all (no peer_cm_kernel)
            push.cm_comm = comm_of(rank_);
            push.cm_nranks = nranks_;
            push.cm_epoch = cm_deferred_epoch_;
            push.cm_inv_mass = c.inv_mass;
            cm_deferred_epoch_ = 0;
        }
        prof_.begin(Prof::VV);
        int grid;
        MB_TRY(integ_grid(grid, own_n_, 2, 5, 0));
        vv_kick_drift_kernel<T, TH_NONE><<<grid, VV_THREADS, 0, stream_>>>(own_s0_, own_n_, c.dt, c.dt_half, c.skin_half2, cm, d_f4_.as<T4>(),
                                                                          d_xref4_.as<T4>(), d_pos4_.as<T4>(), d_vel4_.as<T4>(), c.flag_ptr,
                                                                          ctl, 0, 0, push, ext_map(), thermo_in_k1(c), DpdDrift<T>{});
        prof_.end(Prof::VV);
        launches_++;
        if (o.clear_cm_after_k1) {
            clear_cm_kernel<T><<<1, 1, 0, stream_>>>(cm);
            launches_++;
        }
        if (o.rebuild_hint) {
            // neighbour rebuild on a decomposed box: replicate positions and velocities, rebuild (identical sort on every
            // rank, lists only for the owned slab), then refresh the slot ranges and halo segments
            MB_TRY(allgather_state());
            MB_TRY(set_flag_rebuild());
            MB_TRY(enqueue_rebuild(true, false));
            MB_TRY(update_ownership());
        } else if (p2p_halo) {
            gate_ = make_wait(epoch);  // the force kernel's CTAs wait for the neighbours' pushes of this epoch
        } else {
            MB_TRY(halo_exchange());
        }
        MB_TRY(launch_pairs(false, d_f4_.as<T4>(), true));  // (own_*: after a rebuild, the new ownership)
        MB_TRY(launch_bonded(false));
        const bool p2p_sig = p2p_active();  // (after a rebuild: the new ownership's peers)
        PeerSignal sig;
        memset(&sig, 0, sizeof(sig));
        if (p2p_sig) sig = make_signal(epoch, o.do_cm != 0);
        MB_TRY(integ_grid(grid, own_n_, 2, 8, 3));
        prof_.begin(Prof::VV);
        vv_kick2_kernel<T, false><<<grid, VV_THREADS, 0, stream_>>>(own_s0_, own_n_, c.dt_half, o.do_cm, c.inv_mass, d_f4_.as<T4>(), d_mass_.as<T>(),
                                                                    d_vel4_.as<T4>(), d_partial_.as<double>(), ctl, cm, d_mom_.as<double>(),
                                                                    sig, c.vc);
        prof_.end(Prof::VV);
        launches_++;
        if (p2p_sig && o.do_cm && defer_cm && !c.thermostat) {
            cm_deferred_epoch_ = epoch;  // the next step's K1 adds the slabs' sums itself
        } else if (p2p_sig && o.do_cm) {
            // sum(m v) of all slabs arrived by peer stores: add them in rank order
            peer_cm_kernel<T><<<1, 32, 0, stream_>>>(comm_of(rank_), nranks_, epoch, c.inv_mass, cm);
            launches_++;
        } else if (o.do_cm) {
            // global sum(m v): one 24-byte all-reduce per step, then v_cm for the lazy subtraction
            MB_NCCL(g_nccl.AllReduce(d_mom_.as<double>(), d_mom_.as<double>() + 4, 3, ncclDouble, ncclSum, comm_, stream_));
            cm_from_sum_kernel<T><<<1, 1, 0, stream_>>>(d_mom_.as<double>() + 4, c.inv_mass, cm);
            launches_++;
        }
        if (c.thermostat) {
            andersen_kernel<T><<<std::max(1, (own_n_ + 255) / 256), 256, 0, stream_>>>(own_s0_, own_n_, (int)n_, c.kT, c.ig.andersen_prob, d_orig_.as<int>(), d_mass_.as<T>(), d_vel4_.as<T4>(), cm, ctl);
            launches_++;
        }
        MB_CUDA(cudaGetLastError());
        return MB_OK;
    }
    // The steps of a decomposed run (never captured: the step issues NCCL calls with per-rebuild sizes), between simulate's
    // shared prologue and epilogue. Lists cover the owned slab; the fixed rebuild interval is counted on the host (identical
    // on every rank) and adapted per call from the displacements; every rank returns the whole system.
    int simulate_decomposed(const StepCfg& c, bool cm_pending) {
        const Integrator& ig = c.ig;
        graph_used_ = false;
        cm_deferred_epoch_ = 0;
        adapt_span_ = since_rebuild_;
        // lists built from here on cover only the owned slab
        build_b0_ = own_b0_;
        build_nb_ = own_nb_;
        MB_TRY(p2p_setup());  // collective; falls back to the NCCL transport on every rank if any mapping fails
        MB_TRY(launch_pairs(false, d_f4_.as<T4>(), true));
        MB_TRY(launch_bonded(false));
        const unsigned long long e0 = ++epoch_;  // this force evaluation read the replicated state: tell the pushers
        if (p2p_active()) {
            peer_signal_kernel<<<1, 32, 0, stream_>>>(make_signal(e0, false));
            launches_++;
        }
        for (int64_t k = 1; k <= ig.n_steps; k++) {
            const int64_t step_n = ig.init_step + k;
            const int do_cm = (ig.remove_cm_every != 0 && step_n % ig.remove_cm_every == 0) ? 1 : 0;
            StepOpts o;
            o.do_cm = do_cm;
            o.clear_cm_after_k1 = cm_pending && !do_cm;  // K1 consumed v_cm; nothing overwrites it this step
            o.rebuild_hint = since_rebuild_ >= decomposed_interval();
            since_rebuild_ = o.rebuild_hint ? 1 : since_rebuild_ + 1;
            adapt_span_ = std::max(adapt_span_, since_rebuild_);
            MB_TRY(enqueue_decomposed_step(c, o, k < ig.n_steps));
            cm_pending = (do_cm != 0) && !c.thermostat;  // (the standalone thermostat kernel consumes v_cm)
            n_steps_++;
        }
        MB_TRY(allgather_state());  // every rank returns the whole system
        build_nb_ = -1;
        if (rebuild_every_ == 0) MB_TRY(adapt_interval());
        return MB_OK;
    }

    // The refusals of a simulate call, made before any work; each names the call's C entry point
    int check_simulate(const void* coords, const void* vels, const Integrator& ig) {
        static const char* const entry[] = {"mb_simulate_vv", "mb_simulate_langevin", "mb_simulate_nose_hoover", "mb_simulate_mts",
                                            "mb_simulate_mts", "mb_simulate_langevin_splitting", "mb_simulate_verlet",
                                            "mb_simulate_stormer_verlet", "mb_simulate_overdamped_langevin", "mb_simulate_dpd_vv"};
        static const char* const name[] = {"VelocityVerlet", "Langevin", "Nose-Hoover", "the multiple-time-step integrators",
                                           "the multiple-time-step integrators", "LangevinSplitting", "Verlet", "StormerVerlet",
                                           "OverdampedLangevin", "DPDVelocityVerlet"};
        if (!coords || !vels) return set_error(MB_ERR_INVALID, "null argument");
        if (ig.n_steps < 0 || !(ig.dt > 0)) return set_error(MB_ERR_INVALID, "n_steps < 0 or dt <= 0");
        MB_TRY(check_dpd());
        const std::string who = std::string(entry[ig.kind]) + ": ";
        if (is_mts(ig.kind)) {
            if (ig.n_levels < 1 || ig.n_levels > MB_MTS_MAX_LEVELS)
                return set_error(MB_ERR_INVALID, who + "n_levels must be in 1 .. MB_MTS_MAX_LEVELS");
            if (ig.fractions[0] != 1) return set_error(MB_ERR_INVALID, who + "the first ordered fraction must be 1");
            for (int l = 1; l < ig.n_levels; l++)
                if (!(ig.fractions[l] > ig.fractions[l - 1] && ig.fractions[l] % ig.fractions[l - 1] == 0))
                    return set_error(MB_ERR_INVALID, who + "fraction " + std::to_string(ig.fractions[l]) +
                                                         " is not a larger multiple of fraction " + std::to_string(ig.fractions[l - 1]));
            if (ig.fractions[ig.n_levels - 1] > 1024)
                return set_error(MB_ERR_INVALID, who + "more than 1024 innermost substeps per outer step");
            if (max_specific_level() >= ig.n_levels)
                return set_error(MB_ERR_INVALID, who + "a specific interaction sits at level " + std::to_string(max_specific_level()) +
                                                     " of " + std::to_string(ig.n_levels) + " (mb_set_specific_levels)");
        }
        if (ig.kind == INTEG_SPLIT) {
            if (ig.n_ops < 1 || ig.n_ops > MB_SPLIT_MAX_OPS)
                return set_error(MB_ERR_INVALID, who + "the splitting must have 1 .. MB_SPLIT_MAX_OPS letters");
            for (int k = 0; k < ig.n_ops; k++)
                if (ig.ops[k] != 'A' && ig.ops[k] != 'B' && ig.ops[k] != 'O')
                    return set_error(MB_ERR_INVALID, who + "splitting must contain only A, B, and O steps");
        }
        if (ig.kind == INTEG_LANGEVIN || ig.kind == INTEG_MTS_LANGEVIN || ig.kind == INTEG_SPLIT) {
            if (!(std::isfinite(ig.kT) && ig.kT >= 0)) return set_error(MB_ERR_INVALID, who + "kT must be finite and >= 0");
            if (!(std::isfinite(ig.friction) && ig.friction >= 0)) return set_error(MB_ERR_INVALID, who + "friction must be finite and >= 0");
        }
        if (ig.kind == INTEG_OVERDAMPED) {
            // (friction = 0 would make the noise prefactor sqrt(2 dt / friction) infinite)
            if (!(std::isfinite(ig.kT) && ig.kT >= 0)) return set_error(MB_ERR_INVALID, who + "kT must be finite and >= 0");
            if (!(std::isfinite(ig.friction) && ig.friction > 0)) return set_error(MB_ERR_INVALID, who + "friction must be finite and > 0");
        }
        if (ig.kind == INTEG_DPD_VV && !std::isfinite(ig.lambda)) return set_error(MB_ERR_INVALID, who + "lambda must be finite");
        if (dpd_on_ && ig.kind != INTEG_DPD_VV)
            return set_error(MB_ERR_INVALID, who + "a DPDInteraction is set (mb_set_dpd): only mb_simulate_dpd_vv runs it");
        if (ig.kind == INTEG_NH) {
            // (kT = 0 would make T / T0 infinite)
            if (!(std::isfinite(ig.kT) && ig.kT > 0)) return set_error(MB_ERR_INVALID, who + "kT must be finite and > 0");
            if (!(std::isfinite(ig.damping) && ig.damping > 0)) return set_error(MB_ERR_INVALID, who + "damping must be finite and > 0");
            if (n_ < 2) return set_error(MB_ERR_INVALID, who + "needs at least 2 atoms (Nf = 3N - 3 > 0)");
        }
        if (ig.kind != INTEG_VV) {
            if (vcoupling.kind != MB_VC_NONE)
                return set_error(MB_ERR_INVALID, who + "a velocity coupling is set on the context (couplings with " + name[ig.kind] +
                                                     " are not supported)");
            if (decomposed()) return set_error(MB_ERR_INVALID, who + "not available in decomposed (multi-GPU) runs");
        } else if (vcoupling.kind != MB_VC_NONE) {
            if (ig.andersen_kT > 0 && ig.andersen_prob > 0)
                return set_error(MB_ERR_INVALID, who + "at most one thermostat per call (Andersen and a velocity-rescaling thermostat)");
            if (decomposed())
                return set_error(MB_ERR_INVALID, who + "velocity-rescaling thermostats are not available in decomposed (multi-GPU) runs");
        }
        if (decomposed() && gb_on_) return set_error(MB_ERR_INVALID, "implicit solvent is not available in decomposed (multi-GPU) runs");
        if (decomposed() && path_ == 1 && pme_on_) return set_error(MB_ERR_INVALID, "PME is not available in decomposed (multi-GPU) runs yet");
        return MB_OK;
    }

    // One simulate call in flight on this context, from sim_begin to sim_end (a context runs one call at a time)
    struct SimRun {
        Integrator ig;
        StepCfg c;
        mb_log_t* log = nullptr;
        LogRun lr;
        CallerBuf xb, vb;
        bool dec = false, cm_pending = false;  // cm_pending: host mirror of cm->valid
    } run_;

    // Every mb_simulate_* entry point: the prologue (sim_begin), the steps (sim_step; a decomposed run steps in
    // simulate_decomposed) and the epilogue (sim_end). mb_simulate_group runs the same phases with several contexts'
    // steps interleaved.
    int simulate(void* coords, void* vels, const Integrator& call, mb_log_t* log) override {
        MB_TRY(sim_begin(coords, vels, call, log));
        if (run_.dec) {
            MB_TRY(simulate_decomposed(run_.c, run_.cm_pending));
        } else {
            for (int64_t k = 1; k <= run_.ig.n_steps; k++) MB_TRY(sim_step(k));
        }
        return sim_end();
    }
    bool is_decomposed() const override { return decomposed(); }
    // everything up to the first step: refusals, ingest, the call's Control tail, F0, the loggers at init_step and the
    // step graphs this call launches
    int sim_begin(void* coords, void* vels, const Integrator& call, mb_log_t* log) override {
        MB_TRY(prepare());
        MB_TRY(check_simulate(coords, vels, call));
        run_ = SimRun{};
        run_.dec = decomposed() && path_ == 1;  // a decomposed run: each rank integrates its slab (simulate_decomposed)
        run_.log = log;
        // one level without noise is the VelocityVerlet step: it runs as one (after the refusals, which name mb_simulate_mts)
        Integrator& ig = run_.ig;
        ig = call;
        if (ig.kind == INTEG_MTS && ig.n_levels == 1) {
            ig.kind = INTEG_VV;
            ig.n_levels = 0;
            ig.fractions.fill(0);
        }
        const bool dec = run_.dec;
        LogRun& lr = run_.lr;
        MB_TRY(log_begin(log, ig, lr));
        CallerBuf &xb = run_.xb, &vb = run_.vb;
        MB_TRY(caller_xyz(coords, d_stage_a_, true, xb));
        MB_TRY(caller_xyz(vels, d_stage_c_, true, vb));
        const int nb = (int)((n_ + 255) / 256);
        Control* ctl = d_ctl_.as<Control>();
        CmState<T>* cm = d_cm_.as<CmState<T>>();
        clear_cm_kernel<T><<<1, 1, 0, stream_>>>(cm);
        launches_++;
        if (ig.kind == INTEG_NH) MB_CUDA(cudaMemsetAsync(d_nh_.p, 0, sizeof(NhState), stream_));  // zeta = 0 at the start of every call
        StepCfg& c = run_.c;
        c = step_cfg(ig);
        if (c.ig.n_levels > 1) MB_CUDA(d_f4_mts_.ensure(((size_t)n_ + 16) * sizeof(T4)));
        if (path_ == 0) {
            init_slots(xb.as<T>());
            // velocities + wrap through ingest with an identity order (geometry only needs L)
            ingest_kernel<T><<<nb, 256, 0, stream_>>>((int)n_, g_ap_, xb.as<T>(), vb.as<T>(), d_orig_.as<int>(), d_xref4_.as<T4>(),
                                                      d_pos4_.as<T4>(), d_vel4_.as<T4>(), &ctl->disp);
            wrap_kernel<T><<<nb, 256, 0, stream_>>>((int)n_, g_ap_, d_pos4_.as<T4>());
            launches_ += 2;
            c.skin_half2 = std::numeric_limits<T>::infinity();
            c.flag_ptr = &ctl->disp;
        } else {
            MB_TRY(sync_state_from(xb.as<T>(), vb.as<T>()));
            c.skin_half2 = g_.skin_half2;  // geometry is chosen by the first build
            c.flag_ptr = (rebuild_every_ == 0 && !dec) ? &ctl->rebuild : &ctl->disp;
        }
        // step bookkeeping lives on the device (tail of Control)
        {
            struct Tail { int rebuild_every; long long step, init_step; unsigned int rng[4]; unsigned int max_disp2_bits, call_max_disp2_bits; } t;
            static_assert(sizeof(Tail) == sizeof(Control) - offsetof(Control, rebuild_every), "Control tail layout");
            t.rebuild_every = dec ? 0 : rebuild_every_;  // decomposed: the host counts the interval
            t.step = ig.init_step;
            t.init_step = ig.init_step;
            t.rng[0] = (unsigned int)ig.rng_ctr1; t.rng[1] = (unsigned int)(ig.rng_ctr1 >> 32);
            t.rng[2] = (unsigned int)ig.rng_key; t.rng[3] = (unsigned int)(ig.rng_key >> 32);
            t.max_disp2_bits = 0;
            t.call_max_disp2_bits = 0;
            MB_CUDA(cudaMemcpyAsync(reinterpret_cast<char*>(ctl) + offsetof(Control, rebuild_every), &t, sizeof(t),
                                    cudaMemcpyHostToDevice, stream_));
            MB_CUDA(cudaStreamSynchronize(stream_));  // t is a local
        }
        if (ig.init_step == 0 && ig.remove_cm_every != 0) {
            // remove_CM_motion! before the first force evaluation (simulators.jl:563): zero-length kick
            int grid;
            MB_TRY(integ_grid(grid, (int)n_, 1, 8, 3));
            vv_kick2_kernel<T, false><<<grid, VV_THREADS, 0, stream_>>>(0, (int)n_, (T)0, 1, c.inv_mass, d_f4_.as<T4>(), d_mass_.as<T>(),
                                                                        d_vel4_.as<T4>(), d_partial_.as<double>(), ctl, cm, nullptr,
                                                                        PeerSignal{}, VCouple{});
            launches_++;
            run_.cm_pending = true;
        }
        if (c.ig.kind == INTEG_DPD_VV && dpd_on_) {  // F0 with the current velocities: v_pred = v after the pending v_cm
            dpd_vpred_init_kernel<T><<<nb, 256, 0, stream_>>>((int)n_, d_vel4_.as<T4>(), d_orig_.as<int>(), cm, d_vpred4_.as<T4>());
            launches_++;
        }
        if (dec) return MB_OK;  // (simulate_decomposed evaluates F0 itself)
        MB_TRY(launch_pairs(false, d_f4_.as<T4>()));
        MB_TRY(launch_bonded(false, nullptr, is_mts(c.ig.kind) ? 0 : -1));  // (multiple time steps: F_0 of level 0)
        if (log && log->log_initial) {  // apply_loggers! at init_step (run_loggers == true), after F0
            const int m = log_mask_at(log, ig.init_step);
            if (m) {
                MB_TRY(enqueue_log(c, m));
                MB_TRY(log_step(lr, m));
            }
        }

        // CUDA-graph path: static per-step sequence (remove_CM_motion in {0,1})
        bool use_graph = graphs_usable() && c.do_cm >= 0 && ig.n_steps >= 4;
        if (use_graph) {
            // one executable per log mask this call uses (the plain step and the log steps)
            bool need[8] = {false, false, false, false, false, false, false, false};
            for (int64_t k = 1; k <= ig.n_steps; k++) need[log_mask_at(log, ig.init_step + k)] = true;
            GraphKey key{ig, vcoupling, 0};
            for (int m = 0; m < 8 && use_graph; m++) {
                if (!need[m]) continue;
                key.log_mask = m;
                if (!graphs_[m].exec || !(key == graphs_[m].key)) {
                    if (build_step_graph(c, key) != MB_OK) {
                        graph_failed_ = true;  // stay on the stream path for this context
                        use_graph = false;
                    }
                }
            }
        }
        graph_used_ = use_graph;
        return MB_OK;
    }
    // step k (1 .. n_steps) of the call sim_begin started: one graph launch, or the step enqueued on the stream
    int sim_step(int64_t k) override {
        const Integrator& ig = run_.ig;
        const int64_t step_n = ig.init_step + k;
        if (graph_used_) {
            const int m = log_mask_at(run_.log, step_n);
            MB_CUDA(cudaGraphLaunch(graphs_[m].exec, stream_));
            launches_ += graphs_[m].launches;  // rebuild-body kernels are not counted
            n_force_evals_ += graphs_[m].evals;
            MB_TRY(log_step(run_.lr, m));
        } else {
            const int do_cm = (ig.remove_cm_every != 0 && step_n % ig.remove_cm_every == 0) ? 1 : 0;
            StepOpts o;
            o.do_cm = do_cm;
            o.clear_cm_after_k1 = run_.cm_pending && !do_cm;  // K1 consumed v_cm; nothing overwrites it this step
            o.rebuild_hint = rebuild_every_ > 0 && k > 1 && (step_n - 1) % rebuild_every_ == 0;
            o.log_mask = log_mask_at(run_.log, step_n);
            MB_TRY(enqueue_step(run_.c, o));
            MB_TRY(log_step(run_.lr, o.log_mask));
            run_.cm_pending = do_cm != 0;
        }
        n_steps_++;
        return MB_OK;
    }
    // after the last step: the last step's thermostat, export, copy-back, the loggers' records and the overflow check
    int sim_end() override {
        const StepCfg& c = run_.c;
        const int nb = (int)((n_ + 255) / 256);
        CmState<T>* cm = d_cm_.as<CmState<T>>();
        if (!run_.dec && thermo_in_k1(c).on && c.ig.n_steps > 0) {
            // the thermostat of the last step (the earlier ones ran inside the next step's drift kernel)
            andersen_kernel<T><<<nb, 256, 0, stream_>>>(0, (int)n_, (int)n_, c.kT, c.ig.andersen_prob, d_orig_.as<int>(), d_mass_.as<T>(), d_vel4_.as<T4>(), cm, d_ctl_.as<Control>());
            launches_++;
        }
        // export
        const CallerBuf &xb = run_.xb, &vb = run_.vb;
        export_kernel<T><<<nb, 256, 0, stream_>>>((int)n_, geom(), d_pos4_.as<T4>(), d_vel4_.as<T4>(), d_orig_.as<int>(), cm, xb.as<T>(),
                                                  vb.as<T>());
        launches_++;
        MB_TRY(copy_back_xyz(xb));
        MB_TRY(copy_back_xyz(vb));
        MB_TRY(log_end(run_.lr));
        MB_CUDA(cudaGetLastError());
        if (path_ == 1) MB_TRY(check_overflow_sync());
        else MB_CUDA(cudaStreamSynchronize(stream_));
        return MB_OK;
    }

    // ------------------------------------------------------------------------------------------
    // Steepest-descent minimisation (minimize.cuh). The kept forces and saved positions are in original order: d_sd_f_,
    // d_sd_x_; the trial's forces go to d_f4_ (slot order), so the context's force state is not preserved.
    // The evaluation of the current positions, the decision and the accept pass (init: the starting coordinates)
    int enqueue_sd_eval(bool init, const Capture* cap = nullptr) {
        Partials parts;
        MB_TRY(launch_pairs(true, d_f4_.as<T4>(), false, &parts));
        MB_TRY(launch_bonded(true));
        sd_decide_kernel<<<1, SD_THREADS, 0, stream_>>>(d_sd_st_.as<SdState>(), parts.pe, parts.n,
                                                        has_specific() ? d_sp_energy_.as<double>() : nullptr, init ? 1 : 0,
                                                        cap ? cap->loop : 0, cap ? 1 : 0);
        const int nb = std::max(1, std::min((int)((n_ + SD_THREADS - 1) / SD_THREADS), 4 * sm_count_));
        sd_accept_kernel<T><<<nb, SD_THREADS, 0, stream_>>>((int)n_, path_ == 1 ? d_orig_.as<int>() : nullptr, d_f4_.as<T4>(),
                                                            d_sd_f_.as<T4>(), d_sd_x_.as<T4>(), d_pos4_.as<T4>(), ext_map(),
                                                            d_ctl_.as<Control>(), d_sd_st_.as<SdState>());
        launches_ += 2;
        MB_CUDA(cudaGetLastError());
        return MB_OK;
    }
    // One iteration: trial, [rebuild], evaluation, decision, accept/restore. cap: capture mode, where the rebuild becomes a
    // conditional IF node (splice_rebuild); otherwise the gated pipeline is enqueued.
    int enqueue_sd_iter(Capture* cap = nullptr) {
        const int nb = std::max(1, std::min((int)((n_ + SD_THREADS - 1) / SD_THREADS), 4 * sm_count_));
        sd_trial_kernel<T><<<nb, SD_THREADS, 0, stream_>>>((int)n_, path_ == 1 ? d_orig_.as<int>() : nullptr, d_sd_f_.as<T4>(),
                                                           d_pos4_.as<T4>(), d_sd_x_.as<T4>(), d_xref4_.as<T4>(),
                                                           path_ == 1 ? g_.skin_half2 : (T)0, ext_map(), d_ctl_.as<Control>(),
                                                           d_sd_st_.as<SdState>(), rebuild_handle(cap), cap && path_ == 1 ? 1 : 0);
        launches_++;
        MB_TRY(after_drift(cap, true));  // (the exact displacement trigger whatever rebuild_every says)
        return enqueue_sd_eval(false, cap);
    }
    // The iteration loop: a conditional WHILE node (continue flag set by the decide kernel) whose body is one iteration, with
    // the rebuild as a nested conditional IF node on the cell-list path.
    int build_sd_graph() {
        const int64_t evals_before = n_force_evals_;  // minimize_sd counts the iterations the graph runs
        MB_TRY(capture_graph(sd_graph_, true, [&](Capture& cap) { return enqueue_sd_iter(&cap); }));
        n_force_evals_ = evals_before;
        return MB_OK;
    }

    int minimize_sd(void* coords, mb_sd_params_t* p) override {
        MB_TRY(prepare());
        if (!coords || !p) return set_error(MB_ERR_INVALID, "null argument");
        if (dpd_on_) return set_error(MB_ERR_INVALID, "mb_minimize_sd: a DPDInteraction is set (mb_set_dpd): only mb_simulate_dpd_vv runs it");
        if (p->max_steps < 0 || !(p->step_size > 0) || !(p->tol >= 0))
            return set_error(MB_ERR_INVALID, "mb_minimize_sd: max_steps < 0, step_size <= 0 or tol < 0");
        if (p->trace && p->trace_capacity < p->max_steps + 1)
            return set_error(MB_ERR_INVALID, "mb_minimize_sd: trace capacity too small: this call writes up to " +
                                                 std::to_string(p->max_steps + 1) + " records");
        if (decomposed()) return set_error(MB_ERR_INVALID, "mb_minimize_sd: not available in decomposed (multi-GPU) runs");
        CallerBuf xb, tb;
        MB_TRY(caller_xyz(coords, d_stage_a_, true, xb));
        const size_t rec_bytes = 4 * sizeof(double);
        MB_TRY(caller_buf(p->trace, (size_t)(p->max_steps + 1) * rec_bytes, d_sd_trace_, false, tb));
        const size_t np = (size_t)n_ + 16;
        MB_CUDA(d_sd_f_.ensure(np * sizeof(T4)));
        MB_CUDA(d_sd_x_.ensure(np * sizeof(T4)));
        MB_CUDA(d_sd_st_.ensure(sizeof(SdState)));
        MB_CUDA(d_sp_energy_.ensure(sizeof(double)));
        SdState st;
        memset(&st, 0, sizeof(st));
        st.h = p->step_size;
        st.tol = p->tol;
        st.init_step = p->init_step;
        st.max_steps = p->max_steps;
        st.trace = tb.as<double>();
        if (disp_rc_ > 0) {
            MB_TRY(dispersion_prepare());
            st.pe_const = (disp_f6_ + disp_f12_) / (box_[0] * box_[1] * box_[2]);
        }
        MB_CUDA(cudaMemcpyAsync(d_sd_st_.p, &st, sizeof(st), cudaMemcpyHostToDevice, stream_));
        // start: wrapped coordinates (a forced rebuild wraps them on the cell-list path)
        if (path_ == 0) {
            init_slots(xb.as<T>());
            wrap_kernel<T><<<(int)((n_ + 255) / 256), 256, 0, stream_>>>((int)n_, g_ap_, d_pos4_.as<T4>());
            launches_++;
        } else {
            if (have_list_) MB_TRY(set_flag_rebuild());
            MB_TRY(sync_state_from(xb.as<T>(), nullptr));
        }
        MB_TRY(enqueue_sd_eval(true));
        graph_used_ = false;
        if (graphs_usable() && p->max_steps > 0) {
            if (!sd_graph_.exec && build_sd_graph() != MB_OK) graph_failed_ = true;  // stay on the stream path for this context
            graph_used_ = !graph_failed_;
        }
        SdState out;
        if (graph_used_) {
            MB_CUDA(cudaGraphLaunch(sd_graph_.exec, stream_));
            MB_CUDA(cudaMemcpyAsync(&out, d_sd_st_.p, sizeof(out), cudaMemcpyDeviceToHost, stream_));
            MB_CUDA(cudaStreamSynchronize(stream_));
            launches_ += out.iter * sd_graph_.launches;  // rebuild-body kernels are not counted
            n_force_evals_ += out.iter;
        } else {
            for (int64_t k = 0; k < p->max_steps; k++) {
                int cont = 0;
                MB_CUDA(cudaMemcpyAsync(&cont, &d_sd_st_.as<SdState>()->cont, sizeof(int), cudaMemcpyDeviceToHost, stream_));
                MB_CUDA(cudaStreamSynchronize(stream_));
                if (!cont) break;
                MB_TRY(enqueue_sd_iter());
            }
            MB_CUDA(cudaMemcpyAsync(&out, d_sd_st_.p, sizeof(out), cudaMemcpyDeviceToHost, stream_));
            MB_CUDA(cudaStreamSynchronize(stream_));
        }
        export_kernel<T><<<(int)((n_ + 255) / 256), 256, 0, stream_>>>((int)n_, geom(), d_pos4_.as<T4>(), d_vel4_.as<T4>(),
                                                                      d_orig_.as<int>(), d_cm_.as<CmState<T>>(), xb.as<T>(), nullptr);
        launches_++;
        MB_TRY(copy_back_xyz(xb));
        MB_TRY(copy_back(tb, (size_t)(out.iter + 1) * rec_bytes));
        p->n_iterations = out.iter;
        p->energy = out.E;
        p->max_force = out.m;
        p->final_step_size = out.h;
        p->converged = out.converged;
        MB_CUDA(cudaGetLastError());
        if (path_ == 1) MB_TRY(check_overflow_sync());
        else MB_CUDA(cudaStreamSynchronize(stream_));
        return MB_OK;
    }

    // ------------------------------------------------------------------------------------------
    // Per-CTA partials of `width` doubles each, written by launch(d_partial_) over nblk CTAs, summed on the host in block
    // order per component into out[width]
    template <typename Launch>
    int sum_partials_host(int nblk, int width, Launch launch, double* out) {
        MB_CUDA(d_partial_.ensure((size_t)nblk * width * sizeof(double)));
        launch(d_partial_.as<double>());
        launches_++;
        std::vector<double> part((size_t)nblk * width);
        MB_CUDA(cudaMemcpyAsync(part.data(), d_partial_.p, part.size() * sizeof(double), cudaMemcpyDeviceToHost, stream_));
        MB_CUDA(cudaStreamSynchronize(stream_));
        for (int d = 0; d < width; d++) out[d] = 0;
        for (int b = 0; b < nblk; b++) for (int d = 0; d < width; d++) out[d] += part[(size_t)width * b + d];
        return MB_OK;
    }
    int remove_cm(void* vels) override {
        MB_TRY(prepare());
        if (!vels) return set_error(MB_ERR_INVALID, "null velocities");
        CallerBuf vb;
        MB_TRY(caller_xyz(vels, d_stage_c_, true, vb));
        const int nb = (int)((n_ + 255) / 256);
        double s[3];
        MB_TRY(sum_partials_host(nb, 3, [&](double* part) {
            momentum_kernel<T><<<nb, SUM_THREADS, 0, stream_>>>((int)n_, vb.as<T>(), d_mass_in_.as<T>(), part);
        }, s));
        subtract_velocity_kernel<T><<<nb, 256, 0, stream_>>>((int)n_, (T)(s[0] / total_mass_), (T)(s[1] / total_mass_),
                                                             (T)(s[2] / total_mass_), vb.as<T>());
        launches_++;
        MB_TRY(copy_back_xyz(vb));
        MB_CUDA(cudaStreamSynchronize(stream_));
        return MB_OK;
    }
    int kinetic_energy(const void* vels, double* out) override {
        MB_TRY(prepare());
        if (!vels || !out) return set_error(MB_ERR_INVALID, "null argument");
        CallerBuf vb;
        MB_TRY(caller_xyz(vels, d_stage_c_, true, vb));
        const int nb = (int)((n_ + 255) / 256);
        return sum_partials_host(nb, 1, [&](double* part) {
            kinetic_kernel<T><<<nb, SUM_THREADS, 0, stream_>>>((int)n_, vb.as<T>(), d_mass_in_.as<T>(), part);
        }, out);
    }
    // kinetic energy tensor 1/2 sum m v (x) v (src/energy.jl:56-70) into out9 (3x3, symmetric, host doubles)
    int kinetic_tensor(const void* vels, double* out9) override {
        MB_TRY(prepare());
        if (!vels || !out9) return set_error(MB_ERR_INVALID, "null argument");
        CallerBuf vb;
        MB_TRY(caller_xyz(vels, d_stage_c_, true, vb));
        const int nb = (int)((n_ + 255) / 256);
        double k[6];
        MB_TRY(sum_partials_host(nb, 6, [&](double* part) {
            kinetic_tensor_kernel<T><<<nb, SUM_THREADS, 0, stream_>>>((int)n_, vb.as<T>(), d_mass_in_.as<T>(), part);
        }, k));
        out9[0] = k[0]; out9[4] = k[1]; out9[8] = k[2];
        out9[1] = out9[3] = k[3]; out9[2] = out9[6] = k[4]; out9[5] = out9[7] = k[5];
        return MB_OK;
    }
    // random_velocities!(sys, temp; rng) on the device (src/spatial.jl:819-831): fills vels (n x 3, host or device)
    int random_velocities(void* vels, double kT, uint64_t ctr1, uint64_t key) override {
        MB_TRY(prepare());
        if (!vels || !(kT >= 0)) return set_error(MB_ERR_INVALID, "mb_random_velocities: null velocities or negative kT");
        CallerBuf vb;
        MB_TRY(caller_xyz(vels, d_stage_c_, false, vb));
        const int nb = (int)((n_ + 255) / 256);
        random_velocities_kernel<T><<<nb, 256, 0, stream_>>>((int)n_, (T)kT, d_mass_in_.as<T>(), (uint32_t)ctr1, (uint32_t)(ctr1 >> 32),
                                                             (uint32_t)key, (uint32_t)(key >> 32), vb.as<T>());
        launches_++;
        MB_TRY(copy_back_xyz(vb));
        MB_CUDA(cudaStreamSynchronize(stream_));
        return MB_OK;
    }
    int rebuild(const void* coords) override {
        MB_TRY(prepare());
        if (path_ == 0) return MB_OK;
        CallerBuf xb;
        MB_TRY(caller_xyz(coords, d_stage_a_, true, xb));
        have_list_ = false;
        MB_TRY(sync_state_from(xb.as<T>(), nullptr));
        MB_CUDA(cudaStreamSynchronize(stream_));
        return MB_OK;
    }
    int stats(mb_stats_t* o) override {
        memset(o, 0, sizeof(*o));
        o->n_atoms = n_;
        o->n_force_evals = n_force_evals_;
        o->n_steps = n_steps_;
        o->path = path_;
        o->r_list = r_list_;
        o->kernel_launches = launches_;
        o->graph_mode = graph_used_ ? 1 : (graph_failed_ ? -1 : 0);
        o->reserved_ = decomposed() ? auto_every_ : 0;
        o->peer_transport = (decomposed() && p2p_active()) ? 1 : 0;
        prof_.collect();
        o->force_ms = prof_.ms[Prof::FORCE]; o->force_launches = prof_.count[Prof::FORCE];
        o->vv_ms = prof_.ms[Prof::VV]; o->vv_launches = prof_.count[Prof::VV];
        o->rebuild_ms = prof_.ms[Prof::REBUILD]; o->rebuild_launches = prof_.count[Prof::REBUILD];
        if (d_ctl_.p && !dirty_) {
            Control c;
            MB_TRY(read_ctl(c));
            o->n_rebuilds = (int64_t)c.n_rebuilds;
            o->n_pairs_in_list = (int64_t)c.n_pairs;
            o->max_neighbors = c.max_neighbors;
            o->max_halo = c.max_halo;
            o->violations = c.violations;
            o->n_prunes = 0;
        }
        if (path_ == 1 && have_list_) {
            o->n_list_entries = (int64_t)n_ * g_.stride;
            o->n_bricks = g_.nbricks;
            for (int d = 0; d < 3; d++) { o->n_cells[d] = g_.nc[d]; o->brick_dims[d] = g_.b[d]; }
            o->halo_capacity = g_.halo_cap;
            o->list_stride = g_.stride;
        }
        return MB_OK;
    }

   private:
    cudaStream_t stream_;
    int sm_count_ = 132;
    size_t smem_optin_ = 232448;
    int64_t n_ = 0;
    std::vector<T> h_mass_, h_charge_, h_sigma_, h_eps_, h_eps_raw_;
    double disp_rc_ = 0, disp_f6_ = 0, disp_f12_ = 0;  // LJDispersionCorrection (0 = off)
    bool disp_ready_ = false;
    double box_[3];
    std::vector<mb_inter_t> inters_;
    std::vector<int> ex_ptr_, ex_idx_, sp_ptr_, sp_idx_;
    int max_special_host_ = 0;
    double r_list_ = 0, skin_ = 0, cap_scale_ = 1.0, total_mass_ = 0;
    int rebuild_every_ = 0;
    int user_b_[3] = {0, 0, 0};
    // lower bounds for the capacities of the next first build, from rebuilds that overflowed (check_overflow_sync);
    // cleared when the system changes
    struct CapFloor {
        int ghost = 0, ext = 0, neighbors = 0;
        double halo_per_hcell = 0, icount_per_cell = 0;
    } floor_;
    bool dirty_ = true, have_list_ = false;
    int cutm_ = CUTM_PLAIN;  // cutoff family of the kernel variant (pair.cuh)
    int path_ = 0;
    PairParams<T> P_;
    Geom<T> g_, g_ap_;
    Tric<T> tric_ = {};  // TriclinicBoundary (on = 0: cubic / rectangular box)
    int64_t launches_ = 0, n_force_evals_ = 0, n_steps_ = 0;
    Prof prof_;
    Graph graphs_[8];  // step graphs by log mask
    Graph sd_graph_;   // the minimiser's iteration loop
    bool graph_enabled_ = true, graph_failed_ = false, graph_used_ = false, own_stream_ = false;
    // spatial decomposition (z-slabs of cell layers; one rank per GPU)
    ncclComm_t comm_ = nullptr;
    int rank_ = 0, nranks_ = 1;
    int own_b0_ = 0, own_nb_ = 0;        // this rank's bricks (static for a geometry)
    bool own_valid_ = false;             // ownership derived from the current sort
    int since_rebuild_ = 0;              // MD steps since the last rebuild of a decomposed run (host count, same on every rank)
    int adapt_span_ = 0;                 // longest such count within the current call
    int build_b0_ = 0, build_nb_ = -1;   // brick range the list builder covers (-1 = all)
    int own_s0_ = 0, own_n_ = 0;         // this rank's slots (changes at every rebuild)
    int auto_every_ = 20;                // rebuild interval of decomposed runs when the policy is displacement-triggered
    std::vector<int> layer_start_;       // slot index of the first atom of every cell layer (ncz + 1)
    std::vector<DecompSeg> halo_send_, halo_recv_;
    DevBuf d_layer_start_, d_mom_;
    // peer-memory transport (peer.cuh): IPC-mapped position arrays and PeerComm blocks of the other ranks
    bool p2p_ = false;
    void* p2p_pos_base_ = nullptr;            // the d_pos4_ allocation the peers have mapped
    DevBuf d_comm_, d_ipc_;
    std::vector<void*> peer_pos_, peer_comm_; // [rank]; own entries point at the local buffers
    unsigned long long epoch_ = 0;            // force evaluations of decomposed runs (same on every rank)
    bool plan_fits_ = false;
    PeerWait gate_ = {};
    unsigned long long cm_deferred_epoch_ = 0;
    int plan_key_[3] = {-1, -1, -1};
    int64_t sp_n_[N_SPECIFIC_KINDS] = {};
    DevBuf d_sp_idx_k_[N_SPECIFIC_KINDS], d_sp_par_k_[N_SPECIFIC_KINDS], d_sp_partial_, d_sp_energy_;
    // the terms as mb_set_specific received them, their multiple-time-step levels, and the level ranges of the device arrays
    std::vector<int> h_sp_idx_[N_SPECIFIC_KINDS];
    std::vector<T> h_sp_par_[N_SPECIFIC_KINDS];
    std::vector<int32_t> h_sp_level_[N_SPECIFIC_KINDS];
    int64_t sp_lvl_off_[N_SPECIFIC_KINDS][MTS_MAX_LEVELS + 1] = {};
    DevBuf d_f4_mts_;  // forces of the inner multiple-time-step levels (slot order; fixed address: the step graphs bake it in)
    // PME (pme.cuh)
    bool pme_on_ = false, pme_ready_ = false;
    bool dpd_on_ = false;  // mb_set_dpd: dpd_ replaces the pairwise interactions
    mb_dpd_t dpd_ = {};
    DevBuf d_vpred4_;      // DPD: predicted velocities, original order (dpd.cuh)
    DevBuf d_dpd_args_;    // DPD: the brick kernel's DpdArgs (dpd_args_of)
    double pme_rc_ = 0, pme_tol_ = 0, pme_epsr_ = 1, pme_alpha_ = 0, pme_self_e_ = 0, pme_ke_ = 138.93545764;
    PmeGeom pme_g_ = {{0, 0, 0}, {0, 0, 0}};
    int pme_plan_ = -1;
    std::vector<int> pme_pairs_;
    DevBuf d_pme_grid_, d_pme_bsm_[3], d_pme_partial_, d_pme_pairs_;
    // generalized-Born implicit solvent (gbsa.cuh): parameters, per-atom inputs (original order), per-atom results (slot
    // order), per-split partials, tickets (fixed addresses while set: the step graphs bake them in)
    bool gb_on_ = false;
    int64_t gb_n_ = 0;
    int gb_nsplit_ = 1, gb_chunk_ = GB_CHUNK;
    GbParams<T> gb_p_ = {};
    DevBuf d_gb_par_, d_gb_abg_, d_gb_tab_, d_gb_B_, d_gb_b_, d_gb_st_, d_gb_pd_, d_gb_pf_, d_gb_pe_, d_gb_tk_;
    DevBuf d_mass_in_, d_charge_in_, d_ljp_in_;
    DevBuf d_pos4_, d_vel4_, d_f4_, d_xref4_, d_lj2_, d_orig_, d_inv_orig_, d_mass_;
    DevBuf d_pos4_t_, d_vel4_t_, d_lj2_t_, d_orig_t_, d_mass_t_;
    DevBuf d_nh_;  // NhState of the Nose-Hoover integrator (fixed address: the step graphs bake it in)
    DevBuf d_ctl_, d_cm_, d_stage_a_, d_stage_b_, d_stage_c_, d_scalars_;
    DevBuf d_ex_ptr_, d_ex_idx_, d_sp_ptr_, d_sp_idx_;
    DevBuf d_cid_, d_perm_, d_cell_count_, d_cell_start_, d_cell_fill_;
    DevBuf d_hdrs_, d_runs_, d_irows_, d_hcs_, d_counts_, d_list_, d_slist_;
    DevBuf d_erow_total_, d_erow_start_, d_erow_fill_, d_ecell_start_;  // extended (ghost-padded) grid
    DevBuf d_ext_of_, d_gptr_, d_ghosts_, d_pos4e_, d_lj2e_, d_orig_e_;    // slot -> extended map, ghost table, extended arrays
    DevBuf d_task_tab_, d_sched_;  // per-brick task tables; brick ticket + finished-CTA counter of the force kernel
    DevBuf d_partial_, d_pe_partial_;
    // device-side loggers: descriptor, KE partials, scratch forces of the energy evaluation, energy records and frame rings
    // staged for host outputs
    DevBuf d_log_desc_, d_log_part_, d_f4_log_, d_log_rec_, d_log_frames_[2];
    // steepest-descent minimisation: kept forces and saved positions (original order), state, trace staged for a host output
    DevBuf d_sd_f_, d_sd_x_, d_sd_st_, d_sd_trace_;
};

}  // namespace mb

// ================================================================================================
// C ABI
// ================================================================================================
struct mb_ctx {
    std::unique_ptr<mb::EngineBase> e;
    int device;
};

#define MB_CTX_GUARD(ctx)                                                         \
    if (!(ctx) || !(ctx)->e) return mb::set_error(MB_ERR_INVALID, "null context"); \
    if (cudaSetDevice((ctx)->device) != cudaSuccess) return mb::set_error(MB_ERR_CUDA, "cudaSetDevice failed")

// the fields every mb_simulate_* parameter struct has, and the draws' keys; each kind adds its method's fields
template <typename P>
static mb::Integrator integrator_call(int kind, const P* p, uint64_t rng_ctr1, uint64_t rng_key) {
    mb::Integrator ig;
    ig.kind = kind;
    ig.dt = p->dt;
    ig.n_steps = p->n_steps;
    ig.init_step = p->init_step;
    ig.remove_cm_every = p->remove_cm_every;
    ig.rng_ctr1 = rng_ctr1;
    ig.rng_key = rng_key;
    return ig;
}
// The integrator record of an MB_INTEG_* kind from that kind's mb_simulate_* parameter struct (non-null)
static int integrator_from(int32_t kind, const void* params, mb::Integrator& ig) {
    switch (kind) {
        case MB_INTEG_VV:
        case MB_INTEG_VERLET: {
            const auto* p = static_cast<const mb_vv_params_t*>(params);
            ig = integrator_call(kind == MB_INTEG_VV ? mb::INTEG_VV : mb::INTEG_VERLET, p, p->rng_ctr1, p->rng_key);
            ig.andersen_kT = p->andersen_kT;
            ig.andersen_prob = p->andersen_prob;
            return MB_OK;
        }
        case MB_INTEG_LANGEVIN:
        case MB_INTEG_OVERDAMPED_LANGEVIN: {
            const auto* p = static_cast<const mb_langevin_params_t*>(params);
            ig = integrator_call(kind == MB_INTEG_LANGEVIN ? mb::INTEG_LANGEVIN : mb::INTEG_OVERDAMPED, p, p->rng_ctr1, p->rng_key);
            ig.kT = p->kT;
            ig.friction = p->friction;
            return MB_OK;
        }
        case MB_INTEG_NOSE_HOOVER: {
            const auto* p = static_cast<const mb_nosehoover_params_t*>(params);
            ig = integrator_call(mb::INTEG_NH, p, 0, 0);
            ig.kT = p->kT;
            ig.damping = p->damping;
            return MB_OK;
        }
        case MB_INTEG_MTS: {
            const auto* p = static_cast<const mb_mts_params_t*>(params);
            ig = integrator_call(p->langevin ? mb::INTEG_MTS_LANGEVIN : mb::INTEG_MTS, p, p->rng_ctr1, p->rng_key);
            ig.n_levels = p->n_levels;
            std::copy_n(p->fractions, std::clamp(p->n_levels, 0, MB_MTS_MAX_LEVELS), ig.fractions.begin());
            if (p->langevin) {  // (MTSIntegrator has neither)
                ig.kT = p->kT;
                ig.friction = p->friction;
            }
            return MB_OK;
        }
        case MB_INTEG_LANGEVIN_SPLITTING: {
            const auto* p = static_cast<const mb_splitting_params_t*>(params);
            ig = integrator_call(mb::INTEG_SPLIT, p, p->rng_ctr1, p->rng_key);
            ig.kT = p->kT;
            ig.friction = p->friction;
            ig.n_ops = p->n_ops;
            std::copy_n(p->ops, std::clamp(p->n_ops, 0, MB_SPLIT_MAX_OPS), ig.ops.begin());
            return MB_OK;
        }
        case MB_INTEG_STORMER_VERLET: {
            const auto* p = static_cast<const mb_stormer_params_t*>(params);
            ig = mb::Integrator{};  // (no CM removal anywhere, so the prologue skips it too; no draws)
            ig.kind = mb::INTEG_STORMER;
            ig.dt = p->dt;
            ig.n_steps = p->n_steps;
            ig.init_step = p->init_step;
            return MB_OK;
        }
        case MB_INTEG_DPD_VV: {
            const auto* p = static_cast<const mb_dpd_vv_params_t*>(params);
            ig = integrator_call(mb::INTEG_DPD_VV, p, 0, 0);  // (no draws of its own: the DPD draws are keyed by mb_dpd_t)
            ig.lambda = p->lambda;
            return MB_OK;
        }
        default: return MB_ERR_INVALID;
    }
}
// one mb_simulate_* call: its parameters as an integrator record, then the context's simulate
static int simulate_entry(mb_ctx* ctx, void* coords, void* vels, int32_t kind, const void* p, mb_log_t* log) {
    MB_CTX_GUARD(ctx);
    if (!p) return mb::set_error(MB_ERR_INVALID, "null argument");
    mb::Integrator ig;
    integrator_from(kind, p, ig);
    return ctx->e->simulate(coords, vels, ig, log);
}

extern "C" {

const char* mb_last_error(void) { return mb::g_last_error.c_str(); }

int mb_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

int mb_ctx_create(int device, int dtype, void* cuda_stream, mb_ctx** out) {
    if (!out) return mb::set_error(MB_ERR_INVALID, "out is null");
    *out = nullptr;
    if (dtype != 32 && dtype != 64) return mb::set_error(MB_ERR_INVALID, "dtype must be 32 or 64");
    int n = mb_device_count();
    if (n <= 0) return mb::set_error(MB_ERR_NOGPU, "no CUDA device visible: libmollyb200 has no CPU fallback");
    if (device < 0 || device >= n) return mb::set_error(MB_ERR_INVALID, "device index out of range");
    if (cudaSetDevice(device) != cudaSuccess) return mb::set_error(MB_ERR_CUDA, "cudaSetDevice failed");
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return mb::set_error(MB_ERR_CUDA, "cudaGetDeviceProperties failed");
    if (prop.major != 9 || prop.minor != 0)  // sm_90a code runs on compute capability 9.0 only
        return mb::set_error(MB_ERR_NOGPU, std::string("device ") + prop.name + " is not sm_90 (H100-class); this library is built for sm_90a only");
    mb_ctx* c = new mb_ctx();
    c->device = device;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (dtype == 32) c->e.reset(new mb::Engine<float>(device, s));
    else c->e.reset(new mb::Engine<double>(device, s));
    *out = c;
    return MB_OK;
}
void mb_ctx_destroy(mb_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    delete ctx;
}
int mb_set_atoms(mb_ctx* ctx, int64_t n, const void* atoms_aos) { MB_CTX_GUARD(ctx); return ctx->e->set_atoms_aos(n, atoms_aos); }
int mb_set_atoms_soa(mb_ctx* ctx, int64_t n, const void* mass, const void* charge, const void* sigma, const void* eps) {
    MB_CTX_GUARD(ctx);
    return ctx->e->set_atoms_soa(n, mass, charge, sigma, eps);
}
int mb_set_box(mb_ctx* ctx, const double side[3]) { MB_CTX_GUARD(ctx); return ctx->e->set_box(side); }
int mb_set_box_triclinic(mb_ctx* ctx, const double basis_vectors[9]) {
    MB_CTX_GUARD(ctx);
    if (!basis_vectors) return mb::set_error(MB_ERR_INVALID, "mb_set_box_triclinic: null basis");
    return ctx->e->set_box_triclinic(basis_vectors);
}
int mb_set_inters(mb_ctx* ctx, int n_inters, const mb_inter_t* inters) { MB_CTX_GUARD(ctx); return ctx->e->set_inters(n_inters, inters); }
int mb_set_exceptions(mb_ctx* ctx, int64_t n_excl, const int32_t* ei, const int32_t* ej, int64_t n_spec, const int32_t* si,
                      const int32_t* sj) {
    MB_CTX_GUARD(ctx);
    return ctx->e->set_exceptions(n_excl, ei, ej, n_spec, si, sj);
}
int mb_set_neighbor_policy(mb_ctx* ctx, double r_list, int rebuild_every) {
    MB_CTX_GUARD(ctx);
    return ctx->e->set_neighbor_policy(r_list, rebuild_every);
}
int mb_forces(mb_ctx* ctx, const void* coords, void* fs_mat, void* virial, int64_t step_n) {
    MB_CTX_GUARD(ctx);
    if (!fs_mat) return mb::set_error(MB_ERR_INVALID, "fs_mat is null");
    return ctx->e->forces_energy(coords, fs_mat, nullptr, virial, step_n, false, nullptr);
}
int mb_energy(mb_ctx* ctx, const void* coords, void* pe, int64_t step_n) {
    MB_CTX_GUARD(ctx);
    if (!pe) return mb::set_error(MB_ERR_INVALID, "pe is null");
    return ctx->e->forces_energy(coords, nullptr, pe, nullptr, step_n, false, nullptr);
}
int mb_forces_energy(mb_ctx* ctx, const void* coords, void* fs_mat, void* pe, void* virial, int64_t step_n) {
    MB_CTX_GUARD(ctx);
    return ctx->e->forces_energy(coords, fs_mat, pe, virial, step_n, false, nullptr);
}
int mb_forces_energy_all(mb_ctx* ctx, const void* coords, void* fs_mat, void* pe, int64_t step_n) {
    MB_CTX_GUARD(ctx);
    return ctx->e->forces_energy(coords, fs_mat, pe, nullptr, step_n, true, nullptr);
}
int mb_forces_energy_vel(mb_ctx* ctx, const void* coords, const void* vels, void* fs_mat, void* pe, int64_t step_n) {
    MB_CTX_GUARD(ctx);
    if (!vels) return mb::set_error(MB_ERR_INVALID, "mb_forces_energy_vel: vels is null");
    return ctx->e->forces_energy(coords, fs_mat, pe, nullptr, step_n, true, vels);
}
int mb_set_dpd(mb_ctx* ctx, const mb_dpd_t* p) { MB_CTX_GUARD(ctx); return ctx->e->set_dpd(p); }
int mb_set_specific(mb_ctx* ctx, int kind, int64_t n_terms, const int32_t* atom_idx, const double* params) {
    MB_CTX_GUARD(ctx);
    return ctx->e->set_specific(kind, n_terms, atom_idx, params);
}
int mb_set_specific_levels(mb_ctx* ctx, int kind, int64_t n_terms, const int32_t* level) {
    MB_CTX_GUARD(ctx);
    return ctx->e->set_specific_levels(kind, n_terms, level);
}
int mb_set_pme(mb_ctx* ctx, double r_cut, double error_tol, int order, double eps_r, int64_t n_pairs, const int32_t* pi, const int32_t* pj) {
    MB_CTX_GUARD(ctx);
    return ctx->e->set_pme(r_cut, error_tol, order, eps_r, n_pairs, pi, pj);
}
int mb_set_lj_dispersion_correction(mb_ctx* ctx, double dist_cutoff) { MB_CTX_GUARD(ctx); return ctx->e->set_dispersion(dist_cutoff); }
int mb_set_implicit_solvent(mb_ctx* ctx, const mb_gbsa_t* p, const double* offset_radii, const double* scaled_offset_radii,
                            const double* alpha, const double* beta, const double* gamma, const int32_t* neck_class,
                            const double* d0, const double* m0) {
    MB_CTX_GUARD(ctx);
    return ctx->e->set_implicit_solvent(p, offset_radii, scaled_offset_radii, alpha, beta, gamma, neck_class, d0, m0);
}
int mb_random_velocities(mb_ctx* ctx, void* vels, double kT, uint64_t rng_ctr1, uint64_t rng_key) {
    MB_CTX_GUARD(ctx);
    return ctx->e->random_velocities(vels, kT, rng_ctr1, rng_key);
}
int mb_kinetic_energy_tensor(mb_ctx* ctx, const void* vels, double* ke_tensor9_host) { MB_CTX_GUARD(ctx); return ctx->e->kinetic_tensor(vels, ke_tensor9_host); }
int mb_simulate_vv(mb_ctx* ctx, void* coords, void* vels, const mb_vv_params_t* p) { return mb_simulate_vv_log(ctx, coords, vels, p, nullptr); }
int mb_simulate_vv_log(mb_ctx* ctx, void* coords, void* vels, const mb_vv_params_t* p, mb_log_t* log) {
    return simulate_entry(ctx, coords, vels, MB_INTEG_VV, p, log);
}
int mb_simulate_langevin(mb_ctx* ctx, void* coords, void* vels, const mb_langevin_params_t* p, mb_log_t* log) {
    return simulate_entry(ctx, coords, vels, MB_INTEG_LANGEVIN, p, log);
}
int mb_simulate_nose_hoover(mb_ctx* ctx, void* coords, void* vels, const mb_nosehoover_params_t* p, mb_log_t* log) {
    return simulate_entry(ctx, coords, vels, MB_INTEG_NOSE_HOOVER, p, log);
}
int mb_simulate_mts(mb_ctx* ctx, void* coords, void* vels, const mb_mts_params_t* p, mb_log_t* log) {
    return simulate_entry(ctx, coords, vels, MB_INTEG_MTS, p, log);
}
int mb_simulate_langevin_splitting(mb_ctx* ctx, void* coords, void* vels, const mb_splitting_params_t* p, mb_log_t* log) {
    return simulate_entry(ctx, coords, vels, MB_INTEG_LANGEVIN_SPLITTING, p, log);
}
int mb_simulate_verlet(mb_ctx* ctx, void* coords, void* vels, const mb_vv_params_t* p, mb_log_t* log) {
    return simulate_entry(ctx, coords, vels, MB_INTEG_VERLET, p, log);
}
int mb_simulate_stormer_verlet(mb_ctx* ctx, void* coords, void* vels, const mb_stormer_params_t* p, mb_log_t* log) {
    return simulate_entry(ctx, coords, vels, MB_INTEG_STORMER_VERLET, p, log);
}
int mb_simulate_overdamped_langevin(mb_ctx* ctx, void* coords, void* vels, const mb_langevin_params_t* p, mb_log_t* log) {
    return simulate_entry(ctx, coords, vels, MB_INTEG_OVERDAMPED_LANGEVIN, p, log);
}
int mb_simulate_dpd_vv(mb_ctx* ctx, void* coords, void* vels, const mb_dpd_vv_params_t* p, mb_log_t* log) {
    return simulate_entry(ctx, coords, vels, MB_INTEG_DPD_VV, p, log);
}
int mb_simulate_group(int32_t n, mb_group_member_t* members) {
    if (n <= 0 || !members) return mb::set_error(MB_ERR_INVALID, "mb_simulate_group: n must be > 0 and members non-null");
    for (int32_t i = 0; i < n; i++) members[i].status = MB_ERR_INVALID;  // (a refused group runs no member)
    // every refusal before any work: a member the group cannot run leaves every member's buffers untouched
    std::vector<mb::Integrator> ig(n);
    for (int32_t i = 0; i < n; i++) {
        const mb_group_member_t& m = members[i];
        const std::string who = "mb_simulate_group: member " + std::to_string(i) + ": ";
        if (!m.ctx || !m.ctx->e) return mb::set_error(MB_ERR_INVALID, who + "null context");
        if (!m.params) return mb::set_error(MB_ERR_INVALID, who + "null params");
        if (integrator_from(m.kind, m.params, ig[i]) != MB_OK) return mb::set_error(MB_ERR_INVALID, who + "unknown integrator kind");
        if (m.ctx->device != members[0].ctx->device) return mb::set_error(MB_ERR_INVALID, who + "on another device than member 0");
        if (m.ctx->e->is_decomposed()) return mb::set_error(MB_ERR_INVALID, who + "a decomposed (multi-GPU) context");
        for (int32_t j = 0; j < i; j++)
            if (members[j].ctx == m.ctx) return mb::set_error(MB_ERR_INVALID, who + "the same context as member " + std::to_string(j));
    }
    if (cudaSetDevice(members[0].ctx->device) != cudaSuccess) return mb::set_error(MB_ERR_CUDA, "cudaSetDevice failed");
    // The phases of mb_simulate_* for every member; the steps round-robin, one per member per round, each on its own
    // context's stream, so that the members' kernels may run at the same time. A member that fails drops out where the
    // single call would have returned.
    std::vector<std::string> err(n);
    auto outcome = [&](int32_t i, int rc) {
        members[i].status = rc;
        if (rc != MB_OK) err[i] = mb::g_last_error;
    };
    int64_t rounds = 0;
    for (int32_t i = 0; i < n; i++) {
        outcome(i, members[i].ctx->e->sim_begin(members[i].coords, members[i].vels, ig[i], members[i].log));
        rounds = std::max(rounds, ig[i].n_steps);
    }
    for (int64_t k = 1; k <= rounds; k++)
        for (int32_t i = 0; i < n; i++)
            if (members[i].status == MB_OK && k <= ig[i].n_steps) outcome(i, members[i].ctx->e->sim_step(k));
    for (int32_t i = 0; i < n; i++)
        if (members[i].status == MB_OK) outcome(i, members[i].ctx->e->sim_end());
    for (int32_t i = 0; i < n; i++)
        if (members[i].status != MB_OK)
            return mb::set_error(members[i].status, "mb_simulate_group: member " + std::to_string(i) + ": " + err[i]);
    return MB_OK;
}
int mb_minimize_sd(mb_ctx* ctx, void* coords, mb_sd_params_t* p) { MB_CTX_GUARD(ctx); return ctx->e->minimize_sd(coords, p); }
int mb_set_velocity_coupling(mb_ctx* ctx, const mb_vcoupling_t* c) {
    MB_CTX_GUARD(ctx);
    if (!c) {
        ctx->e->vcoupling = mb_vcoupling_t{MB_VC_NONE, 0, 0.0, 0.0};
        return MB_OK;
    }
    if (c->kind < MB_VC_NONE || c->kind > MB_VC_VRESCALE) return mb::set_error(MB_ERR_INVALID, "mb_set_velocity_coupling: unknown kind");
    if (c->kind != MB_VC_NONE) {
        if (!(std::isfinite(c->kT) && c->kT >= 0)) return mb::set_error(MB_ERR_INVALID, "mb_set_velocity_coupling: kT must be finite and >= 0");
        if (c->kind != MB_VC_IMMEDIATE && !(std::isfinite(c->tau) && c->tau > 0))
            return mb::set_error(MB_ERR_INVALID, "mb_set_velocity_coupling: the coupling constant must be finite and > 0");
        if (c->kind == MB_VC_VRESCALE && c->n_steps < 1) return mb::set_error(MB_ERR_INVALID, "mb_set_velocity_coupling: n_steps < 1");
    }
    ctx->e->vcoupling = *c;
    return MB_OK;
}
int mb_remove_cm_motion(mb_ctx* ctx, void* vels) { MB_CTX_GUARD(ctx); return ctx->e->remove_cm(vels); }
int mb_kinetic_energy(mb_ctx* ctx, const void* vels, double* ke_host) { MB_CTX_GUARD(ctx); return ctx->e->kinetic_energy(vels, ke_host); }
int mb_rebuild_neighbors(mb_ctx* ctx, const void* coords) { MB_CTX_GUARD(ctx); return ctx->e->rebuild(coords); }
int mb_stats(mb_ctx* ctx, mb_stats_t* host_out) {
    MB_CTX_GUARD(ctx);
    if (!host_out) return mb::set_error(MB_ERR_INVALID, "null stats");
    return ctx->e->stats(host_out);
}
int mb_synchronize(mb_ctx* ctx) { MB_CTX_GUARD(ctx); return ctx->e->synchronize(); }
int mb_set_capacity_scale(mb_ctx* ctx, double scale) { MB_CTX_GUARD(ctx); return ctx->e->set_capacity_scale(scale); }
int mb_set_launch_config(mb_ctx* ctx, const int32_t brick_dims[3], int32_t lanes_per_atom) {
    MB_CTX_GUARD(ctx);
    return ctx->e->set_launch_config(brick_dims, lanes_per_atom);
}
int mb_set_profiling(mb_ctx* ctx, int enable) { MB_CTX_GUARD(ctx); return ctx->e->set_profiling(enable); }
int mb_comm_unique_id(void* out128) {
    if (!out128) return mb::set_error(MB_ERR_INVALID, "null output");
    if (!mb::g_nccl.load()) return mb::set_error(MB_ERR_INVALID, "libnccl.so.2 could not be loaded");
    mb::ncclUniqueId id;
    if (mb::g_nccl.GetUniqueId(&id) != mb::ncclSuccess) return mb::set_error(MB_ERR_CUDA, "ncclGetUniqueId failed");
    memcpy(out128, &id, sizeof(id));
    return MB_OK;
}
int mb_decomp_plan(int ncz, int halo_layers, int nranks, int rank, const int32_t* layer_start, int32_t* send_out, int32_t* n_send,
                   int32_t* recv_out, int32_t* n_recv, int capacity) {
    if (ncz < 1 || nranks < 1 || nranks > ncz || rank < 0 || rank >= nranks || !layer_start || !send_out || !recv_out || !n_send || !n_recv)
        return mb::set_error(MB_ERR_INVALID, "mb_decomp_plan: bad arguments");
    std::vector<mb::DecompSeg> snd, rcv;
    mb::decomp_plan(ncz, halo_layers, nranks, rank, layer_start, snd, rcv);
    if ((int)snd.size() > capacity || (int)rcv.size() > capacity) return mb::set_error(MB_ERR_CAPACITY, "mb_decomp_plan: capacity");
    for (size_t k = 0; k < snd.size(); k++) { send_out[3 * k] = snd[k].peer; send_out[3 * k + 1] = snd[k].start; send_out[3 * k + 2] = snd[k].count; }
    for (size_t k = 0; k < rcv.size(); k++) { recv_out[3 * k] = rcv[k].peer; recv_out[3 * k + 1] = rcv[k].start; recv_out[3 * k + 2] = rcv[k].count; }
    *n_send = (int32_t)snd.size();
    *n_recv = (int32_t)rcv.size();
    return MB_OK;
}
int mb_pme_plan(const double box[3], double r_cut, double error_tol, int order, double* alpha_out, int32_t mesh_out[3],
                double* moduli_out, int capacity) {
    if (!box || !alpha_out || !mesh_out || !(r_cut > 0) || !(error_tol > 0 && error_tol < 0.5) || order < 3 || order > 8)
        return mb::set_error(MB_ERR_INVALID, "mb_pme_plan: bad arguments");
    std::vector<double> moduli[3];
    int K[3];
    mb::pme_plan_host(box, r_cut, error_tol, order, alpha_out, K, moduli);
    for (int d = 0; d < 3; d++) mesh_out[d] = K[d];
    if (moduli_out) {
        if (K[0] + K[1] + K[2] > capacity) return mb::set_error(MB_ERR_CAPACITY, "mb_pme_plan: capacity");
        size_t o = 0;
        for (int d = 0; d < 3; d++)
            for (double v : moduli[d]) moduli_out[o++] = v;
    }
    return MB_OK;
}
int mb_comm_init(mb_ctx* ctx, const void* unique_id128, int rank, int nranks) {
    MB_CTX_GUARD(ctx);
    return ctx->e->comm_init(unique_id128, rank, nranks);
}

}  // extern "C"
