/*
 * mollyb200.h — C ABI of libmollyb200.so, the H100-native (sm_90a) engine for
 * Molly.jl's pairwise non-bonded + VelocityVerlet hot path.
 *
 * Every entry point is what a Julia `ccall` (or Python ctypes) binds; no C++ or
 * torch types cross the boundary. Each function cites the reference interface it
 * replaces (paths relative to the Molly.jl v0.23.3 tree). See INTEGRATION.md
 * for the Julia-side shim.
 *
 * Conventions
 *  - All functions return an int32 status: 0 = OK, <0 = error; the message is
 *    available through mb_last_error(). Nothing throws across the boundary
 *    (the reference raises Julia `error(...)`, e.g. ext/MollyCUDAExt.jl:733-739;
 *    the shim turns a non-zero status into the same exception).
 *  - Array arguments may be DEVICE pointers (the Julia shim passes CuPtr) or HOST
 *    pointers (the Python harness, the e2e benchmark): the library detects which
 *    with cudaPointerGetAttributes and stages host buffers itself.
 *  - Element type of coordinate / velocity / force / atom arrays is the
 *    context's dtype (32 -> float, 64 -> double), matching System{D,AT,T}.
 *  - Units are Molly's: nm, ps, g/mol, kJ/mol (force kJ mol^-1 nm^-1); the
 *    accel conversion factor is exactly 1 (SURVEY.md A.7).
 *  - There is no CPU fallback: without a CUDA device every call fails loudly.
 */
#ifndef MOLLYB200_H
#define MOLLYB200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct mb_ctx mb_ctx;

/* interaction kinds: src/interactions/lennard_jones.jl:28-35, coulomb.jl:32-70, :698-747, :1320-1394 */
enum { MB_LJ = 0, MB_COULOMB = 1, MB_CRF = 2, MB_EWALD_REAL = 3 };
/* cutoffs: src/cutoffs.jl:47-253. The two-point cutoffs (CubicSplineCutoff :174-215, PolynomialCutoff :217-253) take
 * dist_activation in r_act and dist_cutoff in r_cut and apply to MB_LJ and MB_COULOMB. */
enum { MB_CUT_NONE = 0, MB_CUT_DISTANCE = 1, MB_CUT_SHIFTED_POTENTIAL = 2, MB_CUT_SHIFTED_FORCE = 3,
       MB_CUT_CUBIC_SPLINE = 4, MB_CUT_POLYNOMIAL = 5 };
/* mixing rules: src/mixing.jl:20-38 */
enum { MB_MIX_LORENTZ = 0, MB_MIX_GEOMETRIC = 1 };

enum {
    MB_OK = 0,
    MB_ERR_INVALID = -1,     /* bad argument / unsupported combination */
    MB_ERR_CUDA = -2,        /* CUDA runtime error */
    MB_ERR_CAPACITY = -3,    /* neighbour/halo capacity overflow (reference: tile overflow error, ext:733-739) */
    MB_ERR_STATE = -4,       /* call order (e.g. forces before atoms were set) */
    MB_ERR_NOGPU = -5        /* no CUDA device: there is no CPU fallback */
};

/* POD descriptor of one PairwiseInteraction (fields of the Julia structs). */
typedef struct {
    int32_t kind;             /* MB_LJ | MB_COULOMB | MB_CRF | MB_EWALD_REAL */
    int32_t cutoff_kind;      /* MB_CUT_* (CRF / Ewald carry their own dist_cutoff in r_cut) */
    double r_cut;             /* inter.cutoff.dist_cutoff or inter.dist_cutoff */
    double r_act;             /* inter.cutoff.dist_activation (MB_CUT_CUBIC_SPLINE / MB_CUT_POLYNOMIAL), else ignored */
    double weight_special;    /* inter.weight_special */
    double coulomb_const;     /* inter.coulomb_const (coulomb.jl:16) */
    double solvent_dielectric;/* CRF (coulomb.jl:676); +inf = conducting */
    double ewald_alpha;       /* CoulombEwald */
    int32_t sigma_mix;        /* MB_MIX_* for sigma (default Lorentz) */
    int32_t eps_mix;          /* MB_MIX_* for epsilon (default geometric) */
    int32_t approx_erfc;      /* CoulombEwald.approximate_erfc (coulomb.jl:1331, default true in the reference): erfc by
                               * calc_erfc's 5-term polynomial (:1384-1393) instead of the exact function */
    int32_t use_neighbors;    /* inter.use_neighbors */
} mb_inter_t;

typedef struct {
    int64_t n_atoms;
    int64_t n_rebuilds;        /* neighbour-structure rebuilds since context creation */
    int64_t n_force_evals;
    int64_t n_steps;           /* VelocityVerlet steps executed */
    int64_t n_list_entries;    /* full-shell list entries (incl. padding) of the last build */
    int64_t n_pairs_in_list;   /* full-shell list entries excluding padding */
    int32_t n_bricks, n_cells[3], brick_dims[3];
    int32_t halo_capacity, list_stride, max_neighbors, max_halo;
    int32_t path;              /* 0 = all-pairs kernel, 1 = cell/brick neighbour-list kernel */
    int32_t violations;        /* fixed-interval policy: steps where an atom moved > skin/2 */
    double r_list;
    int64_t kernel_launches;   /* kernels launched by this context since creation */
    /* device time per category measured with CUDA events on the context's stream while
     * mb_set_profiling(ctx, 1) is active: force kernel, VelocityVerlet kernels, rebuild pipeline */
    double force_ms, vv_ms, rebuild_ms;
    int64_t force_launches, vv_launches, rebuild_launches;
    int32_t graph_mode;        /* last mb_simulate_vv: 1 = CUDA-graph step with conditional rebuild node,
                                * 0 = stream launches, -1 = graph construction failed (stream launches) */
    int32_t n_prunes;          /* always 0 (field kept for ABI stability: the dual-list experiment of round 1 was removed) */
    int32_t peer_transport;    /* decomposed runs: 1 = halo exchange and sum(m v) over NVLink peer memory (IPC-mapped
                                * stores fused into the drift / kick kernels), 0 = NCCL send/recv + all-reduce */
    int32_t reserved_;         /* decomposed runs: the rebuild interval the next call will use (adapted from displacements) */
} mb_stats_t;

const char* mb_last_error(void);
int mb_device_count(void);

/* Context = what BuffersGPU + GPUNeighborFinder hold in the reference
 * (src/force.jl:485-522, src/neighbors.jl:104-115). dtype 32|64. cuda_stream may be NULL. */
int mb_ctx_create(int device, int dtype, void* cuda_stream, mb_ctx** out);
void mb_ctx_destroy(mb_ctx* ctx);

/* Atoms in Molly's bits layout Atom{Int32,T,T,T,T,T} (src/types.jl:466-475):
 * {int32 index; int32 atom_type; T mass; T charge; T sigma; T eps; T lambda; int32 alch_role} =
 * 32 B (f32) / 56 B (f64). Host or device pointer. */
int mb_set_atoms(mb_ctx* ctx, int64_t n, const void* atoms_aos);
/* Same information as plain arrays (what the oracle/tests hold). */
int mb_set_atoms_soa(mb_ctx* ctx, int64_t n, const void* mass, const void* charge, const void* sigma,
                     const void* eps);
/* CubicBoundary side lengths (src/spatial.jl:40). */
int mb_set_box(mb_ctx* ctx, const double side[3]);
/* TriclinicBoundary(bv1, bv2, bv3) (src/spatial.jl:151-215): three basis vectors, row-major (bv1 = basis_vectors[0..2] along
 * x; bv2 in the xy plane; bv3 with a positive z component), approx_images = true. Minimum image as vector() :528-534, wrap
 * as wrap_coords :584-600. Served by the no-list kernel (the reference's triclinic tests are small systems:
 * test/gpu_consistency.jl:287-337). Specific interaction lists use the same vector; they are refused when the system would
 * take the cell-list path in a rectangular box (every interaction on the list, n >= 64, smallest box height >= 2.5 r_list),
 * which does not handle triclinic boxes yet. PME and decomposed runs are refused for such a box. */
int mb_set_box_triclinic(mb_ctx* ctx, const double basis_vectors[9]);
/* sys.pairwise_inters translated to descriptors (dispatch by type in the reference, SURVEY §8b). */
int mb_set_inters(mb_ctx* ctx, int n_inters, const mb_inter_t* inters);
/* GPUNeighborFinder sparse metadata (src/neighbors.jl:104-115, :171-195): 1-based pairs, any order,
 * duplicates allowed; excluded pairs are skipped by every interaction, special pairs are evaluated
 * with special=true; excluded wins over special. Host pointers. */
int mb_set_exceptions(mb_ctx* ctx, int64_t n_excl, const int32_t* excl_i, const int32_t* excl_j,
                      int64_t n_spec, const int32_t* spec_i, const int32_t* spec_j);
/* Neighbour policy: r_list = finder dist_cutoff (+ buffer); rebuild_every = n_steps of the finder
 * (src/neighbors.jl:327, :671); 0 = displacement-triggered (exact: rebuild when an atom moved
 * more than (r_list - max r_cut)/2 since the last build). */
int mb_set_neighbor_policy(mb_ctx* ctx, double r_list, int rebuild_every);

/* pairwise_forces_loop_gpu! (ext/MollyCUDAExt.jl:845; caller src/force.jl:1228): ADD the pairwise
 * forces for coords (n x 3, xyz packed) into fs_mat (3 x n column-major == n x 3 packed, original
 * atom order) and, if non-NULL, dr (x) f into virial (3x3, column-major, type T). */
int mb_forces(mb_ctx* ctx, const void* coords, void* fs_mat, void* virial, int64_t step_n);
/* pairwise_pe_loop_gpu! (ext/MollyCUDAExt.jl:936; caller src/energy.jl:427): ADD sum of pair
 * energies into pe[0] (type T). */
int mb_energy(mb_ctx* ctx, const void* coords, void* pe, int64_t step_n);
/* forces + energy in one traversal (TotalEnergyLogger-style callers). Either output may be NULL. */
int mb_forces_energy(mb_ctx* ctx, const void* coords, void* fs_mat, void* pe, void* virial,
                     int64_t step_n);

/* Specific (bonded) interaction lists, SURVEY.md §8(f)-1: InteractionList{1,2,3,4}Atoms (src/types.jl:89-157) of one
 * element type per kind. atom_idx: n_terms x atoms, 1-based; params: double, n_terms x params, per term in this order:
 *
 *   kind                              atoms  params                    reference (src/interactions/)
 *   0 MB_SPECIFIC_HARMONIC_BOND       2      k, r0                     harmonic_bond.jl
 *   1 MB_SPECIFIC_HARMONIC_ANGLE      3      k, theta0                 harmonic_angle.jl
 *   2 MB_SPECIFIC_PERIODIC_TORSION    4      periodicity, phase, k     periodic_torsion.jl
 *   3 MB_SPECIFIC_POSITION_RESTRAINT  1      k, x0, y0, z0             harmonic_position_restraint.jl
 *   4 MB_SPECIFIC_MORSE_BOND          2      D, a, r0                  morse_bond.jl
 *   5 MB_SPECIFIC_FENE_BOND           2      k, r0, sigma, eps         fene_bond.jl
 *   6 MB_SPECIFIC_COSINE_ANGLE        3      k, theta0                 cosine_angle.jl
 *   7 MB_SPECIFIC_UREY_BRADLEY        3      kangle, theta0, kbond, r0 urey_bradley.jl
 *   8 MB_SPECIFIC_HARMONIC_TORSION    4      k, theta0                 harmonic_torsion.jl
 *   9 MB_SPECIFIC_RB_TORSION          4      f1, f2, f3, f4            rb_torsion.jl
 *
 * PeriodicTorsion has one (periodicity, phase, k) term per entry: a torsion with several terms is listed several times;
 * impropers are the same struct (periodic_torsion.jl:17-142). Angles are in radians. Each call replaces every term of
 * its kind: concatenate the lists of one kind (e.g. propers and impropers) into one call. Host pointers. A kind outside
 * 0 .. MB_SPECIFIC_N_KINDS - 1 or an index outside 1 .. n is refused with MB_ERR_INVALID. The terms are evaluated inside
 * every mb_simulate_* call, the loggers and mb_minimize_sd (specific_forces_gpu!, src/force.jl:1231) and by
 * mb_forces_energy_all; mb_forces / mb_energy stay pairwise-only (the pairwise_*_loop_gpu! seam).
 * Where the engine differs from the reference:
 *  - RBTorsion: the force is -grad E of the reference's own energy, (f1 (1 + cos th) + f2 (1 - cos 2th) + f3 (1 + cos 3th)
 *    + f4) / 2. rb_torsion.jl:30 uses dE/dth = (f1 sin th - 2 f2 sin 2th + 3 f3 sin 3th) / 2, which is minus that
 *    derivative, so its forces push up the energy; the magnitudes agree, the directions are reversed.
 *  - The bend angle of HarmonicAngle, CosineAngle and UreyBradley is theta = atan2(|ba x bc|, ba . bc). It is the
 *    reference's angle (acos of the clamped cosine, bond_angle) computed with the same few-rounding-unit error at every
 *    angle; acos loses most of its digits near 0 and pi, where linear groups (theta0 = pi) sit.
 *  - Collinear angles and torsions (a cross product of exactly zero) keep their energy and get no force. For angles this is
 *    the reference's behaviour (theta is exactly 0 or pi there). For all three torsion kinds the reference divides by zero
 *    in the force. */
enum { MB_SPECIFIC_HARMONIC_BOND = 0, MB_SPECIFIC_HARMONIC_ANGLE = 1, MB_SPECIFIC_PERIODIC_TORSION = 2,
       MB_SPECIFIC_POSITION_RESTRAINT = 3, MB_SPECIFIC_MORSE_BOND = 4, MB_SPECIFIC_FENE_BOND = 5, MB_SPECIFIC_COSINE_ANGLE = 6,
       MB_SPECIFIC_UREY_BRADLEY = 7, MB_SPECIFIC_HARMONIC_TORSION = 8, MB_SPECIFIC_RB_TORSION = 9, MB_SPECIFIC_N_KINDS = 10 };
int mb_set_specific(mb_ctx* ctx, int kind, int64_t n_terms, const int32_t* atom_idx, const double* params);
/* The multiple-time-step level of every term of one kind (mb_simulate_mts): level[t] of the t-th term as mb_set_specific
 * received it, a 0-based index into the integrator's ordered fractions, 0 <= level < MB_MTS_MAX_LEVELS. n_terms must equal
 * the count mb_set_specific set for that kind, which resets every level to 0. The engine stores each kind's terms grouped by
 * level (stable within a level), so a level is one contiguous range of the bonded launch. Every other evaluation
 * (mb_forces_energy_all, mb_simulate_vv and the other integrators, the loggers, the minimiser) sums all levels. Host
 * pointer. Setting an array equal to the current one changes nothing. */
int mb_set_specific_levels(mb_ctx* ctx, int kind, int64_t n_terms, const int32_t* level);
/* forces(sys) / potential_energy(sys) of pairwise + specific + general interactions in one call (ADD semantics). */
int mb_forces_energy_all(mb_ctx* ctx, const void* coords, void* fs_mat, void* pe, int64_t step_n);

/* LJDispersionCorrection general interaction (src/interactions/lennard_jones.jl:163-275; added by setup.jl:2000-2004
 * for cutoff systems): E = (factor_6 + factor_12) / V with the means of eps sigma^6, eps sigma^12 over all i <= j atom
 * pairs (Lorentz sigma, geometric eps), no force, isotropic virial 2 U6 + 4 U12 on the diagonal. The factors are
 * computed once on the host from the atoms (grouped by distinct (sigma, eps), double). dist_cutoff <= 0 switches it
 * off. Added by mb_forces_energy_all (energy) — it is part of OpenMM's lj_only / all_cut energies. */
int mb_set_lj_dispersion_correction(mb_ctx* ctx, double dist_cutoff);

/* Particle-mesh Ewald, SURVEY.md §8(f)-3. GPU parity: tests/test_zz_gpu_pme.py (OpenMM forces_all_pme_exact at the
 * reference's 1e-7 kJ/mol/nm / 1e-5 kJ/mol in f64) and tests/test_gpu_pme_matrix.py (oracle/pme.py in f64 and f32 over
 * meshes, error_tol, charges, eps_r, coordinate and exclusion-pair edges, both force paths and the live-context setters);
 * the per-item arithmetic is also checked on the host (tests/test_pme_host.py), the oracle against a direct Ewald sum
 * (tests/test_pme_direct_ewald.py), the plan by mb_pme_plan's test. Replaces the `PME`
 * general interaction (src/interactions/ewald.jl:363-958; constructor PME(dist_cutoff, atoms, boundary; error_tol,
 * order=5, eps_r)) and the `EwaldExclusion` specific interaction list (:979-1055) that src/setup.jl:1903-1912 builds
 * from find_excluded_pairs(eligible, special): pairs = excluded OR special, 1-based. Use together with an
 * MB_EWALD_REAL pairwise interaction of the same r_cut / error_tol (ewald_alpha = sqrt(-ln(2 error_tol)) / r_cut).
 * Once set, mb_forces_energy_all and mb_simulate_vv add the reciprocal-space + exclusion forces (and energies incl.
 * the self and neutralising-background terms) after the pair kernel. order = 0 switches it off; only order 5 exists.
 * The self and background energy follow later mb_set_atoms calls. If mb_set_atoms lowers the atom count below a pair
 * index, every evaluation and simulate call fails with MB_ERR_STATE, before any launch, until this is called again. */
int mb_set_pme(mb_ctx* ctx, double r_cut, double error_tol, int order, double eps_r, int64_t n_pairs,
               const int32_t* pair_i, const int32_t* pair_j);
/* The host-side PME plan (no GPU needed; what the PME constructor computes, ewald.jl:373, :484-487, :311-361): Ewald
 * alpha, mesh dimensions, and (if moduli_out != NULL, capacity >= K0 + K1 + K2) the B-spline moduli of the three
 * dimensions back to back. */
int mb_pme_plan(const double box[3], double r_cut, double error_tol, int order, double* alpha_out, int32_t mesh_out[3],
                double* moduli_out, int capacity);

/* Generalized-Born implicit solvent: the ImplicitSolventOBC and ImplicitSolventGBN2 general interactions
 * (src/interactions/implicit_solvent.jl). One path for OBC1, OBC2 and GBN2: they differ only in their data. The caller
 * passes what the reference's structs hold (radii derived from elements stay outside the library):
 *   offset_radii, scaled_offset_radii, alpha, beta, gamma: n doubles each, original atom order (OBC broadcasts its three
 *     scalars); scaled radii may be negative (GBN2's sulphur screen);
 *   neck_class: n int32 in [0, n_neck_classes) (NULL when n_neck_classes == 0); d0, m0: row-major n_neck_classes^2 doubles,
 *     entry [c_i * n_neck_classes + c_j] = the reference's d0s[i, j] / m0s[i, j] for atoms i, j of classes c_i, c_j (the
 *     tables are not symmetric). Host pointers; the arrays are copied.
 * Charges come from the atoms. Three all-pairs passes over every ordered pair (O(N^2), no neighbour list; dist_cutoff > 0
 * drops pairs beyond it and shifts the pair energy by -1/dist_cutoff as the reference does), deterministic (no atomics).
 * Once set, mb_forces_energy_all, every integrator's step (inside the captured step graphs), the loggers' energies, the
 * minimiser and level 0 of mb_simulate_mts add the GB forces and energy after the bonded terms; mb_forces / mb_energy stay
 * pairwise-only. Setting it drops the captured graphs. p == NULL switches it off.
 * MB_ERR_STATE: atoms not set. MB_ERR_INVALID: non-finite values, an offset radius <= 0, a negative offset or cutoff, a
 * neck class out of range, n_neck_classes outside 0 .. MB_GB_MAX_NECK_CLASSES, a decomposed (multi-GPU) context. Changing
 * the atom count afterwards makes the next evaluation fail until this is called again. There is no GB virial ("Not
 * currently compatible with virial calculation" in the reference): the virial entry points are pairwise-only. */
#define MB_GB_MAX_NECK_CLASSES 32
typedef struct {
    double dist_cutoff;                   /* inter.dist_cutoff in nm; 0 = none (what setup.jl builds) */
    double offset, probe_radius, sa_factor;
    double factor_solute, factor_solvent; /* as the structs hold them (-k / eps_solute, k / eps_solvent) */
    double kappa;                         /* nm^-1 */
    double neck_scale, neck_cut;          /* used only when n_neck_classes > 0 */
    int32_t use_ace;
    int32_t n_neck_classes;               /* 0: OBC (no neck term); > 0: GBN2 */
} mb_gbsa_t;
int mb_set_implicit_solvent(mb_ctx* ctx, const mb_gbsa_t* p, const double* offset_radii, const double* scaled_offset_radii,
                            const double* alpha, const double* beta, const double* gamma, const int32_t* neck_class,
                            const double* d0, const double* m0);

/* simulate!(sys, VelocityVerlet(dt, coupling, remove_CM_motion), n_steps) hot loop
 * (src/simulators.jl:547-668): wrap, [CM removal when init_step==0], neighbours, F0, then n_steps of
 * kick / drift / wrap / forces / kick / CM removal (every remove_cm_every steps; 0 = never) /
 * Andersen coupling (prob = dt/tau per atom per step; kT<=0 disables) / neighbour policy.
 * coords, vels: n x 3, updated in place (coords returned wrapped into [0,L)). */
typedef struct {
    double dt;
    int64_t n_steps;
    int64_t init_step;        /* simulate!'s init_step; CM motion is removed up front when 0 */
    int32_t remove_cm_every;  /* VelocityVerlet.remove_CM_motion (default 1) */
    double andersen_kT;       /* k*T in kJ/mol, <= 0: no thermostat */
    double andersen_prob;     /* dt / coupling_const */
    uint64_t rng_ctr1, rng_key; /* the two rand(rng, UInt64) of src/coupling.jl:197-212 */
} mb_vv_params_t;
int mb_simulate_vv(mb_ctx* ctx, void* coords, void* vels, const mb_vv_params_t* p);

/* Velocity-rescaling thermostats for mb_simulate_vv and mb_simulate_vv_log (src/coupling.jl:82-168, :227-238), in the
 * reference's order (src/simulators.jl:616-643): after step n's second kick and its CM removal, K = 1/2 sum m v.v of the
 * velocities after that removal, T = 2 K / (Nf k) with Nf = 3N - 3 (the df of `temperature`), and every velocity is
 * scaled by lambda:
 *  - MB_VC_IMMEDIATE (ImmediateThermostat(T0)): lambda = sqrt(T0 / T);
 *  - MB_VC_BERENDSEN (BerendsenThermostat(T0, tau)): lambda^2 = 1 + (dt / tau) (T0 / T - 1);
 *  - MB_VC_VRESCALE (VelocityRescaleThermostat(T0, tau; n_steps), Bussi et al. 2007): only on steps with n % n_steps == 0;
 *    c = exp(-dt n_steps / tau), Kbar = Nf k T0 / 2, A = Kbar / (Nf K), lambda^2 = c + (1 - c) A (R^2 + S) + 2 sqrt(c (1 - c) A) R,
 *    floored at eps(Float64), with R ~ N(0, 1) and S ~ chi^2 with Nf - 1 degrees of freedom.
 * Loggers record after the coupling. K, lambda and the draws are computed on the device by the last CTA of the step's second
 * kick (no host round trip); lambda is applied by the next reader of the velocities (the next step's drift kernel, the
 * loggers, the export at the end of the call). Where the engine differs from the reference:
 *  - random numbers: the reference draws R and the Nf - 1 normals of S from the host rng. The engine draws R and S on the
 *    device from Philox4x32-10 keyed by mb_vv_params_t's rng_ctr1 / rng_key: block j (j = 0, 1, ...) has counter
 *    (0xFFFFFFFF - j, step, ctr1) and key `rng_key`, a range of first words the Andersen thermostat (1..2n) never uses.
 *    Block 0 gives R (Box-Muller of its first two words); S is one chi^2 draw, 2 Gamma((Nf - 1) / 2) by Marsaglia-Tsang
 *    with proposals from blocks 1, 2, ... (shape < 1, i.e. Nf = 2: the shape + 1 draw times U^(1/shape), U from block 0's
 *    third word; Nf = 1: S = 0). Every draw is a function of (keys, step, block) alone. The two agree in distribution
 *    only, as for the Andersen thermostat;
 *  - zero temperature: K = 0 (or Nf <= 0) leaves the velocities unchanged. The reference returns early for
 *    VelocityRescaleThermostat and produces Inf/NaN velocities for the other two;
 *  - Berendsen with dt / tau > 1 can make lambda^2 negative: the velocities become NaN (the reference raises a DomainError).
 * The coupling set here is used by every later call until it is changed; NULL (or kind MB_VC_NONE) switches it off.
 * MB_ERR_INVALID, before any work: an unknown kind, kT not finite or < 0, tau not finite or <= 0 (Berendsen,
 * velocity rescale), n_steps < 1 (velocity rescale); and from mb_simulate_vv, an Andersen thermostat in the same call or a
 * decomposed (multi-GPU) context. */
enum { MB_VC_NONE = 0, MB_VC_IMMEDIATE = 1, MB_VC_BERENDSEN = 2, MB_VC_VRESCALE = 3 };
typedef struct {
    int32_t kind;      /* MB_VC_* */
    int32_t n_steps;   /* MB_VC_VRESCALE: couple every n_steps steps (reference default 1) */
    double kT;         /* k T0 in kJ/mol */
    double tau;        /* coupling_const in ps (MB_VC_BERENDSEN, MB_VC_VRESCALE) */
} mb_vcoupling_t;
int mb_set_velocity_coupling(mb_ctx* ctx, const mb_vcoupling_t* c);

/* Device-side loggers for mb_simulate_vv (apply_loggers!, src/loggers.jl:44-56, called by simulate! at init_step and after
 * every step, src/simulators.jl:575, :657). A step s is recorded when s % interval == 0 (GeneralObservableLogger,
 * src/loggers.jl:96-102): the steps init_step + 1 .. init_step + n_steps, and init_step itself when log_initial != 0
 * (run_loggers == true; false for :skipstart). An interval of 0 records nothing of that kind. At a recorded step:
 *  - energy record (double step, pe, ke): pe = potential_energy(sys) at the positions after the drift of step s
 *    (pairwise + specific + PME + LJDispersionCorrection, as mb_forces_energy_all); ke = 1/2 sum m v.v of the
 *    velocities below, summed in double;
 *  - coordinate frame: n x 3, original atom order, wrapped into the box (as mb_simulate_vv returns them);
 *  - velocity frame: n x 3, after step s's CM removal and coupling: the velocities an unlogged call that stops
 *    at step s returns.
 * Frames have the context's dtype. Outputs may be host or device pointers; host frames are staged through a bounded
 * device ring (at most 64 MiB per kind), not n_frames x n. Logging is an observer: the energy is a second evaluation
 * into a scratch force buffer, so coordinates and velocities are bit-identical to the same call without logging.
 * The energy evaluation runs on every energy step (its cost is one more force evaluation on those steps). */
typedef struct {
    int64_t energy_every;       /* interval of energy records (0 = none) */
    int64_t coords_every;       /* interval of coordinate frames (0 = none) */
    int64_t vels_every;         /* interval of velocity frames (0 = none) */
    int32_t log_initial;        /* also record init_step (run_loggers == true) */
    int32_t reserved_;
    double* energies;           /* energy_capacity x 3 doubles: (step, pe, ke) */
    void* coords;               /* coords_capacity x n x 3 */
    void* vels;                 /* vels_capacity x n x 3 */
    int64_t energy_capacity, coords_capacity, vels_capacity;  /* records the outputs hold */
    int64_t n_energies, n_coords, n_vels;                     /* written back: records of this call */
} mb_log_t;
/* mb_simulate_vv that records into `log` (NULL: mb_simulate_vv). MB_ERR_INVALID, before any work, for a negative
 * interval or capacity, a NULL output with a non-zero interval, a capacity smaller than the records the call writes, and
 * in decomposed (multi-GPU) runs, which do not log. After MB_ERR_CAPACITY the records are invalid, like the coordinates. */
int mb_simulate_vv_log(mb_ctx* ctx, void* coords, void* vels, const mb_vv_params_t* p, mb_log_t* log);

/* simulate!(sys, Langevin(dt, temperature, friction; remove_CM_motion), n_steps) (src/simulators.jl:1065-1210, O step
 * src/kernels.jl:723-756; OpenMM's LangevinMiddleIntegrator, Zhang et al. 2019). c = exp(-dt friction) (vel_scale),
 * sqrt(1 - c^2) (noise_scale), sigma_i = noise_scale sqrt(kT / m_i). Prologue as mb_simulate_vv: wrap, CM removal when
 * init_step == 0 and remove_cm_every != 0, neighbours, F0, loggers at init_step. Step n: v += F/m dt; x += v dt/2;
 * v = c v + sigma_i xi with xi ~ N(0, 1)^3; x += v dt/2; wrap; CM removal when n % remove_cm_every == 0; neighbours;
 * F = forces(x) for step n + 1; loggers. The velocities are half a step behind the positions, and the loggers (mb_log_t, as
 * for mb_simulate_vv_log; NULL: no logging) record that state. One step is one fused kernel plus the force evaluation.
 * Where the engine differs from the reference:
 *  - random numbers: xi of atom i (1-based original index) at step n is the Box-Muller transform of one Philox4x32-10 block
 *    with counter (i, n, ctr1) and key `rng_key` (the first two words give x and y, the last two z). The reference
 *    advances ctr1 by one per step and uses counters i and i + n_atoms. Both are functions of (keys, step, atom) only, so a
 *    run split into calls with the same keys takes the same draws; the two agree in distribution only (PhiloxRNG.jl's
 *    transform is not vendored), as for the Andersen thermostat;
 *  - f32: c v + sigma xi is formed in double and rounded once;
 *  - massless atoms (1/m = 0) get no kick and no noise: v <- c v (the reference's sigma is Inf there);
 *  - sigma_i is formed from the context's 1/m (rounded to the dtype in f32).
 * MB_ERR_INVALID before any work for dt <= 0, n_steps < 0, kT or friction negative or not finite, a velocity coupling set
 * on the context (mb_set_velocity_coupling; couplings with Langevin take the stock path), a decomposed (multi-GPU)
 * context, and the logging errors of mb_simulate_vv_log. MB_ERR_CAPACITY as in mb_simulate_vv. */
typedef struct {
    double dt;
    int64_t n_steps;
    int64_t init_step;
    int32_t remove_cm_every;    /* Langevin.remove_CM_motion (default 1; 0 = never) */
    double kT;                  /* k * temperature in kJ/mol */
    double friction;            /* ps^-1 */
    uint64_t rng_ctr1, rng_key; /* the two rand(rng, UInt64) of src/simulators.jl:1135-1136 */
} mb_langevin_params_t;
int mb_simulate_langevin(mb_ctx* ctx, void* coords, void* vels, const mb_langevin_params_t* p, mb_log_t* log);

/* simulate!(sys, NoseHoover(dt, temperature, damping; remove_CM_motion), n_steps) (src/simulators.jl:1491-1614; Evans and
 * Holian 1985). Q = damping, T0 = kT / k, T(v) = sum m|v|^2 / (Nf k) with Nf = 3N - 3 (the df of `temperature`). Prologue
 * as mb_simulate_vv: wrap, CM removal when init_step == 0 and remove_cm_every != 0, neighbours, F0, loggers at init_step,
 * and zeta = 0 at the start of every call (the reference keeps zeta as a local of simulate!, so two chunked calls differ
 * from one long call). Step n, with a = F/m:
 *   1. v_half = v + (a - v zeta) dt/2
 *   2. x += v_half dt; wrap
 *   3. zeta_half = zeta + dt / (2 Q^2) (T(v) / T0 - 1), with the full-step velocities v before step 1
 *   4. zeta = zeta_half + dt / (2 Q^2) (T(v_half) / T0 - 1)
 *   5. neighbours; F = forces(x)
 *   6. v = (v_half + a dt/2) / (1 + zeta dt/2)
 *   7. CM removal when n % remove_cm_every == 0; loggers (mb_log_t, as for mb_simulate_vv_log; NULL: no logging).
 * zeta and both kinetic sums are double (sums per CTA, added in index order); the per-atom arithmetic is in the context's
 * dtype, in the reference's order of operations, with zeta rounded to it. One step is two kernels around the force
 * evaluation. Where the engine differs from the reference:
 *  - the neighbour rebuild is triggered by the exact displacement test (as for mb_simulate_vv), not by the finder's
 *    fixed interval alone;
 *  - a = F (1/m) with the context's 1/m (massless atoms: no kick; they still feel the friction term).
 * MB_ERR_INVALID before any work for dt <= 0, n_steps < 0, kT not finite or <= 0 (T0 = 0 makes T / T0 infinite), damping
 * not finite or <= 0, fewer than 2 atoms (Nf <= 0), a velocity coupling set on the context (mb_set_velocity_coupling;
 * couplings with NoseHoover take the stock path), a decomposed (multi-GPU) context, and the logging errors of
 * mb_simulate_vv_log. MB_ERR_CAPACITY as in mb_simulate_vv. */
typedef struct {
    double dt;
    int64_t n_steps;
    int64_t init_step;
    int32_t remove_cm_every;  /* NoseHoover.remove_CM_motion (default 1; 0 = never) */
    double kT;                /* k * temperature in kJ/mol */
    double damping;           /* ps (reference default 100 dt) */
} mb_nosehoover_params_t;
int mb_simulate_nose_hoover(mb_ctx* ctx, void* coords, void* vels, const mb_nosehoover_params_t* p, mb_log_t* log);

/* simulate!(sys, MTSIntegrator(dt, pi/si/gi_fractions; remove_CM_motion), n_steps) and, with langevin != 0,
 * simulate!(sys, MTSLangevinIntegrator(dt, temperature, friction, ...), n_steps) (src/simulators.jl:1616-1940; rRESPA,
 * Tuckerman et al. 1992; BAOAB-RESPA, Lagardère et al. 2019). fractions[0 .. n_levels) are the integrator's
 * ordered_fractions: fractions[0] = 1, each one larger than and a multiple of the one before. Level 0 holds all pairwise
 * interactions, PME and the terms of level 0 (mb_set_specific_levels); level l > 0 holds the bonded terms of level l.
 * Prologue as mb_simulate_vv: wrap, CM removal when init_step == 0 and remove_cm_every != 0, neighbours, F_0 (the forces of
 * level 0), loggers at init_step. An outer step runs mts_substeps! from level 0; at level l with dt_x = dt / fractions[l],
 * dt_v = dt_x / 2, repeated fractions[l] / fractions[l - 1] times (once for level 0):
 *   F_l = forces of level l (level 0: only at the start of a call; levels l > 0: on entry to the level);
 *   v += F_l / m dt_v;
 *   innermost level: x += v dt_x (MTSIntegrator) or x += v dt_x/2; v = c v + sigma_i xi; x += v dt_x/2 (langevin), with
 *   c = exp(-dt friction / fractions[n_levels - 1]) and sigma_i = sqrt(1 - c^2) sqrt(kT / m_i); wrap;
 *   other levels: the substeps of level l + 1;
 *   F_l = forces of level l; v += F_l / m dt_v.
 * Then CM removal when n % remove_cm_every == 0 and the loggers (mb_log_t, as for mb_simulate_vv_log), once per outer step.
 * n_steps counts outer steps. The pairwise forces are evaluated once per outer step; level l > 0 is evaluated
 * fractions[l] + fractions[l - 1] times per outer step, as in the reference. With n_levels = 1 and langevin = 0 this is the
 * VelocityVerlet step, and the call runs it. Where the engine differs from the reference:
 *  - neighbours: the exact displacement trigger of mb_simulate_vv, tested once per outer step after the last innermost
 *    drift, so the structure is only rebuilt right before the pair evaluation (the bonded terms need none: they are
 *    evaluated by minimum image). The all-pairs path wraps at that point too, not after every innermost drift;
 *  - random numbers (langevin): xi of atom i (1-based original index) at innermost substep k (0-based within outer step n)
 *    is the Box-Muller transform of one Philox4x32-10 block with counter (i, n, k, low word of ctr1) and key `rng_key`.
 *    A function of (keys, outer step, substep, atom) only, so a run split into calls with the same keys takes the same
 *    draws; the reference's draws agree in distribution only (random_velocities! on the host rng);
 *  - f32 (langevin): c v + sigma xi is formed in double and rounded once;
 *  - massless atoms (1/m = 0) get no kick and no noise;
 *  - the substeps are unrolled into the captured step graph, so fractions[n_levels - 1] is limited to 1024.
 * MB_ERR_INVALID before any work for dt <= 0, n_steps < 0, n_levels outside 1 .. MB_MTS_MAX_LEVELS, fractions that are not
 * ordered as above, a term whose level is n_levels or more, kT or friction negative or not finite (langevin), a velocity
 * coupling set on the context, a decomposed (multi-GPU) context, and the logging errors of mb_simulate_vv_log.
 * MB_ERR_CAPACITY as in mb_simulate_vv. */
#define MB_MTS_MAX_LEVELS 8
typedef struct {
    double dt;                            /* outer time step, ps */
    int64_t n_steps;                      /* outer steps */
    int64_t init_step;
    int32_t remove_cm_every;              /* remove_CM_motion (default 1; 0 = never), in outer steps */
    int32_t n_levels;                     /* length of ordered_fractions */
    int32_t fractions[MB_MTS_MAX_LEVELS]; /* ordered_fractions; fractions[0] = 1 */
    int32_t langevin;                     /* 0: MTSIntegrator, 1: MTSLangevinIntegrator */
    int32_t reserved_;
    double kT;                            /* langevin: k * temperature in kJ/mol */
    double friction;                      /* langevin: ps^-1 */
    uint64_t rng_ctr1, rng_key;           /* langevin: the draws' keys */
} mb_mts_params_t;
int mb_simulate_mts(mb_ctx* ctx, void* coords, void* vels, const mb_mts_params_t* p, mb_log_t* log);

/* simulate!(sys, LangevinSplitting(dt, temperature, friction, splitting; remove_CM_motion), n_steps)
 * (src/simulators.jl:1212-1398; BAOAB is Leimkuhler and Matthews 2013, OBABO Bussi and Parrinello 2007; "BAB" is the
 * VelocityVerlet step and "BAOA" the Langevin step). ops[0 .. n_ops) is the splitting, a string over 'A', 'B' and 'O'. Each
 * letter takes the effective step dt / count(letter, splitting):
 *   A: x += v dt_A;   B: v += F/m dt_B;   O: v = c_i v + sigma_i xi with xi ~ N(0, 1)^3,
 *   c_i = exp(-friction dt / n_O / m_i), sigma_i = sqrt(kT / m_i (1 - c_i^2)) (n_O: the O's in the splitting).
 * The friction is a mass per time (g mol^-1 ps^-1), unlike mb_simulate_langevin's. Prologue as mb_simulate_vv: wrap, CM
 * removal when init_step == 0 and remove_cm_every != 0, neighbours, F0, loggers at init_step. Step n: the letters in
 * order; wrap; CM removal when n % remove_cm_every == 0; neighbours; loggers (mb_log_t, as for mb_simulate_vv_log; NULL: no
 * logging). Forces are recomputed as the reference recomputes them: they are known at the start of a step unless an A
 * follows the last B, an A makes them unknown, and a B recomputes them only when they are unknown. So BAOAB, OBABO, ABOBA,
 * BAOA, AB and BA evaluate the forces once per step, BABAB twice, and a splitting without an A or without a B never. A B that
 * recomputes before any A of its step is served by an evaluation at the end of the step before (the first: F0), at the same
 * positions. Each stretch of letters between two evaluations is one fused kernel. Where the engine differs from the
 * reference:
 *  - random numbers: xi of atom i (1-based original index) at the j-th O (0-based) of step n is the Box-Muller transform of
 *    one Philox4x32-10 block with counter (i, n, ctr1 + j as a 64-bit sum) and key `rng_key`; for j = 0 this is
 *    mb_simulate_langevin's draw. A function of (keys, step, j, atom) only, so a run split into calls with the same keys takes
 *    the same draws; the reference's draws agree in distribution only, as for Langevin;
 *  - neighbours: the exact displacement trigger of mb_simulate_vv, tested after every stretch of letters that moves the
 *    atoms, so every force evaluation reads current lists. The all-pairs path wraps at those points, not after every A;
 *  - f32: c_i and sigma_i are formed in double from the context's 1/m (rounded to the dtype), and c_i v + sigma_i xi is
 *    formed in double and rounded once;
 *  - massless atoms (1/m = 0) get no kick and no noise (c_i = 1, sigma_i = 0);
 *  - at most MB_SPLIT_MAX_OPS letters (the passes are unrolled into the captured step graph).
 * MB_ERR_INVALID before any work for an empty splitting, a letter other than 'A', 'B', 'O', more than MB_SPLIT_MAX_OPS
 * letters, dt <= 0, n_steps < 0, kT or friction negative or not finite, a velocity coupling set on the context, a
 * decomposed (multi-GPU) context, and the logging errors of mb_simulate_vv_log. MB_ERR_CAPACITY as in mb_simulate_vv. */
#define MB_SPLIT_MAX_OPS 32
typedef struct {
    double dt;
    int64_t n_steps;
    int64_t init_step;
    int32_t remove_cm_every;    /* LangevinSplitting.remove_CM_motion (default 1; 0 = never) */
    double kT;                  /* k * temperature in kJ/mol */
    double friction;            /* g mol^-1 ps^-1 (mass per time) */
    uint64_t rng_ctr1, rng_key; /* the draws' keys */
    int32_t n_ops;              /* letters in ops */
    char ops[MB_SPLIT_MAX_OPS]; /* the splitting: 'A', 'B', 'O' (not NUL-terminated) */
} mb_splitting_params_t;
int mb_simulate_langevin_splitting(mb_ctx* ctx, void* coords, void* vels, const mb_splitting_params_t* p, mb_log_t* log);

/* simulate!(sys, Verlet(dt; coupling, remove_CM_motion), n_steps) (src/simulators.jl:858-955), the leapfrog integrator: the
 * velocities are half a step behind the positions. Prologue as mb_simulate_vv: wrap, CM removal when init_step == 0 and
 * remove_cm_every != 0, neighbours, F0, loggers at init_step. Step n, with a = F/m:
 *   1. v += a dt
 *   2. x += v dt (one full drift); wrap
 *   3. CM removal when n % remove_cm_every == 0
 *   4. coupling: the Andersen thermostat of mb_simulate_vv when andersen_kT > 0 and andersen_prob > 0, with the same draws
 *   5. neighbours; F = forces(x) for step n + 1; loggers (mb_log_t, as for mb_simulate_vv_log; NULL: no logging).
 * The parameters are mb_vv_params_t's. One step is one fused kernel plus the force evaluation (and the Andersen kernel).
 * Where the engine differs from the reference:
 *  - the neighbour rebuild is triggered by the exact displacement test (as for mb_simulate_vv);
 *  - massless atoms (1/m = 0) get no kick.
 * MB_ERR_INVALID before any work for dt <= 0, n_steps < 0, a velocity coupling set on the context
 * (mb_set_velocity_coupling; velocity-rescaling couplings with Verlet take the stock path), a decomposed (multi-GPU)
 * context, and the logging errors of mb_simulate_vv_log. MB_ERR_CAPACITY as in mb_simulate_vv. */
int mb_simulate_verlet(mb_ctx* ctx, void* coords, void* vels, const mb_vv_params_t* p, mb_log_t* log);

/* simulate!(sys, StormerVerlet(dt), n_steps) (src/simulators.jl:957-1063). No coupling and no CM removal, not even in the
 * prologue: wrap, neighbours, F0, loggers at init_step. Step n, with a = F/m:
 *   1. d = v dt + a dt^2 / 2 on the first step of every call, d = v dt + a dt^2 on later steps
 *   2. x += d; v = d / dt; wrap
 *   3. neighbours; F = forces(x) for step n + 1; loggers (mb_log_t, as for mb_simulate_vv_log; NULL: no logging).
 * The reference forms the later steps from vector(x_last, x) + a dt^2 and sets v = vector(x_before, x_after) / dt. The
 * engine keeps no second coordinate set: at the end of a step v dt is that displacement, so it carries the previous
 * displacement as the velocity, through cell-list re-sorts and from one call to the next. Where the engine differs from the
 * reference:
 *  - f32: v dt is the displacement up to rounding, where the reference takes `vector` of wrapped coordinates, so the two
 *    differ at the ulp level;
 *  - the neighbour rebuild is triggered by the exact displacement test (as for mb_simulate_vv);
 *  - massless atoms (1/m = 0) feel no force.
 * MB_ERR_INVALID before any work for dt <= 0, n_steps < 0, a velocity coupling set on the context, a decomposed (multi-GPU)
 * context, and the logging errors of mb_simulate_vv_log. MB_ERR_CAPACITY as in mb_simulate_vv. */
typedef struct {
    double dt;
    int64_t n_steps;
    int64_t init_step;
} mb_stormer_params_t;
int mb_simulate_stormer_verlet(mb_ctx* ctx, void* coords, void* vels, const mb_stormer_params_t* p, mb_log_t* log);

/* simulate!(sys, OverdampedLangevin(dt, temperature, friction; remove_CM_motion), n_steps) (src/simulators.jl:1400-1490),
 * Brownian dynamics by Euler-Maruyama. Prologue as mb_simulate_vv: wrap, CM removal when init_step == 0 and
 * remove_cm_every != 0, neighbours, F0, loggers at init_step. Step n, with a = F/m and gamma the friction in ps^-1:
 *   1. x += a / gamma dt + sqrt(2 dt / gamma) sqrt(kT / m_i) xi with xi ~ N(0, 1)^3; wrap
 *   2. CM removal of v when n % remove_cm_every == 0. The velocities are otherwise never changed: as in the reference, the
 *      removal only affects what the loggers see
 *   3. neighbours; F = forces(x) for step n + 1; loggers (mb_log_t, as for mb_simulate_vv_log; NULL: no logging).
 * The parameters are mb_langevin_params_t's. One step is one fused kernel plus the force evaluation. Where the engine
 * differs from the reference:
 *  - random numbers: xi is mb_simulate_langevin's draw (one Philox4x32-10 block with counter (i, n, ctr1) and key
 *    `rng_key`, i the 1-based original index). A function of (keys, step, atom) only, so a run split into calls with the
 *    same keys takes the same draws; the reference's draws agree in distribution only;
 *  - f32: the displacement is formed in double and the new position rounded once;
 *  - massless atoms (1/m = 0) do not move (the reference's noise is Inf there);
 *  - the neighbour rebuild is triggered by the exact displacement test (as for mb_simulate_vv).
 * MB_ERR_INVALID before any work for dt <= 0, n_steps < 0, kT negative or not finite, friction <= 0 or not finite (the
 * reference's noise prefactor is infinite at 0), a velocity coupling set on the context, a decomposed (multi-GPU) context,
 * and the logging errors of mb_simulate_vv_log. MB_ERR_CAPACITY as in mb_simulate_vv. */
int mb_simulate_overdamped_langevin(mb_ctx* ctx, void* coords, void* vels, const mb_langevin_params_t* p, mb_log_t* log);

/* DPDInteraction(a, gamma, sigma, r_c, dt, use_neighbors, key) (src/interactions/dpd.jl:57-142), the pairwise interaction
 * of dissipative particle dynamics. With dr = c_j - c_i, r = |dr|, w = 1 - r / r_c and v_ij = v_i - v_j, the force on i is
 * -(f_C + f_D + f_R) dr with f_C = a w / r, f_D = gamma w^2 (dr . v_ij) / r^2, f_R = sigma w xi_ij dt^(-1/2) / r (dt is this
 * struct's, not the integrator's), and the energy is the conservative part (a / 2) r_c w^2; all zero for r >= r_c and for
 * r == 0. Special pairs get the full force; excluded pairs are skipped when use_neighbors is set (the reference's
 * use_neighbors = false loop visits every pair). xi_ij is symmetric in (i, j), so momentum is conserved exactly: one
 * Philox4x32-10 block with counter (min(i, j), max(i, j), step_lo, step_hi), i and j the 1-based atom indices and step the
 * simulate! step_n, and key (key_lo, key_hi); one N(0, 1) value from its words 0 and 1 by Box-Muller in double (the first
 * output of the O step's transform). The reference draws through PhiloxRNG.jl's randn: the two agree in distribution only.
 * It replaces the pairwise interactions of the context and takes part in the path choice through use_neighbors as an
 * mb_inter_t does: the cell-list path needs use_neighbors and r_list >= r_c (the reference suggests r_list = 1.5 r_c).
 * Bonded lists (mb_set_specific) are allowed. NULL clears it. Drops the captured step graphs.
 * MB_ERR_INVALID for r_c <= 0 or not finite, dt <= 0 or not finite, gamma or sigma < 0 or not finite, a not finite. Checked
 * at the next evaluation or simulate call, before any work: an mb_inter_t interaction, PME, LJDispersionCorrection or
 * implicit solvent on the same context, a decomposed (multi-GPU) context, r_list < r_c on the cell-list path, and an f32
 * context of more than 2^24 atoms (the position records carry the atom index as an exact float). */
typedef struct {
    double a, gamma, sigma, r_c, dt;
    uint64_t key;
    int32_t use_neighbors;
} mb_dpd_t;
int mb_set_dpd(mb_ctx* ctx, const mb_dpd_t* p);

/* forces(sys) of a system with a velocity-dependent pairwise term (mb_set_dpd): ADD the forces of all interactions (DPD +
 * bonded) for coords and vels (n x 3 each, original order) at step step_n into fs_mat and, if non-NULL, the energy (the
 * conservative DPD part + bonded) into pe. fs_mat may be NULL. On a DPD context mb_forces, mb_forces_energy and
 * mb_forces_energy_all return MB_ERR_INVALID with a force output (they have no velocities) and with a virial output (DPD has
 * no virial); mb_energy keeps working. */
int mb_forces_energy_vel(mb_ctx* ctx, const void* coords, const void* vels, void* fs_mat, void* pe, int64_t step_n);

/* simulate!(sys, DPDVelocityVerlet(dt, lambda; remove_CM_motion), n_steps) (src/simulators.jl:670-842), the Groot-Warren
 * modified velocity Verlet. Prologue: wrap, CM removal when init_step == 0 and remove_cm_every != 0, neighbours, F0 at step
 * init_step evaluated with the current velocities, loggers at init_step. Step n, with a = F/m:
 *   1. v += a(t) dt/2
 *   2. x += v dt; wrap
 *   3. v_half = v; v_pred = v_half + (lambda - 1/2) dt a(t)
 *   4. F(t + dt) = forces(x, v_pred) keyed by step n
 *   5. v = v_half + a(t + dt) dt/2
 *   6. CM removal when n % remove_cm_every == 0
 *   7. neighbours; loggers (mb_log_t, as for mb_simulate_vv_log; NULL: no logging).
 * One step is VelocityVerlet's launches: the drift kernel (which also stores v_pred), [rebuild or wrap], forces, bonded, the
 * second kick. Each call's F0 uses v(t), not a v_pred, so a run split into calls differs from one call, as in the
 * reference. On a context without mb_set_dpd the step is mb_simulate_vv's, bit for bit. Where the engine differs from the
 * reference:
 *  - the pairwise draw (mb_set_dpd);
 *  - the neighbour rebuild is triggered by the exact displacement test after the drift (as for mb_simulate_vv);
 *  - massless atoms (1/m = 0) get no kick.
 * MB_ERR_INVALID before any work for dt <= 0, n_steps < 0, lambda not finite, a velocity coupling set on the context
 * (mb_set_velocity_coupling), a decomposed (multi-GPU) context, the refusals of mb_set_dpd, and the logging errors of
 * mb_simulate_vv_log. Every other integrator and the minimiser refuse a DPD context. MB_ERR_CAPACITY as in mb_simulate_vv. */
typedef struct {
    double dt;
    int64_t n_steps;
    int64_t init_step;
    int32_t remove_cm_every;
    double lambda;  /* the velocity prediction parameter (reference default 0.65) */
} mb_dpd_vv_params_t;
int mb_simulate_dpd_vv(mb_ctx* ctx, void* coords, void* vels, const mb_dpd_vv_params_t* p, mb_log_t* log);

/* Several simulate calls on one GPU with their steps in flight at once (temperature replica exchange runs one per
 * thermodynamic state). Member i is the call mb_simulate_<kind>(ctx, coords, vels, params, log) with `params` pointing at
 * that entry's parameter struct:
 *   MB_INTEG_VV                  mb_simulate_vv_log               mb_vv_params_t
 *   MB_INTEG_LANGEVIN            mb_simulate_langevin             mb_langevin_params_t
 *   MB_INTEG_NOSE_HOOVER         mb_simulate_nose_hoover          mb_nosehoover_params_t
 *   MB_INTEG_MTS                 mb_simulate_mts                  mb_mts_params_t
 *   MB_INTEG_LANGEVIN_SPLITTING  mb_simulate_langevin_splitting   mb_splitting_params_t
 *   MB_INTEG_VERLET              mb_simulate_verlet               mb_vv_params_t
 *   MB_INTEG_STORMER_VERLET      mb_simulate_stormer_verlet       mb_stormer_params_t
 *   MB_INTEG_OVERDAMPED_LANGEVIN mb_simulate_overdamped_langevin  mb_langevin_params_t
 *   MB_INTEG_DPD_VV              mb_simulate_dpd_vv               mb_dpd_vv_params_t
 * Every member's prologue runs first (refusals, ingest, F0, the loggers at init_step, graph capture); then the steps,
 * round-robin, one per member per round, each enqueued on its own context's stream (a member with fewer steps drops out
 * early); then every member's epilogue (export, copy-back, the overflow check). Each member computes what its single call
 * computes; the step kernels are the same, and no kernel reads state another context writes.
 * Returns MB_OK when every member succeeded, otherwise the first failing member's status; `status` holds each member's
 * outcome. A failed member leaves its buffers as its single call would have (after MB_ERR_CAPACITY: invalid; retry it
 * with its single call). MB_ERR_INVALID before any work for n <= 0, a null member array, context or params, an unknown
 * kind, one context in two members, members on different devices, and a decomposed (multi-GPU) context; a refused group
 * (n > 0, members non-null) sets every member's status to MB_ERR_INVALID. */
enum {
    MB_INTEG_VV = 0,
    MB_INTEG_LANGEVIN = 1,
    MB_INTEG_NOSE_HOOVER = 2,
    MB_INTEG_MTS = 3,
    MB_INTEG_LANGEVIN_SPLITTING = 4,
    MB_INTEG_VERLET = 5,
    MB_INTEG_STORMER_VERLET = 6,
    MB_INTEG_OVERDAMPED_LANGEVIN = 7,
    MB_INTEG_DPD_VV = 8
};
typedef struct {
    mb_ctx* ctx;
    void* coords;
    void* vels;
    int32_t kind;        /* MB_INTEG_* */
    const void* params;  /* that kind's parameter struct */
    mb_log_t* log;       /* NULL: no logging */
    int32_t status;      /* out: this member's MB_* status */
} mb_group_member_t;
int mb_simulate_group(int32_t n, mb_group_member_t* members);

/* simulate!(sys, SteepestDescentMinimizer(step_size, max_steps, tol)) (src/simulators.jl:183-274) on the device: wrap the
 * coordinates, E = potential energy; then for step n = init_step+1 .. init_step+max_steps: F = forces, m = max |F_i|,
 * x <- wrap(x + h F / m), E_trial = potential energy; E_trial < E accepts (h <- 6h/5, E <- E_trial), otherwise x is restored
 * (h <- h/5); the loop stops after the iteration in which m < tol. Energy and forces are those of mb_forces_energy_all
 * (pairwise + specific + PME + LJDispersionCorrection). coords: n x 3, host or device, updated in place and returned
 * wrapped, original atom order. Where this differs from the reference:
 *  - one evaluation per iteration: forces and energy of the trial together. On accept the trial's forces are the next F;
 *    on reject F is kept (the reference recomputes it at the restored coordinates and gets the same value);
 *  - E and E_trial are the engine's double sums, compared in double; m = sqrt(max |F_i|^2) in double;
 *  - f32: the moved coordinate x + h F / m is formed in double and rounded once (the reference's step size is a Float64);
 *  - neighbours: always the exact displacement trigger (rebuild when an atom is more than skin/2 from its position at the
 *    last build), whatever mb_set_neighbor_policy's rebuild_every says (the reference's GPU finder is exact at every call);
 *  - m = 0 or not finite: the positions stay unchanged and the iteration is recorded as rejected with E_trial = NaN
 *    (the reference's x + h F / m is NaN and is rejected).
 * One iteration is one CUDA graph body (trial, conditional rebuild, evaluation, decision, accept/restore) inside a
 * conditional WHILE node: one graph launch per call. PME, profiling and a failed capture take the stream path (one
 * iteration per host round trip). The context's velocity and force state afterwards is unspecified (mb_simulate_vv starts
 * from a clean one). MB_ERR_INVALID before any work for max_steps < 0, step_size <= 0, tol < 0, a trace capacity below
 * max_steps + 1, and decomposed (multi-GPU) contexts; MB_ERR_CAPACITY as in mb_simulate_vv (results invalid, retry from
 * the starting coordinates). */
typedef struct {
    double step_size;         /* h0 in nm (reference default 0.01) */
    int64_t max_steps;        /* default 1000 */
    double tol;               /* kJ mol^-1 nm^-1 (default 1000) */
    int64_t init_step;
    double* trace;            /* optional (NULL): trace_capacity x 4 doubles (step, E or E_trial, max force, accepted 0/1),
                               * host or device. Record 0 = (init_step, E0, NaN, 1), then one per iteration */
    int64_t trace_capacity;   /* records the trace holds: at least max_steps + 1 */
    /* written back */
    int64_t n_iterations;     /* iterations taken (records written = n_iterations + 1) */
    double energy;            /* E of the returned coordinates */
    double max_force;         /* max |F_i| at the returned coordinates */
    double final_step_size;   /* h after the last iteration */
    int32_t converged;        /* the last iteration's max force was below tol */
    int32_t reserved_;
} mb_sd_params_t;
int mb_minimize_sd(mb_ctx* ctx, void* coords, mb_sd_params_t* p);

/* remove_CM_motion! (ext/MollyCUDAExt.jl:2373; src/spatial.jl:901-929) on an n x 3 velocity array. */
int mb_remove_cm_motion(mb_ctx* ctx, void* vels);
/* kinetic_energy (src/energy.jl:56-70): writes 1/2 sum m v.v to *ke_host (double, host). */
int mb_kinetic_energy(mb_ctx* ctx, const void* vels, double* ke_host);

/* Kinetic energy tensor K = 1/2 sum m v (x) v (src/energy.jl:56-70; the reference copies masses and velocities to the
 * host for it, :58-59): 3x3 symmetric, row-major == column-major, host doubles. */
int mb_kinetic_energy_tensor(mb_ctx* ctx, const void* vels, double* ke_tensor9_host);
/* random_velocities!(sys, temp; rng) (src/spatial.jl:819-831, GPU kernel src/kernels.jl:688-703): fills vels (n x 3, host
 * or device) with Maxwell-Boltzmann velocities, sigma = sqrt(kT / m) per component, zero for massless atoms. Philox4x32-10
 * keyed by the caller's two rand(rng, UInt64); statistical parity with the reference (its uniform -> normal transform
 * lives in PhiloxRNG.jl, which is not vendored: SURVEY.md 8c). kT = k * temp in kJ/mol. */
int mb_random_velocities(mb_ctx* ctx, void* vels, double kT, uint64_t rng_ctr1, uint64_t rng_key);

/* find_neighbors(sys, nf, ..., force=true): force a rebuild from coords now (synchronous; also
 * re-derives capacities). */
int mb_rebuild_neighbors(mb_ctx* ctx, const void* coords);
int mb_stats(mb_ctx* ctx, mb_stats_t* host_out);
int mb_synchronize(mb_ctx* ctx);
/* Multiply the auto-derived halo/list capacities (after MB_ERR_CAPACITY). */
int mb_set_capacity_scale(mb_ctx* ctx, double scale);
/* Tuning overrides (CUDALaunchConfig analogue, src/cuda_config.jl:27-41): brick dims in cells
 * (0 = auto), lanes per i-atom (8, or 0 = default; other values are rejected). */
int mb_set_launch_config(mb_ctx* ctx, const int32_t brick_dims[3], int32_t lanes_per_atom);

/* Per-kernel-category CUDA-event timing (benchmark_gpu_tiles.jl-style stage timers,
 * benchmark/gpu_profile_utils.jl:12-18); results through mb_stats. Resets the accumulators. */
int mb_set_profiling(mb_ctx* ctx, int enable);

/* Spatial decomposition over ranks (one process per GPU; the reference has none, docs/src/documentation.md:1826).
 * The box is cut into z-slabs of whole cell layers; a rank integrates the atoms of its slab and evaluates forces for
 * its bricks. Per step: forward halo exchange of positions between neighbouring slabs (grouped ncclSend/ncclRecv of
 * contiguous slot ranges, 2 cell layers each way; full-shell lists need no reverse force exchange) and one 24-byte
 * all-reduce of sum(m v). At every rebuild (fixed interval, default 20 steps) positions and velocities are all-gathered
 * and every rank re-sorts the replicated system identically. mb_simulate_vv takes and returns the whole system on
 * every rank. rank 0 creates the id, the host runtime (torch.distributed / MPI) broadcasts its 128 bytes. */
int mb_comm_unique_id(void* out128);
int mb_comm_init(mb_ctx* ctx, const void* unique_id128, int rank, int nranks);
/* The host-side plan of the halo exchange (no GPU needed): layer_start = ncz + 1 slot offsets of the cell layers;
 * outputs are (peer, first slot, slot count) triples in the order the exchange posts them. */
int mb_decomp_plan(int ncz, int halo_layers, int nranks, int rank, const int32_t* layer_start, int32_t* send_out,
                   int32_t* n_send, int32_t* recv_out, int32_t* n_recv, int capacity);

#ifdef __cplusplus
}
#endif
#endif /* MOLLYB200_H */
