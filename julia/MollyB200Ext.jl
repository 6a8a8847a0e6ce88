# MollyB200Ext.jl — Julia-side shim that plugs libmollyb200.so in behind Molly.jl's own API.
#
# Written against Molly.jl v0.23.3 (src/force.jl, src/energy.jl, src/simulators.jl, src/neighbors.jl,
# ext/MollyCUDAExt.jl). Julia is not installed in the build image, so this file has only been checked by
# reading; the Python mirror `molly.jl_b200/api.py` binds exactly the same C entry points and is what CI runs.
#
# It overrides the same generic functions that ext/MollyCUDAExt.jl overrides (SURVEY.md §8b):
#   Molly.pairwise_forces_loop_gpu!(buffers, sys, pairwise_inters, nbs::Nothing, Val(needs_vir), step_n)   ext:845
#   Molly.pairwise_pe_loop_gpu!(pe_vec_nounits, buffers, sys, pairwise_inters, nbs::Nothing, step_n)        ext:936
#   Molly.simulate!(sys, sim::VelocityVerlet, n_steps; ...)                                                 simulators.jl:547
#   Molly.simulate!(sys, sim::SteepestDescentMinimizer; ...)                                                simulators.jl:183
#   Molly.simulate!(sys, sim::Langevin, n_steps; ...) with coupling === nothing                              simulators.jl:1101
#   Molly.simulate!(sys, sim::NoseHoover, n_steps; ...) with coupling === nothing                            simulators.jl:1534
#   Molly.simulate!(sys, sim::LangevinSplitting, n_steps; ...) with at most 32 letters                      simulators.jl:1252
#   Molly.simulate!(sys, sim::AbstractMTSIntegrator, n_steps; ...) with coupling === nothing                 simulators.jl:1850
#   Molly.simulate!(sys, sim::Verlet, n_steps; ...) with coupling nothing or one AndersenThermostat           simulators.jl:868
#   Molly.simulate!(sys, sim::StormerVerlet, n_steps; ...)                                                   simulators.jl:970
#   Molly.simulate!(sys, sim::OverdampedLangevin, n_steps; ...)                                              simulators.jl:1427
#   Molly.simulate!(sys, sim::DPDVelocityVerlet, n_steps; ...) with coupling === nothing                     simulators.jl:711
# (Molly.remove_CM_motion! for CuArray Systems is NOT redefined: the stock extension owns that exact signature)
# and falls through to the stock methods (invoke) for anything it does not recognise: non-cubic boundaries,
# constraints, virtual sites, couplings other than one AndersenThermostat, ImmediateThermostat, BerendsenThermostat or
# VelocityRescaleThermostat, interactions outside
# {LennardJones, Coulomb, CoulombReactionField, CoulombEwald} or unsupported cutoffs / mixing rules, general interactions
# other than LJDispersionCorrection and one ImplicitSolventOBC / ImplicitSolventGBN2 (implicit solvent runs in the engine).
# forces(sys) / potential_energy(sys) keep Molly's own evaluation of general interactions, implicit solvent included: the
# seam this file overrides there is the pairwise loop.

module MollyB200Ext

using Molly
using CUDA
using Random
using StaticArrays
using Unitful

const LIB = get(ENV, "MOLLYB200_LIB", joinpath(@__DIR__, "..", "molly.jl_b200", "libmollyb200.so"))

# ---- C structs (include/mollyb200.h) ------------------------------------------------------------------
struct MBInter
    kind::Int32
    cutoff_kind::Int32
    r_cut::Float64
    r_act::Float64
    weight_special::Float64
    coulomb_const::Float64
    solvent_dielectric::Float64
    ewald_alpha::Float64
    sigma_mix::Int32
    eps_mix::Int32
    approx_erfc::Int32
    use_neighbors::Int32
end

struct MBVVParams
    dt::Float64
    n_steps::Int64
    init_step::Int64
    remove_cm_every::Int32
    andersen_kT::Float64
    andersen_prob::Float64
    rng_ctr1::UInt64
    rng_key::UInt64
end

# mb_dpd_t (mb_set_dpd) and mb_dpd_vv_params_t (mb_simulate_dpd_vv)
struct MBDpd
    a::Float64
    gamma::Float64
    sigma::Float64
    r_c::Float64
    dt::Float64
    key::UInt64
    use_neighbors::Int32
end
struct MBDpdVVParams
    dt::Float64
    n_steps::Int64
    init_step::Int64
    remove_cm_every::Int32
    lambda::Float64
end

# mb_langevin_params_t (mb_simulate_langevin)
struct MBLangevinParams
    dt::Float64
    n_steps::Int64
    init_step::Int64
    remove_cm_every::Int32
    kT::Float64
    friction::Float64
    rng_ctr1::UInt64
    rng_key::UInt64
end

# mb_splitting_params_t (mb_simulate_langevin_splitting)
struct MBSplittingParams
    dt::Float64
    n_steps::Int64
    init_step::Int64
    remove_cm_every::Int32
    kT::Float64
    friction::Float64
    rng_ctr1::UInt64
    rng_key::UInt64
    n_ops::Int32
    ops::NTuple{32, UInt8}
end

# mb_nosehoover_params_t (mb_simulate_nose_hoover)
struct MBNoseHooverParams
    dt::Float64
    n_steps::Int64
    init_step::Int64
    remove_cm_every::Int32
    kT::Float64
    damping::Float64
end

# mb_stormer_params_t (mb_simulate_stormer_verlet)
struct MBStormerParams
    dt::Float64
    n_steps::Int64
    init_step::Int64
end

# mb_mts_params_t (mb_simulate_mts)
struct MBMTSParams
    dt::Float64
    n_steps::Int64
    init_step::Int64
    remove_cm_every::Int32
    n_levels::Int32
    fractions::NTuple{8, Int32}
    langevin::Int32
    reserved_::Int32
    kT::Float64
    friction::Float64
    rng_ctr1::UInt64
    rng_key::UInt64
end

# mb_gbsa_t (mb_set_implicit_solvent)
struct MBGbsa
    dist_cutoff::Float64
    offset::Float64
    probe_radius::Float64
    sa_factor::Float64
    factor_solute::Float64
    factor_solvent::Float64
    kappa::Float64
    neck_scale::Float64
    neck_cut::Float64
    use_ace::Int32
    n_neck_classes::Int32
end
const MB_GB_MAX_NECK_CLASSES = 32

# mb_vcoupling_t (mb_set_velocity_coupling)
struct MBVCoupling
    kind::Int32       # 1 Immediate, 2 Berendsen, 3 velocity rescale (MB_VC_*)
    n_steps::Int32
    kT::Float64
    tau::Float64
end

# mb_log_t; mutable so that ccall can write the record counts back
mutable struct MBLog
    energy_every::Int64
    coords_every::Int64
    vels_every::Int64
    log_initial::Int32
    reserved_::Int32
    energies::Ptr{Float64}
    coords::Ptr{Cvoid}
    vels::Ptr{Cvoid}
    energy_capacity::Int64
    coords_capacity::Int64
    vels_capacity::Int64
    n_energies::Int64
    n_coords::Int64
    n_vels::Int64
end

const MB_LJ, MB_COULOMB, MB_CRF, MB_EWALD_REAL = Int32(0), Int32(1), Int32(2), Int32(3)
const MB_CUT_NONE, MB_CUT_DISTANCE, MB_CUT_SHIFTED_POTENTIAL, MB_CUT_SHIFTED_FORCE = Int32(0), Int32(1), Int32(2), Int32(3)
const MB_CUT_CUBIC_SPLINE, MB_CUT_POLYNOMIAL = Int32(4), Int32(5)
const MB_MIX_LORENTZ, MB_MIX_GEOMETRIC = Int32(0), Int32(1)

function check(rc::Integer)
    rc == 0 && return nothing
    msg = unsafe_string(ccall((:mb_last_error, LIB), Cstring, ()))
    error("libmollyb200 error $rc: $msg")   # same failure mode as ext/MollyCUDAExt.jl:733-739
end

# ---- translation of Molly interaction structs to descriptors -----------------------------------------
# (kind, dist_cutoff, dist_activation)
cutoff_desc(::NoCutoff) = (MB_CUT_NONE, 0.0, 0.0)
cutoff_desc(c::DistanceCutoff) = (MB_CUT_DISTANCE, Float64(ustrip(c.dist_cutoff)), 0.0)
cutoff_desc(c::ShiftedPotentialCutoff) = (MB_CUT_SHIFTED_POTENTIAL, Float64(ustrip(c.dist_cutoff)), 0.0)
cutoff_desc(c::ShiftedForceCutoff) = (MB_CUT_SHIFTED_FORCE, Float64(ustrip(c.dist_cutoff)), 0.0)
cutoff_desc(c::CubicSplineCutoff) = (MB_CUT_CUBIC_SPLINE, Float64(ustrip(c.dist_cutoff)), Float64(ustrip(c.dist_activation)))
cutoff_desc(c::PolynomialCutoff) = (MB_CUT_POLYNOMIAL, Float64(ustrip(c.dist_cutoff)), Float64(ustrip(c.dist_activation)))
cutoff_desc(::Any) = nothing

mix_desc(::Molly.LorentzMixing) = MB_MIX_LORENTZ
mix_desc(::Molly.GeometricMixing) = MB_MIX_GEOMETRIC
mix_desc(::Any) = nothing

function descriptor(inter::LennardJones)
    cd = cutoff_desc(inter.cutoff)
    sm, em = mix_desc(inter.σ_mixing), mix_desc(inter.ϵ_mixing)
    (isnothing(cd) || isnothing(sm) || em != MB_MIX_GEOMETRIC) && return nothing
    !(inter.shortcut isa Molly.LJZeroShortcut) && return nothing
    return MBInter(MB_LJ, cd[1], cd[2], cd[3], Float64(inter.weight_special), 138.93545764, 1.0, 0.0, sm, em, 0,
                   Int32(inter.use_neighbors))
end
function descriptor(inter::Coulomb)
    cd = cutoff_desc(inter.cutoff)
    isnothing(cd) && return nothing
    return MBInter(MB_COULOMB, cd[1], cd[2], cd[3], Float64(inter.weight_special), Float64(ustrip(inter.coulomb_const)),
                   1.0, 0.0, 0, 1, 0, Int32(inter.use_neighbors))
end
function descriptor(inter::CoulombReactionField)
    return MBInter(MB_CRF, MB_CUT_DISTANCE, Float64(ustrip(inter.dist_cutoff)), 0.0, Float64(inter.weight_special),
                   Float64(ustrip(inter.coulomb_const)), Float64(inter.solvent_dielectric), 0.0, 0, 1, 0,
                   Int32(inter.use_neighbors))
end
# CoulombEwald (src/interactions/coulomb.jl:1320-1441): alpha and approximate_erfc are fields of the struct
function descriptor(inter::CoulombEwald)
    return MBInter(MB_EWALD_REAL, MB_CUT_DISTANCE, Float64(ustrip(inter.dist_cutoff)), 0.0, Float64(inter.weight_special),
                   Float64(ustrip(inter.coulomb_const)), 1.0, Float64(ustrip(inter.α)), 0, 1,
                   Int32(inter.approximate_erfc), Int32(inter.use_neighbors))
end
descriptor(::Any) = nothing

# ---- per-System context (what BuffersGPU + GPUNeighborFinder caches hold in the reference) ------------
mutable struct Context
    handle::Ptr{Cvoid}
    cache_generation::Int
end
const CONTEXTS = IdDict{Any, Context}()

# a pairwise tuple of exactly one DPDInteraction (src/interactions/dpd.jl): the engine runs it through mb_set_dpd, with no
# mb_inter_t. engine_eligible has no descriptor for it, so every integrator takeover leaves a DPD System to the stock method;
# only the pairwise seams and the DPDVelocityVerlet method ask dpd_eligible instead.
dpd_only(inters) = inters isa Tuple && length(inters) == 1 && inters[1] isa DPDInteraction
# DPD runs in reduced units: parameters with Unitful units are not taken over (nothing)
function dpd_desc(d::DPDInteraction)
    all(x -> x isa Real, (d.a, d.γ, d.σ, d.r_c, d.dt)) || return nothing
    return MBDpd(Float64(d.a), Float64(d.γ), Float64(d.σ), Float64(d.r_c), Float64(d.dt), UInt64(d.key), Int32(d.use_neighbors))
end
# set the tuple's DPDInteraction on the context, or clear it (every caller of context_for with the System's tuple)
function set_dpd!(ctx, inters)
    if dpd_only(inters)
        check(ccall((:mb_set_dpd, LIB), Cint, (Ptr{Cvoid}, Ref{MBDpd}), ctx.handle, Ref(dpd_desc(inters[1]))))
    else
        check(ccall((:mb_set_dpd, LIB), Cint, (Ptr{Cvoid}, Ptr{MBDpd}), ctx.handle, C_NULL))
    end
end

function engine_eligible(sys::System{3, <:CuArray, T}, inters) where T
    T in (Float32, Float64) || return nothing
    (sys.boundary isa CubicBoundary || sys.boundary isa TriclinicBoundary{3, <:Any, <:Any, true}) || return nothing
    length(sys.constraints) == 0 || return nothing
    isempty(sys.virtual_sites) || return nothing
    descs = map(descriptor, inters)
    any(isnothing, descs) && return nothing
    return collect(MBInter, descs)
end

# the System-level conditions of engine_eligible (no pairwise interaction to describe) and a unitless lone DPDInteraction:
# an empty descriptor list for context_for, or nothing
function dpd_eligible(sys::System{3, <:CuArray}, inters)
    dpd_only(inters) && !isnothing(dpd_desc(inters[1])) || return nothing
    return engine_eligible(sys, ())
end

function context_for(sys::System{3, <:CuArray, T}, descs::Vector{MBInter}, inters=sys.pairwise_inters) where T
    nf = sys.neighbor_finder
    gen = nf isa GPUNeighborFinder ? nf.cache_generation : 0
    ctx = get(CONTEXTS, sys.atoms, nothing)
    if isnothing(ctx) || ctx.cache_generation != gen    # exception-list update invalidates cached masks
        isnothing(ctx) || ccall((:mb_ctx_destroy, LIB), Cvoid, (Ptr{Cvoid},), ctx.handle)
        h = Ref{Ptr{Cvoid}}(C_NULL)
        stream = CUDA.stream().handle
        check(ccall((:mb_ctx_create, LIB), Cint, (Cint, Cint, Ptr{Cvoid}, Ref{Ptr{Cvoid}}),
                    CUDA.deviceid(CUDA.device()), T == Float32 ? 32 : 64, stream, h))
        # atoms: Molly's bits layout Atom{Int32,T,T,T,T,T} is read directly from device memory
        check(ccall((:mb_set_atoms, LIB), Cint, (Ptr{Cvoid}, Int64, CuPtr{Cvoid}), h[], length(sys.atoms),
                    pointer(sys.atoms)))
        if sys.boundary isa TriclinicBoundary      # approx_images = true only (engine_eligible); no-list kernel
            bv = sys.boundary.basis_vectors
            basis = Float64[ustrip(bv[i][j]) for i in 1:3 for j in 1:3]   # row-major: bv1, bv2, bv3
            check(ccall((:mb_set_box_triclinic, LIB), Cint, (Ptr{Cvoid}, Ptr{Float64}), h[], basis))
        else
            side = Float64.(ustrip.(sys.boundary.side_lengths))
            check(ccall((:mb_set_box, LIB), Cint, (Ptr{Cvoid}, Ptr{Float64}), h[], collect(side)))
        end
        if nf isa GPUNeighborFinder
            ei, ej = Array(nf.excluded_i), Array(nf.excluded_j)     # sparse 1-based lists, neighbors.jl:104-115
            si, sj = Array(nf.special_i), Array(nf.special_j)
            check(ccall((:mb_set_exceptions, LIB), Cint,
                        (Ptr{Cvoid}, Int64, Ptr{Int32}, Ptr{Int32}, Int64, Ptr{Int32}, Ptr{Int32}),
                        h[], length(ei), ei, ej, length(si), si, sj))
            check(ccall((:mb_set_neighbor_policy, LIB), Cint, (Ptr{Cvoid}, Float64, Cint), h[],
                        Float64(ustrip(nf.dist_cutoff)), 0))
        end
        ctx = Context(h[], gen)
        CONTEXTS[sys.atoms] = ctx
    end
    check(ccall((:mb_set_inters, LIB), Cint, (Ptr{Cvoid}, Cint, Ptr{MBInter}), ctx.handle, length(descs), descs))
    set_dpd!(ctx, inters)
    return ctx
end

# ---- forces / energy seam -----------------------------------------------------------------------------
function Molly.pairwise_forces_loop_gpu!(buffers, sys::System{3, <:CuArray, T}, pairwise_inters::Tuple,
                                         nbs::Nothing, ::Val{needs_vir}, step_n) where {T, needs_vir}
    descs = dpd_only(pairwise_inters) ? dpd_eligible(sys, pairwise_inters) : engine_eligible(sys, pairwise_inters)
    if isnothing(descs)
        # the STOCK method's own signature (ext/MollyCUDAExt.jl:845: System{D, <:CuArray, T}, untyped pairwise_inters);
        # naming this method's System{3, ...} signature here would recurse into itself
        return invoke(Molly.pairwise_forces_loop_gpu!,
                      Tuple{Any, System{D, <:CuArray, T} where D, Any, Nothing, Val{needs_vir}, Any},
                      buffers, sys, pairwise_inters, nbs, Val(needs_vir), step_n)
    end
    ctx = context_for(sys, descs, pairwise_inters)
    if dpd_only(pairwise_inters)
        # the forces depend on the velocities and the step (pairwise_uses_velocity, src/types.jl:50-59). The call adds the
        # context's bonded forces too, so a System with specific lists takes the stock method instead; no virial.
        if !isempty(sys.specific_inter_lists) || needs_vir
            return invoke(Molly.pairwise_forces_loop_gpu!,
                          Tuple{Any, System{D, <:CuArray, T} where D, Any, Nothing, Val{needs_vir}, Any},
                          buffers, sys, pairwise_inters, nbs, Val(needs_vir), step_n)
        end
        check(ccall((:mb_forces_energy_vel, LIB), Cint,
                    (Ptr{Cvoid}, CuPtr{Cvoid}, CuPtr{Cvoid}, CuPtr{Cvoid}, CuPtr{Cvoid}, Int64),
                    ctx.handle, pointer(sys.coords), pointer(sys.velocities), pointer(buffers.fs_mat), CU_NULL, step_n))
        return buffers
    end
    vir = needs_vir ? pointer(buffers.virial_nounits) : CU_NULL
    # contract: ADD into buffers.fs_mat (D x N, original order) and buffers.virial_nounits
    check(ccall((:mb_forces, LIB), Cint, (Ptr{Cvoid}, CuPtr{Cvoid}, CuPtr{Cvoid}, CuPtr{Cvoid}, Int64),
                ctx.handle, pointer(sys.coords), pointer(buffers.fs_mat), vir, step_n))
    return buffers
end

function Molly.pairwise_pe_loop_gpu!(pe_vec_nounits, buffers, sys::System{3, <:CuArray, T}, pairwise_inters::Tuple,
                                     nbs::Nothing, step_n) where T
    descs = dpd_only(pairwise_inters) ? dpd_eligible(sys, pairwise_inters) : engine_eligible(sys, pairwise_inters)
    if isnothing(descs)
        return invoke(Molly.pairwise_pe_loop_gpu!,   # stock: ext/MollyCUDAExt.jl:936
                      Tuple{Any, Any, System{D, <:CuArray, T} where D, Any, Nothing, Any},
                      pe_vec_nounits, buffers, sys, pairwise_inters, nbs, step_n)
    end
    ctx = context_for(sys, descs, pairwise_inters)
    check(ccall((:mb_energy, LIB), Cint, (Ptr{Cvoid}, CuPtr{Cvoid}, CuPtr{Cvoid}, Int64),
                ctx.handle, pointer(sys.coords), pointer(pe_vec_nounits), step_n))
    return pe_vec_nounits
end

# ---- specific (bonded) interaction lists -> mb_set_specific ----------------------------------------------
# InteractionList{1,2,3,4}Atoms (src/types.jl:89-157) whose element type is one of the engine's kinds (MB_SPECIFIC_* in
# include/mollyb200.h). Anything else makes simulate! fall through to the stock path. A PeriodicTorsion with several
# Fourier terms becomes one entry per term (zero-k padding terms are dropped), like src/interactions/periodic_torsion.jl:100-142
# sums them. Units are stripped: the engine works in nm, kJ/mol and radians.
specific_kind(::Type) = nothing
specific_kind(::Type{<:HarmonicBond}) = 0
specific_kind(::Type{<:HarmonicAngle}) = 1
specific_kind(::Type{<:HarmonicPositionRestraint}) = 3
specific_kind(::Type{<:MorseBond}) = 4
specific_kind(::Type{<:FENEBond}) = 5
specific_kind(::Type{<:CosineAngle}) = 6
specific_kind(::Type{<:UreyBradley}) = 7
specific_kind(::Type{<:HarmonicTorsion}) = 8
specific_kind(::Type{<:RBTorsion}) = 9
# the parameters of one term in mb_set_specific's order
specific_params(b::HarmonicBond) = (b.k, b.r0)
specific_params(a::HarmonicAngle) = (a.k, a.θ0)
specific_params(r::HarmonicPositionRestraint) = (r.k, r.x0...)
specific_params(b::MorseBond) = (b.D, b.a, b.r0)
specific_params(b::FENEBond) = (b.k, b.r0, b.σ, b.ϵ)
specific_params(a::CosineAngle) = (a.k, a.θ0)
specific_params(a::UreyBradley) = (a.kangle, a.θ0, a.kbond, a.r0)
specific_params(t::HarmonicTorsion) = (t.k, t.θ0)
specific_params(t::RBTorsion) = (t.f1, t.f2, t.f3, t.f4)

atom_columns(sil::InteractionList1Atoms) = (sil.is,)
atom_columns(sil::InteractionList2Atoms) = (sil.is, sil.js)
atom_columns(sil::InteractionList3Atoms) = (sil.is, sil.js, sil.ks)
atom_columns(sil::InteractionList4Atoms) = (sil.is, sil.js, sil.ks, sil.ls)

# (kind, atom indices atoms x n (1-based, column = one term), params n_params x n), or nothing
function specific_desc(sil::Union{InteractionList1Atoms, InteractionList2Atoms, InteractionList3Atoms, InteractionList4Atoms})
    inters = Array(sil.inters)
    cols = map(Array, atom_columns(sil))
    if sil isa InteractionList4Atoms && eltype(inters) <: PeriodicTorsion
        idx, par = Int32[], Float64[]
        for (t, tor) in enumerate(inters), m in eachindex(tor.periodicities)
            k = Float64(ustrip(tor.ks[m]))
            k == 0 && continue
            append!(idx, (c[t] for c in cols))
            append!(par, (Float64(tor.periodicities[m]), Float64(ustrip(tor.phases[m])), k))
        end
        return (2, reshape(idx, 4, :), reshape(par, 3, :))
    end
    kind = specific_kind(eltype(inters))
    isnothing(kind) && return nothing
    idx = Int32[c[t] for t in eachindex(inters) for c in cols]
    par = Float64[ustrip(p) for b in inters for p in specific_params(b)]
    return (kind, reshape(idx, length(cols), :), reshape(par, :, length(inters)))
end
specific_desc(::Any) = nothing

# The engine holds one array per kind and each mb_set_specific call replaces it, so the lists of one kind (e.g. an Amber
# system's proper and improper PeriodicTorsion lists) are concatenated in list order, as the Python System does.
function set_specific!(ctx::Context, sys)
    descs = collect(map(specific_desc, sys.specific_inter_lists))
    any(isnothing, descs) && return false
    for kind in unique(first.(descs))
        mine = filter(d -> d[1] == kind, descs)
        idx = reduce(hcat, [d[2] for d in mine])
        par = reduce(hcat, [d[3] for d in mine])
        check(ccall((:mb_set_specific, LIB), Cint, (Ptr{Cvoid}, Cint, Int64, Ptr{Int32}, Ptr{Float64}),
                    ctx.handle, kind, size(idx, 2), idx, par))
    end
    return true
end

# ---- implicit solvent: ImplicitSolventOBC / ImplicitSolventGBN2 -> mb_set_implicit_solvent ----------------------------
# The engine adds the GB forces and energy in every integrator's step, the loggers' energies, the minimiser and MTS level 0.
# It takes what the structs hold (src/interactions/implicit_solvent.jl:337-583), with units stripped in the System's units.
# GBN2's n x n d0s / m0s tables become neck classes: atoms of equal radius (offset_radii .+ offset) share a class, and the
# class pair (c_i, c_j) reads d0s[i, j] of one representative pair (the tables are filled by radius, lookup_table :290-320).
is_gb(gi) = gi isa Molly.ImplicitSolventOBC || gi isa Molly.ImplicitSolventGBN2
# the general interactions a takeover accepts: LJDispersionCorrection (no force) and at most one GB term
general_ok(sys) = all(gi -> gi isa Molly.LJDispersionCorrection || is_gb(gi), sys.general_inters) &&
                  count(is_gb, sys.general_inters) <= 1
_f64(x) = Float64(ustrip(x))
_vec(a) = Float64.(ustrip.(Array(a)))

# (MBGbsa, per-atom arrays (offset radii, scaled offset radii, alpha, beta, gamma), neck (classes, d0, m0) or nothing),
# or nothing when the term has more neck classes than the engine takes
function gb_desc(inter)
    or_, sr = _vec(inter.offset_radii), _vec(inter.scaled_offset_radii)
    n = length(or_)
    p = (_f64(inter.dist_cutoff), _f64(inter.offset), _f64(inter.probe_radius), _f64(inter.sa_factor),
         _f64(inter.factor_solute), _f64(inter.factor_solvent), _f64(inter.kappa))
    if inter isa Molly.ImplicitSolventOBC
        abg = [fill(_f64(v), n) for v in (inter.α, inter.β, inter.γ)]
        return MBGbsa(p..., 0.0, 0.0, Int32(inter.use_ACE), Int32(0)), (or_, sr, abg...), nothing
    end
    radii = or_ .+ _f64(inter.offset)
    distinct = sort(unique(radii))
    nc = length(distinct)
    nc <= MB_GB_MAX_NECK_CLASSES || return nothing
    cls = Int32[searchsortedfirst(distinct, r) - 1 for r in radii]
    reps = [findfirst(==(c), cls) for c in Int32(0):Int32(nc - 1)]
    d0 = _vec(inter.d0s[reps, reps])                    # nc x nc gather on the device, then to the host
    m0 = _vec(inter.m0s[reps, reps])
    abg = (_vec(inter.αs), _vec(inter.βs), _vec(inter.γs))
    # row-major for C: entry [c_i * nc + c_j] = d0s[i, j]
    return MBGbsa(p..., Float64(inter.neck_scale), _f64(inter.neck_cut), Int32(inter.use_ACE), Int32(nc)),
           (or_, sr, abg...), (cls, vec(permutedims(d0)), vec(permutedims(m0)))
end
# a GB term the engine cannot take sends the run to the stock path
gb_ok(sys) = all(gi -> !is_gb(gi) || !isnothing(gb_desc(gi)), sys.general_inters)

# set the System's GB term on the context, or clear it when there is none (done on every taken-over call, like
# set_specific!); callers have checked gb_ok
function set_implicit_solvent!(ctx::Context, sys)
    i = findfirst(is_gb, sys.general_inters)
    if isnothing(i)
        check(ccall((:mb_set_implicit_solvent, LIB), Cint,
                    (Ptr{Cvoid}, Ptr{MBGbsa}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64},
                     Ptr{Int32}, Ptr{Float64}, Ptr{Float64}),
                    ctx.handle, C_NULL, C_NULL, C_NULL, C_NULL, C_NULL, C_NULL, C_NULL, C_NULL, C_NULL))
        return nothing
    end
    p, (or_, sr, a, b, g), neck = gb_desc(sys.general_inters[i])
    cls, d0, m0 = isnothing(neck) ? (Int32[0], Float64[0.0], Float64[0.0]) : neck   # (unread when n_neck_classes == 0)
    check(ccall((:mb_set_implicit_solvent, LIB), Cint,
                (Ptr{Cvoid}, Ref{MBGbsa}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64},
                 Ptr{Int32}, Ptr{Float64}, Ptr{Float64}),
                ctx.handle, Ref(p), or_, sr, a, b, g, cls, d0, m0))
    return nothing
end

# ---- multi-GPU: one Julia process per GPU (MPI.jl / Distributed); the reference has nothing here -----------
# rank 0: id = comm_unique_id(); broadcast the 128 bytes; every rank: comm_init!(sys, id, rank, nranks).
function comm_unique_id()
    id = Vector{UInt8}(undef, 128)
    check(ccall((:mb_comm_unique_id, LIB), Cint, (Ptr{UInt8},), id))
    return id
end
function comm_init!(sys::System{3, <:CuArray}, id::Vector{UInt8}, rank::Integer, nranks::Integer)
    descs = engine_eligible(sys, sys.pairwise_inters)
    isnothing(descs) && error("mollyb200: System is not engine-eligible")
    ctx = context_for(sys, descs)
    check(ccall((:mb_comm_init, LIB), Cint, (Ptr{Cvoid}, Ptr{UInt8}, Cint, Cint), ctx.handle, id, rank, nranks))
    return sys
end

# ---- simulate!(sys, ::VelocityVerlet, n) ----------------------------------------------------------------
# Taken over only when nothing but the pairwise path contributes forces and nothing has to run on the host
# every step. When every logger is one the engine records (device_log_kind), the whole run is one mb_simulate_vv_log call
# and the records are pushed into the loggers' histories afterwards; otherwise loggers fire between chunks of
# gcd(logger n_steps) steps (SURVEY.md Appendix A.11). Like the rest of this file, this has only been checked by reading.
function takeover_params(sys, sim::VelocityVerlet, n_steps, init_step, rng)
    # LJDispersionCorrection adds no force (lennard_jones.jl:252-275), implicit solvent runs in the engine
    # (set_implicit_solvent!); anything else (PME) -> stock path
    general_ok(sys) && gb_ok(sys) || return nothing
    all(!isnothing, map(specific_desc, sys.specific_inter_lists)) || return nothing
    kT, prob = 0.0, 0.0
    vc = nothing
    couplings = filter(c -> !(c isa Molly.NoCoupling), sim.coupling isa Tuple ? sim.coupling : (sim.coupling,))
    for c in couplings
        if length(couplings) == 1 && (c isa ImmediateThermostat || c isa BerendsenThermostat || c isa VelocityRescaleThermostat)
            vc = vcoupling_desc(sys, c)
            isnothing(vc) && return nothing
            continue
        end
        c isa AndersenThermostat || return nothing
        kT = Float64(ustrip(sys.k * c.temperature))
        prob = Float64(ustrip(sim.dt / c.coupling_const))
    end
    return MBVVParams(Float64(ustrip(sim.dt)), n_steps, init_step, Int32(sim.remove_CM_motion), kT, prob,
                      rand(rng, UInt64), rand(rng, UInt64)), vc
end

# the velocity-rescaling thermostats with their units stripped: k T0 in the System's energy units, tau in ps
_ps(x) = x isa Unitful.Quantity ? Float64(ustrip(u"ps", x)) : Float64(x)
function vcoupling_desc(sys, c)
    kT = Float64(ustrip(sys.k * c.temperature))
    c isa ImmediateThermostat && return MBVCoupling(Int32(1), Int32(0), kT, 0.0)
    c isa BerendsenThermostat && return MBVCoupling(Int32(2), Int32(0), kT, _ps(c.coupling_const))
    c.n_steps isa Integer && c.n_steps >= 1 || return nothing
    return MBVCoupling(Int32(3), Int32(c.n_steps), kT, _ps(c.coupling_const))
end

# set (or with `nothing`, clear) the context's velocity-rescaling thermostat; done on every taken-over call
function set_velocity_coupling!(ctx, vc)
    if isnothing(vc)
        check(ccall((:mb_set_velocity_coupling, LIB), Cint, (Ptr{Cvoid}, Ptr{MBVCoupling}), ctx.handle, C_NULL))
    else
        check(ccall((:mb_set_velocity_coupling, LIB), Cint, (Ptr{Cvoid}, Ref{MBVCoupling}), ctx.handle, Ref(vc)))
    end
end

function Molly.simulate!(sys::System{3, <:CuArray, T}, sim::VelocityVerlet, n_steps::Integer;
                         init_step=0, rng=Random.default_rng(), run_loggers=true, kwargs...) where T
    descs = engine_eligible(sys, sys.pairwise_inters)
    tp = isnothing(descs) ? nothing : takeover_params(sys, sim, n_steps, init_step, rng)
    if isnothing(tp)
        # stock: simulate!(sys, sim::VelocityVerlet, n_steps_or_time; ...) src/simulators.jl:547
        return invoke(Molly.simulate!, Tuple{Any, VelocityVerlet, Any}, sys, sim, n_steps;
                      init_step=init_step, rng=rng, run_loggers=run_loggers, kwargs...)
    end
    p, vc = tp
    ctx = context_for(sys, descs)
    set_specific!(ctx, sys)
    set_implicit_solvent!(ctx, sys)
    set_velocity_coupling!(ctx, vc)
    if run_loggers != false && !isempty(sys.loggers) && all(l -> !isnothing(device_log_kind(l)), values(sys.loggers))
        return simulate_logged!(sys, ctx, p, n_steps, init_step, run_loggers)
    end
    chunk = run_loggers == false || isempty(sys.loggers) ? n_steps :
            max(1, reduce(gcd, (l.n_steps for l in values(sys.loggers))))
    done = 0
    Molly.apply_loggers!(sys, nothing, nothing, init_step, run_loggers)
    while done < n_steps
        m = min(chunk, n_steps - done)
        pp = MBVVParams(p.dt, m, init_step + done, p.remove_cm_every, p.andersen_kT, p.andersen_prob,
                        rand(rng, UInt64), rand(rng, UInt64))
        check(ccall((:mb_simulate_vv, LIB), Cint, (Ptr{Cvoid}, CuPtr{Cvoid}, CuPtr{Cvoid}, Ref{MBVVParams}),
                    ctx.handle, pointer(sys.coords), pointer(sys.velocities), Ref(pp)))
        done += m
        Molly.apply_loggers!(sys, nothing, nothing, init_step + done, run_loggers)
    end
    return sys
end

# ---- simulate!(sys, ::Langevin, n) (src/simulators.jl:1101-1210) ------------------------------------------------------------
# Taken over when the coupling is nothing, the System is eligible as for VelocityVerlet, and the loggers are none, not run,
# or all ones the engine records; the whole run is then one mb_simulate_langevin call. The velocity coupling of the context
# is cleared first. Anything else (barostats, constraints, virtual sites, host-side loggers) runs the stock method.
function Molly.simulate!(sys::System{3, <:CuArray, T}, sim::Langevin, n_steps::Integer;
                         init_step=0, rng=Random.default_rng(), run_loggers=true, kwargs...) where T
    descs = engine_eligible(sys, sys.pairwise_inters)
    device_logs = run_loggers == false || isempty(sys.loggers) ||
                  all(l -> !isnothing(device_log_kind(l)), values(sys.loggers))
    if isnothing(descs) || !isnothing(sim.coupling) || !device_logs ||
            !general_ok(sys) || !gb_ok(sys) ||
            !all(!isnothing, map(specific_desc, sys.specific_inter_lists))
        # stock: simulate!(sys, sim::Langevin, n_steps_or_time; ...) src/simulators.jl:1101
        return invoke(Molly.simulate!, Tuple{Any, Langevin, Any}, sys, sim, n_steps;
                      init_step=init_step, rng=rng, run_loggers=run_loggers, kwargs...)
    end
    ctx = context_for(sys, descs)
    set_specific!(ctx, sys)
    set_implicit_solvent!(ctx, sys)
    set_velocity_coupling!(ctx, nothing)
    friction = sim.friction isa Unitful.Quantity ? Float64(ustrip(u"ps^-1", sim.friction)) : Float64(sim.friction)
    p = MBLangevinParams(_ps(sim.dt), n_steps, init_step, Int32(sim.remove_CM_motion),
                         Float64(ustrip(sys.k * sim.temperature)), friction,
                         rand(rng, UInt64), rand(rng, UInt64))
    if run_loggers != false && !isempty(sys.loggers)
        return simulate_logged!(sys, ctx, n_steps, init_step, run_loggers) do lg
            ccall((:mb_simulate_langevin, LIB), Cint, (Ptr{Cvoid}, CuPtr{Cvoid}, CuPtr{Cvoid}, Ref{MBLangevinParams}, Ref{MBLog}),
                  ctx.handle, pointer(sys.coords), pointer(sys.velocities), Ref(p), lg)
        end
    end
    check(ccall((:mb_simulate_langevin, LIB), Cint, (Ptr{Cvoid}, CuPtr{Cvoid}, CuPtr{Cvoid}, Ref{MBLangevinParams}, Ptr{MBLog}),
                ctx.handle, pointer(sys.coords), pointer(sys.velocities), Ref(p), C_NULL))
    return sys
end

# ---- simulate!(sys, ::LangevinSplitting, n) (src/simulators.jl:1252-1398) --------------------------------------------------
# Taken over under the conditions of the Langevin method above (LangevinSplitting has no coupling) when the splitting has 1 to
# 32 letters, all of them A, B or O: one mb_simulate_langevin_splitting call. The friction is a mass per time, converted to
# g mol^-1 ps^-1 (a plain number is taken as that). An invalid letter runs the stock method, which raises its ArgumentError.
function Molly.simulate!(sys::System{3, <:CuArray, T}, sim::LangevinSplitting, n_steps::Integer;
                         init_step=0, rng=Random.default_rng(), run_loggers=true, kwargs...) where T
    descs = engine_eligible(sys, sys.pairwise_inters)
    device_logs = run_loggers == false || isempty(sys.loggers) ||
                  all(l -> !isnothing(device_log_kind(l)), values(sys.loggers))
    ops = collect(String(sim.splitting))
    if isnothing(descs) || !device_logs || !general_ok(sys) || !gb_ok(sys) ||
            !all(!isnothing, map(specific_desc, sys.specific_inter_lists)) ||
            !(1 <= length(ops) <= 32) || !all(op -> op in ('A', 'B', 'O'), ops)
        # stock: simulate!(sys, sim::LangevinSplitting, n_steps_or_time; ...) src/simulators.jl:1252
        return invoke(Molly.simulate!, Tuple{Any, LangevinSplitting, Any}, sys, sim, n_steps;
                      init_step=init_step, rng=rng, run_loggers=run_loggers, kwargs...)
    end
    ctx = context_for(sys, descs)
    set_specific!(ctx, sys)
    set_implicit_solvent!(ctx, sys)
    set_velocity_coupling!(ctx, nothing)
    friction = sim.friction isa Unitful.Quantity ? Float64(ustrip(u"g * mol^-1 * ps^-1", sim.friction)) : Float64(sim.friction)
    letters = ntuple(i -> i <= length(ops) ? UInt8(ops[i]) : 0x00, 32)
    p = MBSplittingParams(_ps(sim.dt), n_steps, init_step, Int32(sim.remove_CM_motion),
                          Float64(ustrip(sys.k * sim.temperature)), friction, rand(rng, UInt64), rand(rng, UInt64),
                          Int32(length(ops)), letters)
    if run_loggers != false && !isempty(sys.loggers)
        return simulate_logged!(sys, ctx, n_steps, init_step, run_loggers) do lg
            ccall((:mb_simulate_langevin_splitting, LIB), Cint,
                  (Ptr{Cvoid}, CuPtr{Cvoid}, CuPtr{Cvoid}, Ref{MBSplittingParams}, Ref{MBLog}),
                  ctx.handle, pointer(sys.coords), pointer(sys.velocities), Ref(p), lg)
        end
    end
    check(ccall((:mb_simulate_langevin_splitting, LIB), Cint,
                (Ptr{Cvoid}, CuPtr{Cvoid}, CuPtr{Cvoid}, Ref{MBSplittingParams}, Ptr{MBLog}),
                ctx.handle, pointer(sys.coords), pointer(sys.velocities), Ref(p), C_NULL))
    return sys
end

# ---- simulate!(sys, ::NoseHoover, n) (src/simulators.jl:1534-1614) ---------------------------------------------------------
# Taken over under the conditions of the Langevin method above: one mb_simulate_nose_hoover call, which starts zeta at 0 as
# the stock method does on every call. Units are stripped (dt and damping in ps, k T in kJ/mol). Anything else runs the stock
# method.
function Molly.simulate!(sys::System{3, <:CuArray, T}, sim::NoseHoover, n_steps::Integer;
                         init_step=0, rng=Random.default_rng(), run_loggers=true, kwargs...) where T
    descs = engine_eligible(sys, sys.pairwise_inters)
    device_logs = run_loggers == false || isempty(sys.loggers) ||
                  all(l -> !isnothing(device_log_kind(l)), values(sys.loggers))
    if isnothing(descs) || !isnothing(sim.coupling) || !device_logs ||
            !general_ok(sys) || !gb_ok(sys) ||
            !all(!isnothing, map(specific_desc, sys.specific_inter_lists))
        # stock: simulate!(sys, sim::NoseHoover, n_steps_or_time; ...) src/simulators.jl:1534
        return invoke(Molly.simulate!, Tuple{Any, NoseHoover, Any}, sys, sim, n_steps;
                      init_step=init_step, rng=rng, run_loggers=run_loggers, kwargs...)
    end
    ctx = context_for(sys, descs)
    set_specific!(ctx, sys)
    set_implicit_solvent!(ctx, sys)
    set_velocity_coupling!(ctx, nothing)
    p = MBNoseHooverParams(_ps(sim.dt), n_steps, init_step, Int32(sim.remove_CM_motion),
                           Float64(ustrip(sys.k * sim.temperature)), _ps(sim.damping))
    if run_loggers != false && !isempty(sys.loggers)
        return simulate_logged!(sys, ctx, n_steps, init_step, run_loggers) do lg
            ccall((:mb_simulate_nose_hoover, LIB), Cint, (Ptr{Cvoid}, CuPtr{Cvoid}, CuPtr{Cvoid}, Ref{MBNoseHooverParams}, Ref{MBLog}),
                  ctx.handle, pointer(sys.coords), pointer(sys.velocities), Ref(p), lg)
        end
    end
    check(ccall((:mb_simulate_nose_hoover, LIB), Cint, (Ptr{Cvoid}, CuPtr{Cvoid}, CuPtr{Cvoid}, Ref{MBNoseHooverParams}, Ptr{MBLog}),
                ctx.handle, pointer(sys.coords), pointer(sys.velocities), Ref(p), C_NULL))
    return sys
end

# ---- simulate!(sys, ::Verlet / ::StormerVerlet / ::OverdampedLangevin, n) (src/simulators.jl:858-1063, :1400-1490) -------
# Taken over under the conditions of the Langevin method above; Verlet only with coupling nothing or one AndersenThermostat
# (velocity-rescaling couplings with Verlet run the stock method). One mb_simulate_verlet, mb_simulate_stormer_verlet or
# mb_simulate_overdamped_langevin call; OverdampedLangevin's friction is in ps^-1. Anything else runs the stock method.
function plain_takeover_ok(sys, descs, run_loggers)
    device_logs = run_loggers == false || isempty(sys.loggers) ||
                  all(l -> !isnothing(device_log_kind(l)), values(sys.loggers))
    return !isnothing(descs) && device_logs && general_ok(sys) && gb_ok(sys) &&
           all(!isnothing, map(specific_desc, sys.specific_inter_lists))
end

function Molly.simulate!(sys::System{3, <:CuArray, T}, sim::Verlet, n_steps::Integer;
                         init_step=0, rng=Random.default_rng(), run_loggers=true, kwargs...) where T
    descs = engine_eligible(sys, sys.pairwise_inters)
    couplings = filter(c -> !(c isa Molly.NoCoupling), sim.coupling isa Tuple ? sim.coupling : (sim.coupling,))
    couplings = filter(!isnothing, collect(couplings))
    if !plain_takeover_ok(sys, descs, run_loggers) || length(couplings) > 1 ||
            !all(c -> c isa AndersenThermostat, couplings)
        # stock: simulate!(sys, sim::Verlet, n_steps_or_time; ...) src/simulators.jl:868
        return invoke(Molly.simulate!, Tuple{Any, Verlet, Any}, sys, sim, n_steps;
                      init_step=init_step, rng=rng, run_loggers=run_loggers, kwargs...)
    end
    ctx = context_for(sys, descs)
    set_specific!(ctx, sys)
    set_implicit_solvent!(ctx, sys)
    set_velocity_coupling!(ctx, nothing)
    kT, prob = 0.0, 0.0
    for c in couplings
        kT = Float64(ustrip(sys.k * c.temperature))
        prob = Float64(ustrip(sim.dt / c.coupling_const))
    end
    p = MBVVParams(_ps(sim.dt), n_steps, init_step, Int32(sim.remove_CM_motion), kT, prob, rand(rng, UInt64), rand(rng, UInt64))
    if run_loggers != false && !isempty(sys.loggers)
        return simulate_logged!(sys, ctx, n_steps, init_step, run_loggers) do lg
            ccall((:mb_simulate_verlet, LIB), Cint, (Ptr{Cvoid}, CuPtr{Cvoid}, CuPtr{Cvoid}, Ref{MBVVParams}, Ref{MBLog}),
                  ctx.handle, pointer(sys.coords), pointer(sys.velocities), Ref(p), lg)
        end
    end
    check(ccall((:mb_simulate_verlet, LIB), Cint, (Ptr{Cvoid}, CuPtr{Cvoid}, CuPtr{Cvoid}, Ref{MBVVParams}, Ptr{MBLog}),
                ctx.handle, pointer(sys.coords), pointer(sys.velocities), Ref(p), C_NULL))
    return sys
end

# ---- simulate!(sys, ::DPDVelocityVerlet, n) (src/simulators.jl:711-842) ---------------------------------------------------
# Taken over when the coupling is nothing and the System is eligible as for Verlet with a pairwise tuple of exactly one
# unitless DPDInteraction (dpd_eligible): one mb_simulate_dpd_vv call. Every other integrator leaves a DPD System to its
# stock method (engine_eligible has no DPD descriptor), whose force loop still goes through the DPD seam above. Anything
# else runs the stock method.
function Molly.simulate!(sys::System{3, <:CuArray, T}, sim::DPDVelocityVerlet, n_steps::Integer;
                         init_step=0, rng=Random.default_rng(), run_loggers=true, kwargs...) where T
    descs = dpd_eligible(sys, sys.pairwise_inters)
    if isnothing(descs) || !isnothing(sim.coupling) || !plain_takeover_ok(sys, descs, run_loggers) ||
            !isempty(sys.general_inters)
        # stock: simulate!(sys, sim::DPDVelocityVerlet, n_steps_or_time; ...) src/simulators.jl:711
        return invoke(Molly.simulate!, Tuple{Any, DPDVelocityVerlet, Any}, sys, sim, n_steps;
                      init_step=init_step, rng=rng, run_loggers=run_loggers, kwargs...)
    end
    ctx = context_for(sys, descs)
    set_specific!(ctx, sys)
    set_implicit_solvent!(ctx, sys)
    set_velocity_coupling!(ctx, nothing)
    p = MBDpdVVParams(_ps(sim.dt), n_steps, init_step, Int32(sim.remove_CM_motion), Float64(sim.λ))
    if run_loggers != false && !isempty(sys.loggers)
        return simulate_logged!(sys, ctx, n_steps, init_step, run_loggers) do lg
            ccall((:mb_simulate_dpd_vv, LIB), Cint, (Ptr{Cvoid}, CuPtr{Cvoid}, CuPtr{Cvoid}, Ref{MBDpdVVParams}, Ref{MBLog}),
                  ctx.handle, pointer(sys.coords), pointer(sys.velocities), Ref(p), lg)
        end
    end
    check(ccall((:mb_simulate_dpd_vv, LIB), Cint, (Ptr{Cvoid}, CuPtr{Cvoid}, CuPtr{Cvoid}, Ref{MBDpdVVParams}, Ptr{MBLog}),
                ctx.handle, pointer(sys.coords), pointer(sys.velocities), Ref(p), C_NULL))
    return sys
end

function Molly.simulate!(sys::System{3, <:CuArray, T}, sim::StormerVerlet, n_steps::Integer;
                         init_step=0, rng=Random.default_rng(), run_loggers=true, kwargs...) where T
    descs = engine_eligible(sys, sys.pairwise_inters)
    if !plain_takeover_ok(sys, descs, run_loggers)
        # stock: simulate!(sys, sim::StormerVerlet, n_steps_or_time; ...) src/simulators.jl:970
        return invoke(Molly.simulate!, Tuple{Any, StormerVerlet, Any}, sys, sim, n_steps;
                      init_step=init_step, rng=rng, run_loggers=run_loggers, kwargs...)
    end
    ctx = context_for(sys, descs)
    set_specific!(ctx, sys)
    set_implicit_solvent!(ctx, sys)
    set_velocity_coupling!(ctx, nothing)
    p = MBStormerParams(_ps(sim.dt), n_steps, init_step)
    if run_loggers != false && !isempty(sys.loggers)
        return simulate_logged!(sys, ctx, n_steps, init_step, run_loggers) do lg
            ccall((:mb_simulate_stormer_verlet, LIB), Cint,
                  (Ptr{Cvoid}, CuPtr{Cvoid}, CuPtr{Cvoid}, Ref{MBStormerParams}, Ref{MBLog}),
                  ctx.handle, pointer(sys.coords), pointer(sys.velocities), Ref(p), lg)
        end
    end
    check(ccall((:mb_simulate_stormer_verlet, LIB), Cint,
                (Ptr{Cvoid}, CuPtr{Cvoid}, CuPtr{Cvoid}, Ref{MBStormerParams}, Ptr{MBLog}),
                ctx.handle, pointer(sys.coords), pointer(sys.velocities), Ref(p), C_NULL))
    return sys
end

function Molly.simulate!(sys::System{3, <:CuArray, T}, sim::OverdampedLangevin, n_steps::Integer;
                         init_step=0, rng=Random.default_rng(), run_loggers=true, kwargs...) where T
    descs = engine_eligible(sys, sys.pairwise_inters)
    friction = sim.friction isa Unitful.Quantity ? Float64(ustrip(u"ps^-1", sim.friction)) : Float64(sim.friction)
    if !plain_takeover_ok(sys, descs, run_loggers) || !(isfinite(friction) && friction > 0)
        # stock: simulate!(sys, sim::OverdampedLangevin, n_steps_or_time; ...) src/simulators.jl:1427
        return invoke(Molly.simulate!, Tuple{Any, OverdampedLangevin, Any}, sys, sim, n_steps;
                      init_step=init_step, rng=rng, run_loggers=run_loggers, kwargs...)
    end
    ctx = context_for(sys, descs)
    set_specific!(ctx, sys)
    set_implicit_solvent!(ctx, sys)
    set_velocity_coupling!(ctx, nothing)
    p = MBLangevinParams(_ps(sim.dt), n_steps, init_step, Int32(sim.remove_CM_motion),
                         Float64(ustrip(sys.k * sim.temperature)), friction, rand(rng, UInt64), rand(rng, UInt64))
    if run_loggers != false && !isempty(sys.loggers)
        return simulate_logged!(sys, ctx, n_steps, init_step, run_loggers) do lg
            ccall((:mb_simulate_overdamped_langevin, LIB), Cint,
                  (Ptr{Cvoid}, CuPtr{Cvoid}, CuPtr{Cvoid}, Ref{MBLangevinParams}, Ref{MBLog}),
                  ctx.handle, pointer(sys.coords), pointer(sys.velocities), Ref(p), lg)
        end
    end
    check(ccall((:mb_simulate_overdamped_langevin, LIB), Cint,
                (Ptr{Cvoid}, CuPtr{Cvoid}, CuPtr{Cvoid}, Ref{MBLangevinParams}, Ptr{MBLog}),
                ctx.handle, pointer(sys.coords), pointer(sys.velocities), Ref(p), C_NULL))
    return sys
end

# ---- simulate!(sys, ::MTSIntegrator / ::MTSLangevinIntegrator, n) (src/simulators.jl:1616-1940) ------------------------------
# Taken over under the conditions of the Langevin method above, when every pairwise fraction is 1 (the engine evaluates all
# pairwise interactions in one kernel, once per outer step): one mb_simulate_mts call. The level of every specific term is
# the index of its list's fraction in ordered_fractions; the levels of one kind are concatenated in list order, the order in
# which set_specific! concatenated the terms. Anything else runs the stock method.
function set_specific_levels!(ctx::Context, sys, sim)
    levels = Dict{Int, Vector{Int32}}()
    for (sil, f) in zip(sys.specific_inter_lists, sim.si_fractions)
        kind, idx, _ = specific_desc(sil)
        append!(get!(levels, kind, Int32[]), fill(Int32(findfirst(==(f), sim.ordered_fractions) - 1), size(idx, 2)))
    end
    for (kind, level) in levels
        check(ccall((:mb_set_specific_levels, LIB), Cint, (Ptr{Cvoid}, Cint, Int64, Ptr{Int32}),
                    ctx.handle, kind, length(level), level))
    end
end

function Molly.simulate!(sys::System{3, <:CuArray, T}, sim::Molly.AbstractMTSIntegrator, n_steps::Integer;
                         init_step=0, rng=Random.default_rng(), run_loggers=true, kwargs...) where T
    descs = engine_eligible(sys, sys.pairwise_inters)
    device_logs = run_loggers == false || isempty(sys.loggers) ||
                  all(l -> !isnothing(device_log_kind(l)), values(sys.loggers))
    if isnothing(descs) || !isnothing(sim.coupling) || !device_logs || !all(==(1), sim.pi_fractions) ||
            length(sim.pi_fractions) != length(sys.pairwise_inters) ||
            length(sim.si_fractions) != length(sys.specific_inter_lists) ||
            length(sim.gi_fractions) != length(sys.general_inters) ||
            length(sim.ordered_fractions) > 8 || last(sim.ordered_fractions) > 1024 ||
            !general_ok(sys) || !gb_ok(sys) ||
            any(((gi, f),) -> is_gb(gi) && f != 1, zip(sys.general_inters, sim.gi_fractions)) ||   # GB at level 0 only
            !all(!isnothing, map(specific_desc, sys.specific_inter_lists))
        # stock: simulate!(sys, sim::AbstractMTSIntegrator, n_steps_or_time; ...) src/simulators.jl:1850
        return invoke(Molly.simulate!, Tuple{Any, Molly.AbstractMTSIntegrator, Any}, sys, sim, n_steps;
                      init_step=init_step, rng=rng, run_loggers=run_loggers, kwargs...)
    end
    ctx = context_for(sys, descs)
    set_specific!(ctx, sys)
    set_specific_levels!(ctx, sys, sim)
    set_implicit_solvent!(ctx, sys)
    set_velocity_coupling!(ctx, nothing)
    fr = zeros(Int32, 8)
    fr[1:length(sim.ordered_fractions)] .= sim.ordered_fractions
    lang = sim isa MTSLangevinIntegrator
    kT = lang ? Float64(ustrip(sys.k * sim.temperature)) : 0.0
    friction = !lang ? 0.0 : sim.friction isa Unitful.Quantity ? Float64(ustrip(u"ps^-1", sim.friction)) : Float64(sim.friction)
    p = MBMTSParams(_ps(sim.dt), n_steps, init_step, Int32(sim.remove_CM_motion), Int32(length(sim.ordered_fractions)),
                    NTuple{8, Int32}(fr), Int32(lang), Int32(0), kT, friction, rand(rng, UInt64), rand(rng, UInt64))
    if run_loggers != false && !isempty(sys.loggers)
        return simulate_logged!(sys, ctx, n_steps, init_step, run_loggers) do lg
            ccall((:mb_simulate_mts, LIB), Cint, (Ptr{Cvoid}, CuPtr{Cvoid}, CuPtr{Cvoid}, Ref{MBMTSParams}, Ref{MBLog}),
                  ctx.handle, pointer(sys.coords), pointer(sys.velocities), Ref(p), lg)
        end
    end
    check(ccall((:mb_simulate_mts, LIB), Cint, (Ptr{Cvoid}, CuPtr{Cvoid}, CuPtr{Cvoid}, Ref{MBMTSParams}, Ptr{MBLog}),
                ctx.handle, pointer(sys.coords), pointer(sys.velocities), Ref(p), C_NULL))
    return sys
end

# ---- simulate!(sys, ::SteepestDescentMinimizer) (src/simulators.jl:183-274) ------------------------------------------------
# Taken over when the System is engine-eligible, has no constraints, no general interactions other than one implicit
# solvent term (the engine computes its energy; any other it would need for the log lines) and run_loggers is false: the whole minimisation is one mb_minimize_sd call, and the
# reference's log lines are printed from the trace afterwards. Anything else runs the stock method.
struct MBSDParams
    step_size::Float64
    max_steps::Int64
    tol::Float64
    init_step::Int64
    trace::Ptr{Float64}
    trace_capacity::Int64
    n_iterations::Int64
    energy::Float64
    max_force::Float64
    final_step_size::Float64
    converged::Int32
    reserved_::Int32
end

function Molly.simulate!(sys::System{3, <:CuArray, T}, sim::SteepestDescentMinimizer; init_step=0, run_loggers=false,
                         kwargs...) where T
    descs = engine_eligible(sys, sys.pairwise_inters)
    if isnothing(descs) || run_loggers != false || !all(is_gb, sys.general_inters) || length(sys.general_inters) > 1 ||
            !gb_ok(sys) || !all(!isnothing, map(specific_desc, sys.specific_inter_lists))
        return invoke(Molly.simulate!, Tuple{Any, SteepestDescentMinimizer}, sys, sim;
                      init_step=init_step, run_loggers=run_loggers, kwargs...)
    end
    ctx = context_for(sys, descs)
    set_specific!(ctx, sys)
    set_implicit_solvent!(ctx, sys)
    trace = zeros(Float64, 4, sim.max_steps + 1)   # (step, E or E_trial, max force, accepted) per column
    p = Ref(MBSDParams(Float64(ustrip(sim.step_size)), sim.max_steps, Float64(ustrip(sim.tol)), init_step,
                       pointer(trace), sim.max_steps + 1, 0, 0.0, 0.0, 0.0, Int32(0), Int32(0)))
    GC.@preserve trace begin
        check(ccall((:mb_minimize_sd, LIB), Cint, (Ptr{Cvoid}, CuPtr{Cvoid}, Ref{MBSDParams}),
                    ctx.handle, pointer(sys.coords), p))
    end
    eu, fu = sys.energy_units, sys.force_units
    println(sim.log_stream, "Step ", init_step, " - potential energy ", trace[2, 1] * eu, " - max force N/A - N/A")
    for k in 2:(p[].n_iterations + 1)
        println(sim.log_stream, "Step ", Int(trace[1, k]), " - potential energy ", trace[2, k] * eu, " - max force ",
                trace[3, k] * fu, " - ", trace[4, k] != 0 ? "accepted" : "rejected")
    end
    return sys
end

# The loggers the engine records on the device (src/loggers.jl:134-278): GeneralObservableLoggers whose observable is one
# of these functions. Others return nothing (chunked path).
function device_log_kind(l)
    l isa Molly.GeneralObservableLogger || return nothing
    f = l.observable
    f === Molly.potential_energy_wrapper && return :pe
    f === Molly.kinetic_energy_wrapper && return :ke
    f === Molly.total_energy_wrapper && return :total
    f === Molly.temperature_wrapper && return :temp
    f === Molly.coordinates_wrapper && return :coords
    f === Molly.velocities_wrapper && return :vels
    return nothing
end

# steps a logger of interval `every` is recorded at (simulators.jl:575, :657; loggers.jl:44-56, :96-102)
function record_steps(every, n_steps, init_step, run_loggers)
    every <= 0 && return Int[]
    steps = collect(((init_step ÷ every) + 1) * every:every:(init_step + n_steps))
    run_loggers == true && init_step % every == 0 && pushfirst!(steps, init_step)
    return steps
end

function simulate_logged!(sys::System{3, <:CuArray, T}, ctx, p, n_steps, init_step, run_loggers) where T
    return simulate_logged!(sys, ctx, n_steps, init_step, run_loggers) do lg
        ccall((:mb_simulate_vv_log, LIB), Cint, (Ptr{Cvoid}, CuPtr{Cvoid}, CuPtr{Cvoid}, Ref{MBVVParams}, Ref{MBLog}),
              ctx.handle, pointer(sys.coords), pointer(sys.velocities), Ref(p), lg)
    end
end
function simulate_logged!(run, sys::System{3, <:CuArray, T}, ctx, n_steps, init_step, run_loggers) where T
    kinds = Dict(name => device_log_kind(l) for (name, l) in pairs(sys.loggers))
    gcd_of(sel) = reduce(gcd, (l.n_steps for (name, l) in pairs(sys.loggers) if kinds[name] in sel); init=0)
    e_every, x_every, v_every = gcd_of((:pe, :ke, :total, :temp)), gcd_of((:coords,)), gcd_of((:vels,))
    e_steps = record_steps(e_every, n_steps, init_step, run_loggers)
    x_steps = record_steps(x_every, n_steps, init_step, run_loggers)
    v_steps = record_steps(v_every, n_steps, init_step, run_loggers)
    n = length(sys)
    erec = CUDA.zeros(Float64, 3, max(1, length(e_steps)))   # (step, pe, ke) per column
    xrec = CUDA.zeros(T, 3, n, max(1, length(x_steps)))
    vrec = CUDA.zeros(T, 3, n, max(1, length(v_steps)))
    lg = MBLog(isempty(e_steps) ? 0 : e_every, isempty(x_steps) ? 0 : x_every, isempty(v_steps) ? 0 : v_every,
               Int32(run_loggers == true), Int32(0),
               reinterpret(Ptr{Float64}, pointer(erec)), reinterpret(Ptr{Cvoid}, pointer(xrec)),
               reinterpret(Ptr{Cvoid}, pointer(vrec)), length(e_steps), length(x_steps), length(v_steps), 0, 0, 0)
    GC.@preserve erec xrec vrec begin
        check(run(lg))
    end
    e = Array(erec)
    eu, du, vu = sys.energy_units, unit(eltype(eltype(sys.coords))), unit(eltype(eltype(sys.velocities)))
    for (name, l) in pairs(sys.loggers)
        k = kinds[name]
        if k in (:coords, :vels)
            steps, rec = k == :coords ? (x_steps, xrec) : (v_steps, vrec)
            for (j, s) in enumerate(steps)
                s % l.n_steps == 0 || continue
                frame = reinterpret(SVector{3, T}, vec(rec[:, :, j]))
                push!(l.history, Array(frame) .* (k == :coords ? du : vu))
            end
        else
            for (j, s) in enumerate(e_steps)
                s % l.n_steps == 0 || continue
                pe, ke = e[2, j], e[3, j]
                v = k == :pe ? pe * eu : k == :ke ? ke * eu : k == :total ? (pe + ke) * eu : 2 * ke * eu / (sys.df * sys.k)
                if k == :temp && eu != Unitful.NoUnits
                    v = uconvert(u"K", v)   # temperature(sys), src/energy.jl:158-176
                end
                push!(l.history, v)
            end
        end
    end
    return sys
end

# ---- remove_CM_motion! (ext/MollyCUDAExt.jl:2373) ---------------------------------------------------------
# The stock extension's method has exactly the signature System{3, <:CuArray, T}; defining it again would be a method
# overwrite (an error under precompilation). Inside the taken-over simulate! the engine removes the CM motion itself;
# for stand-alone use this module offers its own function instead of replacing Molly's.
function remove_cm_motion!(sys::System{3, <:CuArray, T}) where T
    descs = engine_eligible(sys, sys.pairwise_inters)
    isnothing(descs) && return Molly.remove_CM_motion!(sys)
    ctx = context_for(sys, descs)
    check(ccall((:mb_remove_cm_motion, LIB), Cint, (Ptr{Cvoid}, CuPtr{Cvoid}), ctx.handle, pointer(sys.velocities)))
    return sys
end

# The launch-config API of the stock extension (optimize_cuda_launch_config!, src/cuda_config.jl:53, ext:594) is left
# alone: it tunes the stock kernels, which stay the fall-through path; the brick shape of this engine is chosen by the
# library (mb_set_launch_config).

end # module
