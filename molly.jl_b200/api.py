"""Host-side mirror of Molly.jl's API for the non-bonded + VelocityVerlet hot path.

Same names and argument meaning as the reference so the parity tests read like the reference's
own tests (Julia is not available in the build image; the Julia shim that binds the same C ABI is
julia/MollyB200Ext.jl, see INTEGRATION.md):

    Atom, CubicBoundary, System                     src/types.jl:466-475, src/spatial.jl:40, src/types.jl:795-979
    NoCutoff, DistanceCutoff, Shifted*Cutoff        src/cutoffs.jl:47-190
    LennardJones, Coulomb, CoulombReactionField     src/interactions/lennard_jones.jl:28-35, coulomb.jl:32-70, :698-747
    GPUNeighborFinder (+ aliases)                   src/neighbors.jl:104-115
    VelocityVerlet, AndersenThermostat, simulate    src/simulators.jl:287-295, :547-668; src/coupling.jl:184-212
    ImmediateThermostat, BerendsenThermostat,       src/coupling.jl:82-168, :227-238 (applied on the device inside
    VelocityRescaleThermostat                       simulate, see mb_set_velocity_coupling)
    SteepestDescentMinimizer                        src/simulators.jl:183-274 (simulate dispatches on the simulator)
    Langevin                                        src/simulators.jl:1065-1210 (mb_simulate_langevin)
    LangevinSplitting                               src/simulators.jl:1212-1398 (mb_simulate_langevin_splitting)
    NoseHoover                                      src/simulators.jl:1491-1614 (mb_simulate_nose_hoover)
    Verlet, StormerVerlet                           src/simulators.jl:858-1063 (mb_simulate_verlet, mb_simulate_stormer_verlet)
    OverdampedLangevin                              src/simulators.jl:1400-1490 (mb_simulate_overdamped_langevin)
    DPDInteraction, DPDVelocityVerlet               src/interactions/dpd.jl:57-142, src/simulators.jl:670-842 (mb_set_dpd,
                                                    mb_simulate_dpd_vv, mb_forces_energy_vel)
    MTSIntegrator, MTSLangevinIntegrator            src/simulators.jl:1616-1940 (mb_simulate_mts)
    forces, forces_virial, potential_energy         src/force.jl:678-720, src/energy.jl:202-248
    kinetic_energy, temperature, remove_CM_motion   src/energy.jl:44-175, src/spatial.jl:901-929
    *EnergyLogger, TemperatureLogger, Coordinates-  src/loggers.jl:44-102, :134-278 (recorded on the device inside
    Logger, VelocitiesLogger, values                simulate)

Everything numerical happens in libmollyb200.so on the GPU; this module only marshals arrays.
Units are Molly's (nm, ps, g/mol, kJ/mol) with the Unitful wrappers stripped.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass, field
from typing import Optional, Sequence

import numpy as np

from . import _capi as capi
from ._capi import MollyB200Error  # noqa: F401

COULOMB_CONST = 138.93545764  # src/interactions/coulomb.jl:16
BOLTZMANN_K = 8.31446261815324e-3  # src/units.jl:186-198


# ------------------------------------------------------------------------------------------------
# types
# ------------------------------------------------------------------------------------------------
@dataclass
class Atom:
    index: int = 1
    atom_type: int = 1
    mass: float = 1.0
    charge: float = 0.0
    sigma: float = 0.0
    eps: float = 0.0
    lam: float = 1.0
    alch_role: int = 0


def atom_dtype(dtype) -> np.dtype:
    """numpy struct dtype with Molly's bits layout Atom{Int32,T,T,T,T,T} (32 B f32 / 56 B f64)."""
    f = np.dtype(dtype)
    return np.dtype([("index", np.int32), ("atom_type", np.int32), ("mass", f), ("charge", f), ("sigma", f),
                     ("eps", f), ("lam", f), ("alch_role", np.int32)], align=True)


def atoms_to_array(atoms: Sequence[Atom], dtype) -> np.ndarray:
    arr = np.zeros(len(atoms), atom_dtype(dtype))
    for k, a in enumerate(atoms):
        arr[k] = (a.index, a.atom_type, a.mass, a.charge, a.sigma, a.eps, a.lam, a.alch_role)
    return arr


def atoms_from_arrays(mass, charge, sigma, eps, dtype) -> np.ndarray:
    n = len(mass)
    arr = np.zeros(n, atom_dtype(dtype))
    arr["index"] = np.arange(1, n + 1)
    arr["atom_type"] = 1
    arr["mass"], arr["charge"], arr["sigma"], arr["eps"], arr["lam"] = mass, charge, sigma, eps, 1.0
    return arr


@dataclass
class CubicBoundary:
    x: float
    y: Optional[float] = None
    z: Optional[float] = None

    def __post_init__(self):
        if self.y is None:
            self.y = self.x
        if self.z is None:
            self.z = self.x

    @property
    def side_lengths(self):
        return np.array([self.x, self.y, self.z], np.float64)


class TriclinicBoundary:
    """TriclinicBoundary(bv1, bv2, bv3) — src/spatial.jl:151-215 (approx_images = true): lower-triangular basis vectors.
    Systems in such a box run on the no-list kernel."""

    def __init__(self, bv1, bv2, bv3):
        self.basis_vectors = np.array([bv1, bv2, bv3], np.float64).reshape(3, 3)
        bv = self.basis_vectors
        if not (bv[0, 0] > 0 and bv[0, 1] == 0 and bv[0, 2] == 0):
            raise ValueError("first basis vector must be along the x-axis with a positive x component")
        if not (bv[1, 1] > 0 and bv[1, 2] == 0):
            raise ValueError("second basis vector must be in the xy plane with a positive y component")
        if not bv[2, 2] > 0:
            raise ValueError("third basis vector must have a positive z component")

    @property
    def side_lengths(self):  # heights (what the engine's geometry code sees)
        return np.array([self.basis_vectors[0, 0], self.basis_vectors[1, 1], self.basis_vectors[2, 2]], np.float64)


@dataclass
class NoCutoff:
    pass


@dataclass
class DistanceCutoff:
    dist_cutoff: float


@dataclass
class ShiftedPotentialCutoff:
    dist_cutoff: float


@dataclass
class ShiftedForceCutoff:
    dist_cutoff: float


@dataclass
class CubicSplineCutoff:
    """CubicSplineCutoff(dist_activation, dist_cutoff) — src/cutoffs.jl:174-215."""
    dist_activation: float
    dist_cutoff: float

    def __post_init__(self):
        if self.dist_cutoff <= self.dist_activation:  # ArgumentError in the reference constructor (:181-187)
            raise ValueError(f"the cutoff radius {self.dist_cutoff} must be larger than the activation radius {self.dist_activation}")


@dataclass
class PolynomialCutoff:
    """PolynomialCutoff(dist_activation, dist_cutoff) — src/cutoffs.jl:217-253 (OpenMM's switching function)."""
    dist_activation: float
    dist_cutoff: float

    def __post_init__(self):
        if self.dist_cutoff <= self.dist_activation:
            raise ValueError(f"the cutoff radius {self.dist_cutoff} must be larger than the activation radius {self.dist_activation}")


def _cutoff_kind(c):
    """-> (kind, dist_cutoff, dist_activation)"""
    if isinstance(c, NoCutoff):
        return capi.MB_CUT_NONE, 0.0, 0.0
    if isinstance(c, DistanceCutoff):
        return capi.MB_CUT_DISTANCE, c.dist_cutoff, 0.0
    if isinstance(c, ShiftedPotentialCutoff):
        return capi.MB_CUT_SHIFTED_POTENTIAL, c.dist_cutoff, 0.0
    if isinstance(c, ShiftedForceCutoff):
        return capi.MB_CUT_SHIFTED_FORCE, c.dist_cutoff, 0.0
    if isinstance(c, CubicSplineCutoff):
        return capi.MB_CUT_CUBIC_SPLINE, c.dist_cutoff, c.dist_activation
    if isinstance(c, PolynomialCutoff):
        return capi.MB_CUT_POLYNOMIAL, c.dist_cutoff, c.dist_activation
    raise TypeError(f"unsupported cutoff {c!r}")


@dataclass
class LennardJones:
    cutoff: object = field(default_factory=NoCutoff)
    use_neighbors: bool = False
    weight_special: float = 1.0
    sigma_mixing: str = "lorentz"
    eps_mixing: str = "geometric"

    def descriptor(self):
        k, rc, ra = _cutoff_kind(self.cutoff)
        return capi.MBInter(capi.MB_LJ, k, rc, ra, self.weight_special, COULOMB_CONST, 1.0, 0.0,
                            capi.MB_MIX_GEOMETRIC if self.sigma_mixing == "geometric" else capi.MB_MIX_LORENTZ,
                            capi.MB_MIX_GEOMETRIC if self.eps_mixing == "geometric" else capi.MB_MIX_LORENTZ, 0,
                            int(self.use_neighbors))


@dataclass
class Coulomb:
    cutoff: object = field(default_factory=NoCutoff)
    use_neighbors: bool = False
    weight_special: float = 1.0
    coulomb_const: float = COULOMB_CONST

    def descriptor(self):
        k, rc, ra = _cutoff_kind(self.cutoff)
        return capi.MBInter(capi.MB_COULOMB, k, rc, ra, self.weight_special, self.coulomb_const, 1.0, 0.0, 0, 1, 0,
                            int(self.use_neighbors))


@dataclass
class CoulombReactionField:
    dist_cutoff: float
    solvent_dielectric: float = 78.3  # coulomb.jl:676
    use_neighbors: bool = False
    weight_special: float = 1.0
    coulomb_const: float = COULOMB_CONST

    def descriptor(self):
        return capi.MBInter(capi.MB_CRF, capi.MB_CUT_DISTANCE, self.dist_cutoff, 0.0, self.weight_special,
                            self.coulomb_const, self.solvent_dielectric, 0.0, 0, 1, 0, int(self.use_neighbors))


@dataclass
class CoulombEwald:
    """Real-space part of Ewald/PME (coulomb.jl:1320-1441); alpha = sqrt(-log(2 tol)) / dist_cutoff.
    approximate_erfc=True (the reference's default, :1331) evaluates erfc with calc_erfc's polynomial (:1384-1393)."""
    dist_cutoff: float
    error_tol: float = 5e-4
    use_neighbors: bool = False
    weight_special: float = 1.0
    coulomb_const: float = COULOMB_CONST
    approximate_erfc: bool = True

    def descriptor(self):
        alpha = np.sqrt(-np.log(2 * self.error_tol)) / self.dist_cutoff
        return capi.MBInter(capi.MB_EWALD_REAL, capi.MB_CUT_DISTANCE, self.dist_cutoff, 0.0, self.weight_special,
                            self.coulomb_const, 1.0, float(alpha), 0, 1, int(self.approximate_erfc), int(self.use_neighbors))


@dataclass
class DPDInteraction:
    """DPDInteraction(a, gamma, sigma, r_c, dt, use_neighbors, key) — src/interactions/dpd.jl:57-142, the pairwise
    interaction of dissipative particle dynamics (conservative, dissipative and random forces), run on the device through
    mb_set_dpd (see include/mollyb200.h). gamma and sigma are the reference's γ and σ (σ² = 2 γ kT for temperature T); dt
    is the step the random force is scaled for (dt^(-1/2)). key=None draws one. It must be the System's only pairwise
    interaction; forces(sys) then uses sys.velocities, and simulate runs it under DPDVelocityVerlet only."""
    a: float = 25.0
    gamma: float = 4.5
    sigma: float = 3.0
    r_c: float = 1.0
    dt: float = 0.01
    use_neighbors: bool = False
    key: Optional[int] = None

    def __post_init__(self):
        if not (math.isfinite(self.r_c) and self.r_c > 0):
            raise ValueError(f"r_c must be finite and positive, found {self.r_c}")
        if not (math.isfinite(self.dt) and self.dt > 0):
            raise ValueError(f"dt must be finite and positive, found {self.dt}")
        for name in ("gamma", "sigma"):
            v = getattr(self, name)
            if not (math.isfinite(v) and v >= 0):
                raise ValueError(f"{name} must be finite and non-negative, found {v}")
        if not math.isfinite(self.a):
            raise ValueError(f"a must be finite, found {self.a}")
        if self.key is None:
            self.key = int(np.random.default_rng().integers(0, 2 ** 64, dtype=np.uint64))
        if not (_is_integer(self.key) and 0 <= int(self.key) < 2 ** 64):
            raise ValueError(f"key must be an integer in [0, 2^64), found {self.key!r}")
        self.key = int(self.key)

    def dpd_descriptor(self):
        return capi.MBDpd(float(self.a), float(self.gamma), float(self.sigma), float(self.r_c), float(self.dt), self.key,
                          int(bool(self.use_neighbors)))


def _dpd_of(sys):
    """The System's DPDInteraction, or None."""
    d = [it for it in sys.pairwise_inters if isinstance(it, DPDInteraction)]
    return d[0] if d else None


def _pairs_from(obj, n, want_true: bool):
    """Accept a dense (n,n) bool matrix or an (m,2) array of 1-based pairs."""
    if obj is None:
        return np.zeros((0, 2), np.int32)
    a = np.asarray(obj)
    if a.ndim == 2 and a.shape == (n, n) and a.dtype == np.bool_:
        m = a if want_true else ~a
        i, j = np.nonzero(np.triu(m, 1) | np.triu(m.T, 1))
        return np.stack([i + 1, j + 1], 1).astype(np.int32)
    return np.ascontiguousarray(a, np.int32).reshape(-1, 2)


@dataclass
class GPUNeighborFinder:
    """Device neighbour finder. `eligible`/`special` may be dense bool matrices (as in the reference
    constructor) or `excluded_pairs`/`special_pairs` sparse 1-based (m,2) arrays (neighbors.jl:104-115).
    n_steps: rebuild interval (reference default 10 CPU / 25 GPU); 0 = displacement-triggered (exact)."""
    dist_cutoff: float = 0.0
    eligible: object = None
    special: object = None
    excluded_pairs: object = None
    special_pairs: object = None
    n_steps: int = 0


# the reference's other finders build the same pair set; here they all map to the device cell list
DistanceNeighborFinder = GPUNeighborFinder
CellListMapNeighborFinder = GPUNeighborFinder
TreeNeighborFinder = GPUNeighborFinder


@dataclass
class PME:
    """PME(dist_cutoff, atoms, boundary; error_tol=0.0005, order=5, ϵr=1.0) general interaction
    (src/interactions/ewald.jl:363-421) together with the EwaldExclusion list that src/setup.jl:1903-1912 builds from
    find_excluded_pairs(eligible, special): `excluded_pairs` here = the excluded OR special pairs, 1-based (m,2).
    Use with CoulombEwald(dist_cutoff, error_tol) as the pairwise interaction. First implementation: see
    include/mollyb200.h (mb_set_pme) for its validation status."""
    dist_cutoff: float
    error_tol: float = 0.0005
    order: int = 5
    eps_r: float = 1.0
    excluded_pairs: object = None


@dataclass
class LJDispersionCorrection:
    """LJDispersionCorrection(atoms, dist_cutoff) general interaction (src/interactions/lennard_jones.jl:163-275): the
    factors are computed by the library from the System's atoms."""
    dist_cutoff: float


class _GBFactors:
    """factor_solute = -k / eps_solute and factor_solvent = k / eps_solvent, zero for a zero dielectric
    (implicit_solvent.jl:399-409), derived from the dielectrics whenever they are read."""

    @property
    def factor_solute(self):
        return -COULOMB_CONST / self.solute_dielectric if self.solute_dielectric != 0 else 0.0

    @property
    def factor_solvent(self):
        return COULOMB_CONST / self.solvent_dielectric if self.solvent_dielectric != 0 else 0.0


@dataclass
class ImplicitSolventOBC(_GBFactors):
    """ImplicitSolventOBC general interaction (src/interactions/implicit_solvent.jl:337-432) at array level: per-atom
    offset_radii (radius - offset) and scaled_offset_radii (screen x offset radius), the OBC alpha, beta, gamma (scalars;
    GBOBCII: 1.0, 0.8, 4.85, GBOBCI: 0.8, 0.0, 2.909125) and the struct's scalars. Radii from elements (mbondi2_radii)
    are the caller's, as the reference's constructor computes them. Run on the device by mb_set_implicit_solvent (three
    all-pairs passes, inside the captured step graphs). No virial."""
    offset_radii: object
    scaled_offset_radii: object
    alpha: float = 0.8
    beta: float = 0.0
    gamma: float = 2.909125
    solvent_dielectric: float = 78.5
    solute_dielectric: float = 1.0
    kappa: float = 0.0
    offset: float = 0.009
    dist_cutoff: float = 0.0
    probe_radius: float = 0.14
    sa_factor: float = 28.3919551
    use_ACE: bool = True

    def __post_init__(self):
        self.offset_radii = np.ascontiguousarray(self.offset_radii, np.float64)
        self.scaled_offset_radii = np.ascontiguousarray(self.scaled_offset_radii, np.float64)
        if self.offset_radii.shape != self.scaled_offset_radii.shape or self.offset_radii.ndim != 1:
            raise ValueError("offset_radii and scaled_offset_radii must be 1-D arrays of the same length")

    def per_atom(self):
        n = len(self.offset_radii)
        return [self.offset_radii, self.scaled_offset_radii] + [np.full(n, float(v)) for v in (self.alpha, self.beta, self.gamma)]

    def neck(self):
        return 0, None, None, None, 0.0, 0.0


@dataclass
class ImplicitSolventGBN2(_GBFactors):
    """ImplicitSolventGBN2 general interaction (src/interactions/implicit_solvent.jl:443-583) at array level: per-atom
    offset_radii, scaled_offset_radii, alphas, betas, gammas, and the neck lookup as classes: neck_class[i] in
    [0, n_classes) and the tables d0[c_i, c_j] = the reference's d0s[i, j], m0 likewise (not symmetric), in nm and nm^-1.
    Atoms of equal radius (offset_radii + offset) share a class. Run on the device by mb_set_implicit_solvent. No virial."""
    offset_radii: object
    scaled_offset_radii: object
    alpha: object
    beta: object
    gamma: object
    neck_class: object
    d0: object
    m0: object
    solvent_dielectric: float = 78.5
    solute_dielectric: float = 1.0
    kappa: float = 0.0
    offset: float = 0.0195141
    dist_cutoff: float = 0.0
    probe_radius: float = 0.14
    sa_factor: float = 28.3919551
    use_ACE: bool = True
    neck_scale: float = 0.826836
    neck_cut: float = 0.68

    def __post_init__(self):
        for name in ("offset_radii", "scaled_offset_radii", "alpha", "beta", "gamma"):
            setattr(self, name, np.ascontiguousarray(getattr(self, name), np.float64))
            if getattr(self, name).shape != np.shape(self.offset_radii) or getattr(self, name).ndim != 1:
                raise ValueError(f"{name}: a 1-D array with one value per atom")
        self.neck_class = np.ascontiguousarray(self.neck_class, np.int32)
        self.d0 = np.ascontiguousarray(self.d0, np.float64)
        self.m0 = np.ascontiguousarray(self.m0, np.float64)
        nc = len(self.d0)
        if self.neck_class.shape != self.offset_radii.shape:
            raise ValueError("neck_class: one class per atom")
        if self.d0.shape != (nc, nc) or self.m0.shape != (nc, nc) or not 0 < nc <= capi.MB_GB_MAX_NECK_CLASSES:
            raise ValueError(f"d0 and m0 must be square tables of the same size, 1 .. {capi.MB_GB_MAX_NECK_CLASSES} classes")
        if self.neck_class.min() < 0 or self.neck_class.max() >= nc:
            raise ValueError("neck_class outside the tables")

    def per_atom(self):
        return [self.offset_radii, self.scaled_offset_radii, self.alpha, self.beta, self.gamma]

    def neck(self):
        return len(self.d0), self.neck_class, self.d0, self.m0, self.neck_scale, self.neck_cut


_GB_TYPES = (ImplicitSolventOBC, ImplicitSolventGBN2)


@dataclass
class InteractionList2Atoms:
    """InteractionList2Atoms of HarmonicBond (src/types.jl:89-157, interactions/harmonic_bond.jl): 1-based is/js,
    per-term k (kJ mol^-1 nm^-2) and r0 (nm)."""
    is_: object
    js: object
    k: object
    r0: object
    kind = 0

    def arrays(self):
        idx = np.stack([np.asarray(self.is_), np.asarray(self.js)], 1).astype(np.int32)
        par = np.stack([np.asarray(self.k, np.float64), np.asarray(self.r0, np.float64)], 1)
        return np.ascontiguousarray(idx), np.ascontiguousarray(par)


@dataclass
class InteractionList3Atoms:
    """InteractionList3Atoms of HarmonicAngle (interactions/harmonic_angle.jl): k (kJ mol^-1 rad^-2), theta0 (rad)."""
    is_: object
    js: object
    ks: object
    k: object
    theta0: object
    kind = 1

    def arrays(self):
        idx = np.stack([np.asarray(self.is_), np.asarray(self.js), np.asarray(self.ks)], 1).astype(np.int32)
        par = np.stack([np.asarray(self.k, np.float64), np.asarray(self.theta0, np.float64)], 1)
        return np.ascontiguousarray(idx), np.ascontiguousarray(par)


@dataclass
class InteractionList4Atoms:
    """InteractionList4Atoms of PeriodicTorsion (interactions/periodic_torsion.jl), flattened to one
    (periodicity, phase, k) term per entry; propers and impropers use the same list type."""
    is_: object
    js: object
    ks: object
    ls: object
    periodicity: object
    phase: object
    k: object
    kind = 2

    def arrays(self):
        idx = np.stack([np.asarray(self.is_), np.asarray(self.js), np.asarray(self.ks), np.asarray(self.ls)], 1).astype(np.int32)
        par = np.stack([np.asarray(self.periodicity, np.float64), np.asarray(self.phase, np.float64),
                        np.asarray(self.k, np.float64)], 1)
        return np.ascontiguousarray(idx), np.ascontiguousarray(par)


def _list_arrays(idx_cols, par_cols):
    idx = np.stack([np.asarray(c).reshape(-1) for c in idx_cols], 1).astype(np.int32)
    par = np.stack([np.broadcast_to(np.asarray(c, np.float64), (len(idx),)) for c in par_cols], 1)
    return np.ascontiguousarray(idx), np.ascontiguousarray(par)


@dataclass
class InteractionList1Atoms:
    """InteractionList1Atoms of HarmonicPositionRestraint (interactions/harmonic_position_restraint.jl): 1-based is_,
    per-term k (kJ mol^-1 nm^-2) and restraint position x0 (n x 3, nm). The displacement to x0 is minimum-image."""
    is_: object
    k: object
    x0: object
    kind = capi.MB_SPECIFIC_POSITION_RESTRAINT

    def arrays(self):
        x0 = np.asarray(self.x0, np.float64).reshape(-1, 3)
        return _list_arrays([self.is_], [self.k, x0[:, 0], x0[:, 1], x0[:, 2]])


@dataclass
class MorseBonds:
    """InteractionList2Atoms of MorseBond (interactions/morse_bond.jl): V = D (1 - exp(-a (r - r0)))^2."""
    is_: object
    js: object
    D: object
    a: object
    r0: object
    kind = capi.MB_SPECIFIC_MORSE_BOND

    def arrays(self):
        return _list_arrays([self.is_, self.js], [self.D, self.a, self.r0])


@dataclass
class FENEBonds:
    """InteractionList2Atoms of FENEBond (interactions/fene_bond.jl): V = -k r0^2 / 2 ln(1 - (r / r0)^2) plus WCA(sigma,
    eps) for r < 2^(1/6) sigma. Undefined (NaN) for r >= r0, as in the reference."""
    is_: object
    js: object
    k: object
    r0: object
    sigma: object
    eps: object
    kind = capi.MB_SPECIFIC_FENE_BOND

    def arrays(self):
        return _list_arrays([self.is_, self.js], [self.k, self.r0, self.sigma, self.eps])


@dataclass
class CosineAngles:
    """InteractionList3Atoms of CosineAngle (interactions/cosine_angle.jl): V = k (1 + cos(theta - theta0)), j in the
    middle, theta0 in radians."""
    is_: object
    js: object
    ks: object
    k: object
    theta0: object
    kind = capi.MB_SPECIFIC_COSINE_ANGLE

    def arrays(self):
        return _list_arrays([self.is_, self.js, self.ks], [self.k, self.theta0])


@dataclass
class UreyBradleys:
    """InteractionList3Atoms of UreyBradley (interactions/urey_bradley.jl): a harmonic angle (kangle, theta0) plus a
    harmonic bond (kbond, r0) between the outer atoms i and k."""
    is_: object
    js: object
    ks: object
    kangle: object
    theta0: object
    kbond: object
    r0: object
    kind = capi.MB_SPECIFIC_UREY_BRADLEY

    def arrays(self):
        return _list_arrays([self.is_, self.js, self.ks], [self.kangle, self.theta0, self.kbond, self.r0])


@dataclass
class HarmonicTorsions:
    """InteractionList4Atoms of HarmonicTorsion (interactions/harmonic_torsion.jl): V = k (theta - theta0)^2, with
    theta - theta0 not wrapped, as in the reference."""
    is_: object
    js: object
    ks: object
    ls: object
    k: object
    theta0: object
    kind = capi.MB_SPECIFIC_HARMONIC_TORSION

    def arrays(self):
        return _list_arrays([self.is_, self.js, self.ks, self.ls], [self.k, self.theta0])


@dataclass
class RBTorsions:
    """InteractionList4Atoms of RBTorsion (interactions/rb_torsion.jl): V = (f1 (1 + cos th) + f2 (1 - cos 2th) +
    f3 (1 + cos 3th) + f4) / 2. The forces are -grad V; the reference's have the opposite sign (include/mollyb200.h)."""
    is_: object
    js: object
    ks: object
    ls: object
    f1: object
    f2: object
    f3: object
    f4: object
    kind = capi.MB_SPECIFIC_RB_TORSION

    def arrays(self):
        return _list_arrays([self.is_, self.js, self.ks, self.ls], [self.f1, self.f2, self.f3, self.f4])


def add_position_restraints(sys, k, atom_selector=None, restrain_coords=None):
    """add_position_restraints (src/setup.jl:2059-2100): a System like `sys` with one more specific interaction list, a
    HarmonicPositionRestraint on every selected atom. k: scalar or one value per atom of the system (kJ mol^-1 nm^-2);
    atom_selector: boolean mask over the atoms or 1-based indices, None for every atom; restrain_coords: n x 3, by default
    a copy of the current coordinates."""
    n = sys.n
    k_arr = np.asarray(k, np.float64)
    if k_arr.ndim > 0 and len(k_arr) != n:
        raise ValueError(f"the system has {n} atoms but there are {len(k_arr)} k values")
    k_arr = np.broadcast_to(k_arr, (n,))
    if restrain_coords is None:
        restrain_coords = sys.coords.cpu().numpy() if hasattr(sys.coords, "data_ptr") else sys.coords
    x0 = np.array(restrain_coords, np.float64).reshape(n, 3)
    if atom_selector is None:
        sel = np.arange(n)
    else:
        a = np.asarray(atom_selector)
        sel = np.flatnonzero(a) if a.dtype == bool else a.astype(np.int64).reshape(-1) - 1
        if a.dtype == bool and len(a) != n:
            raise ValueError(f"atom_selector has {len(a)} entries for {n} atoms")
        if len(sel) and (sel.min() < 0 or sel.max() >= n):
            raise ValueError("atom_selector: an index outside 1 .. n")
    restraints = InteractionList1Atoms(sel + 1, k_arr[sel].copy(), x0[sel])
    def copy(a):
        return a.clone() if hasattr(a, "data_ptr") else np.array(a)
    return System(atoms=sys.atoms.copy(), coords=copy(sys.coords), boundary=sys.boundary, velocities=copy(sys.velocities),
                  pairwise_inters=sys.pairwise_inters, neighbor_finder=sys.neighbor_finder, dtype=sys.dtype, device=sys.device,
                  k=sys.k, specific_inter_lists=sys.specific_inter_lists + (restraints,), general_inters=sys.general_inters,
                  loggers=sys.loggers)


@dataclass
class AndersenThermostat:
    temperature: float
    coupling_const: float


def _check_temperature(t):
    if not (math.isfinite(t) and t >= 0):
        raise ValueError(f"temperature must be finite and non-negative, found {t}")


def _check_coupling_const(tau):
    if not (math.isfinite(tau) and tau > 0):
        raise ValueError(f"coupling_const must be finite and positive, found {tau}")


@dataclass
class ImmediateThermostat:
    """ImmediateThermostat(temperature) — src/coupling.jl:82-91: lambda = sqrt(T0 / T) every step. Temperature in K."""
    temperature: float

    def __post_init__(self):
        _check_temperature(self.temperature)

    def descriptor(self, k):
        return capi.MBVCoupling(capi.MB_VC_IMMEDIATE, 0, k * self.temperature, 0.0)


@dataclass
class BerendsenThermostat:
    """BerendsenThermostat(temperature, coupling_const) — src/coupling.jl:227-238: lambda^2 = 1 + (dt / tau) (T0 / T - 1).
    Temperature in K, coupling_const in ps."""
    temperature: float
    coupling_const: float

    def __post_init__(self):
        _check_temperature(self.temperature)
        _check_coupling_const(self.coupling_const)

    def descriptor(self, k):
        return capi.MBVCoupling(capi.MB_VC_BERENDSEN, 0, k * self.temperature, self.coupling_const)


@dataclass
class VelocityRescaleThermostat:
    """VelocityRescaleThermostat(temperature, coupling_const; n_steps=1) — src/coupling.jl:114-168, the stochastic velocity
    rescaling of Bussi et al. 2007, every n_steps steps. The draws are made on the device (see mb_set_velocity_coupling)."""
    temperature: float
    coupling_const: float
    n_steps: int = 1

    def __post_init__(self):
        _check_temperature(self.temperature)
        _check_coupling_const(self.coupling_const)
        if isinstance(self.n_steps, bool) or int(self.n_steps) != self.n_steps or self.n_steps < 1:
            raise ValueError(f"n_steps must be a positive integer, found {self.n_steps}")

    def descriptor(self, k):
        return capi.MBVCoupling(capi.MB_VC_VRESCALE, int(self.n_steps), k * self.temperature, self.coupling_const)


_SCALING_THERMOSTATS = (ImmediateThermostat, BerendsenThermostat, VelocityRescaleThermostat)


@dataclass
class VelocityVerlet:
    dt: float
    coupling: object = None
    remove_CM_motion: int = 1


@dataclass
class Langevin:
    """Langevin(dt, temperature, friction; coupling=None, remove_CM_motion=1) — src/simulators.jl:1065-1100, Molly's port of
    OpenMM's LangevinMiddleIntegrator, run on the device by mb_simulate_langevin (see include/mollyb200.h for where the
    engine differs from the reference). dt in ps, temperature in K, friction in ps^-1. vel_scale = exp(-dt friction) and
    noise_scale = sqrt(1 - vel_scale^2) as the reference's constructor computes them. A coupling (the reference's barostats)
    is not run by the engine: simulate refuses it."""
    dt: float
    temperature: float
    friction: float
    coupling: object = None
    remove_CM_motion: int = 1
    vel_scale: float = field(init=False)
    noise_scale: float = field(init=False)

    def __post_init__(self):
        if not (math.isfinite(self.dt) and self.dt > 0):
            raise ValueError(f"dt must be finite and positive, found {self.dt}")
        _check_temperature(self.temperature)
        if not (math.isfinite(self.friction) and self.friction >= 0):
            raise ValueError(f"friction must be finite and non-negative, found {self.friction}")
        self.remove_CM_motion = int(self.remove_CM_motion)  # Int(remove_CM_motion): false -> 0
        if self.remove_CM_motion < 0:
            raise ValueError(f"remove_CM_motion must be non-negative, found {self.remove_CM_motion}")
        self.vel_scale = math.exp(-self.dt * self.friction)
        self.noise_scale = math.sqrt(1 - self.vel_scale ** 2)


@dataclass
class LangevinSplitting:
    """LangevinSplitting(dt, temperature, friction, splitting; remove_CM_motion=1) — src/simulators.jl:1212-1398, the
    Langevin integrator with any splitting of A (positions), B (forces) and O (friction and noise) steps, run on the device
    by mb_simulate_langevin_splitting (see include/mollyb200.h for where the engine differs from the reference). dt in ps,
    temperature in K, friction in g mol^-1 ps^-1 (a mass per time, unlike Langevin's). "BAOAB" samples configurations well
    (Leimkuhler-Matthews), "BAB" is the VelocityVerlet step and "BAOA" the Langevin step. Raises ValueError where the
    reference raises ArgumentError (a letter other than A, B, O), and for what the engine refuses: an empty splitting, more
    than MB_SPLIT_MAX_OPS letters, dt, temperature or friction out of range."""
    dt: float
    temperature: float
    friction: float
    splitting: str
    remove_CM_motion: int = 1

    def __post_init__(self):
        if not (math.isfinite(self.dt) and self.dt > 0):
            raise ValueError(f"dt must be finite and positive, found {self.dt}")
        _check_temperature(self.temperature)
        if not (math.isfinite(self.friction) and self.friction >= 0):
            raise ValueError(f"friction must be finite and non-negative, found {self.friction}")
        if not isinstance(self.splitting, str) or not all(op in "ABO" for op in self.splitting):
            raise ValueError("splitting must contain only A, B, and O steps")
        if not 1 <= len(self.splitting) <= capi.MB_SPLIT_MAX_OPS:
            raise ValueError(f"splitting must have 1 to {capi.MB_SPLIT_MAX_OPS} letters, found {len(self.splitting)}")
        self.remove_CM_motion = int(self.remove_CM_motion)  # Int(remove_CM_motion): false -> 0
        if self.remove_CM_motion < 0:
            raise ValueError(f"remove_CM_motion must be non-negative, found {self.remove_CM_motion}")


@dataclass
class NoseHoover:
    """NoseHoover(dt, temperature, damping=100 dt; coupling=None, remove_CM_motion=1) — src/simulators.jl:1491-1614, the
    Nose-Hoover thermostat of Evans and Holian 1985, run on the device by mb_simulate_nose_hoover (see include/mollyb200.h
    for the step and where the engine differs from the reference). dt in ps, temperature in K (> 0: the step divides by
    it), damping in ps. The thermostat variable zeta starts at 0 in every call, as in the reference. A coupling is not run
    by the engine: simulate refuses it."""
    dt: float
    temperature: float
    damping: Optional[float] = None
    coupling: object = None
    remove_CM_motion: int = 1

    def __post_init__(self):
        if not (math.isfinite(self.dt) and self.dt > 0):
            raise ValueError(f"dt must be finite and positive, found {self.dt}")
        if not (math.isfinite(self.temperature) and self.temperature > 0):
            raise ValueError(f"temperature must be finite and positive, found {self.temperature}")
        if self.damping is None:
            self.damping = 100 * self.dt  # the reference's default
        if not (math.isfinite(self.damping) and self.damping > 0):
            raise ValueError(f"damping must be finite and positive, found {self.damping}")
        self.remove_CM_motion = int(self.remove_CM_motion)  # Int(remove_CM_motion): false -> 0
        if self.remove_CM_motion < 0:
            raise ValueError(f"remove_CM_motion must be non-negative, found {self.remove_CM_motion}")


def _check_dt(dt):
    if not (math.isfinite(dt) and dt > 0):
        raise ValueError(f"dt must be finite and positive, found {dt}")


def _check_remove_cm(sim):
    sim.remove_CM_motion = int(sim.remove_CM_motion)  # Int(remove_CM_motion): false -> 0
    if sim.remove_CM_motion < 0:
        raise ValueError(f"remove_CM_motion must be non-negative, found {sim.remove_CM_motion}")


@dataclass
class Verlet:
    """Verlet(dt; coupling=None, remove_CM_motion=1) — src/simulators.jl:858-955, the leapfrog integrator (the velocities
    are half a step behind the positions), run on the device by mb_simulate_verlet (see include/mollyb200.h). dt in ps. The
    coupling may be None or one AndersenThermostat; simulate raises TypeError for any other."""
    dt: float
    coupling: object = None
    remove_CM_motion: int = 1

    def __post_init__(self):
        _check_dt(self.dt)
        _check_remove_cm(self)


@dataclass
class StormerVerlet:
    """StormerVerlet(dt) — src/simulators.jl:957-1063, run on the device by mb_simulate_stormer_verlet (see
    include/mollyb200.h). dt in ps. No coupling and no centre-of-mass motion removal; the first step of every call starts
    from the velocities, later steps from the previous displacement."""
    dt: float

    def __post_init__(self):
        _check_dt(self.dt)


@dataclass
class OverdampedLangevin:
    """OverdampedLangevin(dt, temperature, friction; remove_CM_motion=1) — src/simulators.jl:1400-1490, Brownian dynamics
    by Euler-Maruyama, run on the device by mb_simulate_overdamped_langevin (see include/mollyb200.h). dt in ps,
    temperature in K, friction in ps^-1 (> 0: the noise prefactor is sqrt(2 dt / friction)). The velocities only lose
    their centre-of-mass drift."""
    dt: float
    temperature: float
    friction: float
    remove_CM_motion: int = 1

    def __post_init__(self):
        _check_dt(self.dt)
        _check_temperature(self.temperature)
        if not (math.isfinite(self.friction) and self.friction > 0):
            raise ValueError(f"friction must be finite and positive, found {self.friction}")
        _check_remove_cm(self)


@dataclass
class DPDVelocityVerlet:
    """DPDVelocityVerlet(dt, lam=0.65; coupling=None, remove_CM_motion=1) — src/simulators.jl:670-842, the Groot-Warren
    modified velocity Verlet, run on the device by mb_simulate_dpd_vv (see include/mollyb200.h). lam is the reference's λ:
    the forces of step t + dt are evaluated with v_pred = v(t + dt/2) + (λ - 1/2) dt a(t). No coupling is supported
    (simulate raises TypeError for one)."""
    dt: float
    lam: float = 0.65
    coupling: object = None
    remove_CM_motion: int = 1

    def __post_init__(self):
        _check_dt(self.dt)
        if not math.isfinite(self.lam):
            raise ValueError(f"lam must be finite, found {self.lam}")
        _check_remove_cm(self)


def _is_integer(x) -> bool:
    return isinstance(x, (int, np.integer))


def setup_mts_integrator(pi_fractions, si_fractions, gi_fractions) -> tuple:
    """setup_mts_integrator (src/simulators.jl:1713-1738): the distinct fractions in increasing order, ordered_fractions =
    (1, f1, f2, ...). ValueError where the reference raises ArgumentError."""
    if not (len(pi_fractions) or len(si_fractions) or len(gi_fractions)):
        raise ValueError("MTSIntegrator requires one of pi_fractions, si_fractions or gi_fractions to be provided")
    if not all(_is_integer(f) for f in (*pi_fractions, *si_fractions, *gi_fractions)):
        raise ValueError("MTSIntegrator requires pi_fractions, si_fractions and gi_fractions to consist of integers")
    ordered = tuple(sorted({int(f) for f in (*pi_fractions, *si_fractions, *gi_fractions)}))
    if ordered[0] < 1:
        raise ValueError(f"MTSIntegrator fraction {ordered[0]} cannot be less than 1")
    if ordered[0] > 1:
        raise ValueError(f"MTSIntegrator fractions must include 1, lowest fraction is {ordered[0]}")
    for a, b in zip(ordered, ordered[1:]):
        if b % a != 0:
            raise ValueError(f"MTSIntegrator fraction {b} not a multiple of fraction {a}")
    return ordered


@dataclass
class MTSIntegrator:
    """MTSIntegrator(dt; pi_fractions, si_fractions, gi_fractions, coupling=None, remove_CM_motion=1) —
    src/simulators.jl:1616-1654, 1740-1745: rRESPA multiple time stepping (Tuckerman et al. 1992), run on the device by
    mb_simulate_mts (see include/mollyb200.h). dt is the outer step in ps; an interaction with fraction f is applied f times
    per outer step; n_steps counts outer steps. The engine evaluates every pairwise interaction and PME once per outer step
    (fraction 1); each specific interaction list has a level of its own. A coupling is not run: simulate refuses it."""
    dt: float
    pi_fractions: tuple = ()
    si_fractions: tuple = ()
    gi_fractions: tuple = ()
    coupling: object = None
    remove_CM_motion: int = 1
    ordered_fractions: tuple = field(init=False)

    def __post_init__(self):
        if not (math.isfinite(self.dt) and self.dt > 0):
            raise ValueError(f"dt must be finite and positive, found {self.dt}")
        self.pi_fractions, self.si_fractions, self.gi_fractions = (tuple(self.pi_fractions), tuple(self.si_fractions),
                                                                   tuple(self.gi_fractions))
        self.ordered_fractions = setup_mts_integrator(self.pi_fractions, self.si_fractions, self.gi_fractions)
        self.remove_CM_motion = int(self.remove_CM_motion)  # Int(remove_CM_motion): false -> 0
        if self.remove_CM_motion < 0:
            raise ValueError(f"remove_CM_motion must be non-negative, found {self.remove_CM_motion}")


@dataclass
class MTSLangevinIntegrator:
    """MTSLangevinIntegrator(dt, temperature, friction; pi_fractions, si_fractions, gi_fractions, coupling=None,
    remove_CM_motion=1) — src/simulators.jl:1656-1711, 1747-1757: BAOAB-RESPA (Lagardère et al. 2019), run on the device by
    mb_simulate_mts. The O step runs at every innermost substep with vel_scale = exp(-dt friction / last(ordered_fractions))
    and noise_scale = sqrt(1 - vel_scale^2), as the reference's constructor computes them. Temperature in K, friction in
    ps^-1; the rest as MTSIntegrator."""
    dt: float
    temperature: float
    friction: float
    pi_fractions: tuple = ()
    si_fractions: tuple = ()
    gi_fractions: tuple = ()
    coupling: object = None
    remove_CM_motion: int = 1
    ordered_fractions: tuple = field(init=False)
    vel_scale: float = field(init=False)
    noise_scale: float = field(init=False)

    def __post_init__(self):
        MTSIntegrator.__post_init__(self)
        _check_temperature(self.temperature)
        if not (math.isfinite(self.friction) and self.friction >= 0):
            raise ValueError(f"friction must be finite and non-negative, found {self.friction}")
        self.vel_scale = math.exp(-self.dt * self.friction / self.ordered_fractions[-1])
        self.noise_scale = math.sqrt(1 - self.vel_scale ** 2)


def mts_levels(sys, sim) -> dict:
    """The level of every specific term for mb_set_specific_levels: {kind: int32 array}, in the order System._configure
    concatenates the lists of one kind (e.g. propers then impropers). Checks the fractions against the System as
    mts_interaction_groups does (ValueError), and refuses what the engine does not split (TypeError): a pairwise
    interaction or PME at a fraction other than 1 (LJDispersionCorrection exerts no force: any fraction)."""
    for name, fr, inters in (("pairwise", sim.pi_fractions, sys.pairwise_inters),
                             ("specific", sim.si_fractions, sys.specific_inter_lists),
                             ("general", sim.gi_fractions, sys.general_inters)):
        if len(fr) != len(inters):
            raise ValueError(f"the system has {len(inters)} {name} interactions but there are {len(fr)} in the "
                             f"{type(sim).__name__}")
    if any(f != 1 for f in sim.pi_fractions):
        raise TypeError(f"{type(sim).__name__}: pairwise interactions at a fraction other than 1 are not supported "
                        "(the engine evaluates them in one kernel once per outer step; the stock Molly path handles it)")
    for gi, f in zip(sys.general_inters, sim.gi_fractions):
        if isinstance(gi, PME) and f != 1:
            raise TypeError(f"{type(sim).__name__}: PME at a fraction other than 1 is not supported (the stock Molly "
                            "path handles it)")
        if isinstance(gi, _GB_TYPES) and f != 1:
            raise TypeError(f"{type(sim).__name__}: implicit solvent at a fraction other than 1 is not supported (the "
                            "engine evaluates it with level 0)")
    parts = {}
    for sil, f in zip(sys.specific_inter_lists, sim.si_fractions):
        n = len(sil.arrays()[0])
        parts.setdefault(sil.kind, []).append(np.full(n, sim.ordered_fractions.index(int(f)), np.int32))
    return {kind: np.ascontiguousarray(np.concatenate(p)) for kind, p in parts.items()}


@dataclass
class SteepestDescentMinimizer:
    """SteepestDescentMinimizer(step_size, max_steps, tol, log_stream) — src/simulators.jl:183-274, run on the device by
    mb_minimize_sd (see include/mollyb200.h for where the engine may differ from the reference). step_size in nm, tol in
    kJ mol^-1 nm^-1. log_stream: a text stream that receives the reference's per-step lines after the call (None: none)."""
    step_size: float = 0.01
    max_steps: int = 1000
    tol: float = 1000.0
    log_stream: object = None

    def __post_init__(self):
        if not self.step_size > 0:
            raise ValueError(f"step_size must be positive, found {self.step_size}")
        if int(self.max_steps) < 0:
            raise ValueError(f"max_steps must be non-negative, found {self.max_steps}")
        if not self.tol >= 0:
            raise ValueError(f"tol must be non-negative, found {self.tol}")


# ------------------------------------------------------------------------------------------------
# loggers: recorded on the device inside simulate (mb_simulate_vv_log)
# ------------------------------------------------------------------------------------------------
class _DeviceLogger:
    """GeneralObservableLogger (src/loggers.jl:63-102): records at step s when s % n_steps == 0. `history` grows over
    consecutive simulate calls. For a System with host (numpy) state the entries are numpy values; for a System with
    torch CUDA state they are CUDA tensors the engine wrote."""
    kind = ""  # "energy", "coords" or "vels": which engine record the logger reads

    def __init__(self, n_steps: int):
        if int(n_steps) <= 0:
            raise ValueError(f"n_steps must be positive, found {n_steps}")
        self.n_steps = int(n_steps)
        self.history = []

    def __repr__(self):
        return f"{type(self).__name__}({self.n_steps}) with {len(self.history)} entries"


class PotentialEnergyLogger(_DeviceLogger):
    """potential_energy(sys) of pairwise + specific + general interactions (src/loggers.jl:251-260)."""
    kind = "energy"


class KineticEnergyLogger(_DeviceLogger):
    """kinetic_energy(sys) (src/loggers.jl:225-234)."""
    kind = "energy"


class TotalEnergyLogger(_DeviceLogger):
    """potential + kinetic energy (src/loggers.jl:272-278)."""
    kind = "energy"


class TemperatureLogger(_DeviceLogger):
    """temperature(sys) with the degrees of freedom of `temperature` (src/loggers.jl:134-143)."""
    kind = "energy"


class CoordinatesLogger(_DeviceLogger):
    """Coordinates wrapped into the box, original atom order (src/loggers.jl:153-166)."""
    kind = "coords"


class VelocitiesLogger(_DeviceLogger):
    """Velocities after the step's CM removal and coupling (src/loggers.jl:201-214)."""
    kind = "vels"


def values(logger):
    """values(logger) — src/loggers.jl:85: the stored observations."""
    return logger.history


def _check_run_loggers(run_loggers):
    if not (run_loggers is True or run_loggers is False or run_loggers == "skipstart"):
        raise ValueError(f'run_loggers must be True, False or "skipstart", found {run_loggers!r}')


def record_steps(every: int, n_steps: int, init_step: int = 0, run_loggers=True) -> list:
    """Steps at which simulate(..., n_steps, init_step, run_loggers) records a logger of interval `every`: apply_loggers!
    runs at init_step only when run_loggers is True (src/simulators.jl:575) and after every step unless it is False
    (:657, src/loggers.jl:44-56); a logger keeps step s when s % every == 0 (:96-102)."""
    _check_run_loggers(run_loggers)
    if every <= 0 or run_loggers is False:
        return []
    first = (init_step // every + 1) * every
    steps = list(range(first, init_step + n_steps + 1, every))
    if run_loggers is True and init_step % every == 0:
        steps.insert(0, init_step)
    return steps


_LOG_FIELDS = {"energy": ("energy_every", "energies", "energy_capacity"),
               "coords": ("coords_every", "coords", "coords_capacity"),
               "vels": ("vels_every", "vels", "vels_capacity")}


class _LogPlan:
    """One simulate call's records. The engine records each kind (energies, coordinate frames, velocity frames) at the gcd
    of the intervals of the loggers that read it; each logger then keeps the records of its own steps."""

    def __init__(self, sys, n_steps: int, init_step: int, run_loggers):
        self.sys = sys
        self.loggers = list(sys.loggers.values())
        self.steps, self.buf = {}, {}
        d = capi.MBLog()
        d.log_initial = int(run_loggers is True)
        device = hasattr(sys.coords, "data_ptr")
        for kind in ("energy", "coords", "vels"):
            intervals = [lg.n_steps for lg in self.loggers if lg.kind == kind]
            every = math.gcd(*intervals) if intervals else 0
            steps = record_steps(every, n_steps, init_step, run_loggers)
            shape = (len(steps), 3) if kind == "energy" else (len(steps), sys.n, 3)
            if device:
                import torch
                dt = torch.float64 if kind == "energy" else sys.coords.dtype
                buf = torch.zeros(shape, dtype=dt, device=sys.coords.device)
            else:
                buf = np.zeros(shape, np.float64 if kind == "energy" else sys.dtype)
            self.steps[kind], self.buf[kind] = steps, buf
            if steps:  # (an interval with no record in this call is passed as 0)
                f_every, f_out, f_cap = _LOG_FIELDS[kind]
                setattr(d, f_every, every)
                setattr(d, f_out, _ptr(buf))
                setattr(d, f_cap, len(steps))
        self.desc = d

    def push(self):
        """Append this call's records to the loggers' histories (only after the call succeeded)."""
        e = self.buf["energy"]
        pe, ke = e[:, 1], e[:, 2]
        df = 3 * self.sys.n - 3
        derived = {PotentialEnergyLogger: pe, KineticEnergyLogger: ke, TotalEnergyLogger: pe + ke,
                   TemperatureLogger: 2.0 * ke / (df * self.sys.k)}
        for lg in self.loggers:
            vals = self.buf[lg.kind] if lg.kind != "energy" else derived[type(lg)]
            for k, s in enumerate(self.steps[lg.kind]):
                if s % lg.n_steps == 0:
                    lg.history.append(vals[k])


_LOGGER_TYPES = (PotentialEnergyLogger, KineticEnergyLogger, TotalEnergyLogger, TemperatureLogger, CoordinatesLogger,
                 VelocitiesLogger)


# ------------------------------------------------------------------------------------------------
# System
# ------------------------------------------------------------------------------------------------
class System:
    """System(atoms, coords, boundary, velocities, pairwise_inters, neighbor_finder) — src/types.jl:795-979.

    coords / velocities are numpy arrays (n,3) of `dtype` (host) or torch CUDA tensors (device); the
    engine accepts both through the same C entry points.
    """

    def __init__(self, atoms, coords, boundary, velocities=None, pairwise_inters=(), neighbor_finder=None,
                 dtype=np.float32, device: int = 0, k=BOLTZMANN_K, specific_inter_lists=(), general_inters=(), loggers=None):
        self.dtype = np.dtype(dtype)
        if isinstance(atoms, np.ndarray) and atoms.dtype.names:
            self.atoms = np.ascontiguousarray(atoms.astype(atom_dtype(self.dtype)))
        else:
            self.atoms = atoms_to_array(atoms, self.dtype)
        self.n = len(self.atoms)
        self.boundary = boundary
        self.coords = self._as_state(coords)
        self.velocities = self._as_state(velocities if velocities is not None else np.zeros((self.n, 3)))
        self.pairwise_inters = tuple(pairwise_inters)
        self.neighbor_finder = neighbor_finder
        self.specific_inter_lists = tuple(specific_inter_lists)
        self.general_inters = tuple(general_inters)
        self.device = device
        self.k = k
        self.loggers = dict(loggers or {})
        for name, lg in self.loggers.items():
            if type(lg) not in _LOGGER_TYPES:  # (no silent skip: the engine cannot record it)
                raise TypeError(f"logger {name!r}: {type(lg).__name__} is not supported; the engine records "
                                + ", ".join(t.__name__ for t in _LOGGER_TYPES))
        self._ctx = None

    def _as_state(self, a):
        if hasattr(a, "data_ptr"):  # torch tensor (device resident)
            return a
        return np.ascontiguousarray(np.asarray(a, self.dtype).reshape(self.n, 3))

    @property
    def masses(self):
        return self.atoms["mass"].astype(np.float64)

    # ---- engine context ------------------------------------------------------------------------
    def engine(self):
        if self._ctx is None:
            L = capi.load()
            ctx = C.c_void_p()
            capi.check(L.mb_ctx_create(self.device, 32 if self.dtype == np.float32 else 64, None, C.byref(ctx)))
            self._ctx = ctx
            self._L = L
            self._configure()
        return self._ctx

    def _configure(self):
        L, ctx = self._L, self._ctx
        capi.check(L.mb_set_atoms(ctx, self.n, self.atoms.ctypes.data))
        if isinstance(self.boundary, TriclinicBoundary):
            capi.check(L.mb_set_box_triclinic(ctx, (C.c_double * 9)(*self.boundary.basis_vectors.ravel())))
        else:
            side = (C.c_double * 3)(*self.boundary.side_lengths)
            capi.check(L.mb_set_box(ctx, side))
        dpd = [it for it in self.pairwise_inters if isinstance(it, DPDInteraction)]
        if len(dpd) > 1:
            raise ValueError("at most one DPDInteraction per System")
        descs = [it.descriptor() for it in self.pairwise_inters if not isinstance(it, DPDInteraction)]
        arr = (capi.MBInter * max(1, len(descs)))(*descs)
        capi.check(L.mb_set_inters(ctx, len(descs), arr))
        capi.check(L.mb_set_dpd(ctx, C.byref(dpd[0].dpd_descriptor()) if dpd else None))
        nf = self.neighbor_finder
        if nf is not None:
            if nf.excluded_pairs is not None:
                ex = _pairs_from(nf.excluded_pairs, self.n, want_true=True)
            else:
                ex = _pairs_from(nf.eligible, self.n, want_true=False)
            sp = _pairs_from(nf.special_pairs if nf.special_pairs is not None else nf.special, self.n, want_true=True)
            ei, ej = np.ascontiguousarray(ex[:, 0]), np.ascontiguousarray(ex[:, 1])
            si, sj = np.ascontiguousarray(sp[:, 0]), np.ascontiguousarray(sp[:, 1])
            self._keep = (ei, ej, si, sj)
            capi.check(L.mb_set_exceptions(ctx, len(ei), ei.ctypes.data, ej.ctypes.data, len(si), si.ctypes.data,
                                           sj.ctypes.data))
            capi.check(L.mb_set_neighbor_policy(ctx, float(nf.dist_cutoff), int(nf.n_steps)))
        # specific interaction lists: entries of the same kind are concatenated (e.g. propers + impropers)
        by_kind = {}
        for sil in self.specific_inter_lists:
            idx, par = sil.arrays()
            a, b = by_kind.get(sil.kind, (None, None))
            by_kind[sil.kind] = (idx if a is None else np.concatenate([a, idx]), par if b is None else np.concatenate([b, par]))
        for kind, (idx, par) in by_kind.items():
            idx, par = np.ascontiguousarray(idx), np.ascontiguousarray(par)
            capi.check(L.mb_set_specific(ctx, kind, len(idx), idx.ctypes.data, par.ctypes.data))

        for gi in self.general_inters:
            if isinstance(gi, LJDispersionCorrection):
                capi.check(L.mb_set_lj_dispersion_correction(ctx, float(gi.dist_cutoff)))
                continue
            if isinstance(gi, _GB_TYPES):
                self._set_implicit_solvent(gi)
                continue
            if not isinstance(gi, PME):
                raise ValueError("only PME, LJDispersionCorrection, ImplicitSolventOBC and ImplicitSolventGBN2 are supported "
                                 "as general interactions")
            pairs = np.zeros((0, 2), np.int32) if gi.excluded_pairs is None else np.asarray(gi.excluded_pairs, np.int32).reshape(-1, 2)
            pi, pj = np.ascontiguousarray(pairs[:, 0]), np.ascontiguousarray(pairs[:, 1])
            self._keep_pme = (pi, pj)
            capi.check(L.mb_set_pme(ctx, float(gi.dist_cutoff), float(gi.error_tol), int(gi.order), float(gi.eps_r), len(pi),
                                    pi.ctypes.data, pj.ctypes.data))

    def _set_implicit_solvent(self, gi):
        arrays = [np.ascontiguousarray(a, np.float64) for a in gi.per_atom()]
        if any(len(a) != self.n for a in arrays):
            raise ValueError(f"{type(gi).__name__}: per-atom arrays of {len(arrays[0])} atoms for a system of {self.n}")
        nc, cls, d0, m0, neck_scale, neck_cut = gi.neck()
        p = capi.MBGbsa(dist_cutoff=float(gi.dist_cutoff), offset=float(gi.offset), probe_radius=float(gi.probe_radius),
                        sa_factor=float(gi.sa_factor), factor_solute=float(gi.factor_solute),
                        factor_solvent=float(gi.factor_solvent), kappa=float(gi.kappa), neck_scale=float(neck_scale),
                        neck_cut=float(neck_cut), use_ace=int(bool(gi.use_ACE)), n_neck_classes=int(nc))
        keep = arrays + ([np.ascontiguousarray(cls, np.int32), np.ascontiguousarray(d0, np.float64).ravel(),
                          np.ascontiguousarray(m0, np.float64).ravel()] if nc else [])
        self._keep_gb = keep
        ptr = [a.ctypes.data for a in keep] + ([None] * 3 if not nc else [])
        capi.check(self._L.mb_set_implicit_solvent(self._ctx, C.byref(p), *ptr))

    def close(self):
        if self._ctx is not None:
            self._L.mb_ctx_destroy(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def stats(self) -> dict:
        st = capi.MBStats()
        ctx = self.engine()
        capi.check(self._L.mb_stats(ctx, C.byref(st)))
        out = {}
        for name, _ in capi.MBStats._fields_:
            v = getattr(st, name)
            out[name] = list(v) if hasattr(v, "__len__") else v
        return out

    def set_profiling(self, enable: bool):
        ctx = self.engine()
        capi.check(self._L.mb_set_profiling(ctx, int(enable)))

    def set_launch_config(self, brick_dims=(0, 0, 0), lanes_per_atom=0):
        bd = (C.c_int32 * 3)(*brick_dims)
        ctx = self.engine()
        capi.check(self._L.mb_set_launch_config(ctx, bd, lanes_per_atom))


def _ptr(a):
    return a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data


# ------------------------------------------------------------------------------------------------
# functions
# ------------------------------------------------------------------------------------------------
def _evaluate(call, *outputs):
    """Run one evaluation through the C ABI. MB_ERR_CAPACITY means a neighbour-structure capacity overflowed for these
    coordinates (an atom cloud that moved into a face or gathered since the last call): the outputs are invalid, and the
    engine re-derives its capacities on the next call. The outputs accumulate (ADD semantics), so they are cleared and the
    evaluation runs once more, as simulate does."""
    rc = call()
    if rc == capi.MB_ERR_CAPACITY:
        for a in outputs:
            a[...] = 0
        rc = call()
    capi.check(rc)


def forces(sys: System, neighbors=None, step_n: int = 0) -> np.ndarray:
    """forces(sys[, neighbors, step_n]) — src/force.jl:678-687. Returns (n,3) in kJ mol^-1 nm^-1. With a DPDInteraction the
    forces are those of sys.velocities and of the draws of step step_n (mb_forces_energy_vel)."""
    ctx = sys.engine()
    fs = np.zeros((sys.n, 3), sys.dtype)
    if _dpd_of(sys) is not None:
        _evaluate(lambda: sys._L.mb_forces_energy_vel(ctx, _ptr(sys.coords), _ptr(sys.velocities), fs.ctypes.data, None, step_n), fs)
    elif sys.specific_inter_lists or sys.general_inters:  # forces(sys) sums pairwise + specific + general interactions
        _evaluate(lambda: sys._L.mb_forces_energy_all(ctx, _ptr(sys.coords), fs.ctypes.data, None, step_n), fs)
    else:
        _evaluate(lambda: sys._L.mb_forces(ctx, _ptr(sys.coords), fs.ctypes.data, None, step_n), fs)
    return fs


def forces_virial(sys: System, neighbors=None, step_n: int = 0):
    """forces_virial — src/force.jl:703-720. Returns (forces, virial 3x3). Pairwise interactions only: a System with
    specific or general interactions is refused instead of silently dropping their virial."""
    if sys.specific_inter_lists or sys.general_inters:
        raise NotImplementedError("forces_virial covers the pairwise seam (pairwise_forces_loop_gpu!) only")
    ctx = sys.engine()
    fs = np.zeros((sys.n, 3), sys.dtype)
    vir = np.zeros(9, sys.dtype)
    _evaluate(lambda: sys._L.mb_forces(ctx, _ptr(sys.coords), fs.ctypes.data, vir.ctypes.data, step_n), fs, vir)
    return fs, vir.reshape(3, 3).T.copy()


def potential_energy(sys: System, neighbors=None, step_n: int = 0) -> float:
    """potential_energy(sys[, neighbors, step_n]) — src/energy.jl:202-248 (pairwise part)."""
    ctx = sys.engine()
    pe = np.zeros(1, sys.dtype)
    if sys.specific_inter_lists or sys.general_inters:  # potential_energy(sys): pairwise + specific + general
        _evaluate(lambda: sys._L.mb_forces_energy_all(ctx, _ptr(sys.coords), None, pe.ctypes.data, step_n), pe)
    else:
        _evaluate(lambda: sys._L.mb_energy(ctx, _ptr(sys.coords), pe.ctypes.data, step_n), pe)
    return float(pe[0])


def forces_energy(sys: System, step_n: int = 0):
    """forces(sys) and potential_energy(sys) of all pairwise + specific interactions in one traversal."""
    ctx = sys.engine()
    fs = np.zeros((sys.n, 3), sys.dtype)
    pe = np.zeros(1, sys.dtype)
    if _dpd_of(sys) is not None:
        _evaluate(lambda: sys._L.mb_forces_energy_vel(ctx, _ptr(sys.coords), _ptr(sys.velocities), fs.ctypes.data, pe.ctypes.data,
                                                      step_n), fs, pe)
    elif sys.specific_inter_lists or sys.general_inters:
        _evaluate(lambda: sys._L.mb_forces_energy_all(ctx, _ptr(sys.coords), fs.ctypes.data, pe.ctypes.data, step_n), fs, pe)
    else:
        _evaluate(lambda: sys._L.mb_forces_energy(ctx, _ptr(sys.coords), fs.ctypes.data, pe.ctypes.data, None, step_n), fs, pe)
    return fs, float(pe[0])


def find_neighbors(sys: System, *args, **kwargs):
    """find_neighbors(sys, nf::GPUNeighborFinder, ...) = nothing in the reference (neighbors.jl:364);
    here it forces a device rebuild and returns None."""
    ctx = sys.engine()
    capi.check(sys._L.mb_rebuild_neighbors(ctx, _ptr(sys.coords)))
    return None


def sd_log_lines(trace) -> list:
    """The lines simulate!(sys, ::SteepestDescentMinimizer) prints to its log_stream (src/simulators.jl:227-260), from the
    records (step, E or E_trial, max force, accepted) of steepest_descent."""
    t = np.asarray(trace, np.float64).reshape(-1, 4)
    if len(t) == 0:
        return []
    lines = [f"Step {int(t[0, 0])} - potential energy {t[0, 1]} - max force N/A - N/A"]
    for step, e, m, acc in t[1:]:
        lines.append(f"Step {int(step)} - potential energy {e} - max force {m} - {'accepted' if acc else 'rejected'}")
    return lines


def steepest_descent(sys: System, sim: SteepestDescentMinimizer, init_step: int = 0, max_retries: int = 2):
    """simulate!(sys, sim::SteepestDescentMinimizer; init_step) on the device (mb_minimize_sd). Mutates sys.coords (numpy or
    torch CUDA, in place) and returns (sys, trace): trace is (n_iterations + 1, 4) float64 records (step, E or E_trial,
    max force, accepted), record 0 = (init_step, E0, nan, 1). Also sets sys.minimize_result (the written-back fields)."""
    ctx = sys.engine()
    p = capi.MBSDParams()
    p.step_size = float(sim.step_size)
    p.max_steps = int(sim.max_steps)
    p.tol = float(sim.tol)
    p.init_step = int(init_step)
    trace = np.zeros((p.max_steps + 1, 4), np.float64)
    p.trace = trace.ctypes.data
    p.trace_capacity = len(trace)
    host = not hasattr(sys.coords, "data_ptr")
    backup = sys.coords.copy() if host else None
    scale = 1.0
    for attempt in range(max_retries + 1):
        rc = sys._L.mb_minimize_sd(ctx, _ptr(sys.coords), C.byref(p))
        if rc == capi.MB_ERR_CAPACITY and backup is not None and attempt < max_retries:
            sys.coords[...] = backup
            scale *= 2.0
            capi.check(sys._L.mb_set_capacity_scale(ctx, scale))
            continue
        capi.check(rc)
        break
    trace = trace[:p.n_iterations + 1].copy()
    sys.minimize_result = dict(n_iterations=int(p.n_iterations), energy=float(p.energy), max_force=float(p.max_force),
                               step_size=float(p.final_step_size), converged=bool(p.converged))
    if sim.log_stream is not None:
        for line in sd_log_lines(trace):
            print(line, file=sim.log_stream)
    return sys, trace


# simulator type -> its parameter struct, C entry point and mb_simulate_group kind (each entry takes an optional log plan;
# NULL: no logging)
_SIMULATE_ENTRY = {
    VelocityVerlet: (capi.MBVVParams, "mb_simulate_vv_log", capi.MB_INTEG_VV),
    Langevin: (capi.MBLangevinParams, "mb_simulate_langevin", capi.MB_INTEG_LANGEVIN),
    LangevinSplitting: (capi.MBSplittingParams, "mb_simulate_langevin_splitting", capi.MB_INTEG_LANGEVIN_SPLITTING),
    NoseHoover: (capi.MBNoseHooverParams, "mb_simulate_nose_hoover", capi.MB_INTEG_NOSE_HOOVER),
    MTSIntegrator: (capi.MBMTSParams, "mb_simulate_mts", capi.MB_INTEG_MTS),
    MTSLangevinIntegrator: (capi.MBMTSParams, "mb_simulate_mts", capi.MB_INTEG_MTS),
    Verlet: (capi.MBVVParams, "mb_simulate_verlet", capi.MB_INTEG_VERLET),
    StormerVerlet: (capi.MBStormerParams, "mb_simulate_stormer_verlet", capi.MB_INTEG_STORMER_VERLET),
    OverdampedLangevin: (capi.MBLangevinParams, "mb_simulate_overdamped_langevin", capi.MB_INTEG_OVERDAMPED_LANGEVIN),
    DPDVelocityVerlet: (capi.MBDpdVVParams, "mb_simulate_dpd_vv", capi.MB_INTEG_DPD_VV),
}


class _Call:
    """One simulate call of `sim` on `sys`: the entry point, its parameter struct, the velocity coupling and MTS levels to
    set on the context first, and the log plan (None: no loggers) for the loggers and arrays of `log_sys` (default sys)."""

    def __init__(self, sys, sim, n_steps: int, init_step: int, rng, run_loggers, log_sys=None):
        entry = next((e for t, e in _SIMULATE_ENTRY.items() if isinstance(sim, t)), None)
        if entry is None:
            raise TypeError(f"unsupported simulator {type(sim).__name__}")
        params_t, self.entry, self.kind = entry
        coupling = getattr(sim, "coupling", None)  # (LangevinSplitting, StormerVerlet, OverdampedLangevin have none)
        couplings = coupling if isinstance(coupling, (tuple, list)) else ((coupling,) if coupling else ())
        mts = params_t is capi.MBMTSParams
        p = params_t()  # (zero-filled: no Andersen thermostat, no noise)
        vc = None
        if isinstance(sim, VelocityVerlet):
            for c in couplings:
                if isinstance(c, _SCALING_THERMOSTATS) and len(couplings) == 1:  # (one thermostat per run)
                    vc = c.descriptor(sys.k)
                elif isinstance(c, AndersenThermostat):
                    p.andersen_kT = sys.k * c.temperature
                    p.andersen_prob = sim.dt / c.coupling_const
                else:
                    raise TypeError(f"unsupported coupling {c!r} (the stock Molly path handles it)")
        elif isinstance(sim, Verlet):
            for c in couplings:
                if not (isinstance(c, AndersenThermostat) and len(couplings) == 1):
                    raise TypeError(f"unsupported coupling {c!r} with Verlet (the stock Molly path handles it)")
                p.andersen_kT = sys.k * c.temperature
                p.andersen_prob = sim.dt / c.coupling_const
        elif couplings:
            raise TypeError(f"unsupported coupling {couplings[0]!r} with {type(sim).__name__} (the stock Molly path handles it)")
        self.levels = {}
        if mts:
            self.levels = mts_levels(sys, sim)
            p.n_levels = len(sim.ordered_fractions)
            p.fractions[:p.n_levels] = sim.ordered_fractions
            p.langevin = int(isinstance(sim, MTSLangevinIntegrator))
        if isinstance(sim, (Langevin, NoseHoover, MTSLangevinIntegrator, LangevinSplitting, OverdampedLangevin)):
            p.kT = sys.k * sim.temperature
        if isinstance(sim, (Langevin, MTSLangevinIntegrator, LangevinSplitting, OverdampedLangevin)):
            p.friction = float(sim.friction)
        if isinstance(sim, LangevinSplitting):
            p.n_ops = len(sim.splitting)
            p.ops = sim.splitting.encode()
        if isinstance(sim, NoseHoover):
            p.damping = float(sim.damping)
        if isinstance(sim, DPDVelocityVerlet):
            p.lambda_ = float(sim.lam)
        p.dt = float(sim.dt)
        p.n_steps = int(n_steps)
        p.init_step = int(init_step)
        if not isinstance(sim, StormerVerlet):  # (StormerVerlet never removes it)
            p.remove_cm_every = int(sim.remove_CM_motion)
        if not isinstance(sim, (NoseHoover, StormerVerlet, DPDVelocityVerlet)):  # (these draw nothing of their own)
            rng = rng or np.random.default_rng()
            p.rng_ctr1 = int(rng.integers(0, 2 ** 63))
            p.rng_key = int(rng.integers(0, 2 ** 63))
        self.p, self.vc = p, vc
        log_sys = log_sys or sys
        self.plan = (_LogPlan(log_sys, int(n_steps), int(init_step), run_loggers)
                     if log_sys.loggers and run_loggers is not False else None)

    def configure(self, sys):
        """Set the call's velocity coupling (cleared when it has none) and MTS levels on sys's context."""
        ctx = sys.engine()
        capi.check(sys._L.mb_set_velocity_coupling(ctx, C.byref(self.vc) if self.vc is not None else None))
        for kind, lv in self.levels.items():  # (an unchanged level array leaves the context as it is)
            capi.check(sys._L.mb_set_specific_levels(ctx, kind, len(lv), lv.ctypes.data))

    def log_arg(self):
        return C.byref(self.plan.desc) if self.plan is not None else None

    def run(self, sys, max_retries: int, rc=None, backup=None):
        """Run the call on sys.coords / sys.velocities. rc: the status an attempt made elsewhere (mb_simulate_group) already
        returned, and backup the host state from before it. After MB_ERR_CAPACITY a host state is restored and the call
        repeated with doubled capacities; the records go to the loggers only after success."""
        if rc is None:
            host = not hasattr(sys.coords, "data_ptr")
            backup = (sys.coords.copy(), sys.velocities.copy()) if host else None
        scale = 1.0
        for attempt in range(max_retries + 1):  # (a retry overwrites the records of the failed attempt)
            if rc is None:
                rc = getattr(sys._L, self.entry)(sys.engine(), _ptr(sys.coords), _ptr(sys.velocities), C.byref(self.p),
                                                 self.log_arg())
            if rc == capi.MB_ERR_CAPACITY and backup is not None and attempt < max_retries:
                sys.coords[...], sys.velocities[...] = backup
                scale *= 2.0
                capi.check(sys._L.mb_set_capacity_scale(sys.engine(), scale))
                rc = None
                continue
            capi.check(rc)
            break
        if self.plan is not None:
            self.plan.push()


def simulate(sys, sim, n_steps: Optional[int] = None, init_step: Optional[int] = None, rng=None, max_retries: int = 2,
             run_loggers=None, assign_velocities: bool = False):
    """simulate!(sys, sim, ...) dispatched on the simulator's type.

    VelocityVerlet: simulate!(sys, sim, n_steps; run_loggers=true) — src/simulators.jl:547-668. Mutates sys.coords /
    velocities and appends to the histories of sys.loggers (recorded on the device, see _LogPlan).
    Langevin: simulate!(sys, sim, n_steps; run_loggers=true) — src/simulators.jl:1101-1210, the same arguments and loggers
    as VelocityVerlet; the velocities are half a step behind the positions.
    LangevinSplitting: simulate!(sys, sim, n_steps; run_loggers=true) — src/simulators.jl:1252-1398, the same arguments and
    loggers as VelocityVerlet.
    NoseHoover: simulate!(sys, sim, n_steps; run_loggers=true) — src/simulators.jl:1534-1614, the same arguments and loggers
    as VelocityVerlet; zeta starts at 0 in every call.
    MTSIntegrator, MTSLangevinIntegrator: simulate!(sys, sim, n_steps; run_loggers=true) — src/simulators.jl:1783-1940,
    n_steps outer steps; the same arguments and loggers (once per outer step) as VelocityVerlet. The level of every specific
    term is set on the context (mb_set_specific_levels) before the call.
    Verlet, StormerVerlet, OverdampedLangevin: simulate!(sys, sim, n_steps; run_loggers=true) — src/simulators.jl:868-955,
    :970-1063, :1427-1490, the same arguments and loggers as VelocityVerlet. Verlet's velocities are half a step behind the
    positions; StormerVerlet's first step of every call starts from the velocities.
    DPDVelocityVerlet: simulate!(sys, sim, n_steps; run_loggers=true) — src/simulators.jl:711-842, the same arguments and
    loggers as VelocityVerlet; each call's first force evaluation uses the current velocities.
    SteepestDescentMinimizer: simulate!(sys, sim; run_loggers=false) — src/simulators.jl:183-274, see steepest_descent.
    Loggers are not run during a minimisation (run_loggers must be false).
    ReplicaExchangeMD on a ReplicaSystem: see simulate_remd (init_step defaults to sys.current_step there, and to 0 for
    a System)."""
    if isinstance(sim, ReplicaExchangeMD):
        if not isinstance(sys, ReplicaSystem):
            raise TypeError("simulate(sys, ::ReplicaExchangeMD, n_steps) needs a ReplicaSystem")
        if n_steps is None:
            raise TypeError("simulate(sys, ::ReplicaExchangeMD, n_steps) needs n_steps")
        return simulate_remd(sys, sim, n_steps, init_step=init_step, assign_velocities=assign_velocities,
                             run_loggers=True if run_loggers is None else run_loggers, rng=rng, max_retries=max_retries)
    if isinstance(sys, ReplicaSystem):
        raise TypeError(f"a ReplicaSystem runs with ReplicaExchangeMD, not {type(sim).__name__}")
    if assign_velocities:
        raise TypeError("assign_velocities is an argument of simulate(::ReplicaSystem, ::ReplicaExchangeMD, ...) only")
    init_step = 0 if init_step is None else init_step
    if isinstance(sim, SteepestDescentMinimizer):
        if n_steps is not None:
            raise TypeError("simulate(sys, ::SteepestDescentMinimizer) takes no n_steps (the minimiser's max_steps bounds it)")
        if run_loggers is not None and run_loggers is not False:
            raise NotImplementedError("loggers are not run during a minimisation on the device (run_loggers must be false)")
        steepest_descent(sys, sim, init_step=init_step, max_retries=max_retries)
        return sys
    if not any(isinstance(sim, t) for t in _SIMULATE_ENTRY):
        raise TypeError(f"unsupported simulator {type(sim).__name__}")
    if n_steps is None:
        raise TypeError(f"simulate(sys, ::{type(sim).__name__}, n_steps) needs n_steps")
    if run_loggers is None:
        run_loggers = True
    _check_run_loggers(run_loggers)
    call = _Call(sys, sim, int(n_steps), int(init_step), rng, run_loggers)
    call.configure(sys)  # (Langevin, NoseHoover: the coupling is cleared)
    call.run(sys, max_retries)
    return sys


# ------------------------------------------------------------------------------------------------
# temperature replica exchange (src/types.jl:1183-1427, src/simulators.jl:1942-2206, src/loggers.jl:1170-1218)
# ------------------------------------------------------------------------------------------------
class ThermoState:
    """ThermoState(system, integrator; temperature) — src/types.jl:1211-1280: one thermodynamic state, beta = 1 / (k T)
    with k = system.k. Without `temperature` it is the thermostat coupling's temperature, or else the integrator's.
    Pressure (a barostat's state) is not provided."""

    def __init__(self, system, integrator, temperature=None, pressure=None, name=None):
        if pressure is not None:
            raise TypeError("ThermoState pressure (constant-pressure replica exchange) is not provided; the stock Molly "
                            "path handles it")
        coupling = getattr(integrator, "coupling", None)
        for c in coupling if isinstance(coupling, (tuple, list)) else ((coupling,) if coupling else ()):
            if temperature is None and hasattr(c, "temperature"):
                temperature = c.temperature
        if temperature is None:
            temperature = getattr(integrator, "temperature", None)
        if temperature is None:
            raise ValueError("no temperature provided or inferred from the integrator: give one explicitly, use a "
                             "thermostat, or use an integrator with a temperature")
        self.system, self.integrator, self.name = system, integrator, name
        self.temperature = float(temperature)
        self.beta = 1.0 / (system.k * self.temperature)


class ReplicaExchangeLogger:
    """ReplicaExchangeLogger(n_replicas) — src/loggers.jl:1170-1218: the accepted exchanges (the pair of physical
    replica indices, 0-based, the step and Delta of each) and the number of attempts."""

    def __init__(self, n_replicas: int):
        self.n_replicas = int(n_replicas)
        self.n_attempts = self.n_exchanges = self.end_step = 0
        self.indices, self.steps, self.deltas = [], [], []


class ReplicaExchangeMD:
    """ReplicaExchangeMD(dt, exchange_time) — src/simulators.jl:1953-1963."""

    def __init__(self, dt, exchange_time):
        if not exchange_time > dt:
            raise ValueError(f"exchange time ({exchange_time}) must be greater than the time step ({dt})")
        self.dt, self.exchange_time = float(dt), float(exchange_time)


class ReplicaSystem:
    """ReplicaSystem(thermo_states, replica_coords; replica_velocities, replica_loggers, exchange_logger, initial_step) —
    src/types.jl:1343-1427, for states that share one System (temperature replica exchange). Holds the coordinates and
    velocities of every physical replica (numpy, or torch CUDA tensors), state_indices (physical replica -> state, 0-based,
    starting at the identity), current_step and the exchange logger. replica_loggers[i] is a dict of loggers like
    System.loggers. Each state runs on a private engine context of its own, so its captured step graphs survive every
    exchange."""

    def __init__(self, thermo_states, replica_coords, replica_velocities=None, replica_boundaries=None,
                 replica_neighbor_finders=None, replica_loggers=None, exchange_logger=None, initial_step: int = 0):
        self.thermo_states = list(thermo_states)
        n = self.n_replicas = len(self.thermo_states)
        if n < 1:
            raise ValueError("a ReplicaSystem needs at least one ThermoState")
        if int(initial_step) < 0:
            raise ValueError("initial_step must be non-negative")
        base = self.thermo_states[0].system
        if any(ts.system is not base for ts in self.thermo_states):
            raise TypeError("ThermoStates on different Systems (Hamiltonian replica exchange) are not provided: every "
                            "state must share one System; the stock Molly path handles it")
        if replica_boundaries is not None or replica_neighbor_finders is not None:
            raise TypeError("per-replica boundaries or neighbour finders are not provided; the stock Molly path handles them")
        for ts in self.thermo_states:
            if not any(isinstance(ts.integrator, t) for t in _SIMULATE_ENTRY):
                raise TypeError(f"unsupported integrator {type(ts.integrator).__name__} for replica exchange; the stock Molly "
                                "path handles it")
        for name, arg in (("replica_coords", replica_coords), ("replica_velocities", replica_velocities),
                          ("replica_loggers", replica_loggers)):
            if arg is not None and len(arg) != n:
                raise ValueError(f"{len(arg)} {name} for {n} ThermoStates")
        self.system = base
        self.k, self.n, self.dtype = base.k, base.n, base.dtype
        self.replica_coords = [base._as_state(x) for x in replica_coords]
        if replica_velocities is None:
            replica_velocities = [x.clone().zero_() if hasattr(x, "data_ptr") else np.zeros_like(x) for x in self.replica_coords]
        self.replica_velocities = [base._as_state(v) for v in replica_velocities]
        self.replica_loggers = [dict(lg or {}) for lg in (replica_loggers or [None] * n)]
        for lgs in self.replica_loggers:
            for name, lg in lgs.items():
                if type(lg) not in _LOGGER_TYPES:
                    raise TypeError(f"logger {name!r}: {type(lg).__name__} is not supported")
        self.exchange_logger = exchange_logger if exchange_logger is not None else ReplicaExchangeLogger(n)
        self.state_indices = list(range(n))
        self.betas = [ts.beta for ts in self.thermo_states]
        self.current_step = int(initial_step)
        self.initial_log_pending = True
        self._state_sys = [None] * n

    def state_system(self, s: int) -> System:
        """The private System of state s: the shared System's Hamiltonian on a context of its own, no loggers."""
        if self._state_sys[s] is None:
            import copy
            st = copy.copy(self.system)
            st._ctx, st.loggers = None, {}
            self._state_sys[s] = st
        return self._state_sys[s]

    def close(self):
        for st in self._state_sys:
            if st is not None:
                st.close()


class _ReplicaView:
    """What _LogPlan reads of a System, for one physical replica's arrays and loggers."""

    def __init__(self, repsys, i):
        self.loggers, self.coords = repsys.replica_loggers[i], repsys.replica_coords[i]
        self.n, self.dtype, self.k = repsys.n, repsys.dtype, repsys.k


class _EngineRunner:
    """Runs a cycle's calls (one per state that holds a replica) as one mb_simulate_group call, and evaluates U on a
    state's context. The seam tests substitute to drive simulate_remd with other integrators."""

    def run(self, repsys, calls, max_retries):
        """calls: [(state, _Call)], the state's System holding its replica's arrays. Members that hit MB_ERR_CAPACITY
        are retried one at a time through the single call."""
        L = capi.load()
        members = (capi.MBGroupMember * len(calls))()
        backups = []
        for m, (s, call) in zip(members, calls):
            st = repsys.state_system(s)
            call.configure(st)
            m.ctx, m.coords, m.vels, m.kind = st.engine(), _ptr(st.coords), _ptr(st.velocities), call.kind
            m.params = C.addressof(call.p)
            m.log = C.addressof(call.plan.desc) if call.plan is not None else None
            host = not hasattr(st.coords, "data_ptr")
            backups.append((st.coords.copy(), st.velocities.copy()) if host else None)
        rc = L.mb_simulate_group(len(calls), members)
        if rc == capi.MB_ERR_INVALID and all(m.status == capi.MB_ERR_INVALID for m in members):
            capi.check(rc)  # (refused before any work)
        for m, (s, call), backup in zip(members, calls, backups):
            call.run(repsys.state_system(s), max_retries, rc=m.status, backup=backup)

    def energy(self, repsys, s, coords):
        st = repsys.state_system(s)
        st.coords = coords
        return potential_energy(st)


def _scale_velocities(v, factor, dtype):
    """v *= factor in place, the factor (computed in f64) cast to the state dtype first."""
    if hasattr(v, "data_ptr"):
        v.mul_(float(np.asarray(factor, dtype)))
    else:
        v *= np.asarray(factor, dtype)


def simulate_remd(repsys: ReplicaSystem, sim: ReplicaExchangeMD, n_steps: int, init_step: Optional[int] = None,
                  assign_velocities: bool = False, run_loggers=True, rng=None, max_retries: int = 2, runner=None):
    """simulate!(repsys, ::ReplicaExchangeMD, n_steps; init_step=repsys.current_step, assign_velocities, run_loggers, rng) —
    src/simulators.jl:1965-2206 for temperature replica exchange.

    n_cycles = (n_steps dt) // exchange_time and cycle_length = n_steps // n_cycles; the remaining n_steps % n_cycles
    steps run after the last cycle, with no exchange after them. In cycle c (1-based) physical replica i runs cycle_length
    steps of the integrator of state state_indices[i] from step init_step + (c - 1) cycle_length, on that state's context;
    the states' calls run together (mb_simulate_group). Loggers run with run_loggers = True while
    repsys.initial_log_pending is set and with "skipstart" after that. Then exchanges are attempted between adjacent
    physical replicas (i, i + 1), i = 1, 3, ... (0-based) in odd cycles and i = 0, 2, ... in even ones:
    Delta = (beta_n - beta_m)(U(x_i) - U(x_j)), m and n the states of i and j and U the potential energy of the replica's
    final coordinates, accepted when Delta <= 0 or rng.random() < exp(-Delta). On acceptance the states swap and the
    velocities scale, v_i *= sqrt(beta_m / beta_n), v_j *= sqrt(beta_n / beta_m) (the factor computed in f64 and cast to
    the system dtype); the exchange logger records (i, j), the step init_step + c cycle_length and Delta.

    The draws from `rng`, in order: with assign_velocities, random_velocities of each replica at its state's temperature,
    in physical order; then per cycle (and for the remainder) the integrator keys of each replica in physical order (the
    two rng.integers draws simulate makes, for integrators that draw), and that cycle's exchange uniforms, one per
    attempt with Delta > 0, in pair order."""
    if not isinstance(repsys, ReplicaSystem):
        raise TypeError("simulate_remd needs a ReplicaSystem")
    _check_run_loggers(run_loggers)
    rng = rng or np.random.default_rng()
    runner = runner or _EngineRunner()
    init_step = repsys.current_step if init_step is None else int(init_step)
    n_steps = int(n_steps)
    R = repsys.n_replicas
    repsys.current_step = init_step
    n_cycles = int((n_steps * sim.dt) // sim.exchange_time)
    cycle_length = n_steps // n_cycles if n_cycles > 0 else 0
    remaining = n_steps % n_cycles if n_cycles > 0 else n_steps
    if assign_velocities:
        for i in range(R):
            s = repsys.state_indices[i]
            v = random_velocities(repsys.state_system(s), repsys.thermo_states[s].temperature, rng)
            if hasattr(repsys.replica_velocities[i], "data_ptr"):
                import torch
                repsys.replica_velocities[i].copy_(torch.from_numpy(v))
            else:
                repsys.replica_velocities[i][...] = v

    def run_cycle(length, start):
        rl = False if run_loggers is False else (True if repsys.initial_log_pending else "skipstart")
        calls = []
        for i in range(R):
            s = repsys.state_indices[i]
            st = repsys.state_system(s)
            st.coords, st.velocities = repsys.replica_coords[i], repsys.replica_velocities[i]
            calls.append((s, _Call(st, repsys.thermo_states[s].integrator, length, start, rng, rl, _ReplicaView(repsys, i))))
        runner.run(repsys, calls, max_retries)
        repsys.initial_log_pending = False

    n_attempts = 0
    xl = repsys.exchange_logger
    for cycle in range(1, n_cycles + 1):
        run_cycle(cycle_length, init_step + (cycle - 1) * cycle_length)
        for i in range(cycle % 2, R - 1, 2):
            j = i + 1
            n_attempts += 1
            m, n = repsys.state_indices[i], repsys.state_indices[j]
            bm, bn = repsys.betas[m], repsys.betas[n]
            ui = runner.energy(repsys, m, repsys.replica_coords[i])
            uj = runner.energy(repsys, n, repsys.replica_coords[j])
            delta = (bn - bm) * (float(ui) - float(uj))
            if delta <= 0 or rng.random() < math.exp(-delta):
                repsys.state_indices[i], repsys.state_indices[j] = n, m
                if bm != bn:
                    _scale_velocities(repsys.replica_velocities[i], math.sqrt(bm / bn), repsys.dtype)
                    _scale_velocities(repsys.replica_velocities[j], math.sqrt(bn / bm), repsys.dtype)
                if run_loggers is not False and xl is not None:
                    xl.indices.append((i, j))
                    xl.steps.append(init_step + cycle * cycle_length)
                    xl.deltas.append(delta)
                    xl.n_exchanges += 1
    if remaining > 0:
        run_cycle(remaining, init_step + n_cycles * cycle_length)
    if run_loggers is not False and xl is not None:
        xl.end_step = init_step + n_steps
        xl.n_attempts += n_attempts
    repsys.current_step = init_step + n_steps
    return repsys


def kinetic_energy(sys: System) -> float:
    out = C.c_double(0.0)
    ctx = sys.engine()
    capi.check(sys._L.mb_kinetic_energy(ctx, _ptr(sys.velocities), C.byref(out)))
    return out.value


def temperature(sys: System) -> float:
    """src/energy.jl:158-175 with df = 3N - 3 for a periodic 3-D box."""
    df = 3 * sys.n - 3
    return 2.0 * kinetic_energy(sys) / (df * sys.k)


def remove_CM_motion(sys: System):
    ctx = sys.engine()
    capi.check(sys._L.mb_remove_cm_motion(ctx, _ptr(sys.velocities)))
    return sys


def random_velocities(sys: System, temp: float, rng=None) -> np.ndarray:
    """random_velocities(sys, temp; rng) — src/spatial.jl:803-831: Maxwell-Boltzmann velocities drawn on the device
    (Philox4x32-10 keyed by two 64-bit draws of `rng`, like the reference's GPU kernel src/kernels.jl:688-703)."""
    rng = rng or np.random.default_rng()
    ctx = sys.engine()
    out = np.zeros((sys.n, 3), sys.dtype)
    capi.check(sys._L.mb_random_velocities(ctx, out.ctypes.data, float(sys.k * temp), int(rng.integers(0, 2 ** 63)),
                                           int(rng.integers(0, 2 ** 63))))
    return out


def random_velocities_(sys: System, temp: float, rng=None) -> System:
    """random_velocities!(sys, temp): in place."""
    v = random_velocities(sys, temp, rng)
    if hasattr(sys.velocities, "data_ptr"):
        import torch
        sys.velocities.copy_(torch.from_numpy(v))
    else:
        sys.velocities[...] = v
    return sys


def kinetic_energy_tensor(sys: System) -> np.ndarray:
    """K = 1/2 sum m v (x) v — src/energy.jl:56-70 (3x3, kJ/mol)."""
    out = (C.c_double * 9)()
    ctx = sys.engine()
    capi.check(sys._L.mb_kinetic_energy_tensor(ctx, _ptr(sys.velocities), out))
    return np.array(out[:], np.float64).reshape(3, 3)


def wrap_coords(coords, boundary: CubicBoundary):
    """wrap_coords — src/spatial.jl:573-586 (host helper for test set-up)."""
    L = boundary.side_lengths.astype(coords.dtype)
    return coords - np.floor(coords / L) * L


def comm_unique_id() -> bytes:
    """ncclUniqueId (128 bytes) created on the calling rank; broadcast it to the other ranks with the host runtime."""
    buf = C.create_string_buffer(128)
    capi.check(capi.load().mb_comm_unique_id(buf))
    return buf.raw


def comm_init(sys: System, unique_id: bytes, rank: int, nranks: int):
    """Join the spatial decomposition: z-slabs of cell layers, NCCL halo exchange (see include/mollyb200.h)."""
    ctx = sys.engine()
    capi.check(sys._L.mb_comm_init(ctx, C.c_char_p(unique_id), int(rank), int(nranks)))


def decomp_plan(ncz: int, halo_layers: int, nranks: int, rank: int, layer_start):
    """Host-side halo-exchange plan: (send, recv) lists of (peer, first slot, slot count)."""
    ls = np.ascontiguousarray(layer_start, np.int32)
    cap = 4 * nranks + 8
    snd = np.zeros((cap, 3), np.int32)
    rcv = np.zeros((cap, 3), np.int32)
    ns, nr = C.c_int32(0), C.c_int32(0)
    capi.check(capi.load().mb_decomp_plan(ncz, halo_layers, nranks, rank, ls.ctypes.data, snd.ctypes.data, C.byref(ns),
                                          rcv.ctypes.data, C.byref(nr), cap))
    return snd[:ns.value].tolist(), rcv[:nr.value].tolist()


def device_count() -> int:
    return int(capi.load().mb_device_count())
