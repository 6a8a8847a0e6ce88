"""mollyb200 — H100-native engine for Molly.jl's pairwise non-bonded + VelocityVerlet hot path.

The directory is named after the reference (`molly.jl_b200`); import it through the top-level
`mollyb200` module. Only what the path needs lives here: csrc/ (CUDA kernels + the C ABI), the ctypes
binding and the host-side mirror of the reference interface.
"""
from . import _capi  # noqa: F401
from .api import *  # noqa: F401,F403
from .api import (Atom, CubicBoundary, TriclinicBoundary, System, NoCutoff, DistanceCutoff, ShiftedPotentialCutoff,  # noqa: F401
                  ShiftedForceCutoff, LennardJones, Coulomb, CoulombReactionField, CoulombEwald, GPUNeighborFinder,
                  DistanceNeighborFinder, CellListMapNeighborFinder, TreeNeighborFinder, AndersenThermostat,
                  ImmediateThermostat, BerendsenThermostat, VelocityRescaleThermostat,
                  VelocityVerlet, Langevin, LangevinSplitting, NoseHoover, Verlet, StormerVerlet, OverdampedLangevin, DPDInteraction, DPDVelocityVerlet, MTSIntegrator, MTSLangevinIntegrator, setup_mts_integrator,
                  mts_levels, forces, forces_virial, potential_energy, forces_energy, find_neighbors, simulate,
                  kinetic_energy, temperature, remove_CM_motion, random_velocities, wrap_coords, device_count,
                  atoms_from_arrays, atoms_to_array, atom_dtype, MollyB200Error, COULOMB_CONST, BOLTZMANN_K,
                  comm_unique_id, comm_init, decomp_plan, InteractionList2Atoms, InteractionList3Atoms,
                  InteractionList4Atoms, PotentialEnergyLogger, KineticEnergyLogger, TotalEnergyLogger, TemperatureLogger,
                  CoordinatesLogger, VelocitiesLogger, values, record_steps, SteepestDescentMinimizer, steepest_descent,
                  sd_log_lines, ImplicitSolventOBC, ImplicitSolventGBN2, InteractionList1Atoms, MorseBonds, FENEBonds,
                  CosineAngles, UreyBradleys, HarmonicTorsions, RBTorsions, add_position_restraints, ThermoState,
                  ReplicaSystem, ReplicaExchangeMD, ReplicaExchangeLogger, simulate_remd)
