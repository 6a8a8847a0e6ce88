"""Specific interaction lists (bonds, angles, torsions) in a TriclinicBoundary box. Bonded displacements use
TriclinicBoundary's vector (src/spatial.jl:528-534). Such systems run on the no-list kernel, so they are served where that
kernel is the intended path (box heights below 2.5 r_list, or no neighbour list); larger ones are refused until the
cell-list path handles triclinic boxes."""
import numpy as np
import pytest

import mbhelpers as H
import mollyb200 as mb

pytestmark = pytest.mark.gpu


def _chain_lists(n_mol):
    """Bonds, angles and a torsion along every 4-site molecule of H.molecular_system (1-based indices)."""
    i = np.arange(0, 4 * n_mol, 4) + 1
    one = np.ones(n_mol)
    return (mb.InteractionList2Atoms(np.r_[i, i + 1, i + 2], np.r_[i + 1, i + 2, i + 3], np.full(3 * n_mol, 2e5), np.full(3 * n_mol, 0.11)),
            mb.InteractionList3Atoms(np.r_[i, i + 1], np.r_[i + 1, i + 2], np.r_[i + 2, i + 3], np.full(2 * n_mol, 400.0), np.full(2 * n_mol, 1.9)),
            mb.InteractionList4Atoms(i, i + 1, i + 2, i + 3, 3 * one, 0.3 * one, 5 * one))


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_bonded_sheared_box_equals_rectangular(dtype):
    """LJ + CRF with exclusions and 1-4 specials plus bonds/angles/torsions, in a small rectangular box and in the sheared
    box a = (L,0,0), b = (L,L,0), c = (-L,0,L) that describes the same periodic system: same forces and energy."""
    L, n_mol = 2.4, 100
    sd = H.molecular_system(n_mol, [L, L, L], seed=3)
    lists = _chain_lists(n_mol)
    inters = (mb.LennardJones(cutoff=mb.DistanceCutoff(1.0), use_neighbors=True, weight_special=0.5),
              mb.CoulombReactionField(dist_cutoff=1.0, use_neighbors=True, weight_special=0.8333))

    def fe(boundary, coords):
        atoms = mb.atoms_from_arrays(sd["mass"], sd["charge"], sd["sigma"], sd["eps"], dtype)
        nf = mb.GPUNeighborFinder(dist_cutoff=1.2, excluded_pairs=sd["excluded"] + 1, special_pairs=sd["special"] + 1)
        s = mb.System(atoms=atoms, coords=coords.astype(dtype), boundary=boundary, pairwise_inters=inters, neighbor_finder=nf,
                      dtype=dtype, specific_inter_lists=lists)
        try:
            f, e = mb.forces_energy(s)
            return f.astype(np.float64), e, s.stats()["path"]
        finally:
            s.close()

    bv = np.array([[L, 0, 0], [L, L, 0], [-L, 0, L]])
    x = sd["coords"].astype(np.float64)
    f_ref, e_ref, _ = fe(mb.CubicBoundary(L, L, L), x)
    # every atom moved to another image of the sheared lattice: bonded partners now sit in different images
    x_far = x + np.random.default_rng(4).integers(-1, 2, (len(x), 3)) @ bv
    f, e, path = fe(mb.TriclinicBoundary(*bv), x_far)
    fmax = np.abs(f_ref).max()
    tol = 1e-9 if dtype == np.float64 else 5e-5
    print(f"[sheared vs rectangular {np.dtype(dtype).name}] path={path} max|dF|={np.abs(f - f_ref).max():.3e} "
          f"(max|F| {fmax:.3e}) dE={e - e_ref:.3e}")
    assert path == 0
    assert np.abs(f - f_ref).max() <= tol * fmax + (1e-9 if dtype == np.float64 else 2e-3)
    assert abs(e - e_ref) <= (1e-11 if dtype == np.float64 else 2e-6) * max(abs(e_ref), 1.0) * 10


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_bonds_across_a_triclinic_face(dtype):
    """Bonded partners in different images of a strongly sheared box (the partner's nearest image is a sum of basis
    vectors), no neighbour list: bond, angle and torsion forces and energy equal those of the molecules placed together."""
    bv = np.array([[4.0, 0, 0], [2.0, 4.0, 0], [-2.0, 1.5, 4.0]])
    rng = np.random.default_rng(2)
    n_mol = 40
    start = rng.random((n_mol, 3)) @ bv
    steps = np.array([[0.0, 0, 0], [0.15, 0, 0], [0.2, 0.12, 0], [0.3, 0.15, 0.1]])
    x_in = (start[:, None, :] + steps[None] @ np.linalg.qr(rng.normal(size=(3, 3)))[0]).reshape(-1, 3)
    x_far = x_in + rng.integers(-1, 2, (len(x_in), 3)) @ bv  # every atom moved to another image
    n = len(x_in)
    i = np.arange(0, n, 4) + 1
    lists = (mb.InteractionList2Atoms(i, i + 1, np.full(n_mol, 2e5), np.full(n_mol, 0.14)),
             mb.InteractionList3Atoms(i, i + 1, i + 2, np.full(n_mol, 400.0), np.full(n_mol, 1.9)),
             mb.InteractionList4Atoms(i, i + 1, i + 2, i + 3, np.full(n_mol, 3.0), np.full(n_mol, 0.3), np.full(n_mol, 5.0)))
    atoms = mb.atoms_from_arrays(np.full(n, 12.0), np.zeros(n), np.zeros(n), np.zeros(n), dtype)

    def fe(x):
        s = mb.System(atoms=atoms, coords=x.astype(dtype), boundary=mb.TriclinicBoundary(*bv), dtype=dtype, specific_inter_lists=lists,
                      pairwise_inters=(mb.LennardJones(cutoff=mb.DistanceCutoff(1.0), use_neighbors=False),))
        try:
            return mb.forces_energy(s)
        finally:
            s.close()

    f_ref, e_ref = fe(x_in)
    f, e = fe(x_far)
    tol = 1e-9 if dtype == np.float64 else 2e-3
    print(f"[bonds across faces {np.dtype(dtype).name}] max|dF|={np.abs(f - f_ref).max():.3e} (max|F| {np.abs(f_ref).max():.3e}) dE={e - e_ref:.3e}")
    assert np.abs(f_ref).max() > 1.0
    assert np.abs(f - f_ref).max() <= tol * np.abs(f_ref).max()
    assert abs(e - e_ref) <= tol * abs(e_ref)


def _refused(g, bv, general_inters=(), pairwise=None):
    sd = H.sixmrr_description(g)
    atoms = mb.atoms_from_arrays(sd["mass"], sd["charge"], sd["sigma"], sd["eps"], np.float64)
    nf = mb.GPUNeighborFinder(dist_cutoff=1.2, excluded_pairs=g["excluded"] + 1, special_pairs=g["special"] + 1)
    pairwise = pairwise or (mb.LennardJones(cutoff=mb.DistanceCutoff(1.0), use_neighbors=True, weight_special=0.5),)
    s = mb.System(atoms=atoms, coords=sd["coords"].copy(), boundary=mb.TriclinicBoundary(*bv), neighbor_finder=nf, dtype=np.float64,
                  pairwise_inters=pairwise, general_inters=general_inters, specific_inter_lists=H.sixmrr_specific_lists(g))
    try:
        mb.forces(s)
    finally:
        s.close()


def test_triclinic_refusals(golden_6mrr):
    """6mrr (heights >= 2.5 r_list) with bonded lists in a sheared box would run on the O(N^2) no-list kernel: refused. PME keeps
    an orthorhombic reciprocal grid: refused for a TriclinicBoundary system."""
    g = golden_6mrr
    L = g["box"]
    with pytest.raises(Exception, match="cell-list path"):
        _refused(g, np.array([[L[0], 0, 0], [L[0], L[1], 0], [-L[0], 0, L[2]]]))
    with pytest.raises(Exception, match="PME"):
        _refused(g, np.diag(L), general_inters=(mb.PME(1.0),), pairwise=(mb.CoulombEwald(dist_cutoff=1.0, use_neighbors=True),))
