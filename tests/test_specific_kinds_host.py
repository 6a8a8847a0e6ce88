"""CPU tests of the specific interaction kinds 3-9 (HarmonicPositionRestraint, MorseBond, FENEBond, CosineAngle,
UreyBradley, HarmonicTorsion, RBTorsion): the numpy restatement (tests/bonded_kinds_oracle.py) against the reference's
literal values (test/interactions.jl), its forces against -grad E by central differences, the RBTorsion sign, the Python
list classes, add_position_restraints and the multiple-time-step levels of mixed kinds. The GPU counterpart is
tests/test_gpu_specific_kinds.py."""
import numpy as np
import pytest

import bonded_kinds_oracle as bk
import mollyb200 as mb

KBT = 2.479
C1, C2, C3 = [1.0, 1.0, 1.0], [1.3, 1.0, 1.0], [1.4, 1.0, 1.0]
C3A = [1.0, 1.2, 1.2]
RB_X = [[0.0, 0.0, 0.0], [0.1, 0.0, 0.0], [0.2, 0.1, 0.0], [0.3, 0.1, 0.1]]
HT_X_ANGSTROM = [[27.151, 33.362, 10.650], [28.260, 33.943, 11.096], [28.605, 33.965, 12.503], [28.638, 35.461, 12.900]]

# (kind, coordinates (nm), box side, params, expected forces per atom or None, expected energy, force atol, energy atol):
# the literals of test/interactions.jl, each on its own geometry
LITERALS = {
    "restraint": (bk.POSITION_RESTRAINT, [C2], 2.0, [3e5] + C1, [[-90000.0, 0, 0]], 13500.0, 1e-9, 1e-9),
    "restraint_at_x0": (bk.POSITION_RESTRAINT, [C1], 2.0, [3e5] + C1, [[0.0, 0, 0]], 0.0, 1e-9, 1e-9),
    "morse_1": (bk.MORSE_BOND, [C1, C2], 2.0, [100.0, 10.0, 0.2], [[465.0883158697, 0, 0], [-465.0883158697, 0, 0]],
                39.9576400894, 1e-9, 1e-9),
    "morse_2": (bk.MORSE_BOND, [C1, C3], 2.0, [200.0, 5.0, 0.6], [[-9341.5485409432, 0, 0], [9341.5485409432, 0, 0]],
                590.4984884025, 1e-9, 1e-9),
    "fene_1": (bk.FENE_BOND, [[2.3, 0, 0], [1.0, 0, 0]], 20.0, [10.0 * KBT, 1.6, 1.0, KBT],
               [[-94.8288735632, 0, 0], [94.8288735632, 0, 0]], 34.2465108316, 1e-9, 1e-9),
    "fene_2": (bk.FENE_BOND, [[2.3, 0, 0], [1.0, 0, 0]], 20.0, [0.0, 1.6, 1.0, KBT], [[0.0, 0, 0], [0.0, 0, 0]], 0.0,
               1e-9, 1e-9),
    "cosine_collinear": (bk.COSINE_ANGLE, [[1.0, 0, 0], [2.0, 0, 0], [3.0, 0, 0]], 10.0, [10 * KBT, 0.0], [[0.0, 0, 0]] * 3,
                         0.0, 1e-9, 1e-9),
    "cosine_collinear_pi2": (bk.COSINE_ANGLE, [[1.0, 0, 0], [2.0, 0, 0], [3.0, 0, 0]], 10.0, [10 * KBT, np.pi / 2], None,
                             24.79, 1e-9, 1e-9),
    "cosine_right": (bk.COSINE_ANGLE, [[1.0, 0, 0], [2.0, 0, 0], [2.0, 1.0, 0]], 10.0, [10 * KBT, np.pi / 2],
                     [[0.0, 0, 0]] * 3, 49.58, 1e-9, 1e-9),
    "urey_bradley": (bk.UREY_BRADLEY, [C1, C2, C3A], 2.0, [300.0, 0.8, 10000.0, 0.3],
                     [[0.0, -152.4546720285, -152.4546720285], [-21.9771730369, 14.6514486912, 14.6514486912],
                      [21.9771730369, 137.8032233372, 137.8032233372]], 1.7626664989, 1e-9, 1e-9),
    # forces in kJ mol^-1 A^-1 in the reference: x 10 for nm; a box of infinite side there, a large finite one here
    "harmonic_torsion": (bk.HARMONIC_TORSION, list(np.array(HT_X_ANGSTROM) / 10), 1e3, [1000.0, -1.8],
                         list(10 * np.array([[-228.63867893470425, 398.16345029859656, 49.837063486781354],
                                             [242.87672193557964, -596.3836043695466, -50.228876881052855],
                                             [324.1211893467139, 212.83417983707614, -82.80324255936942],
                                             [-338.3592323475893, -14.614025766126122, 83.19505595364092]])),
                         67.60869243622506, None, None),
}
RB_NORMS = [497.6067743425172, 673.7627575276049, 351.86112450195805, 287.2934051172337]
RB_ENERGY = 47.38033871712585
RB_PARAMS = [10.0, 20.0, 30.0, 5.0]


def _eval(kind, x, side, par, **kw):
    x = np.asarray(x, np.float64)
    idx = np.arange(bk.ATOMS[kind] if kind != bk.POSITION_RESTRAINT else 1)[None, :]
    return bk.FORCES[kind](x, np.full(3, side), idx, np.asarray(par, np.float64)[None, :], **kw)


@pytest.mark.parametrize("name", sorted(LITERALS))
def test_oracle_reproduces_reference_literals(name):
    kind, x, side, par, f_exp, e_exp, fatol, eatol = LITERALS[name]
    f, e = _eval(kind, x, side, par)
    if f_exp is not None:
        if fatol is None:  # isapprox's default: rtol sqrt(eps) on the norm of the difference
            for a, b in zip(f, np.asarray(f_exp)):
                assert np.linalg.norm(a - b) <= np.sqrt(np.finfo(float).eps) * max(np.linalg.norm(a), np.linalg.norm(b))
        else:
            np.testing.assert_allclose(f, np.asarray(f_exp, np.float64), rtol=0, atol=fatol)
    if eatol is None:
        assert abs(e - e_exp) <= np.sqrt(np.finfo(float).eps) * abs(e_exp)
    else:
        assert abs(e - e_exp) <= eatol


def test_rb_torsion_literal_norms_and_energy():
    """The reference pins only the norms of the four forces and the energy: both signs reproduce them."""
    for sign in (False, True):
        f, e = _eval(bk.RB_TORSION, RB_X, 5.0, RB_PARAMS, reference_sign=sign)
        np.testing.assert_allclose(np.linalg.norm(f, axis=1), RB_NORMS, rtol=0, atol=1e-9)
        assert abs(e - RB_ENERGY) <= 1e-9


def _numeric_gradient(fn, x, h=1e-6):
    g = np.zeros_like(x)
    for a in range(x.shape[0]):
        for d in range(3):
            xp, xm = x.copy(), x.copy()
            xp[a, d] += h
            xm[a, d] -= h
            g[a, d] = (fn(xp)[1] - fn(xm)[1]) / (2 * h)
    return g


def _random_terms(kind, rng, n_terms=6):
    """Non-degenerate random geometries: atoms 0.1-0.2 nm apart along a random walk, parameters of the usual sizes."""
    na = bk.ATOMS[kind]
    x = []
    for _ in range(n_terms):
        p = [rng.uniform(0.5, 1.5, 3)]
        for _ in range(na - 1):
            d = rng.normal(size=3)
            p.append(p[-1] + rng.uniform(0.1, 0.2) * d / np.linalg.norm(d))
        x += p
    x = np.array(x)
    idx = np.arange(len(x)).reshape(n_terms, na)
    u = lambda lo, hi: rng.uniform(lo, hi, n_terms)
    par = {bk.POSITION_RESTRAINT: lambda: np.c_[u(1e3, 1e4), x + rng.normal(0, 0.05, x.shape)],
           bk.MORSE_BOND: lambda: np.c_[u(100, 400), u(5, 20), u(0.1, 0.2)],
           bk.FENE_BOND: lambda: np.c_[u(10, 40), u(0.25, 0.35), u(0.12, 0.16), u(1, 3)],
           bk.COSINE_ANGLE: lambda: np.c_[u(10, 50), u(0.5, 2.5)],
           bk.UREY_BRADLEY: lambda: np.c_[u(100, 400), u(1.5, 2.2), u(1e3, 1e4), u(0.2, 0.3)],
           bk.HARMONIC_TORSION: lambda: np.c_[u(10, 100), u(-2.5, 2.5)],
           bk.RB_TORSION: lambda: np.c_[u(-20, 20), u(-20, 20), u(-20, 20), u(-5, 5)]}[kind]()
    return x, idx, par


NEW_KINDS = [bk.POSITION_RESTRAINT, bk.MORSE_BOND, bk.FENE_BOND, bk.COSINE_ANGLE, bk.UREY_BRADLEY, bk.HARMONIC_TORSION,
             bk.RB_TORSION]


@pytest.mark.parametrize("kind", NEW_KINDS)
def test_oracle_force_is_minus_gradient(kind):
    rng = np.random.default_rng(100 + kind)
    box = np.full(3, 10.0)
    x, idx, par = _random_terms(kind, rng)
    fn = lambda y: bk.FORCES[kind](y, box, idx, par)
    f, _ = fn(x)
    g = _numeric_gradient(fn, x)
    assert np.abs(f).max() > 1.0
    assert np.abs(f + g).max() <= 1e-6 * np.abs(f).max()


def test_rb_torsion_reference_sign_is_plus_gradient():
    """rb_torsion.jl:30's dE/dtheta is minus the derivative of its own energy: its forces are +grad E."""
    rng = np.random.default_rng(7)
    box = np.full(3, 10.0)
    x, idx, par = _random_terms(bk.RB_TORSION, rng)
    fn = lambda y: bk.rb_torsion_forces(y, box, idx, par, reference_sign=True)
    f, _ = fn(x)
    g = _numeric_gradient(fn, x)
    assert np.abs(f - g).max() <= 1e-6 * np.abs(f).max()
    assert np.abs(f + g).max() > 0.5 * np.abs(f).max()
    # on the reference's own geometry: the reference sign is far from -grad E, the engine's is not
    x = np.array(RB_X)
    idx, par = np.arange(4)[None, :], np.array([RB_PARAMS])
    for sign, bad in ((True, True), (False, False)):
        fn = lambda y: bk.rb_torsion_forces(y, np.full(3, 5.0), idx, par, reference_sign=sign)
        err = np.abs(fn(x)[0] + _numeric_gradient(fn, x)).max()
        assert (err > 100) if bad else (err < 1e-5), err


def test_list_classes_arrays_and_kinds():
    cases = [
        (mb.InteractionList1Atoms([1, 3], [10.0, 20.0], [[0, 1, 2], [3, 4, 5]]), 3, (2, 1), (2, 4),
         [[10, 0, 1, 2], [20, 3, 4, 5]]),
        (mb.MorseBonds([1], [2], [1.0], [2.0], [3.0]), 4, (1, 2), (1, 3), [[1, 2, 3]]),
        (mb.FENEBonds([1], [2], [1.0], [2.0], [3.0], [4.0]), 5, (1, 2), (1, 4), [[1, 2, 3, 4]]),
        (mb.CosineAngles([1], [2], [3], [1.0], [2.0]), 6, (1, 3), (1, 2), [[1, 2]]),
        (mb.UreyBradleys([1], [2], [3], [1.0], [2.0], [3.0], [4.0]), 7, (1, 3), (1, 4), [[1, 2, 3, 4]]),
        (mb.HarmonicTorsions([1], [2], [3], [4], [1.0], [2.0]), 8, (1, 4), (1, 2), [[1, 2]]),
        (mb.RBTorsions([1], [2], [3], [4], [1.0], [2.0], [3.0], [4.0]), 9, (1, 4), (1, 4), [[1, 2, 3, 4]]),
    ]
    for lst, kind, ishape, pshape, pval in cases:
        idx, par = lst.arrays()
        assert lst.kind == kind
        assert (bk.ATOMS[kind], bk.PARAMS[kind]) == (ishape[1], pshape[1])
        assert idx.shape == ishape and idx.dtype == np.int32 and idx.flags["C_CONTIGUOUS"]
        assert par.shape == pshape and par.dtype == np.float64 and par.flags["C_CONTIGUOUS"]
        np.testing.assert_array_equal(par, pval)
    assert mb.capi.MB_SPECIFIC_N_KINDS == 10
    assert [mb.InteractionList2Atoms.kind, mb.InteractionList3Atoms.kind, mb.InteractionList4Atoms.kind] == [0, 1, 2]


def test_header_kind_table_matches_python():
    import os
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    h = open(os.path.join(root, "include", "mollyb200.h")).read()
    for name, v in re.findall(r"MB_SPECIFIC_(\w+) = (\d+)", h):
        assert getattr(mb.capi, "MB_SPECIFIC_" + name) == int(v)
    src = open(os.path.join(root, "molly.jl_b200", "csrc", "bonded.cuh")).read()
    atoms = re.search(r"SPECIFIC_ATOMS\[N_SPECIFIC_KINDS\] = \{([^}]*)\}", src).group(1)
    params = re.search(r"SPECIFIC_PARAMS\[N_SPECIFIC_KINDS\] = \{([^}]*)\}", src).group(1)
    assert tuple(int(a) for a in atoms.split(",")) == bk.ATOMS
    assert tuple(int(a) for a in params.split(",")) == bk.PARAMS


def _small_system(n=6):
    rng = np.random.default_rng(0)
    atoms = mb.atoms_from_arrays(np.full(n, 12.0), np.zeros(n), np.full(n, 0.3), np.full(n, 0.2), np.float64)
    return mb.System(atoms=atoms, coords=rng.random((n, 3)) * 2, boundary=mb.CubicBoundary(2.0, 2.0, 2.0), dtype=np.float64,
                     pairwise_inters=(mb.LennardJones(),), velocities=rng.normal(size=(n, 3)),
                     specific_inter_lists=(mb.MorseBonds([1], [2], [1.0], [2.0], [0.1]),))


def test_add_position_restraints():
    s = _small_system()
    r = mb.add_position_restraints(s, 100.0)
    assert len(r.specific_inter_lists) == 2 and r.specific_inter_lists[0] is s.specific_inter_lists[0]
    lst = r.specific_inter_lists[1]
    idx, par = lst.arrays()
    assert lst.kind == mb.capi.MB_SPECIFIC_POSITION_RESTRAINT
    np.testing.assert_array_equal(idx[:, 0], np.arange(1, 7))
    np.testing.assert_array_equal(par[:, 0], 100.0)
    np.testing.assert_array_equal(par[:, 1:], s.coords)
    # a copy: moving the new system's atoms moves neither the old system nor the restraint positions
    r.coords[:] += 1.0
    np.testing.assert_array_equal(par[:, 1:], s.coords)
    np.testing.assert_array_equal(r.specific_inter_lists[1].arrays()[1][:, 1:], s.coords)
    # boolean mask and 1-based indices select the same atoms; per-atom k follows the atom
    k = np.arange(6) * 10.0 + 1
    x0 = np.arange(18.0).reshape(6, 3)
    for sel in (np.array([False, True, False, True, True, False]), [2, 4, 5]):
        idx, par = mb.add_position_restraints(s, k, atom_selector=sel, restrain_coords=x0).specific_inter_lists[1].arrays()
        np.testing.assert_array_equal(idx[:, 0], [2, 4, 5])
        np.testing.assert_array_equal(par[:, 0], [11.0, 31.0, 41.0])
        np.testing.assert_array_equal(par[:, 1:], x0[[1, 3, 4]])
    with pytest.raises(ValueError, match="6 atoms but there are 5 k values"):
        mb.add_position_restraints(s, np.ones(5))
    with pytest.raises(ValueError):
        mb.add_position_restraints(s, 1.0, atom_selector=[0])
    with pytest.raises(ValueError):
        mb.add_position_restraints(s, 1.0, atom_selector=np.ones(5, bool))


def test_mts_levels_mixed_old_and_new_kinds():
    s = _small_system()
    lists = (mb.InteractionList2Atoms([1, 2], [2, 3], [1.0, 1.0], [0.1, 0.1]),
             mb.RBTorsions([1], [2], [3], [4], [1.0], [0.0], [0.0], [0.0]),
             mb.add_position_restraints(s, 5.0).specific_inter_lists[1],
             mb.RBTorsions([2, 3], [3, 4], [4, 5], [5, 6], [1.0, 1.0], [0.0, 0.0], [0.0, 0.0], [0.0, 0.0]),
             mb.MorseBonds([5], [6], [1.0], [2.0], [0.1]))
    s2 = mb.System(atoms=s.atoms, coords=s.coords, boundary=s.boundary, dtype=np.float64, pairwise_inters=s.pairwise_inters,
                   specific_inter_lists=lists)
    sim = mb.MTSIntegrator(0.002, pi_fractions=(1,), si_fractions=(1, 2, 4, 1, 2))
    lv = mb.mts_levels(s2, sim)
    assert sorted(lv) == [0, 3, 4, 9]
    assert lv[0].tolist() == [0, 0]
    assert lv[9].tolist() == [1, 0, 0]  # the two RBTorsion lists in list order: fraction 2, then fraction 1
    assert lv[3].tolist() == [2] * 6
    assert lv[4].tolist() == [1]


# ---- energy conservation: the bar of test_gpu_specific_kinds.test_energy_conservation_restraints_rb_morse -----------------
DRIFT_DT, DRIFT_STEPS, DRIFT_SAMPLES = 0.0005, 2000, 10


def drift_system():
    """8 non-interacting 4-site molecules held by Morse bonds, harmonic angles, an RB torsion each and restraints on their
    end atoms, f64."""
    import mbhelpers as H
    sd = H.molecular_system(8, [3.0, 3.0, 3.0], seed=21, stable=True)
    n = sd["n"]
    sd = dict(sd, charge=np.zeros(n), eps=np.zeros(n))
    a = np.arange(0, n, 4) + 1
    b, c, d = a + 1, a + 2, a + 3
    m = np.ones(len(a))
    x = sd["coords"].astype(np.float64)
    x0 = x[np.r_[a, d] - 1] + np.random.default_rng(22).normal(0, 0.03, (2 * len(a), 3))
    bonds = np.stack([np.r_[a, b, c], np.r_[b, c, d]], 1) - 1
    r0 = np.linalg.norm(x[bonds[:, 1]] - x[bonds[:, 0]], axis=1) + 0.01  # near the built geometry, slightly stretched
    angles = np.stack([np.r_[a, b], np.r_[b, c], np.r_[c, d]], 1) - 1
    ba, bc = x[angles[:, 0]] - x[angles[:, 1]], x[angles[:, 2]] - x[angles[:, 1]]
    th0 = np.arccos(np.sum(ba * bc, 1) / np.linalg.norm(ba, axis=1) / np.linalg.norm(bc, axis=1)) + 0.1
    lists = (mb.MorseBonds(bonds[:, 0] + 1, bonds[:, 1] + 1, np.full(3 * len(a), 400.0), np.full(3 * len(a), 10.0), r0),
             mb.InteractionList3Atoms(*(angles.T + 1), np.full(2 * len(a), 300.0), th0),
             mb.RBTorsions(a, b, c, d, 8 * m, -4 * m, 6 * m, 1 * m),
             mb.InteractionList1Atoms(np.r_[a, d], np.full(2 * len(a), 1000.0), x0))
    return sd, lists


def oracle_drift(reference_sign=False):
    """max |E(t) - E(0)| of the numpy VelocityVerlet run (no centre-of-mass removal) at DRIFT_SAMPLES evenly spaced steps."""
    sd, lists = drift_system()
    ol = bk.oracle_lists(lists)
    box = np.asarray(sd["box"], np.float64)
    rest = [t for t in ol if t[0] != bk.RB_TORSION]
    rb = [t for t in ol if t[0] == bk.RB_TORSION]

    def fe(x):
        f, e = bk.specific_forces(x, box, rest)
        for _, idx, par in rb:
            fr, er = bk.rb_torsion_forces(x, box, idx, par, reference_sign=reference_sign)
            f, e = f + fr, e + er
        return f, e
    m = sd["mass"][:, None]
    x, v = sd["coords"].astype(np.float64), sd["velocities"].astype(np.float64)
    f, u = fe(x)
    e0 = u + 0.5 * np.sum(m * v * v)
    drift = 0.0
    for step in range(1, DRIFT_STEPS + 1):
        v = v + f / m * (DRIFT_DT / 2)
        x = x + v * DRIFT_DT
        x = x - np.floor(x / box) * box
        f, u = fe(x)
        v = v + f / m * (DRIFT_DT / 2)
        if step % (DRIFT_STEPS // DRIFT_SAMPLES) == 0:
            drift = max(drift, abs(u + 0.5 * np.sum(m * v * v) - e0))
    return drift


DRIFT_BAR = 2.0  # kJ/mol


def test_drift_bar_separates_the_rb_force_signs():
    good, bad = oracle_drift(False), oracle_drift(True)
    print(f"[drift] -grad E: {good:.3e} kJ/mol; the reference's RB sign: {bad:.3e} kJ/mol (bar {DRIFT_BAR})")
    assert good < DRIFT_BAR / 10
    assert bad > 10 * DRIFT_BAR
