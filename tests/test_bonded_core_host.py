"""CPU tests of the f64 checker of HarmonicBond, HarmonicAngle and PeriodicTorsion (oracle/bonded.py): the reference's
literal values (test/interactions.jl), its forces against -grad E by central differences, its bend angle against a
50-digit evaluation near 0 and pi, and the degenerate geometries with closed forms (collinear and folded angles, collinear
torsions). The GPU counterpart is tests/test_gpu_bonded_core.py."""
import mpmath
import numpy as np
import pytest

import bonded_kinds_oracle as bk
from oracle import bonded as bd
from test_specific_kinds_host import C1, C2, C3, C3A, RB_X, _numeric_gradient

C3_COLIN, C3_90 = [1.6, 1.0, 1.0], [1.3, 1.3, 1.0]
# the reference's PeriodicTorsion on RB_X: periodicities (1, 2, 3), phases (0, pi/2, pi), ks (10, 5, 2), one entry each
PT_PARAMS = [[1.0, 0.0, 10.0], [2.0, np.pi / 2, 5.0], [3.0, np.pi, 2.0]]
PT_NORMS = [139.51649514944324, 188.90622744571394, 98.65305980755139, 80.54988603092418]

# (kind, coordinates (nm), box side, params per entry, expected forces per atom or None, expected force norms or None,
# expected energy): the literals of test/interactions.jl for kinds 0-2, all to atol 1e-9 there
LITERALS = {
    "bond_1": (bk.HARMONIC_BOND, [C1, C2], 2.0, [[3e5, 0.2]], [[30000.0, 0, 0], [-30000.0, 0, 0]], None, 1500.0),
    "bond_2": (bk.HARMONIC_BOND, [C1, C3], 2.0, [[1e5, 0.6]], [[-20000.0, 0, 0], [20000.0, 0, 0]], None, 2000.0),
    "bond_eq": (bk.HARMONIC_BOND, [C1, C2], 2.0, [[1e5, 0.3]], [[0.0, 0, 0], [0.0, 0, 0]], None, 0.0),
    "angle": (bk.HARMONIC_ANGLE, [C1, C2, C3A], 2.0, [[300.0, 0.8]],
              [[0.0, -31.1343284689, -31.1343284689], [-21.9771730369, 14.6514486912, 14.6514486912],
               [21.9771730369, 16.4828797777, 16.4828797777]], None, 0.2908039228),
    "angle_collinear": (bk.HARMONIC_ANGLE, [C1, C2, C3_COLIN], 2.0, [[100.0, np.pi]], [[0.0, 0, 0]] * 3, None, 0.0),
    "angle_90": (bk.HARMONIC_ANGLE, [C1, C2, C3_90], 2.0, [[200.0, np.pi / 2]], None, None, 0.0),
    "torsion": (bk.PERIODIC_TORSION, RB_X, 5.0, PT_PARAMS, None, PT_NORMS, 4.587951202894674),
    "improper": (bk.PERIODIC_TORSION, RB_X, 5.0, [[2.0, np.pi, 15.0]], None, None, 20.0),
}
LIT_ATOL = 1e-9


def literal_terms(name):
    """(kind, x, side, idx (terms x atoms, 0-based), par (terms x params)) of a literal: one entry per term."""
    kind, x, side, par, *_ = LITERALS[name]
    par = np.asarray(par, np.float64)
    return kind, np.asarray(x, np.float64), side, np.tile(np.arange(bk.ATOMS[kind]), (len(par), 1)), par


def check_literal(name, f, e):
    """Assert forces f and energy e against the reference's literals of `name`, to its atol."""
    *_, f_exp, norms, e_exp = LITERALS[name]
    if f_exp is not None:
        np.testing.assert_allclose(f, np.asarray(f_exp, np.float64), rtol=0, atol=LIT_ATOL)
    if norms is not None:
        np.testing.assert_allclose(np.linalg.norm(f, axis=1), norms, rtol=0, atol=LIT_ATOL)
    assert abs(e - e_exp) <= LIT_ATOL, (e, e_exp)


@pytest.mark.parametrize("name", sorted(LITERALS))
def test_oracle_reproduces_reference_literals(name):
    kind, x, side, idx, par = literal_terms(name)
    f, e = bk.FORCES[kind](x, np.full(3, side), idx, par)
    check_literal(name, f, e)


# ---- random non-degenerate terms ------------------------------------------------------------------------------------------
def random_core_terms(kind, rng, n_terms=6, box=10.0):
    """Non-degenerate random terms of kind 0-2, each on its own atoms: a walk of 0.1-0.2 nm steps whose bend angles lie in
    [1.2, 2.6] rad, so no angle or torsion arm comes near 0 or pi; parameters of the usual sizes."""
    na = bk.ATOMS[kind]
    x = []
    for _ in range(n_terms):
        p = [rng.uniform(0.2, box - 0.2, 3)]
        d = rng.normal(size=3)
        d /= np.linalg.norm(d)
        for _ in range(na - 1):
            p.append(p[-1] + rng.uniform(0.1, 0.2) * d)
            w = rng.normal(size=3)
            w -= w.dot(d) * d
            w /= np.linalg.norm(w)
            th = rng.uniform(1.2, 2.6)  # the bend angle at the atom just placed: the next step turns by pi - th
            d = -np.cos(th) * d + np.sin(th) * w
        x += p
    x = np.array(x)
    idx = np.arange(len(x)).reshape(n_terms, na)
    u = lambda lo, hi: rng.uniform(lo, hi, n_terms)
    par = {bk.HARMONIC_BOND: lambda: np.c_[u(1e3, 3e5), u(0.1, 0.2)],
           bk.HARMONIC_ANGLE: lambda: np.c_[u(100, 600), u(1.5, 2.5)],
           bk.PERIODIC_TORSION: lambda: np.c_[rng.integers(1, 7, n_terms).astype(float), u(0, 2 * np.pi), u(1, 20)]}[kind]()
    return x, idx, par


CORE_KINDS = [bk.HARMONIC_BOND, bk.HARMONIC_ANGLE, bk.PERIODIC_TORSION]


@pytest.mark.parametrize("kind", CORE_KINDS)
def test_oracle_force_is_minus_gradient(kind):
    rng = np.random.default_rng(200 + kind)
    box = np.full(3, 10.0)
    x, idx, par = random_core_terms(kind, rng)
    fn = lambda y: bk.FORCES[kind](y, box, idx, par)
    f, _ = fn(x)
    g = _numeric_gradient(fn, x)
    assert np.abs(f).max() > 1.0
    assert np.abs(f + g).max() <= 1e-6 * np.abs(f).max()


def _angle_acos(x, box, idx, par):
    """HarmonicAngle with theta by acos of the clamped cosine, as the checker computed it before (and the reference does)."""
    ba = bd._mic(x[idx[:, 0]] - x[idx[:, 1]], box)
    bc = bd._mic(x[idx[:, 2]] - x[idx[:, 1]], box)
    nba, nbc = np.linalg.norm(ba, axis=1), np.linalg.norm(bc, axis=1)
    th = np.arccos(np.clip(np.sum(ba * bc, 1) / (nba * nbc), -1.0, 1.0))
    n = np.cross(ba, bc)
    pa, pc = np.cross(ba, n), np.cross(-bc, n)
    pa /= np.linalg.norm(pa, axis=1)[:, None]
    pc /= np.linalg.norm(pc, axis=1)[:, None]
    t = -par[:, 0] * (th - par[:, 1])
    f = np.zeros_like(x)
    np.add.at(f, idx[:, 0], (t / nba)[:, None] * pa)
    np.add.at(f, idx[:, 2], (t / nbc)[:, None] * pc)
    np.add.at(f, idx[:, 1], -(t / nba)[:, None] * pa - (t / nbc)[:, None] * pc)
    return f, float(np.sum(0.5 * par[:, 0] * (th - par[:, 1]) ** 2))


def test_oracle_angle_unchanged_away_from_degeneracy():
    """On non-degenerate angles (0.3 .. pi - 0.3) the atan2 form gives the acos form's forces and energy to 1e-12."""
    rng = np.random.default_rng(5)
    box = np.full(3, 10.0)
    x, idx, par = random_core_terms(bk.HARMONIC_ANGLE, rng, n_terms=200)
    f, e = bd.angle_forces(x, box, idx, par)
    f0, e0 = _angle_acos(x, box, idx, par)
    assert np.abs(f - f0).max() <= 1e-12 * np.abs(f0).max()
    assert abs(e - e0) <= 1e-12 * abs(e0)


def _near_linear_vectors(delta, rng, n, folded):
    """n pairs (ba, bc) of 0.1-0.2 nm arms at angle pi - delta (or delta when folded) in random orientations."""
    u = rng.normal(size=(n, 3))
    u /= np.linalg.norm(u, axis=1)[:, None]
    w = rng.normal(size=(n, 3))
    w -= np.sum(w * u, 1)[:, None] * u
    w /= np.linalg.norm(w, axis=1)[:, None]
    th = delta if folded else np.pi - delta
    ba = rng.uniform(0.1, 0.2, (n, 1)) * u
    bc = rng.uniform(0.1, 0.2, (n, 1)) * (np.cos(th) * u + np.sin(th) * w)
    return ba, bc


def _theta_mp(a, b):
    """The angle between two f64 vectors, evaluated with 50 digits from their exact values."""
    a, b = [mpmath.mpf(float(v)) for v in a], [mpmath.mpf(float(v)) for v in b]
    c = [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]
    return mpmath.atan2(mpmath.sqrt(sum(v * v for v in c)), sum(p * q for p, q in zip(a, b)))


@pytest.mark.parametrize("folded", [False, True], ids=["pi-delta", "delta"])
@pytest.mark.parametrize("delta", [1e-2, 1e-3, 1e-4, 1e-5, 1e-6, 1e-7])
def test_oracle_bend_angle_against_mpmath(delta, folded):
    """The checker's theta keeps 1e-14 rad near 0 and pi; the acos form it replaced does not."""
    mpmath.mp.dps = 50
    ba, bc = _near_linear_vectors(delta, np.random.default_rng(int(-np.log10(delta)) + 10 * folded), 50, folded)
    th, _ = bd.bend_angle(ba, bc)
    ref = np.array([float(_theta_mp(a, b)) for a, b in zip(ba, bc)])
    err = np.abs(th - ref).max()
    acos = np.arccos(np.clip(np.sum(ba * bc, 1) / (np.linalg.norm(ba, axis=1) * np.linalg.norm(bc, axis=1)), -1, 1))
    err_acos = np.abs(acos - ref).max()
    print(f"[bend angle delta={delta:g} {'folded' if folded else 'open'}] atan2 {err:.2e} rad, acos {err_acos:.2e} rad")
    assert err <= 1e-14
    if delta <= 1e-4:
        assert err_acos > 1e-12  # the check can tell the two forms apart


# ---- degenerate geometries with closed forms -----------------------------------------------------------------------------
LINE = [[1.0, 1.0, 1.0], [1.3, 1.0, 1.0], [1.6, 1.0, 1.0]]  # on a line parallel to x: every cross product is exactly 0
FOLDED = [[1.3, 1.0, 1.0], [1.0, 1.0, 1.0], [1.6, 1.0, 1.0]]  # i and k on the same side of j: theta = 0


@pytest.mark.parametrize("th0", [np.pi, 1.9], ids=["pi", "1.9"])
@pytest.mark.parametrize("geom", ["collinear", "folded"])
def test_oracle_degenerate_angle_closed_form(geom, th0):
    k = 100.0
    x = np.array(LINE if geom == "collinear" else FOLDED)
    th = np.pi if geom == "collinear" else 0.0
    assert bd.bend_angle(x[[0]] - x[[1]], x[[2]] - x[[1]])[0][0] == th
    f, e = bd.angle_forces(x, np.full(3, 2.0), np.array([[0, 1, 2]]), np.array([[k, th0]]))
    assert np.all(f == 0)
    assert e == 0.5 * k * (th - th0) ** 2
    if geom == "collinear" and th0 == 1.9:
        assert abs(e - 77.07764) < 1e-4  # the case the engine used to report as 0


# i-j-k collinear (l off the line) and j-k-l collinear (i off the line), on lines parallel to x
TORSION_COLLINEAR = {"ijk": [[1.0, 1.0, 1.0], [1.3, 1.0, 1.0], [1.6, 1.0, 1.0], [1.7, 1.2, 1.1]],
                     "jkl": [[0.9, 1.2, 0.9], [1.0, 1.0, 1.0], [1.3, 1.0, 1.0], [1.6, 1.0, 1.0]]}
# theta = atan2(±0, ±0) of those geometries in the engine's operation order (torsion_vectors): signed zeros come out the
# same whatever the order of the sums and whether multiply-adds are fused, because no sum there mixes two nonzero terms
TORSION_COLLINEAR_THETA = {"ijk": 0.0, "jkl": 0.0}


def collinear_torsion_terms():
    """(name, kind, par) of the collinear torsion cases: PeriodicTorsion of even and odd periodicity, HarmonicTorsion and
    RBTorsion."""
    return [("pt_even", bk.PERIODIC_TORSION, [2.0, 0.0, 10.0]), ("pt_odd", bk.PERIODIC_TORSION, [3.0, 0.4, 7.0]),
            ("pt_per1", bk.PERIODIC_TORSION, [1.0, 0.0, 5.0]), ("harmonic", bk.HARMONIC_TORSION, [40.0, 1.0]),
            ("rb", bk.RB_TORSION, [10.0, 20.0, 30.0, 5.0])]


@pytest.mark.parametrize("where", sorted(TORSION_COLLINEAR))
def test_oracle_collinear_torsion_energy_and_no_force(where):
    x = np.array(TORSION_COLLINEAR[where])
    th = bk._torsion(x, np.full(3, 5.0), np.arange(4)[None, :])[-1][0]
    assert th == TORSION_COLLINEAR_THETA[where] and not np.signbit(th)
    for name, kind, par in collinear_torsion_terms():
        f, e = bk.FORCES[kind](x, np.full(3, 5.0), np.arange(4)[None, :], np.array([par]))
        assert np.all(f == 0), name
        if kind == bk.PERIODIC_TORSION:
            assert e == par[2] * (1 + np.cos(par[0] * th - par[1])), name
    # the issue's case: atoms on x plus one off-axis atom, per = 2, phase 0, k = 10 -> E = 20
    f, e = bd.torsion_forces(x, np.full(3, 5.0), np.arange(4)[None, :], np.array([[2.0, 0.0, 10.0]]))
    assert e == 20.0 and np.all(f == 0)
