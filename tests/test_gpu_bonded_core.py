"""HarmonicBond, HarmonicAngle and PeriodicTorsion (kinds 0-2) on the device against the f64 checker (oracle/bonded.py),
f32 and f64, on systems whose pair terms act on nothing (zero-epsilon, uncharged atoms): the reference's literals, exactly
collinear and folded angles and torsions (no force, the energy counted), near-linear angles and near-degenerate torsions
with f32 bars derived from the conditioning, partners in other periodic images, the brick path and a triclinic box, the
edges of the launch's per-kind CTA ranges, a hub atom shared by 8192 terms and the energy records of a captured
VelocityVerlet step graph. The CPU counterpart is tests/test_bonded_core_host.py."""
import numpy as np
import pytest

import bonded_kinds_oracle as bk
import mbhelpers as H
import mollyb200 as mb
import mts_oracle as mo
from oracle import bonded as bd
from test_bonded_core_host import (FOLDED, LINE, LITERALS, TORSION_COLLINEAR, _near_linear_vectors, check_literal,
                                   collinear_torsion_terms, literal_terms, random_core_terms)
from test_gpu_parity import _pos_err

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
DTYPES = pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
EPS32 = float(np.finfo(np.float32).eps)

# f32 bars, in units of the conditioning bounds below: 5x the largest ratio measured on an H100 80GB HBM3 at a 700 W power
# limit (1.59 for the angle kinds, at theta0 = pi; 0.26 for the torsion kinds), rounded up
C_ANGLE = 8.0
C_TORSION = 1.5

_LIST = {bk.HARMONIC_BOND: mb.InteractionList2Atoms, bk.HARMONIC_ANGLE: mb.InteractionList3Atoms,
         bk.PERIODIC_TORSION: mb.InteractionList4Atoms, bk.COSINE_ANGLE: mb.CosineAngles, bk.UREY_BRADLEY: mb.UreyBradleys,
         bk.HARMONIC_TORSION: mb.HarmonicTorsions, bk.RB_TORSION: mb.RBTorsions}


def _lists(terms):
    """(kind, 0-based idx (terms x atoms), par (terms x params)) triples -> the engine's list objects."""
    return tuple(_LIST[kind](*(np.asarray(idx).T + 1), *np.asarray(par, F64).T) for kind, idx, par in terms)


def _system(x, boundary, terms, dtype, nf=None, pairs=None, loggers=None):
    """The atoms of the terms and nothing else: zero-epsilon, uncharged atoms, so only the terms act."""
    n = len(x)
    atoms = mb.atoms_from_arrays(np.full(n, 12.0), np.zeros(n), np.full(n, 0.3), np.zeros(n), dtype)
    return mb.System(atoms=atoms, coords=np.asarray(x, F64).astype(dtype), boundary=boundary, dtype=dtype,
                     pairwise_inters=pairs or (mb.LennardJones(),), neighbor_finder=nf, specific_inter_lists=_lists(terms),
                     loggers=loggers)


def _rounded(terms, dtype):
    """The terms with their parameters as the engine holds them (cast to dtype)."""
    return [(kind, np.asarray(idx), np.asarray(par, F64).astype(dtype).astype(F64)) for kind, idx, par in terms]


def _oracle(x, box, terms, dtype):
    """The checker on the dtype-rounded coordinates and parameters the engine sees."""
    return bk.specific_forces(np.asarray(x, F64).astype(dtype).astype(F64), np.asarray(box, F64), _rounded(terms, dtype))


def _run(s, forces_only=False):
    try:
        f, e = mb.forces_energy(s)
        f0 = mb.forces(s) if forces_only else None
        st = s.stats()
    finally:
        s.close()
    return f.astype(F64), e, f0, st


def _compare(label, f, e, f_ref, e_ref, dtype, scale=1.0):
    fmax = np.abs(f_ref).max()
    err = np.abs(f - f_ref).max()
    print(f"[{label} {np.dtype(dtype).name}] max|dF|={err:.3e} (max|F| {fmax:.3e}) dE={e - e_ref:.3e} (E {e_ref:.6e})")
    assert np.isfinite(f).all()
    assert err <= scale * H.tol(dtype, fmax)
    e_scale = abs(e_ref) if dtype == F64 else max(abs(e_ref), 0.1 * fmax)  # (as test_gpu_specific_kinds)
    assert abs(e - e_ref) <= scale * H.etol(dtype, e_scale)


# ---- 1. the reference's literals ------------------------------------------------------------------------------------------
@DTYPES
@pytest.mark.parametrize("name", sorted(LITERALS))
def test_reference_literal(name, dtype):
    kind, x, side, idx, par = literal_terms(name)
    terms = [(kind, idx, par)]
    f, e, _, _ = _run(_system(x, mb.CubicBoundary(side, side, side), terms, dtype))
    f_ref, e_ref = _oracle(x, np.full(3, side), terms, dtype)
    if dtype == F64:
        check_literal(name, f, e)
    _compare(f"literal {name}", f, e, f_ref, e_ref, dtype)


# ---- 2. exact degeneracies: cross products exactly zero on the device, fused or not --------------------------------------
@DTYPES
@pytest.mark.parametrize("th0", [np.pi, 1.9], ids=["pi", "1.9"])
@pytest.mark.parametrize("geom", ["collinear", "folded"])
def test_degenerate_angle(geom, th0, dtype):
    k = 100.0
    x = LINE if geom == "collinear" else FOLDED
    terms = [(bk.HARMONIC_ANGLE, [[0, 1, 2]], [[k, th0]])]
    f, e, f0, _ = _run(_system(x, mb.CubicBoundary(2.0, 2.0, 2.0), terms, dtype), forces_only=True)
    th = np.pi if geom == "collinear" else 0.0
    e_exp = 0.5 * k * (th - float(dtype(th0))) ** 2  # the closed form with theta0 as the engine holds it
    print(f"[angle {geom} th0={th0:.4f} {np.dtype(dtype).name}] f={f.tolist()} e={e!r} (closed form {e_exp!r})")
    assert np.all(f == 0) and np.all(f0 == 0)  # exactly zero, not NaN, with and without the energy
    assert abs(e - e_exp) <= H.etol(dtype, e_exp)


@DTYPES
@pytest.mark.parametrize("case", [c[0] for c in collinear_torsion_terms()])
@pytest.mark.parametrize("where", sorted(TORSION_COLLINEAR))
def test_collinear_torsion(where, case, dtype):
    _, kind, par = next(c for c in collinear_torsion_terms() if c[0] == case)
    x = TORSION_COLLINEAR[where]
    terms = [(kind, [[0, 1, 2, 3]], [par])]
    f, e, f0, _ = _run(_system(x, mb.CubicBoundary(5.0, 5.0, 5.0), terms, dtype), forces_only=True)
    _, e_ref = _oracle(x, np.full(3, 5.0), terms, dtype)
    print(f"[torsion {where} {case} {np.dtype(dtype).name}] f={f.tolist()} e={e!r} (oracle {e_ref!r})")
    assert np.all(f == 0) and np.all(f0 == 0)
    assert abs(e - e_ref) <= H.etol(dtype, e_ref)


def _line_molecule():
    """Five atoms on a line parallel to x with stretched and compressed bonds, collinear angles (theta0 = 1.9 and pi) and
    collinear torsions of the three torsion kinds."""
    x = [[1.0 + 0.15 * a + (0.02 if a % 2 else 0.0), 1.0, 1.0] for a in range(5)]
    b = np.array([[a, a + 1] for a in range(4)])
    a3 = np.array([[a, a + 1, a + 2] for a in range(3)])
    t4 = np.array([[0, 1, 2, 3], [1, 2, 3, 4]])
    terms = [(bk.HARMONIC_BOND, b, np.c_[np.full(4, 1e4), np.full(4, 0.15)]),
             (bk.HARMONIC_ANGLE, a3, [[100.0, 1.9], [150.0, np.pi], [80.0, 2.2]]),
             (bk.PERIODIC_TORSION, t4, [[2.0, 0.0, 10.0], [3.0, 0.4, 7.0]]),
             (bk.HARMONIC_TORSION, t4, [[40.0, 1.0], [20.0, -0.5]]),
             (bk.RB_TORSION, t4, [[10.0, 20.0, 30.0, 5.0], [1.0, -2.0, 3.0, 0.5]])]
    return x, terms


@DTYPES
def test_collinear_molecule_run_stays_on_its_line_and_logs_its_energy(dtype):
    """A 3-step VelocityVerlet run from rest: the step graph's PotentialEnergyLogger records (the energy launch inside the
    captured graph) equal the checker at the logged frames, and in f64 the molecule moves along its line only."""
    x, terms = _line_molecule()
    lg = {"pe": mb.PotentialEnergyLogger(1), "x": mb.CoordinatesLogger(1)}
    s = _system(x, mb.CubicBoundary(3.0, 3.0, 3.0), terms, dtype, loggers=lg)
    try:
        mb.simulate(s, mb.VelocityVerlet(dt=0.001), 3)
        xs, v = np.array(s.coords, F64), np.array(s.velocities, F64)
    finally:
        s.close()
    frames = np.array([np.asarray(a, F64) for a in lg["x"].history])
    pe = np.array([float(a) for a in lg["pe"].history])
    assert len(frames) == 4 and len(pe) == 4
    for step, (xk, ek) in enumerate(zip(frames, pe)):
        _, e_ref = _oracle(xk, np.full(3, 3.0), terms, dtype)
        print(f"[line molecule {np.dtype(dtype).name} step {step}] pe={ek!r} oracle={e_ref!r}")
        assert abs(ek - e_ref) <= H.etol(dtype, e_ref)
    assert np.abs(frames[-1, :, 0] - frames[0, :, 0]).max() > 1e-6  # the bonds moved the atoms
    if dtype == F64:
        assert np.all(frames[:, :, 1:] == 1.0) and np.all(xs[:, 1:] == 1.0) and np.all(v[:, 1:] == 0.0)


# ---- 3. near-linear angles and near-degenerate torsions ------------------------------------------------------------------
# f32 bars from the conditioning. An angle's theta = atan2(|ba x bc|, ba . bc) carries an absolute error of a few eps32; its
# force k |theta - theta0| / r also turns with the bending plane n = ba x bc, whose direction is known to eps32 / sin(theta)
# only: |dF| <= C eps32 (k + |tau| / sin theta) / r_min with tau = dE/dtheta. A torsion's normals m, n lose digits the same
# way when an arm comes within alpha of the bc axis, and its force scales as 1/(r sin alpha):
# |dF| <= C eps32 (|E'| + max|E''|) / (r_min sin^2 alpha). The f64 runs are held to 1e-9 of the oracle.
DELTAS = [1e-1, 1e-2, 1e-3, 1e-4, 1e-5]
ALPHAS = [1e-2, 1e-3, 1e-4, 1e-5]
BEND_KINDS = {"harmonic_angle": bk.HARMONIC_ANGLE, "cosine_angle": bk.COSINE_ANGLE, "urey_bradley": bk.UREY_BRADLEY}
TORSION_KINDS = {"periodic": bk.PERIODIC_TORSION, "harmonic": bk.HARMONIC_TORSION, "rb": bk.RB_TORSION}
N_SWEEP = 64


def _bend_terms(kind, folded, th0, rng):
    """N_SWEEP terms at each delta, each on its own atoms; returns x, idx, par and the delta of every term."""
    xs, pars, ds = [], [], []
    for d in DELTAS:
        ba, bc = _near_linear_vectors(d, rng, N_SWEEP, folded)
        j = rng.uniform(0.5, 2.5, (N_SWEEP, 3))
        xs.append(np.stack([j + ba, j, j + bc], 1).reshape(-1, 3))
        k = rng.uniform(100, 600, N_SWEEP)
        extra = [rng.uniform(1e3, 1e4, N_SWEEP), rng.uniform(0.2, 0.4, N_SWEEP)] if kind == bk.UREY_BRADLEY else []
        pars.append(np.stack([k, np.full(N_SWEEP, th0)] + extra, 1))
        ds += [d] * N_SWEEP
    x = np.concatenate(xs)
    return x, np.arange(len(x)).reshape(-1, 3), np.concatenate(pars), np.array(ds)


def _bend_bounds(kind, x, idx, par):
    """Per term: the unit force bound eps32 (k + |tau| / sin theta) / r_min (plus eps32 kb r_ik for UreyBradley's bond) and
    the unit energy bound eps32 (|E| + |tau|) (plus eps32 kb r_ik^2)."""
    ba, bc = x[idx[:, 0]] - x[idx[:, 1]], x[idx[:, 2]] - x[idx[:, 1]]
    th, _ = bd.bend_angle(ba, bc)
    k, th0 = par[:, 0], par[:, 1]
    if kind == bk.COSINE_ANGLE:
        tau, e = k * np.abs(np.sin(th - th0)), k * (1 + np.cos(th - th0))
    else:
        tau, e = k * np.abs(th - th0), 0.5 * k * (th - th0) ** 2
    r_min = np.minimum(np.linalg.norm(ba, axis=1), np.linalg.norm(bc, axis=1))
    fb = EPS32 * (k + tau / np.sin(th)) / r_min
    eb = EPS32 * (np.abs(e) + tau)
    if kind == bk.UREY_BRADLEY:
        rik = np.linalg.norm(x[idx[:, 2]] - x[idx[:, 0]], axis=1)
        fb, eb = fb + EPS32 * par[:, 2] * rik, eb + EPS32 * par[:, 2] * rik ** 2
    return fb, eb


def _per_term_err(f, f_ref, idx):
    return np.abs(f - f_ref)[idx].max(axis=(1, 2))


@DTYPES
@pytest.mark.parametrize("th0", [np.pi, 2.0], ids=["th0_pi", "th0_2"])
@pytest.mark.parametrize("folded", [False, True], ids=["pi-delta", "delta"])
@pytest.mark.parametrize("name", sorted(BEND_KINDS))
def test_near_linear_angle_sweep(name, folded, th0, dtype):
    kind = BEND_KINDS[name]
    rng = np.random.default_rng([sorted(BEND_KINDS).index(name), int(folded), int(th0 == np.pi)])
    x, idx, par, ds = _bend_terms(kind, folded, th0, rng)
    terms = [(kind, idx, par)]
    f, e, _, _ = _run(_system(x, mb.CubicBoundary(3.0, 3.0, 3.0), terms, dtype))
    x_in = np.asarray(x, dtype).astype(F64)
    f_ref, e_ref = _oracle(x, np.full(3, 3.0), terms, dtype)
    err = _per_term_err(f, f_ref, idx)
    label = f"{name} {'delta' if folded else 'pi-delta'} th0={th0:.4f} {np.dtype(dtype).name}"
    assert np.isfinite(f).all()
    if dtype == F64:
        fmax = np.abs(f_ref).max()
        print(f"[{label}] max|dF|={err.max():.3e} (max|F| {fmax:.3e}) dE={e - e_ref:.3e} (E {e_ref:.6e})")
        assert err.max() <= 1e-9 * fmax and abs(e - e_ref) <= 1e-9 * abs(e_ref)
        return
    fb, eb = _bend_bounds(kind, x_in, idx, _rounded(terms, dtype)[0][2])
    ratios = {d: (err[ds == d] / fb[ds == d]).max() for d in DELTAS}
    e_ratio = abs(e - e_ref) / eb.sum()
    print(f"[{label}] |dF| / (eps32 (k + |tau|/sin th) / r_min) by delta: "
          + " ".join(f"{d:g}:{r:.3f}" for d, r in ratios.items()) + f"; |dE| / bound {e_ratio:.3f} (bar C = {C_ANGLE})")
    assert max(ratios.values()) <= C_ANGLE
    assert e_ratio <= C_ANGLE


def _unit(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def _torsion_terms(kind, rng):
    """N_SWEEP terms at each alpha: one arm (ab for half the terms, cd for the other half) at alpha from the bc axis, the
    other arm at 1.0 - 2.1 rad from it."""
    xs, ds = [], []
    for a in ALPHAS:
        u = _unit(rng.normal(size=(N_SWEEP, 3)))
        w1, w2 = _unit(np.cross(u, rng.normal(size=(N_SWEEP, 3)))), _unit(np.cross(u, rng.normal(size=(N_SWEEP, 3))))
        wide = rng.uniform(1.0, 2.1, (N_SWEEP, 1))
        near = np.cos(a) * u + np.sin(a) * w1  # at alpha from u
        far = np.cos(wide) * u + np.sin(wide) * w2
        L = rng.uniform(0.1, 0.2, (N_SWEEP, 3))
        first = np.arange(N_SWEEP) % 2 == 0
        ab = L[:, [0]] * np.where(first[:, None], near, far)
        cd = L[:, [2]] * np.where(first[:, None], far, near)
        j = rng.uniform(0.5, 2.5, (N_SWEEP, 3))
        k = j + L[:, [1]] * u
        xs.append(np.stack([j - ab, j, k, k + cd], 1).reshape(-1, 3))
        ds += [a] * N_SWEEP
    x = np.concatenate(xs)
    n = len(x) // 4
    u = lambda lo, hi: rng.uniform(lo, hi, n)
    par = {bk.PERIODIC_TORSION: lambda: np.c_[rng.integers(1, 7, n).astype(float), u(0, 2 * np.pi), u(1, 20)],
           bk.HARMONIC_TORSION: lambda: np.c_[u(10, 100), u(-2.5, 2.5)],
           bk.RB_TORSION: lambda: np.c_[u(-20, 20), u(-20, 20), u(-20, 20), u(-5, 5)]}[kind]()
    return x, np.arange(len(x)).reshape(-1, 4), par, np.array(ds)


def _torsion_bounds(kind, x, idx, par):
    """Per term: eps32 (|E'| + max|E''|) / (r_min sin^2 alpha) and eps32 (|E| + (|E'| + max|E''|) / sin alpha), alpha the
    smaller angle of an arm with the bc axis."""
    ab, bc, cd, m, n, nbc, th = bk._torsion(x, np.full(3, 1e3), idx)
    nab, ncd = np.linalg.norm(ab, axis=1), np.linalg.norm(cd, axis=1)
    sin_a = np.minimum(np.linalg.norm(m, axis=1) / (nab * nbc), np.linalg.norm(n, axis=1) / (nbc * ncd))
    if kind == bk.PERIODIC_TORSION:
        p, ph, k = par.T
        e, d1, d2 = k * (1 + np.cos(p * th - ph)), k * p * np.sin(p * th - ph), k * p * p
    elif kind == bk.HARMONIC_TORSION:
        k, t0 = par.T
        e, d1, d2 = k * (th - t0) ** 2, 2 * k * (th - t0), 2 * k
    else:
        f1, f2, f3, f4 = par.T
        e = (f1 * (1 + np.cos(th)) + f2 * (1 - np.cos(2 * th)) + f3 * (1 + np.cos(3 * th)) + f4) / 2
        d1 = (-f1 * np.sin(th) + 2 * f2 * np.sin(2 * th) - 3 * f3 * np.sin(3 * th)) / 2
        d2 = (np.abs(f1) + 4 * np.abs(f2) + 9 * np.abs(f3)) / 2
    r_min = np.minimum(np.minimum(nab, nbc), ncd)
    return EPS32 * (np.abs(d1) + d2) / (r_min * sin_a ** 2), EPS32 * (np.abs(e) + (np.abs(d1) + d2) / sin_a)


@DTYPES
@pytest.mark.parametrize("name", sorted(TORSION_KINDS))
def test_near_degenerate_torsion_sweep(name, dtype):
    kind = TORSION_KINDS[name]
    x, idx, par, ds = _torsion_terms(kind, np.random.default_rng(31 + kind))
    terms = [(kind, idx, par)]
    f, e, _, _ = _run(_system(x, mb.CubicBoundary(3.0, 3.0, 3.0), terms, dtype))
    f_ref, e_ref = _oracle(x, np.full(3, 3.0), terms, dtype)
    err = _per_term_err(f, f_ref, idx)
    label = f"torsion {name} {np.dtype(dtype).name}"
    assert np.isfinite(f).all()
    if dtype == F64:
        fmax = np.abs(f_ref).max()
        print(f"[{label}] max|dF|={err.max():.3e} (max|F| {fmax:.3e}) dE={e - e_ref:.3e} (E {e_ref:.6e})")
        assert err.max() <= 1e-9 * fmax and abs(e - e_ref) <= 1e-9 * abs(e_ref)
        return
    fb, eb = _torsion_bounds(kind, np.asarray(x, dtype).astype(F64), idx, _rounded(terms, dtype)[0][2])
    ratios = {a: (err[ds == a] / fb[ds == a]).max() for a in ALPHAS}
    e_ratio = abs(e - e_ref) / eb.sum()
    print(f"[{label}] |dF| / (eps32 (|E'| + max|E''|) / (r_min sin^2 a)) by alpha: "
          + " ".join(f"{a:g}:{r:.3f}" for a, r in ratios.items()) + f"; |dE| / bound {e_ratio:.3f} (bar C = {C_TORSION})")
    assert max(ratios.values()) <= C_TORSION
    assert e_ratio <= C_TORSION


# ---- 4. periodic images, the brick path and a triclinic box --------------------------------------------------------------
CORE = [bk.HARMONIC_BOND, bk.HARMONIC_ANGLE, bk.PERIODIC_TORSION]


def _core_terms(n_terms, rng, box):
    """n_terms random non-degenerate terms of each of kinds 0-2, on disjoint atoms of one coordinate array."""
    xs, terms, off = [], [], 0
    for kind in CORE:
        x, idx, par = random_core_terms(kind, rng, n_terms, box)
        xs.append(x)
        terms.append((kind, idx + off, par))
        off += len(x)
    return np.concatenate(xs), terms


@DTYPES
@pytest.mark.parametrize("setup", ["shifted", "brick", "triclinic"])
def test_images_and_paths(setup, dtype):
    rng = np.random.default_rng({"shifted": 1, "brick": 2, "triclinic": 3}[setup])
    L = 4.0 if setup == "brick" else 2.5
    x, terms = _core_terms(300 if setup == "brick" else 60, rng, L)
    x_oracle, scale, nf, pairs, expect_path = x, 1.0, None, None, 0
    if setup == "shifted":  # every atom moved by -3, -1, 0, 1 or 3 box lengths on each axis
        x = x + L * rng.choice([-3, -1, 0, 1, 3], x.shape)
        x_oracle, scale = x, 10.0  # f32: the displacements of atoms 10 nm out carry the rounding of 10 nm coordinates
        bnd = mb.CubicBoundary(L, L, L)
    elif setup == "brick":  # the cell-list path: the bonded kernel maps original indices to slots through slot_of
        x = x - np.floor(x / L) * L
        x_oracle = x
        nf = mb.GPUNeighborFinder(dist_cutoff=1.2)
        pairs = (mb.LennardJones(cutoff=mb.DistanceCutoff(1.0), use_neighbors=True),)
        bnd, expect_path = mb.CubicBoundary(L, L, L), 1
    else:  # every atom moved by lattice vectors: bonded partners sit in different images
        bv = np.array([[L, 0, 0], [L, L, 0], [-L, 0, L]])
        x = x + rng.integers(-1, 2, (len(x), 3)) @ bv
        bnd, scale = mb.TriclinicBoundary(*bv), 10.0
    f, e, _, st = _run(_system(x, bnd, terms, dtype, nf=nf, pairs=pairs))
    f_ref, e_ref = _oracle(x_oracle, np.full(3, L), terms, dtype)
    assert st["path"] == expect_path
    _compare(f"kinds 0-2 {setup}", f, e, f_ref, e_ref, dtype, scale=scale if dtype == F32 else 1.0)


# ---- 5. the launch: the edges of the per-kind CTA ranges -----------------------------------------------------------------
def _rb_terms(n, rng, off, box=6.0):
    x, idx, _ = random_core_terms(bk.PERIODIC_TORSION, rng, n, box)
    return x, (bk.RB_TORSION, idx + off, rng.uniform(-20, 20, (n, 4)))


LAUNCH = {"1": {0: 1, 1: 1, 2: 1}, "127": {0: 127, 1: 127, 2: 127}, "128": {0: 128, 1: 128, 2: 128},
          "129": {0: 129, 1: 129, 2: 129}, "4097": {0: 4097, 1: 4097, 2: 4097}, "127-128-129": {0: 127, 1: 128, 2: 129},
          "kind0_empty": {1: 129, 2: 1, 9: 128}, "only_kind9": {9: 129}}


@DTYPES
@pytest.mark.parametrize("case", list(LAUNCH))
def test_launch_kind_ranges(case, dtype):
    rng = np.random.default_rng(7)
    xs, terms, off = [], [], 0
    for kind, n in LAUNCH[case].items():
        if kind == bk.RB_TORSION:
            x, t = _rb_terms(n, rng, off)
        else:
            x, idx, par = random_core_terms(kind, rng, n, 6.0)
            t = (kind, idx + off, par)
        xs.append(x)
        terms.append(t)
        off += len(x)
    x = np.concatenate(xs)
    f, e, _, _ = _run(_system(x, mb.CubicBoundary(6.0, 6.0, 6.0), terms, dtype))
    f_ref, e_ref = _oracle(x, np.full(3, 6.0), terms, dtype)
    _compare(f"launch {case}", f, e, f_ref, e_ref, dtype)
    # every term's atoms feel their force: a lost CTA leaves whole terms at zero
    for kind, idx, _ in terms:
        moved = np.abs(f_ref[np.asarray(idx)]).max(axis=(1, 2)) > 1e-3
        assert (np.abs(f[np.asarray(idx)]).max(axis=(1, 2))[moved] > 0).all(), kind


def test_mts_level_range_empty_for_one_kind():
    """MTSIntegrator with bonds at both levels, angles at level 0 only and torsions at level 1 only: each level's launch has
    an empty range for one kind (f64 trajectory against the numpy restatement of mts_substeps!)."""
    rng = np.random.default_rng(11)
    x, terms = _core_terms(40, rng, 2.5)
    bonds = terms[0]
    half = len(bonds[1]) // 2
    terms = [(bonds[0], bonds[1][:half], bonds[2][:half]), (bonds[0], bonds[1][half:], bonds[2][half:]), terms[1], terms[2]]
    si = (1, 2, 1, 2)
    sim = mb.MTSIntegrator(0.001, pi_fractions=(1,), si_fractions=si)
    v = rng.normal(0, 0.3, x.shape)
    box = np.full(3, 2.5)
    s = _system(x, mb.CubicBoundary(2.5, 2.5, 2.5), terms, F64)
    s.velocities[:] = v

    def level(lv):
        mine = [t for t, fr in zip(terms, si) if sim.ordered_fractions.index(fr) == lv]
        return lambda y: bk.specific_forces(y, box, _rounded(mine, F64))[0]
    n = 20
    x_ref, v_ref = mo.simulate_mts([level(0), level(1)], x, v, np.full(len(x), 12.0), sim.dt, n, sim.ordered_fractions,
                                   lambda y: y - np.floor(y / box) * box)
    try:
        mb.simulate(s, sim, n)
        ex, ev = _pos_err(s.coords, x_ref, box), np.abs(s.velocities - v_ref).max()
    finally:
        s.close()
    print(f"[MTS empty level ranges f64] dx={ex:.3e} dv={ev:.3e}")
    assert ex < 1e-9 and ev < 1e-8


# ---- 6. contention: one hub atom in 4096 angles and 4096 torsions --------------------------------------------------------
N_HUB = 4096


@DTYPES
def test_hub_atom_shared_by_angles_and_torsions(dtype):
    """The hub is the middle atom j of every angle and the second atom j of every torsion. Its force is a sum of 8192
    atomic adds in no fixed order: the bar is relative to the sum of the per-term forces' magnitudes on it,
    sqrt(8192) eps32 sum |f_t| in f32 (the typical error of a sum in any order), 1e-9 sum |f_t| in f64."""
    rng = np.random.default_rng(17)
    hub = np.array([1.5, 1.5, 1.5])
    copies, parts = [], []  # the same geometry with a private copy of the hub per term: the per-term hub forces
    xs, terms, off = [hub[None, :]], [], 1
    c_off = 0
    for kind in (bk.HARMONIC_ANGLE, bk.PERIODIC_TORSION):
        x, idx, par = random_core_terms(kind, rng, N_HUB, 3.0)
        na = bk.ATOMS[kind]
        x = x.reshape(N_HUB, na, 3)
        x = x - x[:, [1]] + hub  # atom 1 of every term on the hub
        copies.append(x.reshape(-1, 3))
        parts.append((kind, np.arange(N_HUB * na).reshape(N_HUB, na) + c_off, par))
        c_off += N_HUB * na
        rest = np.delete(x, 1, axis=1).reshape(-1, 3)
        own = np.arange(N_HUB * (na - 1)).reshape(N_HUB, na - 1) + off
        terms.append((kind, np.insert(own, 1, 0, axis=1), par))
        xs.append(rest)
        off += len(rest)
    x = np.concatenate(xs)
    f, e, _, _ = _run(_system(x, mb.CubicBoundary(3.0, 3.0, 3.0), terms, dtype))
    f_ref, e_ref = _oracle(x, np.full(3, 3.0), terms, dtype)
    # per-term forces on the hub, from the copies (f32-rounded hub position, as the engine sees it)
    xc = np.concatenate(copies)
    fc, _ = _oracle(xc, np.full(3, 3.0), parts, dtype)
    hub_rows = np.concatenate([p[1][:, 1] for p in parts])
    s_abs = np.linalg.norm(fc[hub_rows], axis=1).sum()
    err_hub = np.linalg.norm(f[0] - f_ref[0])
    unit = np.sqrt(2 * N_HUB) * EPS32 * s_abs if dtype == F32 else 1e-9 * s_abs
    print(f"[hub {np.dtype(dtype).name}] |dF_hub|={err_hub:.3e} |F_hub|={np.linalg.norm(f_ref[0]):.3e} sum|f_t|={s_abs:.3e} "
          f"ratio to bar {err_hub / unit:.3f}")
    assert err_hub <= unit
    _compare("hub, other atoms", f[1:], e, f_ref[1:], e_ref, dtype)
