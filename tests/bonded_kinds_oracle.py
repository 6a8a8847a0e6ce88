"""numpy restatement of the specific interaction kinds beyond HarmonicBond, HarmonicAngle and PeriodicTorsion (which
oracle/bonded.py restates), TEST INFRASTRUCTURE. Float64, rectangular box, minimum-image displacements (`vector`,
src/spatial.jl:491-519). Each function takes 0-based atom indices (n_terms x atoms) and parameters (n_terms x params) in
the layout of mb_set_specific (include/mollyb200.h) and returns forces (n, 3) and the energy.

Formulas: src/interactions/harmonic_position_restraint.jl:18-32, morse_bond.jl:24-38, fene_bond.jl:31-64,
cosine_angle.jl:19-42, urey_bradley.jl:32-61, harmonic_torsion.jl:27-44, rb_torsion.jl:19-43; bond_angle and
torsion_vectors (src/spatial.jl:845-894), with the bend angle and the degenerate geometry of oracle/bonded.py.
RBTorsion's force is -grad E by default; reference_sign=True restates rb_torsion.jl:30 as written, whose dE/dtheta has
the opposite sign."""
import numpy as np

from oracle import bonded as bd

(HARMONIC_BOND, HARMONIC_ANGLE, PERIODIC_TORSION, POSITION_RESTRAINT, MORSE_BOND, FENE_BOND, COSINE_ANGLE, UREY_BRADLEY,
 HARMONIC_TORSION, RB_TORSION) = range(10)
ATOMS = (2, 3, 4, 1, 2, 2, 3, 3, 4, 4)
PARAMS = (2, 2, 3, 4, 3, 4, 2, 4, 2, 4)


def _mic(d, box):
    return d - box * np.round(d / box)


def _rows(a):
    return np.asarray(a, np.float64).reshape(-1)


def restraint_forces(x, box, idx, par):
    f = np.zeros_like(x)
    i = idx[:, 0]
    d = _mic(par[:, 1:4] - x[i], box)  # vector(x_i, x0)
    k = par[:, 0]
    np.add.at(f, i, k[:, None] * d)
    return f, float(np.sum(0.5 * k * np.sum(d * d, 1)))


def morse_forces(x, box, idx, par):
    f = np.zeros_like(x)
    dr = _mic(x[idx[:, 1]] - x[idx[:, 0]], box)
    r = np.linalg.norm(dr, axis=1)
    D, a, r0 = par[:, 0], par[:, 1], par[:, 2]
    ralp = np.exp(-a * (r - r0))
    c = 2 * D * a * (1 - ralp) * ralp
    fi = (c / r)[:, None] * dr
    np.add.at(f, idx[:, 0], fi)
    np.add.at(f, idx[:, 1], -fi)
    return f, float(np.sum(D * (1 - ralp) ** 2))


def fene_forces(x, box, idx, par):
    f = np.zeros_like(x)
    dr = _mic(x[idx[:, 1]] - x[idx[:, 0]], box)
    r2 = np.sum(dr * dr, 1)
    k, r0, sig, eps = par[:, 0], par[:, 1], par[:, 2], par[:, 3]
    sr6 = sig ** 6 / r2 ** 3
    wca = np.sqrt(r2) < sig * 2 ** (1 / 6)
    fwca = np.where(wca, 24 * eps / r2 * (2 * sr6 * sr6 - sr6), 0.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        fj = (fwca - k / (1 - r2 / r0 ** 2))[:, None] * dr
        e = -0.5 * k * r0 ** 2 * np.log(1 - r2 / r0 ** 2) + np.where(wca, 4 * eps * (sr6 * sr6 - sr6) + eps, 0.0)
    np.add.at(f, idx[:, 0], -fj)
    np.add.at(f, idx[:, 1], fj)
    return f, float(np.sum(e))


def _bend(x, box, idx):
    ba = _mic(x[idx[:, 0]] - x[idx[:, 1]], box)
    bc = _mic(x[idx[:, 2]] - x[idx[:, 1]], box)
    nba, nbc = np.linalg.norm(ba, axis=1), np.linalg.norm(bc, axis=1)
    th, n = bd.bend_angle(ba, bc)
    bent = np.sum(n * n, 1) > 0
    pa, pc = np.cross(ba, n), np.cross(-bc, n)
    with np.errstate(divide="ignore", invalid="ignore"):
        pa = np.where(bent[:, None], pa / np.linalg.norm(pa, axis=1)[:, None], 0.0)
        pc = np.where(bent[:, None], pc / np.linalg.norm(pc, axis=1)[:, None], 0.0)
    return th, nba, nbc, pa, pc


def _bend_add(f, idx, t, nba, nbc, pa, pc):
    fa = (t / nba)[:, None] * pa
    fc = (t / nbc)[:, None] * pc
    np.add.at(f, idx[:, 0], fa)
    np.add.at(f, idx[:, 2], fc)
    np.add.at(f, idx[:, 1], -fa - fc)


def cosine_angle_forces(x, box, idx, par):
    f = np.zeros_like(x)
    th, nba, nbc, pa, pc = _bend(x, box, idx)
    k, th0 = par[:, 0], par[:, 1]
    _bend_add(f, idx, k * np.sin(th - th0), nba, nbc, pa, pc)
    return f, float(np.sum(k * (1 + np.cos(th - th0))))


def urey_bradley_forces(x, box, idx, par):
    f = np.zeros_like(x)
    th, nba, nbc, pa, pc = _bend(x, box, idx)
    ka, th0, kb, r0 = par[:, 0], par[:, 1], par[:, 2], par[:, 3]
    _bend_add(f, idx, -ka * (th - th0), nba, nbc, pa, pc)
    ik = _mic(x[idx[:, 2]] - x[idx[:, 0]], box)
    rik = np.linalg.norm(ik, axis=1)
    fb = (kb * (rik - r0) / rik)[:, None] * ik
    np.add.at(f, idx[:, 0], fb)
    np.add.at(f, idx[:, 2], -fb)
    return f, float(np.sum(0.5 * ka * (th - th0) ** 2 + 0.5 * kb * (rik - r0) ** 2))


def _torsion(x, box, idx):
    ab = _mic(x[idx[:, 1]] - x[idx[:, 0]], box)
    bc = _mic(x[idx[:, 2]] - x[idx[:, 1]], box)
    cd = _mic(x[idx[:, 3]] - x[idx[:, 2]], box)
    m, n = np.cross(ab, bc), np.cross(bc, cd)
    nbc = np.linalg.norm(bc, axis=1)
    th = np.arctan2(np.sum(np.cross(m, n) * bc, 1) / nbc, np.sum(m * n, 1))
    return ab, bc, cd, m, n, nbc, th


def _torsion_add(f, idx, geo, dedth):
    ab, bc, cd, m, n, nbc, _ = geo
    fi, fl, v = bd.torsion_arms(ab, bc, cd, m, n, nbc, dedth)
    for col, ff in zip(range(4), (fi, v - fi, -v - fl, fl)):
        np.add.at(f, idx[:, col], ff)


def harmonic_torsion_forces(x, box, idx, par):
    f = np.zeros_like(x)
    geo = _torsion(x, box, idx)
    th = geo[-1]
    k, th0 = par[:, 0], par[:, 1]
    _torsion_add(f, idx, geo, 2 * k * (th - th0))
    return f, float(np.sum(k * (th - th0) ** 2))


def rb_torsion_forces(x, box, idx, par, reference_sign=False):
    f = np.zeros_like(x)
    geo = _torsion(x, box, idx)
    th = geo[-1]
    f1, f2, f3, f4 = par[:, 0], par[:, 1], par[:, 2], par[:, 3]
    dedth = (-f1 * np.sin(th) + 2 * f2 * np.sin(2 * th) - 3 * f3 * np.sin(3 * th)) / 2
    _torsion_add(f, idx, geo, -dedth if reference_sign else dedth)
    return f, float(np.sum((f1 * (1 + np.cos(th)) + f2 * (1 - np.cos(2 * th)) + f3 * (1 + np.cos(3 * th)) + f4) / 2))


FORCES = {HARMONIC_BOND: bd.bond_forces, HARMONIC_ANGLE: bd.angle_forces, PERIODIC_TORSION: bd.torsion_forces,
          POSITION_RESTRAINT: restraint_forces, MORSE_BOND: morse_forces, FENE_BOND: fene_forces,
          COSINE_ANGLE: cosine_angle_forces, UREY_BRADLEY: urey_bradley_forces, HARMONIC_TORSION: harmonic_torsion_forces,
          RB_TORSION: rb_torsion_forces}


def specific_forces(x, box, lists):
    """Sum over (kind, 0-based idx, par) triples, e.g. from oracle_lists(): forces (n, 3) and energy."""
    x = np.asarray(x, np.float64)
    f = np.zeros_like(x)
    e = 0.0
    for kind, idx, par in lists:
        if len(idx):
            ff, ee = FORCES[kind](x, np.asarray(box, np.float64), idx, par)
            f += ff
            e += ee
    return f, e


def oracle_lists(sils):
    """mollyb200 list objects -> (kind, 0-based idx, par) triples."""
    out = []
    for s in sils:
        idx, par = s.arrays()
        out.append((s.kind, idx.astype(np.int64) - 1, par))
    return out
