"""numpy restatement of Molly's bonded terms (TEST INFRASTRUCTURE): HarmonicBond, HarmonicAngle, PeriodicTorsion.

Formulas: SURVEY.md Appendix B.1 — src/interactions/harmonic_bond.jl:13-54, harmonic_angle.jl:45-67,
periodic_torsion.jl:17-142 (dihedral by atan2, spatial.jl:882-894). All displacements are minimum-image
(`vector`, src/spatial.jl:491-519). Returns forces (n,3) and the energy.

Degenerate geometry as in the engine: an angle or torsion whose cross product is exactly zero (collinear atoms) gets no
force and keeps its energy, and the bend angle is atan2(|ba x bc|, ba . bc), which keeps its digits near 0 and pi."""
import numpy as np


def _mic(d, box):
    return d - box * np.round(d / box)


def bond_forces(x, box, idx, par):
    f = np.zeros_like(x)
    ab = _mic(x[idx[:, 1]] - x[idx[:, 0]], box)
    r = np.linalg.norm(ab, axis=1)
    k, r0 = par[:, 0], par[:, 1]
    c = k * (r - r0)
    fi = (c / r)[:, None] * ab
    np.add.at(f, idx[:, 0], fi)
    np.add.at(f, idx[:, 1], -fi)
    return f, float(np.sum(0.5 * k * (r - r0) ** 2))


def bend_angle(ba, bc):
    """theta = atan2(|ba x bc|, ba . bc): the angle of bond_angle (src/spatial.jl:845-853) to full precision at every
    angle; acos of the cosine loses digits near 0 and pi. Exactly collinear vectors give exactly 0 or pi."""
    n = np.cross(ba, bc)
    return np.arctan2(np.sqrt(np.sum(n * n, 1)), np.sum(ba * bc, 1)), n


def angle_forces(x, box, idx, par):
    """No force where ba x bc is exactly zero (harmonic_angle.jl:45-53); the energy is counted there too."""
    f = np.zeros_like(x)
    ba = _mic(x[idx[:, 0]] - x[idx[:, 1]], box)
    bc = _mic(x[idx[:, 2]] - x[idx[:, 1]], box)
    nba, nbc = np.linalg.norm(ba, axis=1), np.linalg.norm(bc, axis=1)
    th, n = bend_angle(ba, bc)
    k, th0 = par[:, 0], par[:, 1]
    bent = np.sum(n * n, 1) > 0
    pa = np.cross(ba, n)
    pc = np.cross(-bc, n)
    with np.errstate(divide="ignore", invalid="ignore"):
        pa = np.where(bent[:, None], pa / np.linalg.norm(pa, axis=1)[:, None], 0.0)
        pc = np.where(bent[:, None], pc / np.linalg.norm(pc, axis=1)[:, None], 0.0)
    t = -k * (th - th0)
    fa = (t / nba)[:, None] * pa
    fc = (t / nbc)[:, None] * pc
    np.add.at(f, idx[:, 0], fa)
    np.add.at(f, idx[:, 2], fc)
    np.add.at(f, idx[:, 1], -fa - fc)
    return f, float(np.sum(0.5 * k * (th - th0) ** 2))


def torsion_arms(ab, bc, cd, m, n, nbc, dedth):
    """The forces fi, fl on the end atoms and the lever term v of dE/dtheta (periodic_torsion_force): f_j = v - fi,
    f_k = -v - fl. All zero where m = ab x bc or n = bc x cd is exactly zero (three collinear atoms), as in the engine;
    the reference divides by zero there."""
    m2, n2 = np.sum(m * m, 1), np.sum(n * n, 1)
    ok = (m2 > 0) & (n2 > 0)
    dedth = np.where(ok, dedth, 0.0)
    m2, n2, nbc2 = np.where(ok, m2, 1.0), np.where(ok, n2, 1.0), np.where(ok, nbc ** 2, 1.0)
    fi = (dedth * nbc / m2)[:, None] * m
    fl = (-dedth * nbc / n2)[:, None] * n
    v = ((-np.sum(ab * bc, 1)) / nbc2)[:, None] * fi - ((-np.sum(cd * bc, 1)) / nbc2)[:, None] * fl
    return fi, fl, v


def torsion_forces(x, box, idx, par):
    """The energy k (1 + cos(n theta - phase)) is counted at every geometry, the force only where torsion_arms gives one."""
    f = np.zeros_like(x)
    if len(idx) == 0:
        return f, 0.0
    ab = _mic(x[idx[:, 1]] - x[idx[:, 0]], box)
    bc = _mic(x[idx[:, 2]] - x[idx[:, 1]], box)
    cd = _mic(x[idx[:, 3]] - x[idx[:, 2]], box)
    m = np.cross(ab, bc)
    n = np.cross(bc, cd)
    nbc = np.linalg.norm(bc, axis=1)
    th = np.arctan2(np.sum(np.cross(m, n) * bc, 1) / nbc, np.sum(m * n, 1))
    per, phase, k = par[:, 0], par[:, 1], par[:, 2]
    dedth = -k * per * np.sin(per * th - phase)
    fi, fl, v = torsion_arms(ab, bc, cd, m, n, nbc, dedth)
    fj = v - fi
    fk = -v - fl
    for col, ff in zip(range(4), (fi, fj, fk, fl)):
        np.add.at(f, idx[:, col], ff)
    return f, float(np.sum(k * (1.0 + np.cos(per * th - phase))))
