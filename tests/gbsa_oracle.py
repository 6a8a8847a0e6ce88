"""numpy restatement (f64) of the reference's generalized-Born implicit solvent, ImplicitSolventOBC and ImplicitSolventGBN2
(src/interactions/implicit_solvent.jl), for per-atom arrays: the Born radii (born_radii_loop_OBC / _GBN2 and
born_radii_sum, :623-725), the forces (gb_force_loop_1 / _2 and forces!, :839-929, :1078-1093) and the energy
(gb_energy_loop, :1095-1150). Minimum image for rectangular boxes and, through oracle/triclinic.py's Triclinic, for
TriclinicBoundary. n x n arrays throughout: meant for systems of a few thousand atoms."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

COULOMB_CONST = 138.93545764  # kJ mol^-1 nm e^-2


@dataclass
class GB:
    """One GB interaction at array level: per-atom offset radii, scaled offset radii and alpha/beta/gamma (OBC passes its
    three scalars broadcast); for GBN2 also per-atom neck classes and the class tables d0[c_i, c_j] = d0s[i, j]."""
    offset_radii: np.ndarray
    scaled_offset_radii: np.ndarray
    alpha: np.ndarray
    beta: np.ndarray
    gamma: np.ndarray
    offset: float
    dist_cutoff: float = 0.0
    probe_radius: float = 0.14
    sa_factor: float = 28.3919551
    factor_solute: float = -COULOMB_CONST / 1.0
    factor_solvent: float = COULOMB_CONST / 78.5
    kappa: float = 0.0
    use_ace: bool = True
    neck_class: np.ndarray = None
    d0: np.ndarray = None
    m0: np.ndarray = None
    neck_scale: float = 0.826836
    neck_cut: float = 0.68
    extra: dict = field(default_factory=dict)

    @property
    def has_neck(self):
        return self.neck_class is not None and self.d0 is not None and len(self.d0) > 0


def displacements(x, box=None, tric=None):
    """d[i, j] = minimum-image x[j] - x[i] (the reference's vector(coords[i], coords[j], boundary))."""
    x = np.asarray(x, np.float64)
    d = x[None, :, :] - x[:, None, :]
    if tric is not None:  # approx_images (src/spatial.jl:528-534): z, then y, then x
        for k in (2, 1, 0):
            d = d - tric.bv[k] * np.floor(d[..., k] * tric.rs[k] + 0.5)[..., None]
    elif box is not None:
        box = np.asarray(box, np.float64)
        d = d - box * np.round(d / box)
    return d


def born_radii(x, p: GB, box=None, tric=None):
    """(B, B', I'_ij, d, r): Born radii, their gradients with respect to I, the neck derivative table and the geometry."""
    d = displacements(x, box, tric)
    r = np.sqrt(np.einsum("ijk,ijk->ij", d, d))
    n = len(r)
    rc = p.dist_cutoff
    valid = (r > 0) & ((rc == 0) | (r <= rc))
    ori = np.asarray(p.offset_radii, np.float64)[:, None]
    srj = np.asarray(p.scaled_offset_radii, np.float64)[None, :]
    with np.errstate(divide="ignore", invalid="ignore"):
        U = r + srj
        L = np.maximum(ori, np.abs(r - srj))
        t = (1 / L - 1 / U + (r - srj ** 2 / r) * (1 / U ** 2 - 1 / L ** 2) / 4 + np.log(L / U) / (2 * r)) / 2
        t = t + np.where(ori < srj - r, 2 * (1 / ori - 1 / L), 0.0)
        Iij = np.where(valid & (ori < U), t, 0.0)
        ig = np.zeros((n, n))
        if p.has_neck:
            rad = np.asarray(p.offset_radii, np.float64) + p.offset
            cond = valid & (r < rad[:, None] + rad[None, :] + p.neck_cut)
            c = np.asarray(p.neck_class)
            d0 = np.asarray(p.d0, np.float64)[c[:, None], c[None, :]]
            m0 = np.asarray(p.m0, np.float64)[c[:, None], c[None, :]]
            s = 10 * (r - d0)  # the integral uses Angstrom
            denom = 1 + s ** 2 + 3 * s ** 6 / 10
            Iij = Iij + np.where(cond, p.neck_scale * m0 / denom, 0.0)
            ig = np.where(cond, -10 * p.neck_scale * m0 * (2 * s + 9 * s ** 5 / 5) / denom ** 2, 0.0)
    I = Iij.sum(1)
    orr = np.asarray(p.offset_radii, np.float64)
    radius = orr + p.offset
    psi = I * orr
    a, b, g = (np.broadcast_to(np.asarray(v, np.float64), orr.shape) for v in (p.alpha, p.beta, p.gamma))
    th = np.tanh(a * psi - b * psi ** 2 + g * psi ** 3)
    B = 1 / (1 / orr - th / radius)
    Bg = (1 - th ** 2) * orr * (a - 2 * b * psi + 3 * g * psi ** 2) / radius
    return B, Bg, ig, d, r


def _pre(p: GB, den, with_derivative):
    if p.kappa == 0:
        return p.factor_solute + p.factor_solvent
    e = np.exp(-p.kappa * den)
    pre = p.factor_solute + e * p.factor_solvent
    return pre + p.kappa * den * e * p.factor_solvent if with_derivative else pre


def forces_energy(x, charge, p: GB, box=None, tric=None):
    """GB forces (n, 3) and energy (kJ/mol) of coordinates x with charges `charge`."""
    q = np.asarray(charge, np.float64)
    B, Bg, ig, d, r = born_radii(x, p, box, tric)
    n = len(q)
    rc = p.dist_cutoff
    r2 = r * r
    off = ~np.eye(n, dtype=bool)
    orr = np.asarray(p.offset_radii, np.float64)
    radius = orr + p.offset
    # gb_force_loop_1 for every ordered pair (the self pair at r2 = 0 feeds the Born force only)
    inside = (rc == 0) | (r2 <= rc * rc)
    a2 = B[:, None] * B[None, :]
    D = r2 / (4 * a2)
    ex = np.exp(-D)
    den2 = r2 + a2 * ex
    den = np.sqrt(den2)
    G = _pre(p, den, True) * q[:, None] * q[None, :] / den
    dGdr = np.where(inside & off, -G * (1 - ex / 4) / den2, 0.0)
    dGda = np.where(inside, -G * ex * (1 + D) / (2 * den2), 0.0)
    f = np.einsum("ijk,ij->ik", d, dGdr)
    if p.use_ace:
        sa = p.sa_factor * (radius + p.probe_radius) ** 2 * (radius / B) ** 6
        bf = np.where(B > 0, -6 * sa / B, 0.0)
    else:
        sa = np.zeros(n)
        bf = np.zeros(n)
    bf = bf + (dGda * B[None, :]).sum(1)
    bi = bf * B ** 2 * Bg
    # gb_force_loop_2: de_ij = b_i (t3_ij - I'_ij) / r, zero unless or_i < r + sr_j
    srj = np.asarray(p.scaled_offset_radii, np.float64)[None, :]
    ori = orr[:, None]
    valid = (r > 0) & ((rc == 0) | (r <= rc)) & (ori < r + srj)
    with np.errstate(divide="ignore", invalid="ignore"):
        Li = 1 / np.maximum(ori, np.abs(r - srj))
        Ui = 1 / (r + srj)
        r2inv = 1 / r2
        t3 = (1 + srj ** 2 * r2inv) * (Li ** 2 - Ui ** 2) / 8 + np.log(Ui / Li) * r2inv / 4
        de = np.where(valid, bi[:, None] * (t3 - ig) / r, 0.0)
    f = f - np.einsum("ijk,ij->ik", d, de + de.T)
    # gb_energy_loop
    self_pre = p.factor_solute + p.factor_solvent if p.kappa == 0 else p.factor_solute + np.exp(-p.kappa * B) * p.factor_solvent
    e = np.sum(self_pre * q ** 2 / (2 * B))
    if p.use_ace:
        e += np.sum(np.where(B > 0, sa, 0.0))
    iu = np.triu(np.ones((n, n), bool), 1) & inside
    fe = np.sqrt(r2 + a2 * np.exp(-r2 / (4 * a2)))
    fc = 1 / fe - (1 / rc if rc > 0 else 0.0)
    e += np.sum(np.where(iu, _pre(p, fe, False) * q[:, None] * q[None, :] * fc, 0.0))
    return f, float(e)


def energy(x, charge, p: GB, box=None, tric=None):
    return forces_energy(x, charge, p, box, tric)[1]


def from_golden(g, model: str, **over) -> GB:
    """The GB interaction of tests/golden/6mrr_gb.npz for model "obc2" or "gbn2" (keyword overrides: kappa, dist_cutoff, ...)."""
    kw = dict(offset_radii=g[f"{model}_offset_radii"], scaled_offset_radii=g[f"{model}_scaled_offset_radii"],
              alpha=g[f"{model}_alpha"], beta=g[f"{model}_beta"], gamma=g[f"{model}_gamma"], offset=float(g[f"{model}_offset"]),
              kappa=float(g["kappa"]))
    if model == "gbn2":
        kw.update(neck_class=g["gbn2_neck_class"], d0=g["gbn2_d0"], m0=g["gbn2_m0"])
    kw.update(over)
    return GB(**kw)
