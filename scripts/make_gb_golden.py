"""Generate tests/golden/6mrr_gb.npz: 6mrr without water (data/6mrr_nowater.pdb, ff99SBildn) with the per-atom
generalized-Born arrays of ImplicitSolventOBC(use_OBC2=true) and ImplicitSolventGBN2, and OpenMM's forces and energies of
the reference's "Implicit solvent" test (test/protein.jl:663-707: 100 nm box, LJ + Coulomb with DistanceCutoff(5 nm),
kappa = 1 nm^-1).

Run where a checkout of the reference is available: python scripts/make_gb_golden.py /path/to/Molly.jl
The element-to-radius, element-to-screen and GBN2 parameter dictionaries and the 21 x 21 d0/m0 tables are read from the
reference's src/interactions/implicit_solvent.jl at generation time; only the arrays derived from them are written.
mbondi2_radii / mbondi3_radii and lookup_table (:253-320) are restated below."""
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ffreader as fr  # noqa: E402

NUCLEIC = ("A", "C", "G", "U", "DA", "DC", "DG", "DT")
OBC_OFFSET, GBN2_OFFSET = 0.009, 0.0195141


def _dicts(src):
    out = {}
    for m in re.finditer(r"const (\w+) = Dict\((.*?)\n\)", src, re.S):
        out[m.group(1)] = {k: float(v) for k, v in re.findall(r'"([^"]+)"\s*=>\s*([-0-9.eE]+)', m.group(2))}
    return out


def _table(src, name):
    """A 21 x 21 table in nm units: the literal list with the unit conversion written after it (`]u"nm" ./ 10`)."""
    m = re.search(rf"const {name} = \[(.*?)\][^\n]*?\.([*/])\s*([0-9.]+)\n", src, re.S)
    vals = np.array([float(v) for v in re.findall(r"[-0-9.eE]+", m.group(1))])
    assert len(vals) == 21 * 21, name
    return vals / float(m.group(3)) if m.group(2) == "/" else vals * float(m.group(3))


def mbondi_radii(elements, types, atom_names, res_names, bonds, radius, mbondi3):
    n = len(elements)
    to_n = np.zeros(n, bool)
    for i, j in bonds:
        if elements[i] == "N":
            to_n[j] = True
        if elements[j] == "N":
            to_n[i] = True
    out = np.zeros(n)
    for k in range(n):
        if mbondi3 and res_names[k] == "ARG" and (atom_names[k].startswith("HH") or atom_names[k].startswith("HE")):
            out[k] = radius["H_ARG"]
        elif mbondi3 and types[k] == "O2":
            out[k] = radius["O_CAR"]
        elif elements[k] in ("H", "D"):
            out[k] = radius["H_N"] if to_n[k] else radius["H"]
        else:
            out[k] = radius.get(elements[k], radius["-"])
    return out


def _lookup_weights(r):
    p = (r - 0.1) * 200
    if p <= 0:
        return [(0, 1.0)]
    if p >= 20:
        return [(20, 1.0)]
    i1 = int(np.floor(p))
    w1 = (i1 + 1) - p
    return [(i1, w1), (i1 + 1, 1.0 - w1)]


def class_table(full, radii_of_class):
    """t[c_i, c_j] = the reference's lookup_table(full, radii)[i, j] for atoms i, j of classes c_i, c_j: the entry
    table[j, i] sums full[idx(i) * 21 + idx(j)], so t[c_i, c_j] reads full[idx(c_j) * 21 + idx(c_i)]."""
    nc = len(radii_of_class)
    t = np.zeros((nc, nc))
    for ci in range(nc):
        for cj in range(nc):
            s = 0.0
            for a, wa in _lookup_weights(radii_of_class[cj]):
                for b, wb in _lookup_weights(radii_of_class[ci]):
                    s += wa * wb * full[a * 21 + b]
            t[ci, cj] = s
    return t


def main(ref):
    data = os.path.join(ref, "data")
    src = open(os.path.join(ref, "src", "interactions", "implicit_solvent.jl")).read()
    D = _dicts(src)
    ff = fr.read_force_field(f"{data}/force_fields/ff99SBildn.xml")
    atoms, _ = fr.read_pdb(f"{data}/6mrr_nowater.pdb")
    top = fr.build_topology(atoms, ff)
    types = top["types"]
    elements = [ff.type_element.get(t, "") for t in types]
    names = [a.name for a in atoms]
    res = [a.resname for a in atoms]
    bonds = top["bonds"]
    out = dict(box=np.array([100.0, 100.0, 100.0]), coords=np.array([a.xyz for a in atoms], np.float64), mass=top["mass"],
               charge=top["charge"], sigma=top["sigma"], eps=top["eps"], excluded=top["excluded"], special=top["special"],
               lj14scale=np.float64(ff.lj14scale), coulomb14scale=np.float64(ff.coulomb14scale), dist_cutoff=np.float64(5.0),
               kappa=np.float64(1.0))
    for key in ("bond_idx", "bond_par", "angle_idx", "angle_par", "proper_idx", "proper_par", "improper_idx", "improper_par"):
        out[key] = top[key]
    radius = D["mbondi2_element_to_radius"]
    # ImplicitSolventOBC(...; use_OBC2=true)
    r2 = mbondi_radii(elements, types, names, res, bonds, radius, False)
    or2 = r2 - OBC_OFFSET
    scr = D["obc_element_to_screen"]
    out["obc2_offset_radii"] = or2
    out["obc2_scaled_offset_radii"] = np.array([scr.get(e, scr["-"]) for e in elements]) * or2
    out["obc2_alpha"], out["obc2_beta"], out["obc2_gamma"] = (np.full(len(or2), v) for v in (1.0, 0.8, 4.85))
    out["obc2_offset"] = np.float64(OBC_OFFSET)
    # ImplicitSolventGBN2(...)
    r3 = mbondi_radii(elements, types, names, res, bonds, radius, True)
    or3 = r3 - GBN2_OFFSET
    sp, spn = D["gbn2_element_to_screen"], D["gbn2_element_to_screen_nucleic"]
    ap, apn = D["gbn2_atom_params"], D["gbn2_atom_params_nucleic"]
    nuc = [r in NUCLEIC for r in res]
    out["gbn2_offset_radii"] = or3
    out["gbn2_scaled_offset_radii"] = np.array([(spn if u else sp).get(e, (spn if u else sp)["-"])
                                                for e, u in zip(elements, nuc)]) * or3
    for g in ("α", "β", "γ"):
        key = {"α": "alpha", "β": "beta", "γ": "gamma"}[g]
        out[f"gbn2_{key}"] = np.array([(apn if u else ap).get(f"{e}_{g}", (apn if u else ap)[f"-_{g}"])
                                       for e, u in zip(elements, nuc)])
    out["gbn2_offset"] = np.float64(GBN2_OFFSET)
    # neck classes: the distinct radii (offset_radii + offset) in increasing order
    cls_r, cls = np.unique(r3, return_inverse=True)
    out["gbn2_neck_class"] = cls.astype(np.int32)
    out["gbn2_d0"] = class_table(_table(src, "gbn2_data_d0"), cls_r)
    out["gbn2_m0"] = class_table(_table(src, "gbn2_data_m0"), cls_r)
    amber = f"{data}/openmm_6mrr/amber"
    for m in ("obc2", "gbn2"):
        out[f"forces_{m}"] = np.loadtxt(f"{amber}/forces_{m}.txt")
        out[f"energy_{m}"] = np.float64(open(f"{amber}/energy_{m}.txt").read())
    path = os.path.join(ROOT, "tests", "golden", "6mrr_gb.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path) / 1e3, "kB;", len(or3), "atoms,", len(cls_r), "neck classes,",
          int(np.sum(r3 != r2)), "radii changed by mbondi3")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit("usage: python scripts/make_gb_golden.py /path/to/Molly.jl")
    main(sys.argv[1])
