"""Implicit solvent in decomposed (multi-GPU) contexts (needs >= 2 GPUs): mb_set_implicit_solvent refuses a decomposed
context, and a context that had GB set before mb_comm_init refuses the run, both with MB_ERR_INVALID and before any work."""
import os
import socket

import numpy as np
import pytest

import mbhelpers as H
import mollyb200 as mb

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _gb(n):
    return mb.ImplicitSolventOBC(offset_radii=np.full(n, 0.15), scaled_offset_radii=np.full(n, 0.12), alpha=1.0, beta=0.8,
                                 gamma=4.85)


def _worker(rank, world, port, out_dir):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    sd = H.lj_fluid(10, seed=9, dtype=np.float64, temp=120.0)
    inter = (mb.LennardJones(cutoff=mb.ShiftedForceCutoff(1.0), use_neighbors=True),)
    atoms = mb.atoms_from_arrays(sd["mass"], sd["charge"], sd["sigma"], sd["eps"], np.float64)
    out = []
    for gb_first in (False, True):
        nf = mb.GPUNeighborFinder(dist_cutoff=1.15, n_steps=20)
        s = mb.System(atoms=atoms, coords=sd["coords"].copy(), boundary=mb.CubicBoundary(*sd["box"]),
                      velocities=sd["velocities"].copy(), pairwise_inters=inter, neighbor_finder=nf, dtype=np.float64,
                      device=rank, general_inters=(_gb(sd["n"]),) if gb_first else ())
        s.engine()
        uid = [mb.comm_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(uid, src=0)
        mb.comm_init(s, uid[0], rank, world)
        x0 = s.coords.copy()
        try:
            if gb_first:
                mb.simulate(s, mb.VelocityVerlet(dt=0.002), 5)
            else:
                s._set_implicit_solvent(_gb(sd["n"]))
            out.append((0, ""))
        except mb.MollyB200Error as e:
            out.append((e.args[0] if e.args else 0, str(e)))
        assert np.array_equal(s.coords, x0)  # refused before any work
        s.close()
    np.save(os.path.join(out_dir, f"rank{rank}.npy"), np.array([str(o) for o in out]))
    dist.destroy_process_group()


def test_decomposed_context_refuses_implicit_solvent(tmp_path):
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    for rank in range(2):
        res = np.load(tmp_path / f"rank{rank}.npy")
        print(rank, res)
        assert len(res) == 2
        for r in res:
            assert str(mb.capi.MB_ERR_INVALID) in r and "decomposed" in r, r
