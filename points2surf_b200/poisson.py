"""Screened Poisson surface reconstruction from oriented points (the SPSR baseline the paper compares against, which
the reference runs through meshlabserver with poisson.mlx): the solve on the GPU (ops.poisson_solve,
csrc/poisson.cu), the iso-surface by marching cubes (ops.marching_cubes, csrc/mc.cu), then world coordinates."""
import numpy as np
import torch

from . import ops
from . import sdf


def reconstruct(pts, normals, depth=8, point_weight=4.0, scale=1.1, iters=8):
    """pts, normals [N,3] (NumPy arrays or CUDA tensors) -> (verts [V,3] float32 world, faces [F,3] int32, report).
    The mesh is the zero level of iso - chi on the (2^depth + 1)^3 node grid, outward oriented (marching_cubes flips
    every face when the signed volume is negative).  report: ops.poisson_solve's dict plus 'mc_ms', the CUDA-event
    time of marching cubes and the world transform."""
    dev = sdf._device()
    p = torch.as_tensor(np.asarray(pts, np.float32) if not torch.is_tensor(pts) else pts, dtype=torch.float32).to(dev)
    n = torch.as_tensor(np.asarray(normals, np.float32) if not torch.is_tensor(normals) else normals,
                        dtype=torch.float32).to(dev)
    values, report = ops.poisson_solve(p, n, depth, point_weight, scale, iters)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    verts, faces = ops.marching_cubes(values, 0.0)
    # marching_cubes writes ((i + 0.5) / R - 0.5) * 2 for grid index i; node i lies at origin + edge * i / 2^depth
    R = values.shape[0]
    i = (verts.double() * 0.5 + 0.5) * R - 0.5
    origin = torch.tensor(report['origin'], dtype=torch.float64, device=dev)
    world = (origin[None, :] + i * (report['edge'] / (R - 1))).float()
    t1.record()
    t1.synchronize()
    report['mc_ms'] = t0.elapsed_time(t1)
    return world.cpu().numpy(), faces.cpu().numpy(), report
