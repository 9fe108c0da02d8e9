"""Measure the tensor-core path's logit error against the fp32 path on the benchmark workload and the number
of sign-class mismatches that a guard band of a given width would leave (run on the GPU):
    python tools/guard_study.py [n_queries]
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from points2surf_b200 import ops, synth  # noqa: E402


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 16384
    dev = torch.device('cuda', 0)
    for variant, seed in (('vanilla', 6), ('max', 4)):
        v = synth.VARIANTS[variant]
        sd = synth.make_state_dict(variant, seed)
        cloud = synth.make_cloud('sphere', 10000, seed=0)
        pts = torch.from_numpy(cloud).to(dev)
        lin = ops.query_grid(pts, 256, 3)
        sel = torch.linspace(0, lin.numel() - 1, n, device=dev).long()
        q = ops.query_points(lin[sel].contiguous(), 256)
        _, patch, radius = ops.knn_patch(pts, q, 300)
        sub = ops.gather_points(pts, ops.subsample(pts, q, 1000, bool(v['uniform_subsample']), 1))
        e32 = ops.Engine(sd, v['use_point_stn'], v['shared_transformer'], precision='fp32')
        ref = torch.cat([e32.forward(patch[i:i + 2048], sub[i:i + 2048], q[i:i + 2048]) for i in range(0, n, 2048)])
        # centre the sign logit like bench.py does (mixed sign classes)
        bias = ref.median(dim=0).values
        etc = ops.Engine(sd, v['use_point_stn'], v['shared_transformer'], precision='tc', guard_band=0.0)
        out = torch.cat([etc.forward(patch[i:i + 8192], sub[i:i + 8192], q[i:i + 8192]) for i in range(0, n, 8192)])
        ref, out = (ref - bias).cpu().numpy(), (out - bias).cpu().numpy()
        err = np.abs(out - ref)
        print('%s: n=%d  logit scale (std) %.2f / %.2f' % (variant, n, ref[:, 0].std(), ref[:, 1].std()))
        print('  |err| sign logit: mean %.4f  p99 %.4f  p99.9 %.4f  max %.4f ; magnitude logit max %.4f'
              % (err[:, 1].mean(), np.percentile(err[:, 1], 99), np.percentile(err[:, 1], 99.9), err[:, 1].max(), err[:, 0].max()))
        for band in (0.0, 0.02, 0.05, 0.1):
            inside = np.abs(out[:, 1]) < band
            mism = ((out[:, 1] >= 0) != (ref[:, 1] >= 0)) & ~inside
            print('  band %.2f: %.2f %% of queries recomputed, %d sign mismatches left outside the band' % (band, 100 * inside.mean(), int(mism.sum())))


if __name__ == '__main__':
    main()
