#!/usr/bin/env python
"""Phase trace of the fp16 pass kernel (pointnet_pass_kernel<false>, csrc/net_tc.cu) on the bench workload.

Builds a traced copy of the library in a temporary directory: net_tc.cu is recompiled with the build's nvcc flags plus
-DP2S_PASS_TRACE and linked with the other objects of the in-tree build (run `python -m points2surf_b200.build` first).
Then it loads that copy instead of the package's library, runs one reconstruction of bench.py's headline workload
(vanilla model, one synthetic 10k-point sphere, grid_res 256, epsilon 3) after one warm-up, and prints, per pass class,
each phase's share of the warpgroups' clock cycles.  In the traced kernel thread 0 of each warpgroup reads clock64() at
every phase boundary, so the traced kernel itself runs a little slower than the default build.

    python tools/pass_trace.py [--grid_res 256] [--epsilon 3] [--points 10000]
"""
import argparse
import ctypes as C
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PHASES = ['query start', 'point load + first layer', 'mid layers', 'wait on empty', 'send', 'big layer, own tile',
          'wait on full', 'receive', 'big layer, received tile', 'query end: reduction + store']
CLASSES = ['pass A', 'pass B/C local', 'pass B/C global']


def build_traced(out_dir):
    from points2surf_b200 import build as b
    objs = sorted(os.path.join(b.OBJ, f) for f in os.listdir(b.OBJ) if f.endswith('.o') and f != 'net_tc.o')
    if not objs or not os.path.exists(os.path.join(b.OBJ, 'net_tc.o')):
        raise SystemExit('no in-tree objects under %s: run `python -m points2surf_b200.build` first' % b.OBJ)
    obj = os.path.join(out_dir, 'net_tc_trace.o')
    lib = os.path.join(out_dir, 'libp2s_b200.so')
    for cmd in ([b.NVCC] + b.FLAGS + ['-DP2S_PASS_TRACE', '-c', os.path.join(b.CSRC, 'net_tc.cu'), '-o', obj],
                [b.NVCC, '-shared', '-o', lib, obj] + objs + ['-lcudart']):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise SystemExit('traced build failed')
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--grid_res', type=int, default=256)
    ap.add_argument('--epsilon', type=int, default=3)
    ap.add_argument('--points', type=int, default=10000)
    ap.add_argument('--seed', type=int, default=40938661)
    args = ap.parse_args()

    tmp = tempfile.mkdtemp(prefix='p2s_pass_trace_')
    lib_path = build_traced(tmp)
    from points2surf_b200 import _lib
    _lib.LIB_PATH = lib_path                     # every later _lib.load() opens the traced copy
    lib = _lib.load()
    lib.p2s_pass_trace_read.restype = C.c_int
    lib.p2s_pass_trace_read.argtypes = [C.c_void_p, C.c_int]

    import numpy as np
    import torch
    from points2surf_b200 import ops, synth
    v = synth.VARIANTS['vanilla']
    sd = synth.make_state_dict('vanilla', 6)
    eng = ops.Engine(sd, v['use_point_stn'], v['shared_transformer'], device=0, precision='tc', guard_band=0.0)
    pts = torch.from_numpy(synth.make_cloud('sphere', args.points, seed=0)).cuda()
    table = np.zeros((len(CLASSES), len(PHASES)), dtype=np.uint64)

    def read(reset):
        if lib.p2s_pass_trace_read(table.ctypes.data, reset) != 0:
            raise SystemExit('p2s_pass_trace_read failed')

    eng.reconstruct(pts, args.grid_res, args.epsilon, v['uniform_subsample'], args.seed)   # warm-up
    read(1)
    eng.reconstruct(pts, args.grid_res, args.epsilon, v['uniform_subsample'], args.seed)
    read(0)
    eng.close()

    gpu = torch.cuda.get_device_name(0)
    print('pass kernel phase trace: %s, vanilla model, %d-pt sphere, grid_res %d, epsilon %d'
          % (gpu, args.points, args.grid_res, args.epsilon))
    tot = table.astype(np.float64)
    print('%-30s' % 'phase' + ''.join('%18s' % c for c in CLASSES))
    for j, name in enumerate(PHASES):
        print('%-30s' % name + ''.join('%17.1f%%' % (100.0 * tot[i, j] / max(tot[i].sum(), 1.0)) for i in range(len(CLASSES))))
    print('%-30s' % 'warpgroup Gcycles' + ''.join('%18.2f' % (tot[i].sum() * 1e-9) for i in range(len(CLASSES))))


if __name__ == '__main__':
    main()
