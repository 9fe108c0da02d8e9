"""Time of the training step's column reductions (the BatchNorm statistics, p2s_op_bn_stats; p2s_op_bn_backward: the
dgamma / dbeta sums and dz) at the shapes training runs, with CUDA events over many launches.  `--ref-lib` times a second
build of the library (for instance one built from an earlier commit) in the same process, alternating with this tree's,
so the two numbers come from the same card in the same session.  A library without p2s_op_bn_stats is timed on
p2s_op_col_stats + p2s_op_bn_finalize, the two launches that computed the statistics before it.

    python tools/train_prims_bench.py [--reps 50] [--ref-lib /path/to/libp2s_b200.so]

Prints the card's name and power limit, one line per shape and library, and a JSON summary line."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from points2surf_b200 import _lib  # noqa: E402

# (M, C): conv layers of a 1024-query batch (300-point patches, 1000-point sub-samples) and an FC BatchNorm
SHAPES = [(307200, 64), (307200, 128), (1024000, 64), (1024000, 1024), (307200, 1024), (1024, 512)]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = 'unknown'
    return name, power or 'unknown'


def open_lib(path):
    lib = C.CDLL(path)
    vp, i64, i32 = C.c_void_p, C.c_int64, C.c_int
    f32 = C.c_float
    lib.p2s_op_col_stats.argtypes = [vp, i64, i32, vp, vp, vp]
    lib.p2s_op_bn_finalize.argtypes = [vp, vp, i64, i32, f32, f32, vp, vp, vp, vp, vp]
    if hasattr(lib, 'p2s_op_bn_stats'):
        lib.p2s_op_bn_stats.argtypes = [vp, i64, i32, f32, f32, vp, vp, vp, vp, vp, vp, vp]
    lib.p2s_op_bn_backward.argtypes = [vp, vp, vp, i64, i32, vp, vp, vp, vp, vp, vp, vp]
    return lib


def bn_stats(lib, z, s, mean, inv, st):
    """The BatchNorm statistics as the library's BatchNorm wrappers compute them: p2s_op_bn_stats where the library has
    it, else p2s_op_col_stats + p2s_op_bn_finalize (the same two launches)."""
    M, Cc = z.shape
    if hasattr(lib, 'p2s_op_bn_stats'):
        lib.p2s_op_bn_stats(z.data_ptr(), M, Cc, 1e-5, 0.1, s[0].data_ptr(), s[1].data_ptr(), mean.data_ptr(), inv.data_ptr(),
                            None, None, st)
    else:
        lib.p2s_op_col_stats(z.data_ptr(), M, Cc, s[0].data_ptr(), s[1].data_ptr(), st)
        lib.p2s_op_bn_finalize(s[0].data_ptr(), s[1].data_ptr(), M, Cc, 1e-5, 0.1, mean.data_ptr(), inv.data_ptr(), None, None, st)


def time_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--ref-lib', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('train_prims_bench: needs a CUDA device')
    libs = {'this tree': open_lib(_lib.LIB_PATH)}
    if a.ref_lib:
        libs['ref'] = open_lib(a.ref_lib)
    name, power = card()
    print('card: %s, power limit %s' % (name, power))
    st = torch.cuda.current_stream().cuda_stream
    out = []
    for M, Cc in SHAPES:
        z = torch.randn(M, Cc, device='cuda') * 0.5 + 3.0
        dy, y = torch.randn_like(z), torch.randn_like(z)
        s = torch.empty(2, Cc, dtype=torch.float64, device='cuda')
        mean, inv, gamma = torch.full((Cc,), 3.0, device='cuda'), torch.full((Cc,), 2.0, device='cuda'), torch.ones(Cc, device='cuda')
        mo, io = torch.empty_like(mean), torch.empty_like(inv)
        dz = torch.empty_like(z)
        best = {}
        for _ in range(a.rounds):                      # alternate the libraries; keep each one's best round
            for key, lib in libs.items():
                t_stats = time_ms(lambda: bn_stats(lib, z, s, mo, io, st), a.reps)
                t_bwd = time_ms(lambda: lib.p2s_op_bn_backward(dy.data_ptr(), z.data_ptr(), y.data_ptr(), M, Cc, mean.data_ptr(),
                                                               inv.data_ptr(), gamma.data_ptr(), s[0].data_ptr(),
                                                               s[1].data_ptr(), dz.data_ptr(), st), a.reps)
                b = best.setdefault(key, [float('inf'), float('inf')])
                b[0], b[1] = min(b[0], t_stats), min(b[1], t_bwd)
        for key, (t_stats, t_bwd) in best.items():
            gbs = M * Cc * 4 / (t_stats * 1e-3) / 1e9
            print('M %8d C %5d  %-9s  bn_stats %.4f ms (%.0f GB/s read)  bn_backward %.4f ms'
                  % (M, Cc, key, t_stats, gbs, t_bwd))
            out.append(dict(M=M, C=Cc, lib=key, bn_stats_ms=round(t_stats, 5), bn_backward_ms=round(t_bwd, 5)))
        del z, dy, y, dz
    print(json.dumps(dict(card=name, power_limit=power, results=out)))


if __name__ == '__main__':
    main()
