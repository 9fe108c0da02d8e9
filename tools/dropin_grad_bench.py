"""Cost of autograd through PointsToSurfModel in eval mode on one GPU (prints one JSON line).

* eager forward + backward of the module (vanilla, B queries, P patch points, S sub-sample points, fp32 engine) with
  every parameter requiring grad: median over --iters timed iterations (CUDA events) after --warmup, and the peak of
  torch.cuda.max_memory_allocated over one iteration;
* the backward of one conv3 layer (feat_global: 128 -> 1024 over B * S rows, eval BatchNorm, max over the S points)
  with the fused gather / scatter kernel (p2s_op_bn_maxpool_eval_bwd) against the dense path on the same tensors:
  maxpool_bwd into a dense [B*S, 1024] gradient, the eval BatchNorm backward, gemm_tn for the weight gradient and
  gemm_nt for the input gradient, both medians over the same number of alternating runs.
The card's name and power limit are read in the same run and printed with the numbers.

    python tools/dropin_grad_bench.py [--batch 1024 --points 300 --sub 1000 --iters 7 --warmup 2]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from points2surf_b200 import synth  # noqa: E402
from points2surf_b200.model import PointsToSurfModel  # noqa: E402
from points2surf_b200.train_ops import CudaPrims  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = 'unknown'
    return name, out


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=1024)
    ap.add_argument('--points', type=int, default=300)
    ap.add_argument('--sub', type=int, default=1000)
    ap.add_argument('--iters', type=int, default=7)
    ap.add_argument('--warmup', type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    B, P, S = a.batch, a.points, a.sub
    dev = torch.device('cuda', 0)
    m = PointsToSurfModel(num_points=P, output_dim=2, use_point_stn=True, sub_sample_size=S, shared_transformation=True,
                          precision='fp32')
    m.load_state_dict(synth.make_state_dict('vanilla', 0))
    m.to(dev).eval()
    inp = {k: torch.from_numpy(v).to(dev) for k, v in synth.make_model_inputs(B, P, S, 0).items()}
    dl = torch.randn(B, 2, device=dev)

    def step():
        x = {k: t.clone() for k, t in inp.items()}
        m.zero_grad(set_to_none=True)
        m(x).backward(dl)

    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    m.zero_grad(set_to_none=True)
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)
    step()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(dev)
    fb = [timed(step) for _ in range(a.iters)]

    # one conv3 layer's backward, fused against dense, alternating
    p = CudaPrims()
    g = torch.Generator(device=dev).manual_seed(0)
    C, K = 1024, 128
    x = torch.randn(B * S, K, device=dev, generator=g)
    W = torch.randn(C, K, device=dev, generator=g) * 0.1
    bias = torch.randn(C, device=dev, generator=g) * 0.1
    mean = torch.randn(C, device=dev, generator=g) * 0.2
    invstd = torch.rsqrt(torch.rand(C, device=dev, generator=g) + 0.5)
    gamma, beta = torch.rand(C, device=dev, generator=g) + 0.5, torch.randn(C, device=dev, generator=g) * 0.1
    z = p.gemm_nt(x, W, bias)
    out, arg = p.bn_maxpool_apply(z, B, S, mean, invstd, gamma, beta, False)
    dout = torch.randn(B, C, device=dev, generator=g)
    dW = torch.zeros(C, K, device=dev)

    def fused():
        p.bn_maxpool_eval_backward(dout, arg, out, z, x, W, mean, invstd, gamma, False, B, S, dW)

    parts = {}

    def dense():
        e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        e[0].record()
        dy = p.maxpool_bwd(dout, arg, S)
        dz = p.bn_eval_backward(dy, z, None, mean, invstd, gamma)[0]
        del dy
        p.gemm_tn(dz, x, out=dW)
        e[1].record()
        p.gemm_nt(dz, p.transpose(W))
        e[2].record()
        e[2].synchronize()
        parts.setdefault('w', []).append(e[0].elapsed_time(e[1]))

    for _ in range(a.warmup):
        fused()
        dense()
    tf, td = [], []
    for _ in range(a.iters):
        tf.append(timed(fused))
        td.append(timed(dense))
    name, power = card()
    res = {
        'card': name, 'power_limit': power, 'batch': B, 'points_per_patch': P, 'sub_sample_size': S,
        'forward_backward_ms_median': statistics.median(fb), 'forward_backward_ms_all': fb,
        'peak_memory_gib': (peak - base) / 2 ** 30,
        'conv3_bwd_fused_ms_median': statistics.median(tf),
        'conv3_bwd_dense_ms_median': statistics.median(td),
        'conv3_bwd_dense_without_dx_ms_median': statistics.median(parts['w'][a.warmup:]),
        'iters': a.iters, 'warmup': a.warmup,
    }
    print(json.dumps(res))


if __name__ == '__main__':
    main()
