"""Training-step benchmark (BASELINE config 4 / SURVEY.md section 8d): vanilla model, kNN 300 patch + 1000-point
sub-sample, synthetic batch, SGD(momentum).  One process per GPU; under torchrun the global batch is split over the
ranks and gradients are averaged with one all_reduce per step.

    python tools/train_bench.py --batch 1024 --steps 5 --warmup 2 [--profile]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 tools/train_bench.py --batch 1024
"""
import argparse
import json
import os
import sys
import time

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from points2surf_b200 import synth, ops  # noqa: E402
from points2surf_b200.train import TrainStep  # noqa: E402
from helpers_train import make_train_batch  # noqa: E402
from helpers_train_regression import make_regression_train_batch  # noqa: E402

# SURVEY.md section 8d, per query; 'regression' is the `uniform` network with a 128 -> 1 head (256 FLOP less per query)
FLOP_FWD = {'vanilla': 1.1407e9, 'max': 0.7768e9, 'uniform': 1.1407e9, 'regression': 1.1407e9}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=1024, help='global batch (queries per step over all ranks)')
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--model', default='vanilla', help='vanilla | max | uniform | regression (one-output head, imp_surf loss)')
    ap.add_argument('--cpu_sample', type=int, default=0, help='queries of one CPU-oracle iteration timed beside it (0 = skip)')
    ap.add_argument('--graph', action='store_true', help='replay the step as CUDA graphs (TrainStep.capture_graph)')
    ap.add_argument('--profile', action='store_true', help='per-primitive time table (synchronising; slower)')
    a = ap.parse_args()
    rank, world = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1))
    local = int(os.environ.get('LOCAL_RANK', 0))
    torch.cuda.set_device(local)
    dev = torch.device('cuda', local)
    if world > 1:
        os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
        dist.init_process_group('nccl', device_id=dev)
    v = synth.VARIANTS[a.model]
    regression = v.get('output_dim', 2) == 1
    make_batch = make_regression_train_batch if regression else make_train_batch
    outputs = ('imp_surf',) if regression else ('imp_surf_magnitude', 'imp_surf_sign')
    per_rank = a.batch // world
    sd = {k: t.to(dev) for k, t in synth.make_state_dict(a.model, seed=0).items()}
    batch = {k: t.to(dev) for k, t in make_batch(per_rank, seed=100 + rank).items()}
    ts = TrainStep(sd, v['use_point_stn'], v['shared_transformer'], lr=1e-4, outputs=outputs)
    if a.graph:
        ts.capture_graph(batch)
    prof, shapes = {}, {}
    if a.profile:
        p = ts.p
        for name in ('gemm_nt', 'gemm_tn', 'transpose', 'bn_forward', 'bn_backward', 'bn_maxpool_forward', 'bn_maxpool_backward',
                     'col_sum', 'maxpool_fwd', 'maxpool_bwd',
                     'axpy_', 'center', 'loss', 'loss_distance', 'sgd_', 'add_row_', 'quat_to_rot', 'quat_to_rot_bwd'):
            fn = getattr(p, name)

            def wrap(fn=fn, name=name):
                def inner(*args, **kw):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    out = fn(*args, **kw)
                    torch.cuda.synchronize()
                    dt = (time.perf_counter() - t0) * 1e3
                    d = prof.setdefault(name, [0, 0.0])
                    d[0] += 1
                    d[1] += dt
                    if name in ('gemm_nt', 'gemm_tn'):
                        key = '%s %s x %s' % (name, tuple(args[0].shape), tuple(args[1].shape))
                        d = shapes.setdefault(key, [0, 0.0])
                        d[0] += 1
                        d[1] += dt
                    return out
                return inner
            setattr(p, name, wrap())
    for _ in range(a.warmup):
        ts.step(batch)
    prof.clear()
    shapes.clear()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    ops.launch_count(reset=True)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        losses = ts.step(batch)
    e1.record()
    torch.cuda.synchronize()
    ms = torch.tensor([e0.elapsed_time(e1)], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    ms = float(ms.item()) / a.steps
    if rank == 0:
        out = {'workload': '%s training step, global batch %d (%d per rank), P 300, S 1000, fp32' % (a.model, a.batch, per_rank),
               'n_gpus': world, 'ms_per_step': ms, 'steps_per_s': 1e3 / ms, 'queries_per_s': a.batch * 1e3 / ms,
               'tflops_algorithmic': 3 * FLOP_FWD[a.model] * a.batch / (ms * 1e-3) / 1e12,
               'launches_per_step': ops.launch_count() / a.steps, 'cuda_graph': bool(a.graph), 'loss': [float(l) for l in losses],
               'peak_mem_GB': torch.cuda.max_memory_allocated() / 1e9}
        if a.cpu_sample > 0 and world == 1:
            import train_regression_oracle as train_oracle
            cb = make_batch(a.cpu_sample, seed=100)
            csd = synth.make_state_dict(a.model, seed=0)
            best = (0.0, 0)
            for th in sorted({min(os.cpu_count() or 1, c) for c in (16, 32, os.cpu_count() or 1)}):   # give the CPU arm its best thread count
                torch.set_num_threads(th)
                train_oracle.train_iteration(csd, cb, v['use_point_stn'], v['shared_transformer'], outputs=outputs)   # warm-up
                t0 = time.perf_counter()
                train_oracle.train_iteration(csd, cb, v['use_point_stn'], v['shared_transformer'], outputs=outputs)
                rate = a.cpu_sample / (time.perf_counter() - t0)
                if rate > best[0]:
                    best = (rate, th)
            out['cpu_baseline'] = {'value': best[0], 'unit': 'queries/s', 'cores': best[1], 'kind': 'port',
                                   'sample': 'one training iteration of %d queries with the oracle port (torch CPU autograd, best of 16 / 32 / all threads)' % a.cpu_sample}
        print(json.dumps(out))
        if prof:
            tot = sum(d[1] for d in prof.values())
            for name, d in sorted(prof.items(), key=lambda kv: -kv[1][1]):
                print('  %-16s %5d calls  %9.2f ms/step  %5.1f %%' % (name, d[0] // a.steps, d[1] / a.steps, 100 * d[1] / tot))
            for key, d in sorted(shapes.items(), key=lambda kv: -kv[1][1])[:24]:
                print('    %-64s %3d calls  %8.3f ms/step' % (key, d[0] // a.steps, d[1] / a.steps))
    if world > 1:
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
