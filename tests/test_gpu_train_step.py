"""GPU test of the whole training step per element: every logit, both losses, every gradient and, after the update, every
parameter, momentum buffer and running mean / var of points2surf_b200.train.TrainStep on the CUDA primitives are held to
the conditioned float64 step of tests/train_step_bound.py, |x - v| <= LAMBDA e (LAMBDA = 4).  The float64 step runs on
the same device, takes the CUDA step's own ReLU masks, max-pool args and sign of p0 from its tapes, and starts from the
state the CUDA step held before each step, so two consecutive steps are two independent checks.
num_batches_tracked must match exactly.

Each case prints the worst ratio per tensor in layer order, so the first tensor out of bound points at the faulty primitive.
Cases: the four variants at the real P = 300, S = 1000 (B = 2, where the FC BatchNorms run over two rows; 32; 128),
fixed_radius, B = 1024 at P = 64, S = 128 (dZ in the split GEMMs' small-operand regime), a ragged shape; the same on the
fp32 FMA GEMMs (P2S_TRAIN_GEMM_FP32=1, read once per process: a subprocess); and two CUDA-graph replays whose decisions
are read from the replay's own tapes."""
import json
import os
import subprocess
import sys

import pytest
import torch

import train_step_bound as tsb
from points2surf_b200 import synth
from points2surf_b200.train import TrainStep
from helpers_train import make_train_batch
from helpers_train_regression import make_regression_train_batch

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
SEEDS = {'vanilla': 21, 'max': 22, 'uniform': 23, 'regression': 24}

# name -> (variant, B, P, S, fixed_radius)
CASES = {
    'vanilla-B2': ('vanilla', 2, 300, 1000, False),
    'vanilla-B32': ('vanilla', 32, 300, 1000, False),
    'max-B32': ('max', 32, 300, 1000, False),
    'uniform-B32': ('uniform', 32, 300, 1000, False),
    'regression-B32': ('regression', 32, 300, 1000, False),
    'regression-B32-fixed-radius': ('regression', 32, 300, 1000, True),
    'vanilla-B128': ('vanilla', 128, 300, 1000, False),
    'vanilla-B1024-P64-S128': ('vanilla', 1024, 64, 128, False),
    'uniform-B7-P75-S130': ('uniform', 7, 75, 130, False),
}
FMA_CASES = ['vanilla-B2', 'max-B32', 'regression-B32', 'vanilla-B1024-P64-S128', 'uniform-B7-P75-S130']


class StashingTrainStep(TrainStep):
    """backward() drops the tape; inside a captured graph its tensors would go back to the graph's pool.  Keeping a
    reference keeps them alive, and every replay rewrites them in place with that replay's own decisions."""

    def backward(self, dlogits):
        self._stash = self._rec
        super().backward(dlogits)


def make_step(variant, B, P, S, fixed_radius, cls=TrainStep):
    v = synth.VARIANTS[variant]
    kw = dict(outputs=('imp_surf',)) if variant == 'regression' else {}
    sd = {k: t.to(DEV) for k, t in synth.make_state_dict(variant, seed=SEEDS[variant]).items()}
    return cls(sd, v['use_point_stn'], v['shared_transformer'], points_per_patch=P, sub_sample_size=S, lr=0.01,
               momentum=0.9, fixed_radius=fixed_radius, **kw)


def make_batch(variant, B, P, S, seed):
    mk = make_regression_train_batch if variant == 'regression' else make_train_batch
    return {k: t.to(DEV) for k, t in mk(B, P, S, seed=seed).items()}


def check(case, step, ts, run, fp32_only):
    """Holds one step to the bound; prints the per-tensor worst ratios in layer order -> the worst (ratio, tensor)."""
    ref = tsb.reference(ts, run, run['batch'], fp32_only)
    items = tsb.checks(ts, run, ref)
    rs = tsb.ratios(items)
    del ref, items
    print('%s step %d (%s GEMMs):' % (case, step, 'FMA' if fp32_only else 'tensor-core'))
    print('  ' + '  '.join('%s %.3g@%s' % (n, r, ','.join(map(str, i))) for n, r, i in rs))
    name, r, idx = max(rs, key=lambda x: x[1])
    print('  worst %.3f at %s %s' % (r, name, idx))
    assert tsb.num_batches_tracked_ok(run), case
    return r, name, [x for x in rs if not x[1] <= 1.0]


def run_case(case, fp32_only):
    """Two consecutive eager steps -> [(worst ratio, tensor, out-of-bound list)] per step."""
    variant, B, P, S, fixed = CASES[case]
    ts = make_step(variant, B, P, S, fixed)
    out = []
    for k in range(2):
        batch = make_batch(variant, B, P, S, seed=200 + k)
        run = tsb.drive(ts, batch)
        run['batch'] = batch
        out.append(check(case, k + 1, ts, run, fp32_only))
        del run, batch
        torch.cuda.empty_cache()
    del ts
    torch.cuda.empty_cache()
    return out


@pytest.mark.parametrize('case', list(CASES))
def test_train_step_per_element_bound(case):
    torch.cuda.reset_peak_memory_stats()
    res = run_case(case, fp32_only=False)
    print('%s: peak device memory %.1f GB' % (case, torch.cuda.max_memory_allocated() / 2 ** 30))
    bad = [(k + 1, b) for k, (_, _, b) in enumerate(res) if b]
    assert not bad, bad


_FMA_SCRIPT = r'''
import json, sys
sys.path[:0] = [%r, %r]
import test_gpu_train_step as t
res = {}
for c in t.FMA_CASES:
    res[c] = [(r, n, b) for r, n, b in t.run_case(c, fp32_only=True)]
print('RESULT ' + json.dumps(res))
'''


def test_train_step_per_element_bound_fp32_fma_kernels():
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, P2S_TRAIN_GEMM_FP32='1')
    r = subprocess.run([sys.executable, '-c', _FMA_SCRIPT % (os.path.dirname(here), here)], env=env, capture_output=True,
                       text=True, timeout=1800)
    print(r.stdout)
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    res = json.loads([l for l in r.stdout.splitlines() if l.startswith('RESULT ')][-1][7:])
    assert set(res) == set(FMA_CASES)
    bad = {c: [s[2] for s in steps if s[2]] for c, steps in res.items() if any(s[2] for s in steps)}
    assert not bad, bad


def test_cuda_graph_replay_per_element_bound():
    """Two replayed steps under the same bound, each read from the replay's own tapes (the forward is not bitwise
    repeatable: the BatchNorm column sums finish with float64 atomicAdd across blocks, train_ops.cu:135-136, :251-252,
    and the weight-gradient GEMMs accumulate with fp32 atomics, train_ops.cu:74, gemm_tn_tc.cu:144-145)."""
    variant, B, P, S = 'vanilla', 32, 300, 1000
    ts = make_step(variant, B, P, S, False, cls=StashingTrainStep)
    ts.step(make_batch(variant, B, P, S, seed=300))               # one eager step: momentum buffers are non-zero
    ts.capture_graph(make_batch(variant, B, P, S, seed=301))
    bad = []
    for k in range(2):
        batch = make_batch(variant, B, P, S, seed=302 + k)
        before = tsb.state_of(ts)
        losses = ts.step(batch)
        assert ts._graph is not None and ts._graph_matches(batch)
        logits = ts.last_logits
        run = dict(before=before, dec=tsb.decisions(ts._stash, logits), logits=logits.detach().clone(),
                   losses=torch.stack([l.reshape(()) for l in losses]),
                   grads={n: g.detach().clone() for n, g in ts.grads.items()}, after=tsb.state_of(ts), batch=batch)
        r, name, b = check('graph-replay', k + 1, ts, run, fp32_only=False)
        bad += b
        del run
        torch.cuda.empty_cache()
    assert not bad, bad
