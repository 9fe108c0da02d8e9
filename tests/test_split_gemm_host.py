"""CPU tests of oracle/split_gemm.py, the float64 model of the split-precision training GEMMs: the hi/lo split applied
to raw operands breaks the per-element bound once operands leave fp16's normal range (tiny, as the backward pass's dZ
is, or huge); with the per-row / per-column power-of-two scaling the kernels apply, it meets the bound at every scale."""
import numpy as np
import pytest
import torch

from oracle import split_gemm
from points2surf_b200 import synth
from points2surf_b200.train import TrainStep
from helpers_train import TorchPrims, make_train_batch

SCALES = [2.0 ** -30, 2.0 ** -20, 2.0 ** -14, 1.0, 2.0 ** 14, 2.0 ** 17]


def _randn(*shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g, dtype=torch.float64) * scale).float()


def _excess_nt(A, W, scaled):
    return split_gemm.excess(split_gemm.gemm_nt(A, W, scaled), A.double() @ W.double().t(), split_gemm.bound_nt(A, W))


def _excess_tn(A, B, scaled):
    return split_gemm.excess(split_gemm.gemm_tn(A, B, scaled), A.double().t() @ B.double(),
                             split_gemm.bound_nt(A.t(), B.t()))


def test_split_exp_puts_the_maximum_in_the_fp16_top_binade():
    amax = np.concatenate([np.float32(2.0) ** np.arange(-149, 128, dtype=np.float32),
                           np.array([65504, 65505, 65519, 65520, 65535.9, 32767.99, 1e-45, 3.4028235e38, 1.0, 0.999999], np.float32),
                           np.random.RandomState(0).lognormal(0, 20, 1000).astype(np.float32)])
    amax = amax[np.isfinite(amax) & (amax > 0)]
    s = split_gemm.split_exp(amax)
    scaled = amax.astype(np.float64) * 2.0 ** s
    assert (scaled >= 2.0 ** 15 * (1 - 2 ** -10)).all() and (scaled <= 65504).all()
    assert ((scaled >= 2.0 ** 15) | (amax.astype(np.float64) * 2.0 ** (s + 1) > 65504)).all()
    # |s| / 2 stays inside the normal exponent range: the kernels apply 2^s as two exact fp32 factors
    assert s.min() >= -126 and s.max() <= 2 * 82
    assert (split_gemm.split_exp(np.array([0.0, np.inf, np.nan], np.float32)) == 0).all()
    # the scaled maximum never rounds to fp16 infinity
    assert np.isfinite(torch.from_numpy(scaled.astype(np.float32)).half().float().numpy()).all()


@pytest.mark.parametrize('scale', SCALES)
def test_scaled_split_meets_the_bound_at_every_scale(scale):
    A, W = _randn(300, 256, seed=1, scale=scale), _randn(96, 256, seed=2, scale=scale)
    assert _excess_nt(A, W, True) <= 1.0
    Bx = _randn(300, 64, seed=3)
    assert _excess_tn(A, Bx, True) <= 1.0
    assert _excess_tn(Bx, A, True) <= 1.0


@pytest.mark.parametrize('scale', [2.0 ** -20, 2.0 ** 17])
def test_unscaled_split_breaks_the_bound_outside_fp16_range(scale):
    A, W = _randn(300, 256, seed=1, scale=scale), _randn(96, 256, seed=2, scale=scale)
    assert _excess_nt(A, W, False) > 10.0
    assert _excess_tn(A, _randn(300, 64, seed=3), False) > 10.0


def test_scaled_split_mixed_magnitudes_zero_and_tiny_rows():
    g = torch.Generator().manual_seed(4)
    A = _randn(256, 128, seed=5)
    A = A * torch.pow(2.0, torch.randint(-30, 18, (256, 1), generator=g).float())        # rows of very different size
    A[:8] = 0.0                                                                           # rows that are all zero
    A[8:16] = _randn(8, 128, seed=6, scale=2.0 ** -100)                                   # rows whose entries are all tiny
    W = _randn(64, 128, seed=7) * torch.pow(2.0, torch.randint(-30, 11, (1, 128), generator=g).float())   # columns
    assert _excess_nt(A, W, True) <= 1.0
    assert _excess_nt(W, A, True) <= 1.0
    assert _excess_tn(A.t().contiguous(), W.t().contiguous(), True) <= 1.0
    assert (split_gemm.gemm_nt(A, W)[:8] == 0).all()


class _RecordingPrims(TorchPrims):
    """TorchPrims that keeps the operands of every GEMM the CUDA library would send to its tensor-core kernels
    (the shape conditions of gemm_nt_tc_ok / gemm_tn_tc_ok), tagged forward or backward."""

    def __init__(self):
        self.calls, self.backward = [], False

    def gemm_nt(self, A, W, bias=None, relu=False):
        if A.dim() == 2 and A.shape[0] >= 128 and W.shape[0] % 4 == 0 and 64 <= W.shape[0] <= 4096 and A.shape[1] % 32 == 0:
            self.calls.append(('nt', self.backward, A.detach().clone(), W.detach().clone()))
        return super().gemm_nt(A, W, bias, relu)

    def gemm_tn(self, A, B, out=None):
        if A.dim() == 2 and A.shape[0] >= 4096 and A.shape[1] >= 64 and B.shape[1] >= 64 and A.shape[1] % 4 == 0 and B.shape[1] % 4 == 0:
            self.calls.append(('tn', self.backward, A.detach().clone(), B.detach().clone()))
        return super().gemm_tn(A, B, out)

    def loss(self, *args, **kw):
        self.backward = True
        return super().loss(*args, **kw)


def test_backward_gemms_of_a_training_step():
    # one fp32 TrainStep of the `max` variant on the CPU; its backward dZ operands lie mostly below fp16's normal range
    torch.manual_seed(0)
    prims = _RecordingPrims()
    sd = synth.make_state_dict('max', seed=3)
    ts = TrainStep(sd, 0, 0, points_per_patch=128, sub_sample_size=256, lr=0.01, momentum=0.9, device='cpu', prims=prims)
    ts.step(make_train_batch(32, 128, 256, seed=1))
    bwd = [c for c in prims.calls if c[1]]
    assert len(bwd) >= 6 and any(c[0] == 'tn' for c in bwd) and any(c[0] == 'nt' for c in bwd)
    unscaled = []
    for kind, _, X, Y in prims.calls:
        f = _excess_nt if kind == 'nt' else _excess_tn
        assert f(X, Y, True) <= 1.0, (kind, tuple(X.shape), tuple(Y.shape))
    for kind, _, X, Y in bwd:
        f = _excess_nt if kind == 'nt' else _excess_tn
        unscaled.append(f(X, Y, False))
    assert max(unscaled) > 10.0, unscaled
