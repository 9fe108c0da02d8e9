"""CPU restatement of the regression head's post-process (outputs imp_surf, experiments/eval_p2s_regression.sh), for the
tests and tests/golden/make_regression_golden.py: the reference's own torch CPU operations in its order, so that it equals
the reference bit for bit (make_regression_golden.py asserts that on the fixture's logits)."""
import numpy as np


def post_process_distance(logits, patch_radius):
    """logits [B,1] -> d = tanh(l)^2 * sign(l) (sign(0) = 0), then * r unless patch_radius is None (the fixed-radius case)
    (source/sdf_nn.py:6-8, points_to_surf_eval.py:176-183).  float32.  NaN -> 1.0 as in save_reconstruction_data
    (points_to_surf_eval.py:205-207)."""
    import torch
    lg = torch.from_numpy(np.asarray(logits, dtype=np.float32).reshape(-1, 1))
    d = torch.tanh(lg).pow(2) * torch.sign(lg)
    if patch_radius is not None:
        d = d * torch.from_numpy(np.asarray(patch_radius, dtype=np.float32)).unsqueeze(1)
    sdf = d[:, 0].numpy().copy()
    sdf[np.isnan(sdf)] = 1.0
    return sdf
