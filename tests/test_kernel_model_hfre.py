"""The separable-window algorithm the CUDA kernels implement == the oracle's
interpolate -> concat -> roi_align -> mean (CPU-only check of the math)."""
import os

import numpy as np
import pytest
import torch

from oracle import hfre as O
from tests import kernel_models as KM


@pytest.mark.parametrize("tag", ["small", "rect"])
def test_separable_weights_equal_oracle(golden_dir, tag):
    z = np.load(os.path.join(golden_dir, f"hfre_{tag}.npz"))
    aux = [z[f"aux{i}"] for i in range(4)]
    boxes = z["boxes"]
    H, W = aux[0].shape[1:]
    got = np.concatenate([KM.hfre_level(a.transpose(1, 2, 0), boxes, 0.25, 7, (H, W)) for a in aux], axis=1)
    ref = O.hfre_aux_branch([torch.from_numpy(a) for a in aux], torch.from_numpy(boxes)).numpy()
    scale = np.abs(ref).max()
    assert np.abs(got - ref).max() <= 2e-5 * scale
    pyr = [z[f"pyr{i}"] for i in range(4)]
    vtb = z["vt_boxes"]
    got = np.concatenate([KM.hfre_level(p.transpose(1, 2, 0), vtb, 1.0 / s, 7, p.shape[1:]) for p, s in zip(pyr, O.FPN_STRIDES)], axis=1)
    ref = O.hfre_vt_branch([torch.from_numpy(p) for p in pyr], torch.from_numpy(vtb), "fpn").numpy()
    assert np.abs(got - ref).max() <= 2e-5 * np.abs(ref).max()


@pytest.mark.parametrize("tag", ["small", "rect"])
def test_tensor_sweep_weight_split_stays_inside_the_parity_budget(golden_dir, tag):
    """The sweep feeds the fp32 column weights to the tensor pipe as hi + lo bf16 halves: on bf16-exact maps that must agree
    with the fp64 separable sum to ~1e-5 (two orders inside the 1e-3 parity tolerance); a single bf16 half would not."""
    z = np.load(os.path.join(golden_dir, f"hfre_{tag}.npz"))
    aux = [KM._bf16_round(z[f"aux{i}"]) for i in range(4)]
    boxes = z["boxes"]
    H, W = aux[0].shape[1:]
    for a in aux[:2]:
        hwc = a.transpose(1, 2, 0)
        exact = KM.hfre_level(hwc, boxes, 0.25, 7, (H, W))
        split = KM.hfre_level_tensor_sweep(hwc, boxes, 0.25, 7, (H, W))
        scale = np.abs(exact).max()
        assert np.abs(split - exact).max() <= 2e-5 * scale
