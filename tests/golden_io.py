"""Load tests/golden/*.npz fixtures (weights are stored as bf16 bit patterns under 'w::<name>').  A fixture too large for one file
continues in <name>.part1.npz, <name>.part2.npz, ... (oracle/gen_golden.py: save)."""
import json
import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load(name):
    z = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    i = 1
    while os.path.exists(os.path.join(GOLDEN, f"{name}.part{i}.npz")):
        z.update(np.load(os.path.join(GOLDEN, f"{name}.part{i}.npz")))
        i += 1
    sd, rest = {}, {}
    for k in z:
        if k.startswith("w::"):
            sd[k[3:]] = torch.from_numpy(z[k].copy()).view(torch.bfloat16).float()
        elif k == "cfg_json":
            rest["cfg"] = json.loads(bytes(z[k]).decode())
        else:
            rest[k] = z[k]
    return sd, rest


def nerr(got: torch.Tensor, ref: torch.Tensor) -> float:
    """max |got - ref| / max |ref| -- the normalised error every parity test bounds by 1e-3 (fp32 stages)."""
    return float((got.float() - ref.float()).abs().max() / ref.float().abs().max().clamp_min(1e-30))


def rerr(got: torch.Tensor, ref: torch.Tensor) -> float:
    """||got - ref||_2 / ||ref||_2 -- the relative (RMS) error.  Under bf16 storage the MAX-norm error of a tensor with millions of
    elements is an extreme-value statistic of single-ulp rounding flips at its largest elements; the RMS error is what stays
    at the 1e-3 level when two implementations agree."""
    g, r = got.double(), ref.double()
    return float((g - r).norm() / r.norm().clamp_min(1e-30))
