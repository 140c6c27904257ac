"""The attention bounds (tests/attention_bounds.py) on CPU models of the kernels' rounding (tests/kernel_models.py):
the faithful model satisfies the bound, and every modelled kernel mistake breaks it by at least 4x on the same inputs.
Each control also reports whether the flat tolerance the GPU tests used before accepted it."""
import numpy as np
import pytest
import torch

from tests import attention_bounds as AB
from tests import kernel_models as KM

CONTROL_MIN = 4.0
SOUND_MAX = 1.0 / AB.SAFETY        # the faithful model stays inside the bound without its safety factor


def _report(kernel, defect, name, r, idx, old_ok, r_plain, old_plain):
    verdict = lambda ok: "accepted" if ok else "rejected"
    print(f"control {kernel} {defect} on {name}: ratio {r:.3g} at {idx}, old tolerance {verdict(old_ok)}; "
          f"on plain random data: ratio {r_plain:.3g}, old tolerance {verdict(old_plain)}")


def _np(t):
    return t.float().numpy()


# ------------------------------------------------------------------------------------------------------------- varlen
VARLEN_CASES = {
    # name: (lens, qh, kvh, hd, causal)
    "gqa_causal": ([63, 129, 65, 1, 257], 8, 2, 128, True),
    "vit_windows": ([64, 64, 48, 36, 127, 65], 4, 4, 80, False),
    "davit_g4": ([144, 144, 100, 1, 256], 8, 2, 32, False),
    "offset_causal": ([1, 255, 128, 64], 4, 1, 64, True),
}


def _varlen(name, defect=None, seed=0, plain=False):
    lens, qh, kvh, hd, causal = VARLEN_CASES[name]
    buf, q, k, v, cu = AB.varlen_inputs(lens, qh, kvh, hd, causal, seed, plain=plain)
    scale = hd ** -0.5
    out = KM.attn_varlen_model(_np(q), _np(k), _np(v), cu, qh, kvh, hd, scale, causal, defect)
    ref, bound = AB.varlen_reference(q, k, v, cu, qh, kvh, hd, scale, causal)
    old_ok = bool(np.abs(out - ref.reshape(len(out), -1).float().numpy()).max() < 3e-2)   # the former flat tolerance
    return torch.from_numpy(out), ref, bound, old_ok


@pytest.mark.parametrize("name", list(VARLEN_CASES))
def test_varlen_model_within_bound(name):
    out, ref, bound, _ = _varlen(name)
    r = AB.check(out, ref, bound, f"varlen model {name}")
    print(f"varlen model {name}: max ratio {r:.3f}")
    assert r < SOUND_MAX


def test_varlen_model_lazy_rescale_within_bound():
    """Keys rising by just under / just over kAtRescale log2 units per 64-key tile: the rescale is skipped and taken."""
    for step in (7.75, 8.25):
        buf, q, k, v, cu = AB.varlen_inputs([700], 2, 2, 128, False, 3, tile_step_log2=step)
        out = KM.attn_varlen_model(_np(q), _np(k), _np(v), cu, 2, 2, 128, 128 ** -0.5, False)
        ref, bound = AB.varlen_reference(q, k, v, cu, 2, 2, 128, 128 ** -0.5, False)
        r = AB.check(torch.from_numpy(out), ref, bound, f"lazy rescale step {step}")
        print(f"varlen model rescale step {step}: max ratio {r:.3f}")
        assert r < SOUND_MAX


VARLEN_CONTROLS = [
    ("past_end", "vit_windows"), ("past_end", "davit_g4"),
    ("neighbour", "vit_windows"), ("neighbour", "gqa_causal"),
    ("tile_last", "vit_windows"), ("tile_last", "gqa_causal"),
    ("diag", "gqa_causal"), ("diag", "offset_causal"),
    ("future", "gqa_causal"), ("future", "offset_causal"),
    ("gqa_mod", "gqa_causal"), ("gqa_mod", "davit_g4"),
]


@pytest.mark.parametrize("defect,name", VARLEN_CONTROLS)
def test_varlen_control_breaks_bound(defect, name):
    out, ref, bound, old_ok = _varlen(name, defect)
    r, idx = AB.ratio(out, ref, bound)
    out, ref, bound, old_plain = _varlen(name, defect, plain=True)
    _report("attn_tc_kernel", defect, name, r, idx, old_ok, AB.ratio(out, ref, bound)[0], old_plain)
    assert r >= CONTROL_MIN


# ------------------------------------------------------------------------------------------------------------- decode
DECODE_CASES = {
    # name: (lens, qh, kvh, n_splits)
    "gqa8_s8": ([1, 15, 16, 17, 600, 257], 16, 2, 8),
    "g7_s3": ([47, 48, 49, 145, 300], 14, 2, 3),
    "mha_s1": ([33, 64, 65, 200], 4, 4, 1),
    "g8_s2": ([31, 32, 33, 400], 8, 1, 2),
}


def _decode(name, poison, defect=None, seed=0):
    lens, qh, kvh, S = DECODE_CASES[name]
    cap = max(lens) + 2
    q, kc, vc = AB.decode_inputs(lens, qh, kvh, cap, seed, poison)
    scale = 128 ** -0.5
    out = KM.decode_attn_model(_np(q), _np(kc), _np(vc), lens, qh, kvh, scale, S, defect)
    ref, bound = AB.decode_reference(q, kc, vc, lens, qh, kvh, scale)
    refm = ref.reshape(len(lens), -1).float().numpy()
    old_ok = all(np.abs(out[b] - refm[b]).max() <= 2e-2 * max(1.0, np.abs(refm[b]).max()) for b in range(len(lens)))
    return torch.from_numpy(out), ref, bound, old_ok


@pytest.mark.parametrize("poison", ["nan", "adversarial"])
@pytest.mark.parametrize("name", list(DECODE_CASES))
def test_decode_model_within_bound(name, poison):
    out, ref, bound, _ = _decode(name, poison)
    r = AB.check(out, ref, bound, f"decode model {name} {poison}")
    print(f"decode model {name} ({poison}): max ratio {r:.3f}")
    assert r < SOUND_MAX


DECODE_CONTROLS = [
    ("past_end", "gqa8_s8"), ("past_end", "mha_s1"),
    ("own_key", "gqa8_s8"), ("own_key", "g7_s3"),
    ("tile_last", "gqa8_s8"), ("tile_last", "g8_s2"),
    ("chunk_last", "g7_s3"), ("chunk_last", "gqa8_s8"),
    ("gqa_mod", "gqa8_s8"), ("gqa_mod", "g7_s3"),
    ("combine_drop_last", "gqa8_s8"), ("combine_drop_last", "g7_s3"),
]


@pytest.mark.parametrize("defect,name", DECODE_CONTROLS)
def test_decode_control_breaks_bound(defect, name):
    out, ref, bound, old_ok = _decode(name, "adversarial", defect)
    r, idx = AB.ratio(out, ref, bound)
    out, ref, bound, old_plain = _decode(name, "random", defect)
    _report("decode_attn", defect, name, r, idx, old_ok, AB.ratio(out, ref, bound)[0], old_plain)
    assert r >= CONTROL_MIN


# ------------------------------------------------------------------------------------------------------------ channel
CHAN_CASES = {"n513_c64": (2, 513, 64), "n4097_c256": (1, 4097, 256), "n1000_c96": (1, 1000, 96)}


def _chan(name, defect=None, seed=0, plain=False):
    B, N, C = CHAN_CASES[name]
    qkv = AB.chan_inputs(B, N, C, seed, plain)
    nc, tpc = AB.chan_plan(N, C)
    out = KM.chan_attn_model(_np(qkv), C // 32, nc, tpc, AB.chan_constants()[0], defect)
    ref, bound = AB.channel_reference(qkv, C // 32)
    refm = ref.float().numpy()
    old_ok = bool(np.abs(out - refm).max() / np.abs(refm).max() < 1e-3 + 2 * 2.0 ** -8)
    return torch.from_numpy(out), ref.reshape(B * N, C // 32, 32), bound.reshape(B * N, C // 32, 32), old_ok


@pytest.mark.parametrize("name", list(CHAN_CASES))
def test_chan_model_within_bound(name):
    out, ref, bound, _ = _chan(name)
    r = AB.check(out, ref, bound, f"channel model {name}")
    print(f"channel model {name}: max ratio {r:.3f}")
    assert r < SOUND_MAX


CHAN_CONTROLS = [("scale_tile_n", "n513_c64"), ("scale_tile_n", "n1000_c96"), ("drop_last_chunk", "n513_c64"),
                 ("drop_last_chunk", "n4097_c256"), ("transposed", "n1000_c96")]


@pytest.mark.parametrize("defect,name", CHAN_CONTROLS)
def test_chan_control_breaks_bound(defect, name):
    out, ref, bound, old_ok = _chan(name, defect)
    r, idx = AB.ratio(out, ref, bound)
    out, ref, bound, old_plain = _chan(name, defect, plain=True)
    _report("channel_attention", defect, name, r, idx, old_ok, AB.ratio(out, ref, bound)[0], old_plain)
    assert r >= CONTROL_MIN

