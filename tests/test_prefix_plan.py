"""CPU checks of shared-prefix generation: the pipeline's grouping of samples by encoder-input content and its prefix planner (pure
Python), and fo1_llm_generate's host-side argument checks of d.prefix, which run before the model or the device is touched."""
import ctypes
from importlib import import_module

import pytest
import torch


def _pipeline():
    return import_module("vlm-fo1_b200.pipeline")


def _sample(seed, ids=(1, 2, 3), n_boxes=2, grid=(4, 4)):
    P = _pipeline()
    g = torch.Generator().manual_seed(seed)
    return P.SampleInputs(list(ids), torch.rand(grid[0] * grid[1], 8, generator=g), grid, torch.rand(3, 16, 16, generator=g),
                          torch.rand(n_boxes, 4, generator=g) * 16)


def _copy(s, ids=None):
    """The same encoder inputs in fresh tensors (what prepare_inputs builds on every call)."""
    P = _pipeline()
    return P.SampleInputs(list(ids if ids is not None else s.input_ids), s.pixel_values.clone(), s.grid_hw, s.image_aux.clone(), s.boxes.clone())


def test_groups_by_content_not_identity():
    P = _pipeline()
    a, b = _sample(0), _sample(1)
    assert P.encoder_groups([a, _copy(a), b, _copy(b, ids=[9]), _copy(a)]) == [0, 0, 2, 2, 0]


def test_groups_non_adjacent_members_and_loners():
    P = _pipeline()
    a, b, c = _sample(0), _sample(1), _sample(2, n_boxes=3)
    assert P.encoder_groups([b, a, c, _copy(b), _sample(3), _copy(a)]) == [0, 1, 2, 0, 4, 1]


def test_groups_need_equal_boxes_and_pixels():
    P = _pipeline()
    a = _sample(0)
    other_boxes = _copy(a)
    other_boxes.boxes[0, 0] += 1.0
    other_aux = _copy(a)
    other_aux.image_aux[0, 0, 0] += 1.0
    other_px = _copy(a)
    other_px.pixel_values[0, 0] += 1.0
    other_grid = _sample(0, grid=(2, 8))
    assert P.encoder_groups([a, other_boxes, other_aux, other_px, other_grid]) == [0, 1, 2, 3, 4]


def test_groups_uint8_images():
    P = _pipeline()
    img = torch.randint(0, 256, (28, 28, 3), dtype=torch.uint8)
    bx = torch.tensor([[1.0, 2.0, 10.0, 12.0]])
    mk = lambda im, b: P.SampleInputs([1], None, None, None, b, image_u8=im)
    img2 = img.clone()
    img2[0, 0, 0] ^= 1
    assert P.encoder_groups([mk(img, bx), mk(img2, bx), mk(img.clone(), bx.clone())]) == [0, 1, 0]


IMG, REG = -200, -300


def test_prefix_identical_prompts_keep_one_row():
    P = _pipeline()
    ids = [5, 6, IMG, 7, REG, REG, 8, 9]
    L = len(ids) - 1 + 16                    # the image placeholder expands to 16 rows
    assert P.shared_prefix_groups([ids, ids, ids], [0, 0, 0], [16] * 3, [L] * 3) == [([0, 1, 2], L - 1)]


def test_prefix_through_image_and_regions_counts_spliced_rows():
    P = _pipeline()
    a = [5, 6, IMG, 7, REG, REG, 8, 40, 41]
    b = [5, 6, IMG, 7, REG, REG, 8, 50]
    lens = [len(a) - 1 + 16, len(b) - 1 + 16]
    # common ids: 5 6 <image> 7 <r> <r> 8 -> 2 + 16 + 4 rows
    assert P.shared_prefix_groups([a, b], [0, 0], [16, 16], lens) == [([0, 1], 22)]


def test_prefix_ending_before_the_image():
    P = _pipeline()
    a = [5, 6, 7, IMG, 8]
    b = [5, 6, 9, IMG, 8]
    assert P.shared_prefix_groups([a, b], [0, 0], [16, 16], [20, 20]) == [([0, 1], 2)]


def test_prefix_sets_without_a_common_row_and_loners_are_left_out():
    P = _pipeline()
    prompts = [[1, IMG, 2], [7, IMG, 2], [1, IMG, 3], [1, IMG, 3], [4, 4]]
    rep = [0, 0, 2, 2, 4]          # 0 / 1 share the image but no first token; 4 is alone
    lens = [18, 18, 18, 18, 2]
    assert P.shared_prefix_groups(prompts, rep, [16] * 5, lens) == [([2, 3], 17)]


def test_prefix_groups_with_non_adjacent_members():
    P = _pipeline()
    prompts = [[1, 2, 3], [8, 9], [1, 2, 4], [8, 9, 9], [1, 5]]
    assert P.shared_prefix_groups(prompts, [0, 1, 0, 1, 0], [1] * 5, [3, 2, 3, 3, 2]) == [([0, 2, 4], 1), ([1, 3], 1)]


# ---------------------------------------------------------------------------------------------------------------- C ABI
def _lib():
    import fo1_b200
    return fo1_b200._lib, fo1_b200.lib(), import_module("vlm-fo1_b200.engine")


PREFIX_CASES = ["group_range", "group_below", "one_member", "prefix_too_long", "prefix_zero", "null_lens", "null_embeds", "null_pos",
                "null_groups", "all_logits", "null_model"]


@pytest.mark.parametrize("case", PREFIX_CASES)
def test_generate_prefix_desc_validation_without_gpu(case):
    F, L, E = _lib()
    d = E.GenerateDescC()
    d.n_seqs = 3
    lens = (ctypes.c_int32 * 3)(10, 12, 9)
    d.seq_lens = lens
    groups = [0, -1, 0]
    plens = [8]
    if case == "group_range":
        groups = [0, 1, 0]
    elif case == "group_below":
        groups = [0, -2, 0]
    elif case == "one_member":
        groups = [0, -1, -1]
    elif case == "prefix_too_long":
        plens = [9]                   # sequence 2 has 9 rows: no own row left
    elif case == "prefix_zero":
        plens = [0]
    if case == "all_logits":
        d.all_logits = 16
    px = F.PrefixDesc(1, None if case == "null_lens" else (ctypes.c_int32 * 1)(*plens), None if case == "null_embeds" else 16,
                      None if case == "null_pos" else 16, None if case == "null_groups" else (ctypes.c_int32 * 3)(*groups))
    d.prefix = ctypes.pointer(px)
    model = None if case == "null_model" else ctypes.c_void_p(16)      # never dereferenced: the checks come first
    rc = L.fo1_llm_generate(model, ctypes.byref(d), None)
    assert rc == -1
    msg = L.fo1_last_error().decode()
    assert ("fo1_llm_generate: null argument" if case == "null_model" else "fo1_llm_generate: prefix: ") in msg, msg


def test_prefix_attention_argument_validation_without_gpu():
    F, L, _ = _lib()
    pre, own = (ctypes.c_int32 * 2)(60, 0), (ctypes.c_int32 * 2)(10, 3)
    d = F.PrefixAttnDesc(16, 512, 16, 16, 2, 96, pre, own, 16, 2, 128, 0.1, 16, 2048)
    assert L.fo1_prefix_attention(ctypes.byref(d), None) == -1           # cap not a multiple of 64
    d.cap = 64
    assert L.fo1_prefix_attention(ctypes.byref(d), None) == -1           # 60 + 10 rows exceed the slot
    d.cap, d.head_dim = 128, 64
    assert L.fo1_prefix_attention(ctypes.byref(d), None) == -1           # head_dim
    assert "fo1_prefix_attention" in L.fo1_last_error().decode()
