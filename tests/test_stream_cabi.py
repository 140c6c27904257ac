"""CPU checks of fo1_llm_generate's decoding options (include/fo1.h): it refuses missing stream buffers, and every pair of options
its combination table refuses, before it touches the model or the device; and the host-side progress / cancel accessors of the
streamed-decoding ABI (fo1_stream_desc) work on ordinary host memory."""
import ctypes
from importlib import import_module

import pytest


def _mods():
    import fo1_b200
    return fo1_b200._lib, fo1_b200.lib(), import_module("vlm-fo1_b200.engine")


@pytest.mark.parametrize("case", ["null_model", "null_desc", "null_tokens", "null_lens", "null_progress"])
def test_generate_stream_desc_rejects_null_buffers_without_gpu(case):
    F, L, E = _mods()
    d = E.GenerateDescC()
    d.n_seqs = 1
    buf = (ctypes.c_int32 * 64)()
    p = ctypes.addressof(buf)
    fields = dict(tokens=p, lens=p + 32 * 4, progress=p + 48 * 4, cancel=None)
    if case.startswith("null_") and case[5:] in fields:
        fields[case[5:]] = None
    st = F.StreamDesc(**fields)
    d.stream = ctypes.pointer(st)
    model = None if case == "null_model" else ctypes.c_void_p(16)         # never dereferenced: the check comes first
    desc = None if case == "null_desc" else ctypes.byref(d)
    rc = L.fo1_llm_generate(model, desc, None)
    assert rc == -1
    msg = L.fo1_last_error().decode()
    assert ("fo1_llm_generate: null argument" if case in ("null_model", "null_desc") else "fo1_llm_generate: stream: null") in msg, msg


# every pair of options fo1_llm_generate refuses (include/fo1.h, the combination table)
REFUSED = [("beam", "sampling"), ("beam", "scores"), ("beam", "stream"), ("beam", "prefix"), ("beam", "processors"), ("beam", "lookup"),
           ("lookup", "stream"), ("lookup", "processors")]


def _options(F):
    """One non-empty descriptor per option (contents past the emptiness test are never read when the pair is refused)."""
    one = (ctypes.c_int32 * 2)(0, 0)
    return dict(sampling=F.SamplingDesc(), scores=F.ScoreDesc(16, None, None, None), stream=F.StreamDesc(16, 16, 16, None),
                prefix=F.PrefixDesc(n_groups=1), processors=F.ProcessorDesc(n_sets=1, seq_set=one), lookup=F.LookupDesc(num_tokens=4),
                beam=F.BeamDesc(num_beams=4)), one


@pytest.mark.parametrize("a,b", REFUSED)
def test_generate_refuses_each_pair_of_the_table_without_gpu(a, b):
    F, L, E = _mods()
    opts, _keep = _options(F)
    d = E.GenerateDescC()
    d.n_seqs = 2
    setattr(d, a, ctypes.pointer(opts[a]))
    setattr(d, b, ctypes.pointer(opts[b]))
    rc = L.fo1_llm_generate(ctypes.c_void_p(16), ctypes.byref(d), None)    # never dereferenced: the table comes first
    assert rc == -3                                                         # FO1_ERR_UNSUPPORTED
    msg = L.fo1_last_error().decode()
    assert msg.startswith("fo1_llm_generate: ") and a in msg and b in msg, msg


def test_generate_empty_options_are_the_call_without_them_without_gpu():
    """An option that asks for nothing does not take part in the table: beam search with an empty score desc, a prefix of no group
    and processors in which no sequence has a set reaches the beam checks (here: max_new_tokens 0)."""
    F, L, E = _mods()
    cfg = E.ModelConfigC()
    cfg.llm_vocab = 1000
    m = ctypes.c_void_p()
    assert L.fo1_model_create(ctypes.byref(cfg), ctypes.byref(m)) == 0     # host only
    none = (ctypes.c_int32 * 2)(-1, -1)
    sc, px, pr = F.ScoreDesc(), F.PrefixDesc(n_groups=0), F.ProcessorDesc(n_sets=1, seq_set=none)
    bm = F.BeamDesc(num_beams=4, n_keep=8, num_return=1, sequence_scores=16, beam_indices=16, steps_run=16)
    d = E.GenerateDescC()
    d.n_seqs, d.out_tokens, d.out_lens = 2, 16, 16
    d.beam, d.scores, d.prefix, d.processors = ctypes.pointer(bm), ctypes.pointer(sc), ctypes.pointer(px), ctypes.pointer(pr)
    rc = L.fo1_llm_generate(m, ctypes.byref(d), None)
    msg = L.fo1_last_error().decode()
    assert rc == -1 and "fo1_llm_generate: beam: max_new_tokens 0" in msg, msg
    L.fo1_model_destroy(m)


def test_stream_progress_and_cancel_on_host_memory():
    F, L, _ = _mods()
    cell = (ctypes.c_int32 * 2)(0, 0)
    prog, cancel = ctypes.addressof(cell), ctypes.addressof(cell) + 4
    assert L.fo1_stream_progress(prog) == 0
    cell[0] = 17 | F.FO1_STREAM_DONE
    got = L.fo1_stream_progress(prog)
    assert got & F.FO1_STREAM_DONE and got & (F.FO1_STREAM_DONE - 1) == 17
    assert cell[1] == 0
    L.fo1_stream_cancel(cancel)
    assert cell[1] == 1 and cell[0] == 17 | F.FO1_STREAM_DONE
    assert F.FO1_STREAM_DONE == 1 << 30
