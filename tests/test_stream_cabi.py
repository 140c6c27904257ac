"""CPU checks of the streamed-decoding C ABI (include/fo1.h, fo1_stream_desc): fo1_llm_generate_streamed refuses missing stream
buffers before it touches the model or the device, and the host-side progress / cancel accessors work on ordinary host memory."""
import ctypes
from importlib import import_module

import pytest


def _mods():
    import fo1_b200
    return fo1_b200._lib, fo1_b200.lib(), import_module("vlm-fo1_b200.engine")


@pytest.mark.parametrize("case", ["null_model", "null_desc", "null_tokens", "null_lens", "null_progress"])
def test_generate_streamed_rejects_null_buffers_without_gpu(case):
    F, L, E = _mods()
    d = E.GenerateDescC()
    d.n_seqs = 1
    buf = (ctypes.c_int32 * 64)()
    p = ctypes.addressof(buf)
    fields = dict(tokens=p, lens=p + 32 * 4, progress=p + 48 * 4, cancel=None)
    if case.startswith("null_") and case[5:] in fields:
        fields[case[5:]] = None
    st = F.StreamDesc(**fields)
    model = None if case == "null_model" else ctypes.c_void_p(16)         # never dereferenced: the check comes first
    desc = None if case == "null_desc" else ctypes.byref(d)
    rc = L.fo1_llm_generate_streamed(model, desc, None, None, ctypes.byref(st), None)
    assert rc == -1
    msg = L.fo1_last_error().decode()
    assert "fo1_llm_generate_streamed" in msg and ("null" in msg), msg


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
