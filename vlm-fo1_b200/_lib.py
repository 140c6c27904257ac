"""ctypes binding of libfo1.so (the C ABI in include/fo1.h).  No CPU fallback: if the library is
missing or a call fails, this raises."""
from __future__ import annotations

import ctypes as C
import os

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "libfo1.so")

FO1_HFRE_MAX_LEVELS = 8
FO1_BF16, FO1_F32, FO1_I32, FO1_I64, FO1_U8, FO1_F16 = range(6)
EPI_NONE, EPI_GELU, EPI_SILU = range(3)


class Fo1Error(RuntimeError):
    pass


class HfreLevel(C.Structure):
    _fields_ = [("data", C.c_void_p), ("H", C.c_int32), ("W", C.c_int32), ("C", C.c_int32),
                ("up_H", C.c_int32), ("up_W", C.c_int32), ("spatial_scale", C.c_float),
                ("box_set", C.c_int32), ("out_offset", C.c_int32)]


class HfreImage(C.Structure):
    _fields_ = [("levels", HfreLevel * FO1_HFRE_MAX_LEVELS), ("n_levels", C.c_int32), ("n_boxes", C.c_int32),
                ("boxes_aux", C.c_void_p), ("boxes_vt", C.c_void_p), ("out", C.c_void_p),
                ("out_bf16", C.c_void_p), ("pos_img_w", C.c_float), ("pos_img_h", C.c_float),
                ("pos_box_set", C.c_int32)]


class HfreParams(C.Structure):
    _fields_ = [("out_dim", C.c_int32), ("roi_size", C.c_int32), ("apply_pos_embed", C.c_int32)]


class GemmDesc(C.Structure):
    _fields_ = [("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32),
                ("A", C.c_void_p), ("lda", C.c_int64), ("W", C.c_void_p), ("ldw", C.c_int64),
                ("D", C.c_void_p), ("ldd", C.c_int64), ("d_dtype", C.c_int32),
                ("bias", C.c_void_p), ("bias_dtype", C.c_int32), ("act", C.c_int32),
                ("residual", C.c_void_p), ("ldr", C.c_int64), ("gated", C.c_int32), ("tile_n", C.c_int32), ("split_k", C.c_int32)]


class AttnDesc(C.Structure):
    _fields_ = [("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p), ("o", C.c_void_p),
                ("ldq", C.c_int64), ("ldk", C.c_int64), ("ldv", C.c_int64), ("ldo", C.c_int64),
                ("cu_seqlens", C.c_void_p), ("n_seqs", C.c_int32), ("max_seqlen", C.c_int32),
                ("q_heads", C.c_int32), ("kv_heads", C.c_int32), ("head_dim", C.c_int32),
                ("scale", C.c_float), ("causal", C.c_int32), ("total_rows", C.c_int32)]


class DecodeAttnDesc(C.Structure):
    _fields_ = [("q", C.c_void_p), ("ldq", C.c_int64), ("k_cache", C.c_void_p), ("v_cache", C.c_void_p), ("cache_len", C.c_void_p),
                ("n_seqs", C.c_int32), ("cap", C.c_int32), ("q_heads", C.c_int32), ("kv_heads", C.c_int32), ("head_dim", C.c_int32),
                ("scale", C.c_float), ("out", C.c_void_p), ("ldo", C.c_int64), ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t)]


class SamplingDesc(C.Structure):
    """fo1_sampling_desc: HOST arrays of per-row temperature, top_p, top_k, seed."""
    _fields_ = [("temperature", C.POINTER(C.c_float)), ("top_p", C.POINTER(C.c_float)), ("top_k", C.POINTER(C.c_int32)),
                ("seed", C.POINTER(C.c_uint64))]


def sampling_desc(temperature, top_p, top_k, seed):
    """-> (SamplingDesc, the ctypes arrays it points into: keep them alive for the call)."""
    n = len(temperature)
    assert len(top_p) == n and len(top_k) == n and len(seed) == n, "one temperature / top_p / top_k / seed per row"
    arrs = ((C.c_float * n)(*[float(x) for x in temperature]), (C.c_float * n)(*[float(x) for x in top_p]),
            (C.c_int32 * n)(*[int(x) for x in top_k]), (C.c_uint64 * n)(*[int(x) & 0xFFFFFFFFFFFFFFFF for x in seed]))
    return SamplingDesc(*arrs), arrs


class ScoreDesc(C.Structure):
    """fo1_score_desc: optional DEVICE outputs logprobs [n][max_new], scores / logits [max_new][n][V]; HOST raw_rows [n]."""
    _fields_ = [("logprobs", C.c_void_p), ("scores", C.c_void_p), ("logits", C.c_void_p), ("raw_rows", C.POINTER(C.c_int32))]


class StreamDesc(C.Structure):
    """fo1_stream_desc: HOST pointers to pinned, mapped memory: tokens [n][max_new], lens [n], progress [1], cancel [1] (optional)."""
    _fields_ = [("tokens", C.c_void_p), ("lens", C.c_void_p), ("progress", C.c_void_p), ("cancel", C.c_void_p)]


class PrefixDesc(C.Structure):
    """fo1_prefix_desc: HOST prefix_lens [n_groups], seq_group [n_seqs]; DEVICE prefix_embeds bf16 [sum P][hidden], position ids [3][sum P]."""
    _fields_ = [("n_groups", C.c_int32), ("prefix_lens", C.POINTER(C.c_int32)), ("prefix_embeds", C.c_void_p),
                ("prefix_position_ids", C.c_void_p), ("seq_group", C.POINTER(C.c_int32))]


class PrefixAttnDesc(C.Structure):
    _fields_ = [("q", C.c_void_p), ("ldq", C.c_int64), ("k_cache", C.c_void_p), ("v_cache", C.c_void_p), ("n_seqs", C.c_int32),
                ("cap", C.c_int32), ("prefix_lens", C.POINTER(C.c_int32)), ("own_lens", C.POINTER(C.c_int32)), ("q_heads", C.c_int32),
                ("kv_heads", C.c_int32), ("head_dim", C.c_int32), ("scale", C.c_float), ("out", C.c_void_p), ("ldo", C.c_int64)]


class LoglikDesc(C.Structure):
    """fo1_loglik_desc: HOST seq_lens [n] and targets [sum L]; DEVICE embeddings, positions [3][rows], outputs logprobs / greedy
    [sum L], seq_logprob fp64 / seq_count [n], all_logits [sum L][V], lse / target_logits [n_scored]."""
    _fields_ = [("n_seqs", C.c_int32), ("seq_lens", C.POINTER(C.c_int32)), ("inputs_embeds", C.c_void_p), ("position_ids", C.c_void_p),
                ("prefix", C.POINTER(PrefixDesc)), ("targets", C.POINTER(C.c_int32)), ("logprobs", C.c_void_p), ("greedy", C.c_void_p),
                ("seq_logprob", C.c_void_p), ("seq_count", C.c_void_p), ("all_logits", C.c_void_p), ("lse", C.c_void_p),
                ("target_logits", C.c_void_p)]


class BeamDesc(C.Structure):
    """fo1_beam_desc: HOST parameters; DEVICE outputs sequence_scores [n * num_return], beam_indices [n * num_return][max_new],
    steps_run [n], optional scores / logits [max_new][n * num_beams][V] and logprobs [n * num_return][max_new]."""
    _fields_ = [("num_beams", C.c_int32), ("n_keep", C.c_int32), ("length_penalty", C.c_double), ("early_stopping", C.c_int32),
                ("num_return", C.c_int32), ("sequence_scores", C.c_void_p), ("beam_indices", C.c_void_p), ("steps_run", C.c_void_p),
                ("scores", C.c_void_p), ("logits", C.c_void_p), ("logprobs", C.c_void_p)]


class LookupDesc(C.Structure):
    """fo1_lookup_desc: HOST num_tokens, max_ngram, packed corpus int32 and offsets [n + 1]; optional DEVICE int32 [n] outputs steps /
    accepted."""
    _fields_ = [("num_tokens", C.c_int32), ("max_ngram", C.c_int32), ("corpus", C.POINTER(C.c_int32)),
                ("corpus_offsets", C.POINTER(C.c_int32)), ("steps", C.c_void_p), ("accepted", C.c_void_p)]


class SlotsDesc(C.Structure):
    """fo1_slots_desc: HOST parameters and stop ids; DEVICE int32 outputs tokens [n_slots][max_new], lens [n_slots], finished [n_slots]."""
    _fields_ = [("n_slots", C.c_int32), ("cap", C.c_int32), ("max_new_tokens", C.c_int32), ("stop_ids", C.POINTER(C.c_int32)),
                ("n_stop_ids", C.c_int32), ("pad_id", C.c_int32), ("sampled", C.c_int32), ("early_exit_interval", C.c_int32),
                ("out_tokens", C.c_void_p), ("out_lens", C.c_void_p), ("finished", C.c_void_p)]


class ProcessorDesc(C.Structure):
    """fo1_processor_desc: every array HOST; per sequence its set (-1: none) and prompt ids, per set its settings and id lists."""
    _fields_ = [("n_sets", C.c_int32), ("seq_set", C.POINTER(C.c_int32)), ("prompt", C.POINTER(C.c_int32)),
                ("prompt_offsets", C.POINTER(C.c_int32)), ("no_repeat_ngram_size", C.POINTER(C.c_int32)), ("min_length", C.POINTER(C.c_int32)),
                ("min_new_tokens", C.POINTER(C.c_int32)), ("eos_offsets", C.POINTER(C.c_int32)), ("suppress_offsets", C.POINTER(C.c_int32)),
                ("begin_suppress_offsets", C.POINTER(C.c_int32)), ("bias_offsets", C.POINTER(C.c_int32)), ("bad_offsets", C.POINTER(C.c_int32)),
                ("n_sequences", C.c_int32), ("seq_offsets", C.POINTER(C.c_int32)), ("bias", C.POINTER(C.c_float)), ("n_ids", C.c_int32),
                ("ids", C.POINTER(C.c_int32))]


class SlotsAdmitDesc(C.Structure):
    """fo1_slots_admit_desc: HOST slots / seq_lens / max_new_tokens [n]; DEVICE embeddings, positions [3][sum L], rope deltas [n]."""
    _fields_ = [("n", C.c_int32), ("slots", C.POINTER(C.c_int32)), ("seq_lens", C.POINTER(C.c_int32)), ("inputs_embeds", C.c_void_p),
                ("position_ids", C.c_void_p), ("rope_deltas_device", C.c_void_p), ("max_new_tokens", C.POINTER(C.c_int32)),
                ("sampling", C.POINTER(SamplingDesc)), ("processors", C.POINTER(ProcessorDesc))]


FO1_STREAM_DONE = 1 << 30

_lib = None


def lib() -> C.CDLL:
    """Load libfo1.so once.  Raises Fo1Error if it has not been built (``__graft_entry__.build()``)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise Fo1Error(f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                       "(there is no CPU or PyTorch fallback for the FO1 hot path)")
    L = C.CDLL(LIB_PATH)
    L.fo1_abi_version.restype = C.c_int
    L.fo1_last_error.restype = C.c_char_p
    L.fo1_launch_count.restype = C.c_uint64
    L.fo1_last_decode_path.restype = C.c_int
    L.fo1_last_decode_path.argtypes = [C.c_void_p]
    L.fo1_launch_count_reset.restype = None
    L.fo1_hfre_workspace_bytes.restype = C.c_size_t
    L.fo1_hfre_workspace_bytes.argtypes = [C.POINTER(HfreImage), C.c_int32, C.POINTER(HfreParams)]
    L.fo1_hfre_forward.restype = C.c_int
    L.fo1_hfre_forward.argtypes = [C.POINTER(HfreImage), C.c_int32, C.POINTER(HfreParams), C.c_void_p,
                                   C.c_size_t, C.c_void_p]
    L.fo1_decode_attention_workspace_bytes.restype = C.c_size_t
    L.fo1_decode_attention_workspace_bytes.argtypes = [C.c_int32, C.c_int32]
    L.fo1_decode_attention.restype = C.c_int
    L.fo1_decode_attention.argtypes = [C.POINTER(DecodeAttnDesc), C.c_void_p]
    L.fo1_gemm_bf16.restype = C.c_int
    L.fo1_gemm_bf16.argtypes = [C.POINTER(GemmDesc), C.c_void_p]
    L.fo1_attention_varlen.restype = C.c_int
    L.fo1_attention_varlen.argtypes = [C.POINTER(AttnDesc), C.c_void_p]
    L.fo1_sample_tokens_workspace_bytes.restype = C.c_size_t
    L.fo1_sample_tokens_workspace_bytes.argtypes = [C.c_int32]
    L.fo1_sample_tokens.restype = C.c_int
    L.fo1_sample_tokens.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.POINTER(SamplingDesc), C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_size_t, C.c_void_p]
    L.fo1_llm_generate.restype = C.c_int
    L.fo1_llm_generate.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.fo1_llm_loglik.restype = C.c_int
    L.fo1_llm_loglik.argtypes = [C.c_void_p, C.POINTER(LoglikDesc), C.c_void_p]
    L.fo1_logits_process.restype = C.c_int
    L.fo1_logits_process.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.POINTER(ProcessorDesc), C.c_void_p, C.c_int64,
                                     C.POINTER(C.c_int32), C.c_void_p]
    L.fo1_slots_open.restype = C.c_int
    L.fo1_slots_open.argtypes = [C.c_void_p, C.POINTER(SlotsDesc), C.c_void_p]
    L.fo1_slots_admit.restype = C.c_int
    L.fo1_slots_admit.argtypes = [C.c_void_p, C.POINTER(SlotsAdmitDesc), C.c_void_p]
    L.fo1_slots_decode.restype = C.c_int
    L.fo1_slots_decode.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.c_void_p]
    L.fo1_slots_close.restype = C.c_int
    L.fo1_slots_close.argtypes = [C.c_void_p]
    L.fo1_lookup_drafts.restype = C.c_int
    L.fo1_lookup_drafts.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p,
                                    C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.fo1_prefix_attention.restype = C.c_int
    L.fo1_prefix_attention.argtypes = [C.POINTER(PrefixAttnDesc), C.c_void_p]
    L.fo1_stream_progress.restype = C.c_int32
    L.fo1_stream_progress.argtypes = [C.c_void_p]
    L.fo1_stream_cancel.restype = None
    L.fo1_stream_cancel.argtypes = [C.c_void_p]
    L.fo1_score_rows.restype = C.c_int
    L.fo1_score_rows.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.POINTER(SamplingDesc), C.POINTER(C.c_int32), C.c_void_p,
                                 C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    _lib = L
    return L


def check(status: int, what: str) -> None:
    if status != 0:
        msg = lib().fo1_last_error().decode("utf-8", "replace")
        raise Fo1Error(f"{what} failed with status {status}: {msg}")


def exported_symbols() -> list:
    """Every symbol include/fo1.h declares (used by the CPU test that the library loads)."""
    import re
    hdr = os.path.join(os.path.dirname(_PKG), "include", "fo1.h")
    text = open(hdr).read()
    return sorted(set(re.findall(r"\b(fo1_[a-z0-9_]+)\s*\(", text)))
