"""Stateless operator wrappers over the C ABI (device pointers in, device pointers out).
torch tensors are only the memory handles; every computation happens inside libfo1.so."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib
from ._lib import GemmDesc, check, lib

_ACT = {None: _lib.EPI_NONE, "none": _lib.EPI_NONE, "gelu": _lib.EPI_GELU, "silu": _lib.EPI_SILU}
_DT = {torch.bfloat16: _lib.FO1_BF16, torch.float32: _lib.FO1_F32}


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _require_cuda(*ts) -> None:
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _lib.Fo1Error("libfo1 operators take CUDA tensors only (no CPU fallback)")


def gemm(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, act: Optional[str] = None,
         residual: Optional[torch.Tensor] = None, out_dtype: torch.dtype = torch.bfloat16, gated: bool = False,
         out: Optional[torch.Tensor] = None, tile_n: int = 0, split_k: int = 0) -> torch.Tensor:
    """out[M, N] = act(a[M, K] @ w[N, K]^T + bias) + residual   (nn.Linear semantics).
    ``gated``: w/bias rows interleave [32 gate | 32 up] blocks -> out[M, N/2] = act(gate) * up.
    ``tile_n`` / ``split_k`` pin the tile width and the in-kernel K split (0 = the library's choice)."""
    _require_cuda(a, w, bias, residual)
    assert a.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and a.dim() == 2 and w.dim() == 2
    assert a.stride(1) == 1 and w.stride(1) == 1 and a.shape[1] == w.shape[1]
    M, K = a.shape
    N = w.shape[0]
    n_out = N // 2 if gated else N
    if out is None:
        out = torch.empty((M, n_out), dtype=out_dtype, device=a.device)
    assert out.shape == (M, n_out) and out.stride(1) == 1
    d = GemmDesc()
    d.M, d.N, d.K = M, N, K
    d.A, d.lda = a.data_ptr(), a.stride(0)
    d.W, d.ldw = w.data_ptr(), w.stride(0)
    d.D, d.ldd, d.d_dtype = out.data_ptr(), out.stride(0), _DT[out.dtype]
    if bias is not None:
        assert bias.shape == (N,) and bias.is_contiguous()
        d.bias, d.bias_dtype = bias.data_ptr(), _DT[bias.dtype]
    d.act = _ACT[act]
    if residual is not None:
        assert residual.dtype == torch.bfloat16 and residual.shape == (M, n_out) and residual.stride(1) == 1
        d.residual, d.ldr = residual.data_ptr(), residual.stride(0)
    d.gated = 1 if gated else 0
    d.tile_n, d.split_k = int(tile_n), int(split_k)
    check(lib().fo1_gemm_bf16(C.byref(d), C.c_void_p(_stream())), "fo1_gemm_bf16")
    return out


def interleave_gate_up(gate: torch.Tensor, up: torch.Tensor, block: int = 32) -> torch.Tensor:
    """Host-side weight prep for the gated epilogue: rows (or bias entries) of gate/up interleaved in
    blocks of ``block``; the row count is zero-padded to a multiple of ``block`` first."""
    n = gate.shape[0]
    pad = (-n) % block
    if pad:
        z = torch.zeros((pad,) + tuple(gate.shape[1:]), dtype=gate.dtype, device=gate.device)
        gate = torch.cat([gate, z]); up = torch.cat([up, z])
    g = gate.reshape(-1, block, *gate.shape[1:])
    u = up.reshape(-1, block, *up.shape[1:])
    return torch.stack([g, u], dim=1).reshape(-1, *gate.shape[1:]).contiguous()


def attention_varlen(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, cu_seqlens: torch.Tensor, max_seqlen: int,
                     q_heads: int, kv_heads: int, head_dim: int, scale: float, causal: bool = False,
                     out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """q/k/v: bf16 [T, heads*head_dim] views (any row pitch, unit column stride); cu_seqlens int32 [n+1] on device."""
    _require_cuda(q, k, v, cu_seqlens)
    T = q.shape[0]
    if out is None:
        out = torch.empty((T, q_heads * head_dim), dtype=torch.bfloat16, device=q.device)
    d = _lib.AttnDesc()
    d.q, d.k, d.v, d.o = q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr()
    d.ldq, d.ldk, d.ldv, d.ldo = q.stride(0), k.stride(0), v.stride(0), out.stride(0)
    assert cu_seqlens.dtype == torch.int32
    d.cu_seqlens = cu_seqlens.data_ptr()
    d.n_seqs, d.max_seqlen = cu_seqlens.numel() - 1, max_seqlen
    d.q_heads, d.kv_heads, d.head_dim = q_heads, kv_heads, head_dim
    d.scale, d.causal = scale, 1 if causal else 0
    d.total_rows = T
    check(lib().fo1_attention_varlen(C.byref(d), C.c_void_p(_stream())), "fo1_attention_varlen")
    return out


def decode_attention(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, cache_len: torch.Tensor, q_heads: int, kv_heads: int,
                     scale: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """One decode step of GQA attention over the cache: q bf16 [B, q_heads*128]; k_cache / v_cache bf16 [B, cap, kv_heads*128];
    cache_len int32 [B] on the device (keys 0..cache_len[b] inclusive are attended)."""
    _require_cuda(q, k_cache, v_cache, cache_len)
    B, cap = k_cache.shape[0], k_cache.shape[1]
    assert q.dtype == torch.bfloat16 and k_cache.dtype == torch.bfloat16 and v_cache.dtype == torch.bfloat16 and cache_len.dtype == torch.int32
    assert k_cache.is_contiguous() and v_cache.is_contiguous() and q.stride(1) == 1
    if out is None:
        out = torch.empty((B, q_heads * 128), dtype=torch.bfloat16, device=q.device)
    L = lib()
    need = L.fo1_decode_attention_workspace_bytes(B, q_heads)
    ws = torch.empty(max(need, 16), dtype=torch.uint8, device=q.device)
    d = _lib.DecodeAttnDesc()
    d.q, d.ldq, d.k_cache, d.v_cache, d.cache_len = q.data_ptr(), q.stride(0), k_cache.data_ptr(), v_cache.data_ptr(), cache_len.data_ptr()
    d.n_seqs, d.cap, d.q_heads, d.kv_heads, d.head_dim, d.scale = B, cap, q_heads, kv_heads, 128, scale
    d.out, d.ldo, d.workspace, d.workspace_bytes = out.data_ptr(), out.stride(0), ws.data_ptr(), ws.numel()
    check(L.fo1_decode_attention(C.byref(d), C.c_void_p(_stream())), "fo1_decode_attention")
    return out


def dwconv3x3_residual(x: torch.Tensor, w9: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """DaViT conv position encoding: x bf16 [B, H, W, C] (NHWC), w9 bf16 [9, C], bias bf16 [C] -> x + dwconv3x3(x) + bias (fo1_dwconv3x3_residual)."""
    _require_cuda(x)
    assert x.dtype == torch.bfloat16 and x.dim() == 4 and x.is_contiguous() and w9.is_contiguous() and bias.is_contiguous()
    B, H, W, Cc = x.shape
    assert tuple(w9.shape) == (9, Cc) and tuple(bias.shape) == (Cc,)
    y = torch.empty_like(x)
    L = lib()
    L.fo1_dwconv3x3_residual.restype = C.c_int
    L.fo1_dwconv3x3_residual.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
    check(L.fo1_dwconv3x3_residual(C.c_void_p(x.data_ptr()), C.c_void_p(w9.data_ptr()), C.c_void_p(bias.data_ptr()), C.c_void_p(y.data_ptr()),
                                   B, H, W, Cc, C.c_void_p(_stream())), "fo1_dwconv3x3_residual")
    return y


NORM_WARP, NORM_BLOCK = 0, 1      # fo1_row_norm's kernel: one warp per row / one block per row


def row_norm(x: torch.Tensor, gamma: Optional[torch.Tensor], beta: Optional[torch.Tensor], eps: float, rms: bool, kernel: int,
             out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """RMSNorm (``rms``; beta None) or LayerNorm of the rows of x bf16 [rows, cols] (any row pitch, unit column stride) with the named
    kernel (fo1_row_norm).  ``out``: optional bf16 [rows, cols] view (any row pitch) written in place."""
    _require_cuda(x, gamma, beta, out)
    assert x.dtype == torch.bfloat16 and x.dim() == 2 and x.stride(1) == 1
    rows, cols = x.shape
    for t in (gamma, beta):
        assert t is None or (t.dtype == torch.bfloat16 and tuple(t.shape) == (cols,) and t.is_contiguous())
    if out is None:
        out = torch.empty((rows, cols), dtype=torch.bfloat16, device=x.device)
    assert out.dtype == torch.bfloat16 and tuple(out.shape) == (rows, cols) and out.stride(1) == 1
    L = lib()
    L.fo1_row_norm.restype = C.c_int
    L.fo1_row_norm.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_float,
                               C.c_int32, C.c_int32, C.c_void_p]
    ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    check(L.fo1_row_norm(ptr(x), x.stride(0), ptr(gamma), ptr(beta), ptr(out), out.stride(0), rows, cols, eps, 1 if rms else 0, kernel,
                         C.c_void_p(_stream())), "fo1_row_norm")
    return out


def channel_attention(qkv: torch.Tensor, groups: int) -> torch.Tensor:
    """DaViT channel-group attention: qkv bf16 [B, N, 3C] -> bf16 [B, N, C] (fo1_channel_attention)."""
    _require_cuda(qkv)
    assert qkv.dtype == torch.bfloat16 and qkv.dim() == 3 and qkv.is_contiguous() and qkv.shape[2] % 3 == 0
    B, N, C3 = qkv.shape
    Cc = C3 // 3
    out = torch.empty((B, N, Cc), dtype=torch.bfloat16, device=qkv.device)
    L = lib()
    L.fo1_channel_attention_workspace_bytes.restype = C.c_size_t
    L.fo1_channel_attention_workspace_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32]
    L.fo1_channel_attention.restype = C.c_int
    L.fo1_channel_attention.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    need = L.fo1_channel_attention_workspace_bytes(B, N, Cc)
    ws = torch.empty(max(need, 16), dtype=torch.uint8, device=qkv.device)
    check(L.fo1_channel_attention(C.c_void_p(qkv.data_ptr()), B, N, Cc, groups, C.c_void_p(out.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(),
                                  C.c_void_p(_stream())), "fo1_channel_attention")
    return out
