"""A/B two builds of libfo1.so on the same box: time fo1_gemm_bf16 on a list of (M, N, K, act) shapes through each
library (ctypes, CUDA-event timing, L2 flushed), with torch.matmul (cuBLAS) on the same operands as the rate the card
reaches.  Usage: python scripts/ab_gemm.py <libA.so> [<libB.so> ...]

Three sections, one JSON line per row:
  shapes : the engine's large GEMMs (ViT, LLM prefill incl. the gated gate/up, DaViT) at the library's own tile choice;
  tile_n : the largest shapes with the tile width pinned to 128 / 192 / 256.  If TFLOP/s tracks the operand bytes a CTA
           loads per FMA (64 : 77 : 85 FLOP per byte), the operand feed bounds the k-loop;
  ksweep : K, 2K, 4K at fixed M and N.  The slope of ms over K is the k-loop rate, the intercept the fixed cost per tile
           (prologue and epilogue)."""
import ctypes as C
import json
import os
import sys

import numpy as np
import torch


class GemmDesc(C.Structure):
    _fields_ = [("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32),
                ("A", C.c_void_p), ("lda", C.c_int64), ("W", C.c_void_p), ("ldw", C.c_int64),
                ("D", C.c_void_p), ("ldd", C.c_int64), ("d_dtype", C.c_int32),
                ("bias", C.c_void_p), ("bias_dtype", C.c_int32), ("act", C.c_int32),
                ("residual", C.c_void_p), ("ldr", C.c_int64), ("gated", C.c_int32), ("tile_n", C.c_int32), ("split_k", C.c_int32)]


# (M, N, K, act, gated, resid)
SHAPES = [(100352, 4096, 1024, 1, 0, 0), (131072, 3840, 1280, 0, 0, 0), (131072, 1280, 1280, 0, 0, 1), (38240, 2048, 2048, 0, 0, 1),
          (38240, 2048, 11008, 0, 0, 1), (131072, 1280, 3424, 0, 0, 1), (131072, 6848, 1280, 2, 1, 0), (100352, 1024, 4096, 0, 0, 1),
          (38240, 2560, 2048, 0, 0, 0), (38240, 22016, 2048, 2, 1, 0)]
TILE_SWEEP = [(131072, 3840, 1280, 0, 0, 0), (38240, 22016, 2048, 2, 1, 0)]
K_SWEEP = [(131072, 3840, 1280), (38240, 2560, 2048)]


def time_ms(fn, flush, iters=8, skip=3):
    ts = []
    for i in range(iters):
        flush.zero_()
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record(); torch.cuda.synchronize()
        if i >= skip:
            ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def run(section, libs, flush, M, N, K, act=0, gated=0, resid=0, tile_n=0):
    a = (torch.randn(M, K, device="cuda") * 0.5).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda") * 0.05).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda").to(torch.bfloat16)
    out = torch.empty(M, N // 2 if gated else N, device="cuda", dtype=torch.bfloat16)
    d = GemmDesc()
    d.M, d.N, d.K = M, N, K
    d.A, d.lda, d.W, d.ldw, d.D, d.ldd, d.d_dtype = a.data_ptr(), K, w.data_ptr(), K, out.data_ptr(), out.shape[1], 0
    d.bias, d.bias_dtype, d.act, d.gated, d.tile_n = bias.data_ptr(), 0, act, gated, tile_n
    if resid:
        res = torch.randn_like(out)
        d.residual, d.ldr = res.data_ptr(), out.shape[1]
    fl = 2.0 * M * N * K
    row = {"section": section, "M": M, "N": N, "K": K, "act": act, "gated": gated, "resid": resid, "tile_n": tile_n}
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for path, lib in libs:
        def call():
            rc = lib.fo1_gemm_bf16(C.byref(d), st)
            assert rc == 0, rc
        ms = time_ms(call, flush)
        row[path] = {"ms": round(ms, 3), "tflops": round(fl / ms / 1e9, 1)}
    if tile_n == 0:
        full = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)   # the plain product: cuBLAS has no fused gate
        ms = time_ms(lambda: torch.matmul(a, w.t(), out=full), flush)
        row["cublas"] = {"ms": round(ms, 3), "tflops": round(fl / ms / 1e9, 1)}
        del full
    print(json.dumps(row), flush=True)


def main():
    libs = [(p, C.CDLL(os.path.abspath(p))) for p in sys.argv[1:]]
    for _, lib in libs:
        lib.fo1_gemm_bf16.restype = C.c_int
    print(json.dumps({"device": torch.cuda.get_device_name(0)}), flush=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for M, N, K, act, gated, resid in SHAPES:
        run("shapes", libs, flush, M, N, K, act, gated, resid)
    for M, N, K, act, gated, resid in TILE_SWEEP:
        for tn in (128, 192, 256):
            run("tile_n", libs, flush, M, N, K, act, gated, resid, tile_n=tn)
    for M, N, K in K_SWEEP:
        for k in (K, 2 * K, 4 * K):
            run("ksweep", libs, flush, M, N, k)


if __name__ == "__main__":
    main()
