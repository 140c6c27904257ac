"""CPU: the C-ABI library builds, loads, and exports every symbol include/fo1.h declares."""
import ctypes


def test_library_loads_abi_4_and_exports_header_symbols():
    import __graft_entry__ as G
    G.build()
    import fo1_b200
    L = fo1_b200.lib()
    assert L.fo1_abi_version() == 4
    syms = fo1_b200._lib.exported_symbols()
    assert "fo1_hfre_forward" in syms and "fo1_gemm_bf16" in syms
    for s in syms:
        assert hasattr(L, s), f"libfo1.so does not export {s}"
    assert L.fo1_last_error() in (b"",) or isinstance(L.fo1_last_error(), bytes)


def test_hfre_argument_validation_without_gpu():
    """Host-side argument checks run before any CUDA call, so they are testable on a CPU box."""
    import fo1_b200
    HfreImage, HfreParams = fo1_b200._lib.HfreImage, fo1_b200._lib.HfreParams
    L = fo1_b200.lib()
    imgs = (HfreImage * 1)()
    imgs[0].n_levels = 0
    imgs[0].n_boxes = 1
    p = HfreParams(64, 7, 1)
    rc = L.fo1_hfre_forward(imgs, 1, ctypes.byref(p), None, 0, None)
    assert rc != 0 and len(L.fo1_last_error()) > 0
    p2 = HfreParams(66, 7, 1)   # out_dim not a multiple of 4
    assert L.fo1_hfre_forward(imgs, 1, ctypes.byref(p2), None, 0, None) == -1
