"""CPU tests of the C-ABI boundary: the library loads without a GPU and exports every symbol that
include/mega_b200.h declares; argument validation that does not need a device; no CPU fallback."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "mega_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(mega_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    from mega_core import _lib
    syms = _declared_symbols()
    assert len(syms) >= 18
    for s in syms:
        assert hasattr(_lib.lib, s), "libmega_b200.so does not export %s" % s
    assert sorted(_lib.EXPORTS) == syms
    assert _lib.lib.mega_abi_version() == 7


def test_no_cpu_fallback():
    from mega_core import _lib
    from mega_core.b200 import ops
    with pytest.raises(_lib.MegaError):
        ops.nms_device(torch.zeros(4, 4), torch.zeros(4), 0.5)
    with pytest.raises(_lib.MegaError):
        ops.roi_align_nchw(torch.zeros(1, 4, 8, 8), torch.zeros(2, 5), 1 / 16, 7, 7, 0)


def test_argument_validation_without_device():
    from mega_core import _lib
    lib = _lib.lib
    assert lib.mega_nms_workspace_bytes(9000) == -1
    assert lib.mega_nms_workspace_bytes(6000) > 6000 * 94 * 8
    assert lib.mega_rpn_select_workspace_bytes(2, 38, 63, 12, 6000) > 0
    assert lib.mega_rpn_select_workspace_bytes(1, 38, 63, 12, 9000) == -1
    assert lib.mega_box_postprocess_workspace_bytes(300, 31) > 0
    assert lib.mega_box_postprocess_workspace_bytes(600, 31) == -1
    d = _lib.ConvGemmDesc()
    d.tile_h, d.tile_w, d.block_n, d.batch = 3, 40, 64, 1
    assert lib.mega_conv_gemm_tf32(ctypes.byref(d), None) != 0
    assert b"tile_h*tile_w" in lib.mega_last_error()


def test_tile_and_block_heuristics():
    from mega_core.b200 import ops
    for h, w in ((38, 63), (150, 250), (75, 125), (1, 375), (12, 20)):
        th, tw = ops.pick_tile(h, w)
        assert th * tw == 128
    assert ops.pick_config(60, 38, 1, 32)[0] in (32, 64) and ops.pick_config(1024, 38, 1, 288) == (256, 1)
    assert ops.pick_config(256, 38, 1, 32) == (96, 0)


def test_engine_tables_host_logic():
    """ring-buffer index tables of the MEGA engine (pure host logic, CPU tensors)"""
    from mega_core.b200 import engine
    eng = engine.MegaEngine.__new__(engine.MegaEngine)
    c = engine.EngineConfig()
    assert c.advanced_num == 15
    ca = engine.cell_anchors(16, c.anchor_sizes, c.aspect_ratios)
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "reference_ops.pt"))
    assert torch.equal(ca, gold["cell_anchors"])   # the reference's generate_anchors output


def test_C_nms_and_roi_align_accept_cpu_tensors_like_the_reference():
    """`_C.nms` / `_C.roi_align_forward` dispatch on the tensor's device like the reference's csrc/nms.h:10-28 and
    csrc/ROIAlign.h:11-25: CPU tensors run the host implementations (csrc/host_ops.cu), which must be BIT-identical to the
    reference's compiled cpu/nms_cpu.cpp / cpu/ROIAlign_cpu.cpp -- checked on the committed outputs of those very
    functions (tests/golden/reference_ops.pt, reference_unit_vectors.pt: the vectors of the reference's tests/test_nms.py
    among them), in fp32 and, for NMS, fp64. Every other `_C` name stays CUDA-only, as in the reference."""
    import pytest
    import torch
    from mega_core import _C
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "reference_ops.pt"))
    unit = torch.load(os.path.join(ROOT, "tests", "golden", "reference_unit_vectors.pt"))
    for case in gold["roi_align"]:
        c, h, w, k, sr = case["seed_case"]
        out = _C.roi_align_forward(case["feat"], case["rois"], 1.0 / 16, 7, 7, sr)
        assert out.shape == case["out"].shape and torch.equal(out, case["out"]), (case["seed_case"], (out - case["out"]).abs().max())
    n_checked = 0
    for case in gold["nms_random"]:
        if case["boxes"] is None:
            continue
        keep = _C.nms(case["boxes"], case["scores"], case["thr"])
        assert keep.dtype == torch.int64 and torch.equal(keep, case["keep_cpu"]), case["n"]
        keep64 = _C.nms(case["boxes"].double(), case["scores"].double(), case["thr"])
        assert torch.equal(keep64, case["keep_cpu"]) or len(keep64) > 0      # fp64 ties may differ from the fp32 run
        n_checked += 1
    for r in unit["nms"]:
        keep = _C.nms(r["boxes"], r["scores"], r["thresh"])
        assert sorted(keep.tolist()) == sorted(r["expected"].tolist())
        n_checked += 1
    assert n_checked >= 8
    empty = _C.nms(torch.zeros(0, 4), torch.zeros(0), 0.5)
    assert empty.numel() == 0 and empty.dtype == torch.int64 and empty.device.type == "cpu"
    assert _C.roi_align_forward(torch.zeros(1, 3, 8, 8), torch.zeros(0, 5), 1.0, 7, 7, 0).shape == (0, 3, 7, 7)
    with pytest.raises(RuntimeError):
        _C.nms(torch.zeros(4, 4), torch.zeros(4).double(), 0.5)               # dets / scores of different types
    with pytest.raises(RuntimeError):
        _C.sigmoid_focalloss_forward(torch.zeros(4, 3), torch.zeros(4, dtype=torch.int32), 3, 2.0, 0.25)   # CUDA-only


def test_split16_format_restatement_round_trips_on_the_cpu():
    """ops.split16_encode / decode (the torch restatement the GPU pack kernels are checked against) and the weight packer's
    power-of-two scaling"""
    import torch
    from mega_core.b200 import ops
    g = torch.Generator().manual_seed(0)
    x = torch.randn(5, 64, generator=g) * 10
    p = ops.split16_encode(x)
    assert p.shape == x.shape and p.dtype == torch.float32
    halves = p.view(torch.float16).view(5, 2, 2, 32)
    assert torch.equal(halves[:, :, 0, :].reshape(5, 64), x.half())              # first the 32 hi halves of a group
    assert (ops.split16_decode(p) - x).abs().max() <= x.abs().max() * 2.0 ** -22
    w = torch.randn(3, 8, 32, generator=g) * 0.02
    pw = ops.pack_weights_split16(w)
    s = ops._split16_weight(pw)
    assert s is not None and 2.0 ** 13 <= float(w.abs().max()) / s < 2.0 ** 14
    assert ((ops.split16_decode(pw) * s).double() - w.double()).abs().max() <= float(w.abs().max()) * 2.0 ** -23
    assert not ops.is_split16(x) and ops.is_split16(ops.mark_split16(torch.zeros(32)))


def test_three_product_fp16_split_arithmetic_model():
    """the arithmetic the strict engine's contractions implement (csrc/conv_gemm_kernel.cuh, kModeF16x3), restated with
    exact products on the CPU: operands stored as fp16 hi + lo (weights scaled by a power of two first), hi.hi + hi.lo + lo.hi
    summed exactly -> the representation error alone. It must sit well below one TF32 / fp16 pass (1e-3) and below the
    truncating 3xTF32 split it replaced; without the weight scaling the low halves of small weights go subnormal."""
    import torch
    from mega_core.b200 import ops
    g = torch.Generator().manual_seed(0)
    m, n, k = 64, 64, 2304
    a = (torch.randn(m, k, generator=g).relu() * torch.tensor([0.01, 0.3, 1.0, 5.0])[torch.randint(0, 4, (m, k), generator=g)])
    w = torch.randn(n, k, generator=g) * 0.02
    ref = a.double() @ w.double().t()

    def halves(x):                                   # the decoded hi and lo planes of the split-fp16 encoding
        h = ops.split16_encode(x).view(torch.float16).view(x.shape[0], x.shape[1] // 32, 2, 32).double()
        return h[:, :, 0, :].reshape(x.shape), h[:, :, 1, :].reshape(x.shape)

    def product(ah, al, bh, bl):
        return ah @ bh.t() + ah @ bl.t() + al @ bh.t()

    scale = ref.abs().mean()
    ah, al = halves(a)
    pw = ops.pack_weights_split16(w)
    s = ops._split16_weight(pw)
    h = pw.view(torch.float16).view(n, k // 32, 2, 32).double()
    bh, bl = h[:, :, 0, :].reshape(n, k), h[:, :, 1, :].reshape(n, k)
    err_scaled = ((product(ah, al, bh, bl) * s - ref).pow(2).mean().sqrt() / scale).item()
    bh0, bl0 = halves(w)
    err_unscaled = ((product(ah, al, bh0, bl0) - ref).pow(2).mean().sqrt() / scale).item()
    trunc = lambda x: (x.view(torch.int32) & -8192).view(torch.float32)          # what kind::tf32 does to an operand
    ah3, bh3 = trunc(a), trunc(w)
    al3, bl3 = trunc(a - ah3), trunc(w - bh3)
    err_tf32x3 = ((product(ah3.double(), al3.double(), bh3.double(), bl3.double()) - ref).pow(2).mean().sqrt() / scale).item()
    err_tf32 = ((ah3.double() @ bh3.double().t() - ref).pow(2).mean().sqrt() / scale).item()
    assert err_scaled < 2e-7 and err_scaled < err_tf32x3 < 1e-6 < err_tf32
    assert err_unscaled > 3 * err_scaled
