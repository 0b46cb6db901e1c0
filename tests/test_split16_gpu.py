"""GPU parity of the strict "3xFP16" path: the split-fp16 storage format (include/mega_b200.h), its pack / unpack kernels
and the precision-3 implicit GEMM (three kind::f16 MMAs per k-step over hi / lo halves) against fp64 references.

Stated tolerance of the contraction: max|err| <= 3e-6 x RMS(output) (measured 3.2e-6 .. 4.3e-6; the format keeps 22 mantissa bits, a plain TF32 or
fp16 contraction sits at ~1e-3), the same bar the 3xTF32 kernel is held to in test_conv_gemm_gpu.py.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL = 1e-5


def _rel_err(got, ref):
    ref = ref.double()
    return ((got.double().cpu() - ref).abs().max() / ref.pow(2).mean().sqrt().clamp_min(1e-12)).item()


def test_pack_unpack_kernels_match_the_torch_restatement_bit_for_bit(cuda_dev):
    from mega_core.b200 import ops
    g = torch.Generator().manual_seed(3)
    x = torch.randn(37, 96, generator=g) * torch.tensor([1e-6, 1e-3, 1.0, 300.0, 7e4, 1e-9]).repeat(16)
    x[0, :4] = torch.tensor([0.0, -0.0, 65504.0, -1e6])
    xd = x.to(cuda_dev)
    want = ops.split16_encode(x)
    got = torch.empty_like(xd)
    ops.pack_split16(xd, out=got)
    assert torch.equal(got.cpu().view(torch.int32), want.view(torch.int32))
    back = ops.unpack_split16(got, torch.empty_like(xd))
    assert torch.equal(back.cpu(), ops.split16_decode(want))
    inplace = xd.clone()
    ops.pack_split16(inplace)
    assert ops.is_split16(inplace) and torch.equal(inplace.view(torch.int32), got.view(torch.int32))
    # the format itself: 22+ mantissa bits for |x| >= 2^-3, absolute 2^-25 below, saturation at the fp16 range
    fin = x.abs() <= 65504
    err = (ops.split16_decode(want).double() - x.double()).abs()
    bound = torch.maximum(x.double().abs() * 2.0 ** -22, torch.tensor(2.0 ** -25, dtype=torch.float64))
    assert (err[fin] <= bound[fin]).all()


def _conv_case(dev, n, h, w, cin, cout, ks, dil, relu, res_mode, out_split, seed, block_n=None, stream_k=None, wscale=1.0,
               want_output=False):
    from mega_core.b200 import ops
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, cin, h, w, generator=g).relu() * 3.0
    wt = torch.randn(cout, cin, ks, ks, generator=g) / (cin * ks * ks) ** 0.5 * wscale
    scale = torch.rand(cout, generator=g) + 0.5
    bias = torch.randn(cout, generator=g)
    res = torch.randn(n, cout, h, w, generator=g) if res_mode else None
    pad = dil * (ks - 1) // 2
    ref = F.conv2d(x.double(), wt.double(), None, 1, pad, dil) * scale.double().view(1, -1, 1, 1) + bias.double().view(1, -1, 1, 1)
    if res_mode:
        ref = ref + res.double()
    if relu:
        ref = ref.relu()
    a = ops.pack_split16(x.permute(0, 2, 3, 1).contiguous().to(dev))
    wp = ops.pack_weights_split16(wt.permute(2, 3, 0, 1).reshape(ks * ks, cout, cin).contiguous().to(dev), scale=scale.to(dev))
    out = torch.full((n, h, w, cout), float("nan"), device=dev)
    if out_split:
        ops.mark_split16(out)
    r = None
    if res_mode:
        r = res.permute(0, 2, 3, 1).contiguous().to(dev)
        if res_mode == "split":
            ops.pack_split16(r)
    with ops.precision("fp32x3"):
        ops.conv_gemm(a, wp, out, taps=(ks, ks), dil=dil, pad=pad, bias=bias.to(dev),      # (the scale is in the packed weights)
                      residual=r, relu=relu, block_n=block_n, stream_k=stream_k)
    torch.cuda.synchronize()
    if out_split:
        out = ops.unpack_split16(out, torch.empty_like(out))
    got = out.permute(0, 3, 1, 2)
    assert torch.isfinite(got).all(), "kernel left unwritten / non-finite outputs"
    if want_output:
        return _rel_err(got, ref), got.clone()
    return _rel_err(got, ref)


@pytest.mark.parametrize("case", [
    # n, h, w, cin, cout, ks, dil, relu, residual, out_split, block_n, stream_k, weight magnitude
    (1, 16, 16, 64, 64, 1, 1, False, None, False, 64, 0, 1.0),
    (1, 38, 63, 256, 256, 3, 1, True, None, True, 128, 0, 1.0),
    (2, 38, 63, 1024, 256, 1, 1, True, None, True, 128, 1, 1e-3),
    (1, 38, 63, 256, 1024, 1, 1, True, "split", True, 128, 0, 1.0),
    (1, 38, 63, 512, 2048, 1, 1, True, "split", False, 128, 0, 30.0),
    (1, 38, 63, 512, 512, 3, 2, True, "fp32", True, 128, 1, 1.0),
    (1, 19, 21, 96, 80, 3, 1, False, None, False, 64, 0, 1.0),
    (1, 38, 63, 1024, 1024, 3, 1, True, None, True, 128, 1, 1.0),
])
def test_conv_3xfp16_matches_fp64(cuda_dev, case):
    n, h, w, cin, cout, ks, dil, relu, res, osplit, bn, sk, ws = case
    err = _conv_case(cuda_dev, n, h, w, cin, cout, ks, dil, relu, res, osplit, seed=sum(map(hash, map(str, case))) % 1000,
                     block_n=bn, stream_k=sk, wscale=ws)
    assert err < TOL, err


def test_deep_reduction_as_taps_matches_fp64(cuda_dev):
    """the l_fcs[0] form: [rows, K] x [K/64 taps][1024][64] with K = 64 x 392, stream-K over a 12544-deep reduction"""
    from mega_core.b200 import ops
    from mega_core.b200.engine import WindowedEngine
    g = torch.Generator().manual_seed(5)
    rows, k, n_out = 300, 64 * 392, 256
    x = torch.randn(rows, k, generator=g).relu()
    w = torch.randn(n_out, k, generator=g) / k ** 0.5
    bias = torch.randn(n_out, generator=g)
    ref = (x.double() @ w.double().t() + bias.double()).relu()
    xd = ops.pack_split16(x.to(cuda_dev))
    wd = ops.pack_weights_split16(WindowedEngine.pack_fc0(w).to(cuda_dev))
    out = torch.full((rows, n_out), float("nan"), device=cuda_dev)
    with ops.precision("fp32x3"):
        ops.conv_gemm(xd.view(1, rows, k // 64, 64), wd, out.view(1, rows, 1, n_out), taps=(1, k // 64), pad=0,
                      bias=bias.to(cuda_dev), relu=True, tile=(128, 1), out_hw=(rows, 1))
    torch.cuda.synchronize()
    assert _rel_err(out, ref) < TOL


def test_relation_products_in_split16(cuda_dev):
    """the relation module's GEMM forms: V'^T = Wv . refs^T (packed WEIGHT as the A operand, activation as B, ragged cout
    rounded up to whole groups), per-head Q.K^T (both operands activations, fp32 logits out) and P.V' + bias + residual"""
    from mega_core.b200 import ops
    g = torch.Generator().manual_seed(9)
    nq, nref, D, ld = 200, 150, 1024, 160
    xq, refs = torch.randn(nq, D, generator=g), torch.randn(nref, D, generator=g)
    wv = torch.randn(D, D, generator=g) / 32
    bv = torch.randn(D, generator=g)
    dev = cuda_dev
    xq_d, refs_d = ops.pack_split16(xq.to(dev)), ops.pack_split16(refs.to(dev))
    wv_d = ops.pack_weights_split16(wv.to(dev))
    vt = ops.mark_split16(torch.zeros(D, ld, device=dev))
    s = torch.zeros(16, nq, ld, device=dev)
    out = ops.mark_split16(torch.zeros(nq, D, device=dev))
    with ops.precision("fp32x3"):
        ops.linear(wv_d, refs_d, vt)
        ops.conv_gemm(xq_d.view(1, 1, nq, D), refs_d.view(1, nref, D), s.view(16, 1, nq, ld), tile=(1, 128), cout=nref,
                      k=64, batch=16, a_c_off=64, b_k_off=64, out_n_off=1, n_img=1)
        torch.cuda.synchronize()
        logits_ref = torch.einsum("qhd,khd->hqk", xq.double().view(nq, 16, 64), refs.double().view(nref, 16, 64))
        assert _rel_err(s[:, :, :nref], logits_ref) < TOL
        assert (s[:, :, nref:] == 0).all()
        probs = torch.softmax(s[:, :, :nref].double().cpu() / 8, dim=-1)
        s.zero_()
        s[:, :, :nref] = probs.float().to(dev)
        ops.pack_split16(s)
        ops.conv_gemm(s.view(16, 1, nq, ld), vt.view(1, D, ld), out.view(1, 1, nq, D), tile=(1, 128), cout=64, k=ld,
                      batch=16, a_n_off=1, b_n_off=64, out_c_off=64, res_c_off=64, bias_z_off=64, bias=bv.to(dev),
                      residual=xq_d.view(1, 1, nq, D), block_n=64)
    torch.cuda.synchronize()
    vt_ref = wv.double() @ refs.double().t()                                   # [D, nref]
    got_vt = ops.unpack_split16(vt, torch.empty_like(vt))
    assert _rel_err(got_vt[:, :nref], vt_ref) < TOL and (got_vt[:, nref:] == 0).all()
    pv = torch.einsum("hqk,hdk->qhd", probs, vt_ref.view(16, 64, nref)).reshape(nq, D)
    want = xq.double() + pv + bv.double()
    assert _rel_err(ops.unpack_split16(out, torch.empty_like(out)), want) < TOL


def test_mixed_formats_are_refused(cuda_dev):
    from mega_core.b200 import ops
    a = torch.zeros(1, 8, 16, 64, device=cuda_dev)
    w = ops.pack_weights_split16(torch.zeros(1, 64, 64, device=cuda_dev))
    out = torch.zeros(1, 8, 16, 64, device=cuda_dev)
    with pytest.raises(AssertionError):
        ops.conv_gemm(a, w, out)                     # packed weights, plain fp32 activations
    with pytest.raises(AssertionError):
        ops.conv_gemm(ops.pack_split16(a), torch.zeros(1, 64, 64, device=cuda_dev), out)   # the other way round


def test_roi_align_over_a_split16_map_matches_the_fp32_kernel(cuda_dev):
    """the separable split-fp16 ROIAlign against the bit-exact fp32 kernel on the same (decoded) map: fused multiply-adds in a
    different association order, so the bar is 2e-6 x max|map| instead of equality"""
    from mega_core.b200 import ops
    g = torch.Generator().manual_seed(11)
    n, h, w, c = 2, 38, 63, 256
    feat = (torch.randn(n, h, w, c, generator=g).relu() * 4).to(cuda_dev)
    packed = ops.pack_split16(feat.clone())
    plain = ops.unpack_split16(packed, torch.empty_like(feat))
    k = 40
    xy = torch.rand(k, 2, generator=g) * torch.tensor([900.0, 500.0])
    wh = torch.rand(k, 2, generator=g) * torch.tensor([600.0, 400.0]) + 8
    boxes = torch.cat([xy, xy + wh], 1).to(cuda_dev)
    boxes[0] = torch.tensor([-50.0, -30.0, 1200.0, 700.0])          # larger than the image
    boxes[1] = torch.tensor([10.0, 10.0, 11.0, 11.0])               # a single cell
    bidx = (torch.arange(k) % n).int().to(cuda_dev)
    want = torch.zeros(k, 49 * c, device=cuda_dev)
    ops.roi_align_nhwc(plain, boxes, bidx, 1.0 / 16, 7, 7, 2, want)
    got_p = torch.zeros(k, 49 * c, device=cuda_dev)
    ops.roi_align_nhwc(packed, boxes, bidx, 1.0 / 16, 7, 7, 2, got_p)
    assert ops.is_split16(got_p)
    got = ops.unpack_split16(got_p, torch.empty_like(want))
    torch.cuda.synchronize()
    assert (got - want).abs().max().item() <= 2e-6 * plain.abs().max().item()
