"""GPU parity of the wgmma implicit-GEMM kernel against torch fp32 (CPU) references.

TF32 operands (10-bit mantissa, round-to-nearest on load) with fp32 accumulation: the stated
tolerance is max|err| <= 4e-3 x RMS(output) (observed 1.5e-3..2.1e-3, identical to cuBLAS TF32).
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL = 4e-3


def _rel_err(got, ref):
    ref = ref.double()
    return ((got.double().cpu() - ref).abs().max() / ref.pow(2).mean().sqrt().clamp_min(1e-12)).item()


def _conv_case(dev, n, h, w, cin, cout, ks, dil, relu, use_res, seed, block_n=None, tile=None):
    from mega_core.b200 import ops
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, cin, h, w, generator=g)
    wt = torch.randn(cout, cin, ks, ks, generator=g) / (cin * ks * ks) ** 0.5
    scale = torch.rand(cout, generator=g) + 0.5
    bias = torch.randn(cout, generator=g)
    res = torch.randn(n, cout, h, w, generator=g) if use_res else None
    pad = dil * (ks - 1) // 2
    ref = F.conv2d(x, wt, None, 1, pad, dil) * scale.view(1, -1, 1, 1) + bias.view(1, -1, 1, 1)
    if use_res:
        ref = ref + res
    if relu:
        ref = ref.relu()
    a = x.permute(0, 2, 3, 1).contiguous().to(dev)
    wp = wt.permute(2, 3, 0, 1).reshape(ks * ks, cout, cin).contiguous().to(dev)
    out = torch.full((n, h, w, cout), float("nan"), device=dev)
    r = res.permute(0, 2, 3, 1).contiguous().to(dev) if use_res else None
    ops.conv_gemm(a, wp, out, taps=(ks, ks), dil=dil, pad=pad, scale=scale.to(dev), bias=bias.to(dev),
                  residual=r, relu=relu, block_n=block_n, tile=tile)
    torch.cuda.synchronize()
    got = out.permute(0, 3, 1, 2)
    assert torch.isfinite(got).all(), "kernel left unwritten / non-finite outputs"
    return _rel_err(got, ref)


@pytest.mark.parametrize("case", [
    # n, h, w, cin, cout, ks, dil, relu, res, block_n, tile
    (1, 16, 16, 64, 64, 1, 1, False, False, 64, (8, 16)),
    (1, 38, 63, 256, 256, 3, 1, True, False, None, None),
    (2, 38, 63, 1024, 256, 1, 1, True, False, None, None),
    (1, 38, 63, 256, 1024, 1, 1, True, True, 128, None),
    (1, 38, 63, 512, 512, 3, 2, True, False, 256, None),
    (1, 19, 21, 96, 60, 3, 1, False, False, 64, (4, 32)),
    (1, 75, 125, 128, 128, 3, 1, True, False, 32, (16, 8)),
])
def test_conv_matches_fp32(cuda_dev, case):
    n, h, w, cin, cout, ks, dil, relu, res, bn, tile = case
    err = _conv_case(cuda_dev, n, h, w, cin, cout, ks, dil, relu, res, seed=hash(case) % 1000, block_n=bn,
                     tile=tile)
    assert err < TOL, err


@pytest.mark.parametrize("m,k,n,splits", [(75, 1024, 1024, 1), (300, 4096, 1024, 4), (450, 100352, 1024, 16),
                                         (1, 64, 31, 1), (675, 1024, 124, 1)])
def test_linear_matches_fp32(cuda_dev, m, k, n, splits):
    from mega_core.b200 import ops
    g = torch.Generator().manual_seed(m + k + n)
    x = torch.randn(m, k, generator=g)
    w = torch.randn(n, k, generator=g) / k ** 0.5
    b = torch.randn(n, generator=g)
    ref = (x.double() @ w.double().t() + b.double()).relu().float()
    n_pad = (n + 3) // 4 * 4                      # output rows are written by TMA: pitch multiple of 4 floats
    out = torch.full((m, n_pad), float("nan"), device=cuda_dev)
    bias = torch.zeros(n_pad)
    bias[:n] = b
    ops.linear(x.to(cuda_dev), w.to(cuda_dev), out, bias=bias.to(cuda_dev), relu=True,
               max_ctas=(0 if splits > 1 else 3))
    torch.cuda.synchronize()
    assert torch.isfinite(out[:, :n]).all()
    assert _rel_err(out[:, :n], ref) < TOL


def test_batched_heads(cuda_dev):
    """per-head Q.K^T through the batch offsets: S[g] = Q[:, g*64:(g+1)*64] @ K[:, g*64:(g+1)*64].T"""
    from mega_core.b200 import ops
    g = torch.Generator().manual_seed(7)
    nq, mk, heads, dh = 300, 750, 16, 64
    q = torch.randn(nq, heads * dh, generator=g)
    k = torch.randn(mk, heads * dh, generator=g)
    ref = torch.einsum("ngd,mgd->gnm", q.view(nq, heads, dh).double(), k.view(mk, heads, dh).double()).float()
    mk_pad = 752
    out = torch.zeros(heads, nq, mk_pad, device=cuda_dev)
    qd, kd = q.to(cuda_dev), k.to(cuda_dev)
    a4 = qd.view(1, 1, nq, heads * dh)
    w3 = kd.view(1, mk, heads * dh)
    o4 = out.view(heads, 1, nq, mk_pad)
    ops.conv_gemm(a4, w3, o4, tile=(1, 128), cout=mk, k=dh, batch=heads, a_c_off=dh, b_k_off=dh,
                  out_n_off=1, n_img=1, block_n=128)
    torch.cuda.synchronize()
    assert _rel_err(out[:, :, :mk], ref) < TOL
    assert (out[:, :, mk:] == 0).all()


@pytest.mark.parametrize("bn,sk", [(96, 0), (96, 1), (160, 0), (160, 1), (192, 1), (256, 0), (64, 1), (32, 1)])
def test_stream_k_and_wide_tiles(cuda_dev, bn, sk):
    """every N-tile width in both scheduling modes on a 3x3 conv whose tile count (57) does not divide the SMs"""
    from mega_core.b200 import ops
    g = torch.Generator().manual_seed(bn + sk)
    n, h, w, cin, cout = 1, 38, 63, 160, 320
    x = torch.randn(n, cin, h, w, generator=g)
    wt = torch.randn(cout, cin, 3, 3, generator=g) / (cin * 9) ** 0.5
    ref = F.conv2d(x, wt, None, 1, 1).relu()
    a = x.permute(0, 2, 3, 1).contiguous().to(cuda_dev)
    wp = wt.permute(2, 3, 0, 1).reshape(9, cout, cin).contiguous().to(cuda_dev)
    out = torch.full((n, h, w, cout), float("nan"), device=cuda_dev)
    for _ in range(2):          # twice: the tile counters must come back to zero
        ops.conv_gemm(a, wp, out, taps=(3, 3), pad=1, relu=True, block_n=bn, stream_k=sk)
    torch.cuda.synchronize()
    assert _rel_err(out.permute(0, 3, 1, 2), ref) < TOL


@pytest.mark.parametrize("bn,sk", [(64, 0), (128, 0), (128, 1)])
def test_fp32x3_split_precision(cuda_dev, bn, sk):
    """strict mode: hi*hi + hi*lo + lo*hi with TF32 MMAs -> near-fp32 (bound asserted: max|err| <= 5e-5 x RMS, measured 2.0e-5;
    plain TF32 gives ~1.5e-3 on the same problem)"""
    from mega_core.b200 import ops
    g = torch.Generator().manual_seed(17)
    n, h, w, cin, cout = 1, 38, 63, 256, 200
    x = torch.randn(n, cin, h, w, generator=g)
    wt = torch.randn(cout, cin, 3, 3, generator=g) / (cin * 9) ** 0.5
    bias = torch.randn(cout, generator=g)
    res = torch.randn(n, cout, h, w, generator=g)
    ref = (F.conv2d(x.double(), wt.double(), bias.double(), 1, 2, 2) + res.double()).relu().float()
    a = x.permute(0, 2, 3, 1).contiguous().to(cuda_dev)
    wp = wt.permute(2, 3, 0, 1).reshape(9, cout, cin).contiguous().to(cuda_dev)
    out = torch.full((n, h, w, cout), float("nan"), device=cuda_dev)
    r = res.permute(0, 2, 3, 1).contiguous().to(cuda_dev)
    with ops.precision("fp32x3"):
        ops.conv_gemm(a, wp, out, taps=(3, 3), dil=2, pad=2, bias=bias.to(cuda_dev), residual=r, relu=True,
                      block_n=bn, stream_k=sk)
    torch.cuda.synchronize()
    err = _rel_err(out.permute(0, 3, 1, 2), ref)
    assert err < 5e-5, err


# ------------------------------------------------------------------ fp16-operand mode (kind::f16)
def _f16_conv_case(dev, n, h, w, cin, cout, ks, dil, relu, use_res, out16, seed, block_n=None, stream_k=None, tile=None):
    """operands rounded to fp16 up front, so the fp64 reference isolates the kernel's own error:
    fp32 accumulation (<= 1e-5 x RMS) plus, for fp16 outputs, one final rounding (2^-11 relative)."""
    from mega_core.b200 import ops
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, cin, h, w, generator=g).half()
    wt = (torch.randn(cout, cin, ks, ks, generator=g) / (cin * ks * ks) ** 0.5).half()
    scale = torch.rand(cout, generator=g) + 0.5
    bias = torch.randn(cout, generator=g)
    res = torch.randn(n, cout, h, w, generator=g).half() if use_res else None
    pad = dil * (ks - 1) // 2
    ref = F.conv2d(x.double(), wt.double(), None, 1, pad, dil) * scale.double().view(1, -1, 1, 1) + bias.double().view(1, -1, 1, 1)
    if use_res:
        ref = ref + res.double()
    if relu:
        ref = ref.relu()
    a = x.permute(0, 2, 3, 1).contiguous().to(dev)
    wp = wt.permute(2, 3, 0, 1).reshape(ks * ks, cout, cin).contiguous().to(dev)
    out = torch.full((n, h, w, cout), float("nan"), device=dev, dtype=torch.float16 if out16 else torch.float32)
    r = None
    if use_res:
        r = res.permute(0, 2, 3, 1).contiguous().to(dev)
        if not out16:
            r = r.float()
            ref = ref   # same values (fp16-representable), passed as fp32
    for _ in range(2):
        ops.conv_gemm(a, wp, out, taps=(ks, ks), dil=dil, pad=pad, scale=scale.to(dev), bias=bias.to(dev),
                      residual=r, relu=relu, block_n=block_n, stream_k=stream_k, tile=tile)
    torch.cuda.synchronize()
    got = out.float().permute(0, 3, 1, 2)
    assert torch.isfinite(got).all(), "kernel left unwritten / non-finite outputs"
    if out16:
        # one rounding to fp16 of the fp32 result: |err| <= 2^-11 |ref| (+ the accumulation error, <= 2e-5 x RMS)
        err = (got.double().cpu() - ref).abs()
        bound = ref.abs() * 2.0 ** -11 + 2e-5 * ref.pow(2).mean().sqrt()
        assert (err <= bound * 1.01).all(), (err / bound).max().item()
        return 0.0
    return _rel_err(got, ref.float())


@pytest.mark.parametrize("case", [
    # n, h, w, cin, cout, ks, dil, relu, res, out16, block_n, stream_k
    (2, 38, 63, 1024, 256, 1, 1, True, False, True, None, None),
    (2, 38, 63, 256, 256, 3, 1, True, False, True, 128, 0),
    (2, 38, 63, 256, 1024, 1, 1, True, True, True, 256, 0),
    (2, 38, 63, 256, 1024, 1, 1, True, True, True, 192, 1),
    (1, 38, 63, 512, 512, 3, 2, True, False, True, 64, 1),
    (1, 38, 63, 1024, 60, 1, 1, False, False, False, 64, 0),       # RPN head: fp16 operands, fp32 logits
    (1, 19, 21, 96, 200, 3, 1, False, True, False, 96, 0),        # fp32 out + fp32 residual, odd tile width
    (1, 75, 125, 160, 64, 1, 1, True, False, True, 64, 0),         # K tail (160 = 2.5 slabs of 64)
])
def test_f16_conv_matches_fp64(cuda_dev, case):
    n, h, w, cin, cout, ks, dil, relu, res, out16, bn, sk = case
    err = _f16_conv_case(cuda_dev, n, h, w, cin, cout, ks, dil, relu, res, out16, seed=hash(case) % 1000, block_n=bn,
                         stream_k=sk)
    assert err < (2e-3 if out16 else 2e-5), err


def test_f16_linear_and_batched_heads(cuda_dev):
    """l_fcs[0]-shaped GEMM (K = 100352, stream-K) and the per-head Q.K^T / P.V' batch offsets with fp16 operands"""
    from mega_core.b200 import ops
    g = torch.Generator().manual_seed(5)
    m, k, n = 375, 100352, 1024
    x = (torch.randn(m, k, generator=g)).half()
    w = (torch.randn(n, k, generator=g) / k ** 0.5).half()
    b = torch.randn(n, generator=g)
    xd, wd = x.to(cuda_dev), w.to(cuda_dev)
    ref = (xd.double() @ wd.double().t() + b.to(cuda_dev).double()).relu().float().cpu()
    out = torch.full((m, n), float("nan"), device=cuda_dev, dtype=torch.float16)
    ops.linear(xd, wd, out, bias=b.to(cuda_dev), relu=True)
    torch.cuda.synchronize()
    assert _rel_err(out.float(), ref) < 4e-3       # fp16 output: 2^-11 relative at ~6 sigma
    nq, mk, heads, dh = 300, 750, 16, 64
    q = torch.randn(nq, heads * dh, generator=g).half()
    kk = torch.randn(mk, heads * dh, generator=g).half()
    ref = torch.einsum("ngd,mgd->gnm", q.view(nq, heads, dh).double(), kk.view(mk, heads, dh).double()).float()
    mk_pad = 768
    s = torch.zeros(heads, nq, mk_pad, device=cuda_dev)
    ops.conv_gemm(q.to(cuda_dev).view(1, 1, nq, heads * dh), kk.to(cuda_dev).view(1, mk, heads * dh),
                  s.view(heads, 1, nq, mk_pad), tile=(1, 128), cout=mk, k=dh, batch=heads, a_c_off=dh, b_k_off=dh,
                  out_n_off=1, n_img=1)
    torch.cuda.synchronize()
    assert _rel_err(s[:, :, :mk], ref) < 2e-5
    # P.V'^T with the residual / bias / channel-offset batching of the attention epilogue
    p = torch.rand(heads, nq, mk_pad, generator=g).half()
    p[:, :, mk:] = 0
    vt = torch.randn(heads * dh, mk_pad, generator=g).half()
    xq = torch.randn(nq, heads * dh, generator=g).half()
    bv = torch.randn(heads * dh, generator=g)
    ref = torch.einsum("gnm,gdm->ngd", p.double(), vt.view(heads, dh, mk_pad).double()).reshape(nq, heads * dh) \
        + bv.double() + xq.double()
    out = torch.full((nq, heads * dh), float("nan"), device=cuda_dev, dtype=torch.float16)
    ops.conv_gemm(p.to(cuda_dev).view(heads, 1, nq, mk_pad), vt.to(cuda_dev).view(1, heads * dh, mk_pad),
                  out.view(1, 1, nq, heads * dh), tile=(1, 128), cout=dh, k=mk_pad, batch=heads, a_n_off=1, b_n_off=dh,
                  out_c_off=dh, res_c_off=dh, bias_z_off=dh, bias=bv.to(cuda_dev),
                  residual=xq.to(cuda_dev).view(1, 1, nq, heads * dh), block_n=64)
    torch.cuda.synchronize()
    assert _rel_err(out.float(), ref.float()) < 4e-3


def test_f16_layer_chain_matches_per_layer_launches(cuda_dev):
    """three bottleneck blocks (1x1 -> 3x3 -> 1x1 + residual, the res4 pattern at 2 x 38 x 63) + a 1x1 head with fp32
    output, once as 10 separate launches and once as ONE persistent chain kernel (csrc/conv_chain.cu): with the tile
    configuration pinned the two must agree bit for bit (same MMAs in the same order); replayed three times to
    exercise the grid-barrier reset; also checked against an fp64 reference of the whole chain."""
    from mega_core.b200 import ops
    g = torch.Generator().manual_seed(21)
    n, h, w, c, mid = 2, 38, 63, 512, 128
    x0 = torch.randn(n, h, w, c, generator=g).half().to(cuda_dev)
    blocks = []
    for b in range(3):
        w1 = (torch.randn(1, mid, c, generator=g) / c ** 0.5).half().to(cuda_dev)
        w2 = (torch.randn(9, mid, mid, generator=g) / (9 * mid) ** 0.5).half().to(cuda_dev)
        w3 = (torch.randn(1, c, mid, generator=g) / mid ** 0.5).half().to(cuda_dev)
        sb = [(torch.rand(k, generator=g) * 0.5 + 0.75).to(cuda_dev) for k in (mid, mid, c)]
        bb = [(torch.randn(k, generator=g) * 0.1).to(cuda_dev) for k in (mid, mid, c)]
        blocks.append((w1, w2, w3, sb, bb))
    wh = (torch.randn(1, 60, c, generator=g) / c ** 0.5).half().to(cuda_dev)

    def run(bufs, stream_k):
        x = x0
        for b, (w1, w2, w3, sb, bb) in enumerate(blocks):
            t1, t2, y = bufs["t1%d" % b], bufs["t2%d" % b], bufs["y%d" % b]
            ops.conv_gemm(x, w1, t1, scale=sb[0], bias=bb[0], relu=True, block_n=128, stream_k=0)
            ops.conv_gemm(t1, w2, t2, taps=(3, 3), pad=1, scale=sb[1], bias=bb[1], relu=True, block_n=64, stream_k=stream_k)
            ops.conv_gemm(t2, w3, y, scale=sb[2], bias=bb[2], residual=x, relu=True, block_n=128, stream_k=0)
            x = y
        ops.conv_gemm(x, wh, bufs["head"], cout=60, block_n=64, stream_k=0)
        return x, bufs["head"]

    def mkbufs():
        d = {}
        for b in range(3):
            d["t1%d" % b] = torch.full((n, h, w, mid), float("nan"), device=cuda_dev, dtype=torch.float16)
            d["t2%d" % b] = torch.full((n, h, w, mid), float("nan"), device=cuda_dev, dtype=torch.float16)
            d["y%d" % b] = torch.full((n, h, w, c), float("nan"), device=cuda_dev, dtype=torch.float16)
        d["head"] = torch.full((n, h, w, 60), float("nan"), device=cuda_dev)
        return d

    for sk in (0, 1):
        ref_bufs, ch_bufs = mkbufs(), mkbufs()
        y_ref, head_ref = run(ref_bufs, sk)
        cache = {}
        for rep in range(3):
            with ops.chain(cache, "k", cuda_dev):
                y_ch, head_ch = run(ch_bufs, sk)
        torch.cuda.synchronize()
        assert len(cache) == 1 and cache["k"].n == 10
        assert torch.equal(y_ch, y_ref) and torch.equal(head_ch, head_ref), (sk, (y_ch.float() - y_ref.float()).abs().max())
    # fp64 reference of the chain (fp16 storage between layers reproduced)
    x = x0.double().cpu()
    for (w1, w2, w3, sb, bb) in blocks:
        xin = x
        t = F.conv2d(x.permute(0, 3, 1, 2), w1.double().cpu().reshape(mid, c, 1, 1))
        t = (t * sb[0].double().cpu().view(1, -1, 1, 1) + bb[0].double().cpu().view(1, -1, 1, 1)).relu().half().double()
        t = F.conv2d(t, w2.double().cpu().reshape(3, 3, mid, mid).permute(2, 3, 0, 1), padding=1)
        t = (t * sb[1].double().cpu().view(1, -1, 1, 1) + bb[1].double().cpu().view(1, -1, 1, 1)).relu().half().double()
        t = F.conv2d(t, w3.double().cpu().reshape(c, mid, 1, 1))
        t = t * sb[2].double().cpu().view(1, -1, 1, 1) + bb[2].double().cpu().view(1, -1, 1, 1)
        x = (t.permute(0, 2, 3, 1) + xin).relu().half().double()
    assert _rel_err(y_ch.float(), x.float()) < 1e-2      # fp16 storage of 9 chained layers


def test_fp32x3_presplit_weights_are_bit_identical(cuda_dev):
    """strict mode with the weights' low parts stored behind them once (ops.presplit: the kernel fetches lo by TMA,
    mega_conv_gemm_desc.b_lo_tap_off) against the same launches splitting the staged weight tile on the fly: identical bits,
    for a 3x3 convolution (9 taps), a Linear (1 tap, rows not a multiple of the tile) and a stream-K deep reduction"""
    from mega_core.b200 import ops
    g = torch.Generator().manual_seed(31)
    x = torch.randn(2, 19, 31, 96, generator=g).to(cuda_dev)
    w = (torch.randn(9, 160, 96, generator=g) / 30).to(cuda_dev)
    xl = torch.randn(300, 1024, generator=g).to(cuda_dev)
    wl = (torch.randn(155, 1024, generator=g) / 32).to(cuda_dev)
    bias = torch.randn(160, generator=g).to(cuda_dev)
    with ops.precision("fp32x3"):
        for bn, sk in ((64, 0), (128, 1)):
            ref = torch.zeros(2, 19, 31, 160, device=cuda_dev)
            ops.conv_gemm(x, w, ref, taps=(3, 3), pad=1, bias=bias, relu=True, block_n=bn, stream_k=sk)
            wp = ops.presplit(w)
            assert torch.equal(wp, w) and wp.data_ptr() != w.data_ptr()
            got = torch.zeros_like(ref)
            ops.conv_gemm(x, wp, got, taps=(3, 3), pad=1, bias=bias, relu=True, block_n=bn, stream_k=sk)
            torch.cuda.synchronize()
            assert torch.equal(got, ref), (bn, sk, (got - ref).abs().max())
            refl = torch.zeros(300, 156, device=cuda_dev)
            ops.linear(xl, wl, refl[:, :155], block_n=bn, stream_k=sk)
            wlp = ops.presplit(wl)
            gotl = torch.zeros_like(refl)
            ops.linear(xl, wlp, gotl[:, :155], block_n=bn, stream_k=sk)
            torch.cuda.synchronize()
            assert torch.equal(gotl, refl), (bn, sk)
    ref64 = F.conv2d(x.double().cpu().permute(0, 3, 1, 2), w.double().cpu().reshape(3, 3, 160, 96).permute(2, 3, 0, 1), padding=1)
    ref64 = (ref64 + bias.double().cpu().view(1, -1, 1, 1)).relu().permute(0, 2, 3, 1)
    assert _rel_err(got.cpu(), ref64.float()) < 1e-5


def test_f16_interleaved_chain_matches_per_layer_launches(cuda_dev):
    """barrier depth 2 (ops.chain(interleave=True)): the res4 pattern on the two halves of a batch of four 38 x 63 maps as
    two interleaved lanes A0 B0 A1 B1 ... of ONE chain kernel, every layer waiting only for the layer two positions back.
    With the tile configuration pinned the result must be bit-identical to the separate launches of the same layers
    (stream-K on and off: odd layers keep their partial sums / tile counters in the second half of the workspace);
    replayed several times (barrier reset) and with unequal work per lane position (3x3 vs 1x1) back to back."""
    from mega_core.b200 import ops
    g = torch.Generator().manual_seed(22)
    n, h, w, c, mid = 4, 38, 63, 512, 128
    x0 = torch.randn(n, h, w, c, generator=g).half().to(cuda_dev)
    blocks = []
    for b in range(4):
        w1 = (torch.randn(1, mid, c, generator=g) / c ** 0.5).half().to(cuda_dev)
        w2 = (torch.randn(9, mid, mid, generator=g) / (9 * mid) ** 0.5).half().to(cuda_dev)
        w3 = (torch.randn(1, c, mid, generator=g) / mid ** 0.5).half().to(cuda_dev)
        sb = [(torch.rand(k, generator=g) * 0.5 + 0.75).to(cuda_dev) for k in (mid, mid, c)]
        bb = [(torch.randn(k, generator=g) * 0.1).to(cuda_dev) for k in (mid, mid, c)]
        blocks.append((w1, w2, w3, sb, bb))
    wh = (torch.randn(1, 60, c, generator=g) / c ** 0.5).half().to(cuda_dev)

    def run(bufs, x, lane, stream_k):
        """the layer sequence on one half of the batch; scratch per lane, outputs into the lane's half of `y` / `head`"""
        hn = x.shape[0]
        sl = slice(lane * hn, (lane + 1) * hn)
        for b, (w1, w2, w3, sb, bb) in enumerate(blocks):
            t1, t2 = bufs["t1_%d" % lane], bufs["t2_%d" % lane]
            y = bufs["y%d" % (b & 1)][sl]
            ops.conv_gemm(x, w1, t1, scale=sb[0], bias=bb[0], relu=True, block_n=128, stream_k=stream_k)
            ops.conv_gemm(t1, w2, t2, taps=(3, 3), pad=1, scale=sb[1], bias=bb[1], relu=True, block_n=64, stream_k=stream_k)
            ops.conv_gemm(t2, w3, y, scale=sb[2], bias=bb[2], residual=x, relu=True, block_n=128, stream_k=0)
            x = y
        ops.conv_gemm(x, wh, bufs["head"][sl], cout=60, block_n=64, stream_k=stream_k)

    def mkbufs():
        d = {}
        for lane in range(2):
            d["t1_%d" % lane] = torch.full((n // 2, h, w, mid), float("nan"), device=cuda_dev, dtype=torch.float16)
            d["t2_%d" % lane] = torch.full((n // 2, h, w, mid), float("nan"), device=cuda_dev, dtype=torch.float16)
        for b in range(2):
            d["y%d" % b] = torch.full((n, h, w, c), float("nan"), device=cuda_dev, dtype=torch.float16)
        d["head"] = torch.full((n, h, w, 60), float("nan"), device=cuda_dev)
        return d

    for sk in (0, 1):
        ref = mkbufs()
        for lane in range(2):
            run(ref, x0[lane * 2:(lane + 1) * 2], lane, sk)
        torch.cuda.synchronize()
        got = mkbufs()
        cache = {}
        for rep in range(4):
            with ops.chain(cache, "k", cuda_dev, interleave=True) as ch:
                run(got, x0[0:2], 0, sk)
                ch.next_lane()
                run(got, x0[2:4], 1, sk)
        torch.cuda.synchronize()
        assert len(cache) == 1 and cache["k"].n == 26 and cache["k"].depth == 2
        for name in ("y1", "head"):
            assert torch.isfinite(got[name].float()).all()
            assert torch.equal(got[name], ref[name]), (sk, name, (got[name].float() - ref[name].float()).abs().max())


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_strided_conv_leaky_and_transposed_conv(cuda_dev, dtype):
    """the generalisations FlowNetS needs (backbone/flownet.py): stride-2 k x k convolutions through TMA element
    strides, LeakyReLU(0.1) in the epilogue, ConvTranspose2d(4, stride 2) + crop_like as four parity-class 2x2
    convolutions writing every other pixel of a channel slice of a wider (concat) buffer, 2-channel outputs."""
    from mega_core.b200 import engine, ops
    g = torch.Generator().manual_seed(3)
    tol = 4e-3 if dtype == torch.float16 else TOL
    rnd = lambda *s: torch.randn(*s, generator=g)
    q = (lambda t: t.half().float()) if dtype == torch.float16 else (lambda t: t)
    # ---- 5x5 stride 2 conv + leaky relu, odd sizes
    n, h, w, cin, cout = 2, 37, 45, 64, 128
    x, wt, b = q(rnd(n, cin, h, w)), q(rnd(cout, cin, 5, 5) / (cin * 25) ** 0.5), rnd(cout)
    ref = F.leaky_relu(F.conv2d(x, wt, b, 2, 2), 0.1)
    out = torch.full((n, ref.shape[2], ref.shape[3], cout), float("nan"), device=cuda_dev, dtype=dtype)
    ops.conv_gemm(x.permute(0, 2, 3, 1).contiguous().to(cuda_dev).to(dtype), engine.pack_conv(wt, cuda_dev, dtype), out,
                  taps=(5, 5), pad=2, stride=(2, 2), bias=b.to(cuda_dev), relu="leaky")
    torch.cuda.synchronize()
    assert _rel_err(out.float().permute(0, 3, 1, 2), ref) < tol
    # ---- ConvTranspose2d(cin, cout, 4, 2) + crop_like + leaky into channels [16, 16+cout) of a 72-channel buffer
    sd = {"flownet.flow_conv1.weight": torch.zeros(64, 6, 7, 7)}
    n, hi, wi, cin, cout = 2, 9, 13, 24, 40
    xi = q(rnd(n, cin, hi, wi))
    wd, bd = q(rnd(cin, cout, 4, 4) / (4 * cin) ** 0.5), rnd(cout)
    full = F.conv_transpose2d(xi, wd, bd, stride=2)                       # [n, cout, 2hi+2, 2wi+2]
    for ht, wt_ in ((2 * hi, 2 * wi), (2 * hi - 1, 2 * wi + 1), (2 * hi + 2, 2 * wi + 2)):
        ref = full if (ht, wt_) == tuple(full.shape[2:]) else full[:, :, 1:ht + 1, 1:wt_ + 1]
        ref = F.leaky_relu(ref, 0.1)
        fl = engine.FlowNetS.__new__(engine.FlowNetS)
        fl.dev, fl.dtype = cuda_dev, dtype
        cls = {}
        for py in (0, 1):
            for px in (0, 1):
                wp = torch.zeros(4, cout, cin)
                for r in (0, 1):
                    for s_ in (0, 1):
                        wp[r * 2 + s_] = wd[:, :, py + 2 * (1 - r), px + 2 * (1 - s_)].t()
                cls[(py, px)] = wp.contiguous().to(cuda_dev).to(dtype)
        fl.w, fl.b = {"d": cls}, {"d": bd.to(cuda_dev)}
        target = torch.full((n, ht, wt_, 72), 7.0, device=cuda_dev, dtype=dtype)
        fl._deconv("d", xi.permute(0, 2, 3, 1).contiguous().to(cuda_dev).to(dtype), target, 16, cout, "leaky")
        torch.cuda.synchronize()
        assert (target[..., :16] == 7).all() and (target[..., 16 + cout:] == 7).all()
        assert _rel_err(target[..., 16:16 + cout].float().permute(0, 3, 1, 2), ref) < tol, (ht, wt_)
    # ---- 3x3 conv to 2 channels written into an 8-channel-padded buffer (channel-clipped TMA store)
    xc, wc, bc = q(rnd(2, 200, 19, 32)), q(rnd(2, 200, 3, 3) / 1800 ** 0.5), rnd(2)
    ref = F.conv2d(xc, wc, bc, 1, 1)
    buf = torch.zeros(2, 19, 32, 8, device=cuda_dev, dtype=dtype)
    ops.conv_gemm(xc.permute(0, 2, 3, 1).contiguous().to(cuda_dev).to(dtype), engine.pack_conv(wc, cuda_dev, dtype), buf[..., 0:2],
                  taps=(3, 3), pad=1, bias=bc.to(cuda_dev), cout=2)
    torch.cuda.synchronize()
    assert (buf[..., 2:] == 0).all()
    assert _rel_err(buf[..., 0:2].float().permute(0, 3, 1, 2), ref) < tol
