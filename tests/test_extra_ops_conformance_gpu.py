"""Conformance of the kernels of csrc/deform.cu and csrc/train_ops.cu against the fp64 references of extra_ops_ref.py,
element by element: every output lies within A[output] * bound of the reference.

A (extra_ops_ref.A) is >= 2x the largest value the whole file measures, where "measured" is the smallest A every output
still passes with. Measured on an NVIDIA H100 80GB HBM3 (700 W power limit, max SM clock 1980 MHz):
    output              measured A      A
    focal_fwd           0.52            2
    focal_bwd           0.71            2
    im2col              1.00            2      (tile and scalar kernels through mega_deform_im2col)
    deform_conv         0.81            2      (end to end through _C in fp32x3, GEMM term 1.6e-6 P)
    psroi_fwd           0.37            1
    psroi_grad_input    0.96            2
    psroi_grad_trans    0.35            1
    roi_align_bwd       0.85            2
    channel_sum         0.37            1
    im2col_kq           1.00            2
    roi_pool_bwd        1.00            2
    dcn_grad_input      0.79            2
    dcn_grad_offset     0.60            2
    dcn_grad_mask       0.64            2
Where the measured value reaches 1.0 the kernel meets its rigorous bound with equality in the worst element (the
rounding of an atomic sum or of a single blend); no kernel exceeded the A = 1 bound.
ROIPool forward values and argmax are compared bit for bit.

Every case also checks: outputs written into NaN-filled buffers (im2col padding columns past C * taps, the K-major
columns' padding past Ho * Wo) keep their NaN where nothing may be written; accumulation targets (grad_input,
grad_trans, the channel sum) are seeded with nonzero values, so an assignment fails; inputs come back bit-unchanged.
The profiler records which kernel instantiation each call launched, in a child process of its own (fixture
`observed`), so the pytest process never opens a profiler session. The last test asserts that all fourteen
instantiations ran in cases that passed.
"""
import json
import os
import re
import subprocess
import sys
import time

import pytest
import torch

import extra_ops_ref as R

pytestmark = pytest.mark.gpu

TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
SEEN = set()
MEASURED = {}
NAMES = {}


# ------------------------------------------------------------------------------------------------ case table
def make_cases():
    cases = []
    for c in (1, 3, 4, 30, 80, 81):
        for gamma, alpha in ((0.0, 0.25), (1.0, 1.0), (1.5, 0.25), (2.0, 0.25)):
            for off in ((0, 1, 2) if c % 4 == 0 else (0, 1)):
                cases.append(dict(kind="focal", id="focal_c%d_g%g_a%g_off%d" % (c, gamma, alpha, off), c=c, n=64,
                                  gamma=gamma, alpha=alpha, off=off, seed=len(cases)))
    cases.append(dict(kind="focal", id="focal_cap_c80", c=80, n=28000, gamma=2.0, alpha=0.25, off=0, seed=1))
    cases.append(dict(kind="focal", id="focal_cap_c81", c=81, n=28000, gamma=2.0, alpha=0.25, off=0, seed=2))
    for k, cpg, wo, dg, st, dil, mask in ((1, 16, 33, 1, 1, 1, "rand"), (3, 1, 31, 1, 1, 1, "rand"),
                                          (3, 3, 32, 2, 1, 1, "zero_one"), (3, 16, 65, 1, 2, 1, "rand"),
                                          (3, 20, 33, 4, 1, 2, None), (3, 64, 1, 1, 1, 1, "rand"),
                                          (7, 20, 33, 1, 1, 1, "rand"), (7, 64, 32, 1, 1, 1, None),
                                          ((8, 7), 3, 31, 2, 1, 1, "rand"), (9, 16, 33, 1, 1, 1, None)):
            cases.append(dict(kind="im2col", id="im2col_k%s_cpg%d_wo%d_dg%d_s%d_d%d_%s" % (k, cpg, wo, dg, st, dil, mask),
                              k=k, cpg=cpg, wo=wo, dg=dg, stride=st, dil=dil, mask=mask, seed=len(cases)))
    for modulated, dtype, alias in ((True, "f32", True), (True, "f64", False), (False, "f64", False),
                                    (False, "f32", False)):
        cases.append(dict(kind="deform_conv", id="deform_conv_%s_%s%s" % ("v2" if modulated else "v1", dtype,
                                                                         "_aliased" if alias else ""),
                          modulated=modulated, dtype=dtype, alias=alias, seed=len(cases)))
    for gs, ps, part, spp, ncls, no_trans in ((1, 3, 2, 1, 1, True), (3, 3, 3, 4, 2, False), (7, 7, 4, 4, 3, False),
                                              (3, 6, 3, 1, 1, False)):
        cases.append(dict(kind="psroi", id="psroi_g%d_p%d_part%d_s%d_cls%d%s" % (gs, ps, part, spp, ncls,
                                                                                 "_notrans" if no_trans else ""),
                          gs=gs, ps=ps, part=part, spp=spp, ncls=ncls, no_trans=no_trans, seed=len(cases)))
    for c, k, sr, same in ((1, 6, 0, False), (7, 6, 2, False), (8, 6, 0, False), (9, 6, 2, False), (256, 4, 0, False),
                           (8, 300, 2, True), (256, 400, 2, False)):
        cases.append(dict(kind="roi_align_bwd", id="roi_align_bwd_c%d_k%d_sr%d%s" % (c, k, sr, "_same" if same else ""),
                          c=c, k=k, sr=sr, same=same, seed=len(cases)))
    for c, k, plane in ((3, 8, "const"), (5, 8, "neg"), (256, 100, "randn")):
        cases.append(dict(kind="roi_pool", id="roi_pool_c%d_k%d_%s" % (c, k, plane), c=c, k=k, plane=plane,
                          seed=len(cases)))
    for b, cpg, k, dg, h, w, mod in ((1, 1, 3, 1, 5, 7, True), (3, 4, 3, 2, 6, 5, True), (2, 2, 7, 1, 9, 9, False),
                                     (2, 16, 3, 1, 33, 70, True)):
        cases.append(dict(kind="dcn_bwd", id="dcn_bwd_b%d_cpg%d_k%d_dg%d_%dx%d%s" % (b, cpg, k, dg, h, w,
                                                                                     "_v2" if mod else "_v1"),
                          b=b, cpg=cpg, k=k, dg=dg, h=h, w=w, modulated=mod, seed=len(cases)))
    for b, c, p in ((2, 33, 50), (1, 9000, 7), (3, 20, 1000)):
        cases.append(dict(kind="channel_sum", id="channel_sum_b%d_c%d_p%d" % (b, c, p), b=b, c=c, p=p,
                          seed=len(cases)))
    return cases


CASES = make_cases()


def expected(c):
    k = c["kind"]
    if k == "focal":
        vec = "true" if c["c"] % 4 == 0 and c["off"] % 4 == 0 else "false"
        return {"focal_loss_kernel<false, %s>" % vec, "focal_loss_kernel<true, %s>" % vec}
    if k in ("im2col", "deform_conv"):
        kh, kw = (c.get("k", 3),) * 2 if not isinstance(c.get("k", 3), tuple) else c["k"]
        return {"deform_im2col_tile_kernel" if kh * kw <= R.K_DCN_MAX_TAPS else "deform_im2col_kernel"}
    return {"psroi": {"deform_psroi_fwd_kernel", "deform_psroi_bwd_kernel"}, "roi_align_bwd": {"roi_align_bwd_kernel"},
            "roi_pool": {"roi_pool_fwd_kernel", "roi_pool_bwd_kernel"},
            "dcn_bwd": {"dcn_im2col_kq_kernel", "dcn_col2im_fused_kernel"},
            "channel_sum": {"channel_sum_nchw_kernel"}}[k]


# ------------------------------------------------------------------------------------------------ checks
def _bits(t):
    return t.contiguous().view(torch.int64 if t.element_size() == 8 else torch.int32)


def _check(cid, name, got, ref, bound):
    a = R.A[name]
    got = got.double().to(ref.device)
    ok = R.inside(got, ref, bound, a)
    if not bool(ok.all()):
        i = tuple((~ok).nonzero()[0].tolist())
        raise AssertionError("%s %s: %d of %d elements outside the bound, first %s: got %r fp64 %r bound %r (A %g)"
                             % (cid, name, int((~ok).sum()), ok.numel(), i, got[i].item(), ref[i].item(),
                                bound[i].item(), a))
    return name, R.needed_a(got, ref, bound)


def _profiled(fn, want):
    """the kernel instantiations fn launched. A session now and then delivers only part of its kernel records; the call
    is then repeated (only the names of the repeats are used) until every expected name or no new one shows up"""
    from torch.profiler import ProfilerActivity, profile
    names = set()
    for attempt in range(8):
        if attempt:
            time.sleep(0.05 * 2 ** attempt)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names |= {m[0] + m[1] for e in prof.events()
                  for m in re.findall(r"mega::(\w+_kernel)(<[^>()]*>)?\(", e.name)} & set(R.INSTANTIATIONS)
        if names >= want:
            break
    return names


def _offsets(shape, g, dev):
    """offsets that land on integers, on -1, H and W, one ulp on either side of the gate, at +-1e4, and random"""
    special = torch.tensor([0.0, 1.0, -1.0, 0.5, -0.5, 2.0, -2.0, 3.0, 5.0, 1e4, -1e4, 1.0000001, 0.99999994,
                            -0.99999994, -1.0000001, 4.0, 6.0, 33.0, 64.0, 65.0])
    pick = torch.randint(0, len(special) + 8, shape, generator=g)
    rnd = torch.randn(shape, generator=g) * 3
    return torch.where(pick < len(special), special[pick.clamp(max=len(special) - 1)], rnd).float().to(dev)


def run_case(c, dev, profile=False):
    from mega_core import _C, _lib
    from mega_core.b200 import ops
    g = torch.Generator().manual_seed(1000 + c["seed"])
    rec = []
    calls = []
    k = c["kind"]

    def launch(fn):
        calls.append(fn)
    if k == "focal":
        n, cc = c["n"], c["c"]
        buf = (torch.randn(n * cc + 8, generator=g) * 6).float()
        edges = torch.tensor([0.0, 1e-3, -1e-3, 20, -20, 87.3, -87.3, 88, -88, 100, -100])
        buf[:len(edges) * 4:4] = edges
        buf = buf.to(dev)
        x = buf[c["off"]:c["off"] + n * cc].view(n, cc)
        dbuf = torch.randn(n * cc + 8, generator=g).float().to(dev)
        dl = dbuf[c["off"]:c["off"] + n * cc].view(n, cc)
        t = torch.tensor([-1, 0, 1, cc], dtype=torch.int32).repeat(n // 4 + 1)[:n]
        t = t[torch.randperm(n, generator=g)].to(dev)
        keep = [(buf, buf.clone()), (dbuf, dbuf.clone()), (t, t.clone())]
        res = {}
        launch(lambda: res.update(f=_C.sigmoid_focalloss_forward(x, t, cc, c["gamma"], c["alpha"]),
                                  b=_C.sigmoid_focalloss_backward(x, t, dl, cc, c["gamma"], c["alpha"])))
        checks = lambda: [_check(c["id"], "focal_fwd", res["f"], *R.focal_reference(x, t, c["gamma"], c["alpha"])),  # noqa
                          _check(c["id"], "focal_bwd", res["b"], *R.focal_reference(x, t, c["gamma"], c["alpha"], dl))]
    elif k == "im2col":
        kh, kw = c["k"] if isinstance(c["k"], tuple) else (c["k"], c["k"])
        dg, cpg, st, dil = c["dg"], c["cpg"], c["stride"], c["dil"]
        ch = dg * cpg
        wo = c["wo"]
        pad_h, pad_w = dil * (kh - 1) // 2, dil * (kw - 1) // 2
        width = (wo - 1) * st + dil * (kw - 1) + 1 - 2 * pad_w
        height = max(3, dil * (kh - 1) + 1 - 2 * pad_h)
        ho = (height + 2 * pad_h - (dil * (kh - 1) + 1)) // st + 1
        b = 2
        x = torch.randn(b, ch, height, width, generator=g).float().to(dev)
        off = _offsets((b, dg * 2 * kh * kw, ho, wo), g, dev)
        if c["mask"] == "rand":
            m = torch.rand(b, dg * kh * kw, ho, wo, generator=g).float().to(dev)
        elif c["mask"] == "zero_one":
            m = (torch.rand(b, dg * kh * kw, ho, wo, generator=g) > 0.5).float().to(dev)
        else:
            m = None
        kpad = ch * kh * kw + 5
        cols = torch.full((b, ho * wo, kpad), float("nan"), device=dev)
        keep = [(t, t.clone()) for t in (x, off, m) if t is not None]
        launch(lambda: _lib.check(_lib.lib.mega_deform_im2col(
            _lib.ptr(x), _lib.ptr(off), _lib.ptr(m), b, ch, height, width, kh, kw, pad_h, pad_w, st, st, dil, dil, dg,
            kpad, _lib.ptr(cols), _lib.stream_ptr()), "mega_deform_im2col"))

        def checks():
            ref, bnd = R.im2col_reference(x, off, m, kh, kw, pad_h, pad_w, st, st, dil, dil, dg)
            got = cols[..., :ch * kh * kw].view(b, ho, wo, ch, kh * kw).permute(0, 3, 4, 1, 2)
            assert bool(cols[..., ch * kh * kw:].isnan().all()), "%s: wrote past C * taps" % c["id"]
            return [_check(c["id"], "im2col", got, ref, bnd)]
    elif k == "deform_conv":
        td = torch.float64 if c["dtype"] == "f64" else torch.float32
        b, ch, height, width, cout, dg = 2, 16, 9, 11, 32, 2
        x = torch.randn(b, ch, height, width, generator=g).to(td).to(dev)
        wt = (torch.randn(cout, ch, 3, 3, generator=g) / 12).float().to(dev)
        bias = torch.randn(cout, generator=g).float().to(dev)
        om = _offsets((b, dg * 27, height, width), g, dev).to(td)
        om[:, dg * 18:] = torch.rand(b, dg * 9, height, width, generator=g).to(td).to(dev)
        if c["alias"]:
            off, m = om[:, :dg * 18], om[:, dg * 18:]
        else:
            off, m = om[:, :dg * 18].contiguous(), om[:, dg * 18:].contiguous()
        if not c["modulated"]:
            m = None
        out = torch.full((b, cout, height, width), float("nan"), device=dev)
        keep = [(t, t.clone()) for t in (x, wt, bias, om)]

        def call():
            with ops.precision("fp32x3"):
                if c["modulated"]:
                    _C.modulated_deform_conv_forward(x, wt, bias, None, off, m, out, None, 3, 3, 1, 1, 1, 1, 1, 1, 1,
                                                     dg, True)
                else:
                    _C.deform_conv_forward(x, wt, off, out, None, None, 3, 3, 1, 1, 1, 1, 1, 1, 1, dg, 64)
        launch(call)

        def checks():
            cols, cb = R.im2col_reference(x.float(), off.float(), m.float() if m is not None else None, 3, 3, 1, 1, 1, 1,
                                          1, 1, dg)
            w2 = wt.double().reshape(cout, -1)
            cols, cb = cols.reshape(b, ch * 9, -1), cb.reshape(b, ch * 9, -1)
            ref = torch.einsum("ok,bkp->bop", w2, cols)
            if c["modulated"]:
                ref = ref + bias.double().view(1, -1, 1)
            p = torch.einsum("ok,bkp->bop", w2.abs(), cols.abs())
            bnd = 1.6e-6 * p + R.A["im2col"] * torch.einsum("ok,bkp->bop", w2.abs(), cb) + 2 * R.U * ref.abs()
            return [_check(c["id"], "deform_conv", out.view(b, cout, -1), ref, bnd)]
    elif k == "psroi":
        gs, ps, part, spp, ncls, no_trans = c["gs"], c["ps"], c["part"], c["spp"], c["ncls"], c["no_trans"]
        od = 2 * ncls
        height, width, scale = 12, 14, 0.25
        x = torch.randn(2, od * gs * gs, height, width, generator=g).float().to(dev)
        nr = 12
        x1 = torch.randint(-30, 60, (nr, 2), generator=g).float()
        ext = torch.randint(0, 40, (nr, 2), generator=g).float()
        rois = torch.cat([torch.randint(0, 2, (nr, 1), generator=g).float(), x1, x1 + ext], 1)
        rois[0] = torch.tensor([0, 80.0, 80.0, 90.0, 90.0])           # outside the map: count 0
        rois[1] = torch.tensor([1, 10.0, 10.0, 7.0, 7.0])             # degenerate: width clamped to 0.1
        rois[2] = torch.tensor([0, 2.5, 3.5, 20.5, 30.5])             # corners at x.5
        rois = rois.to(dev)
        trans = (torch.randn(nr, 2 * ncls, part, part, generator=g) * 0.6).float().to(dev)
        std = 0.1
        out = torch.full((nr, od, ps, ps), float("nan"), device=dev)
        cnt = torch.full((nr, od, ps, ps), float("nan"), device=dev)
        og = torch.randn(nr, od, ps, ps, generator=g).float().to(dev)
        gi0 = torch.randn(x.shape, generator=g).float().to(dev)
        gt0 = torch.randn(trans.shape, generator=g).float().to(dev)
        gi, gt = gi0.clone(), gt0.clone()
        keep = [(t, t.clone()) for t in (x, rois, trans, og)]

        def call():
            _C.deform_psroi_pooling_forward(x, rois, trans, out, cnt, int(no_trans), scale, od, gs, ps, part, spp, std)
            _C.deform_psroi_pooling_backward(og, x, rois, trans, cnt, gi, gt, int(no_trans), scale, od, gs, ps, part,
                                             spp, std)
        launch(call)

        def checks():
            xc, rc, tc = x.cpu(), rois.cpu(), trans.cpu()
            ref, bnd, rcnt, dec = R.psroi_fwd_reference(xc, rc, tc, no_trans, scale, od, gs, ps, part, spp, std)
            assert R.decisions_stable(dec), "%s: a sample position is ambiguous" % c["id"]
            assert torch.equal(cnt.cpu(), rcnt.float()), "%s: top_count differs" % c["id"]
            r = [_check(c["id"], "psroi_fwd", out.cpu(), ref, bnd)]
            (ri, bi), tg = R.psroi_bwd_reference(og.cpu(), rcnt.float(), xc, rc, tc, no_trans, scale, od, gs, ps, part,
                                                 spp, std, gi0.cpu(), gt0.cpu())
            r.append(_check(c["id"], "psroi_grad_input", gi.cpu(), ri, bi))
            if tg is not None:
                r.append(_check(c["id"], "psroi_grad_trans", gt.cpu(), *tg))
            else:
                assert torch.equal(_bits(gt), _bits(gt0)), "%s: grad_trans written without trans" % c["id"]
            return r
    elif k == "roi_align_bwd":
        cc, nr, sr = c["c"], c["k"], c["sr"]
        height, width, scale, php = 20, 24, 0.5, 7
        x1 = torch.rand(nr, 2, generator=g) * 50 - 4
        ext = torch.rand(nr, 2, generator=g) * 40 + (20 if sr == 0 else 1)
        rois = torch.cat([torch.randint(0, 2, (nr, 1), generator=g).float(), x1, x1 + ext], 1).float()
        if c["same"]:
            rois[:] = torch.tensor([1, 30.0, 20.0, 47.0, 39.0])
        rois[0] = torch.tensor([0, 30.0, 25.0, 60.0, 48.0])           # past the right and bottom border
        rois = rois.to(dev)
        grad = torch.randn(nr, cc, php, php, generator=g).float().to(dev)
        seed = torch.randn(2, cc, height, width, generator=g).float().to(dev)
        gi = seed.clone()
        keep = [(t, t.clone()) for t in (rois, grad)]
        launch(lambda: _lib.check(_lib.lib.mega_roi_align_backward_nchw(
            _lib.ptr(grad), _lib.ptr(rois), nr, scale, php, php, 2, cc, height, width, sr, _lib.ptr(gi),
            _lib.stream_ptr()), "mega_roi_align_backward_nchw"))

        def checks():
            ref, bnd, dec = R.roi_align_bwd_reference(grad, rois, scale, php, php, 2, cc, height, width, sr, seed)
            assert R.decisions_stable(dec), "%s: a sample position is ambiguous" % c["id"]
            return [_check(c["id"], "roi_align_bwd", gi, ref, bnd)]
    elif k == "roi_pool":
        cc, nr, php = c["c"], c["k"], 7
        height, width, scale = 15, 17, 0.5
        if c["plane"] == "const":
            x = torch.full((2, cc, height, width), 0.75)
        elif c["plane"] == "neg":
            x = -torch.rand(2, cc, height, width, generator=g) - 1
        else:
            x = torch.randn(2, cc, height, width, generator=g)
        x = x.float().to(dev)
        x1 = torch.randint(-10, 60, (nr, 2), generator=g).float() + 0.5 * torch.randint(0, 2, (nr, 2), generator=g)
        ext = torch.randint(0, 30, (nr, 2), generator=g).float() + 0.5
        rois = torch.cat([torch.randint(0, 2, (nr, 1), generator=g).float(), x1, x1 + ext], 1).float()
        rois[0] = torch.tensor([0, 1.0, 1.0, 3.0, 3.0])               # 2x2 cells into 7x7 bins: repeated cells
        rois[1] = torch.tensor([1, 40.0, 40.0, 50.0, 50.0])           # outside the map: empty bins
        rois = rois.to(dev)
        out = torch.full((nr, cc, php, php), float("nan"), device=dev)
        arg = torch.full((nr, cc, php, php), -7, dtype=torch.int32, device=dev)
        grad = torch.randn(nr, cc, php, php, generator=g).float().to(dev)
        seed = torch.randn(2, cc, height, width, generator=g).float().to(dev)
        gi = seed.clone()
        keep = [(t, t.clone()) for t in (x, rois, grad)]

        def call():
            _lib.check(_lib.lib.mega_roi_pool_forward(_lib.ptr(x), _lib.ptr(rois), nr, scale, cc, height, width, php,
                                                      php, _lib.ptr(out), _lib.ptr(arg), _lib.stream_ptr()), "fwd")
            _lib.check(_lib.lib.mega_roi_pool_backward(_lib.ptr(grad), _lib.ptr(arg), _lib.ptr(rois), nr, cc, height,
                                                       width, php, php, _lib.ptr(gi), _lib.stream_ptr()), "bwd")
        launch(call)

        def checks():
            ro, ra = R.roi_pool_reference(x, rois, scale, php, php)
            assert torch.equal(_bits(out.cpu()), _bits(ro)), "%s: ROIPool values differ" % c["id"]
            assert torch.equal(arg.cpu(), ra), "%s: ROIPool argmax differs" % c["id"]
            ref, bnd = R.roi_pool_bwd_reference(grad, ra.to(dev), rois, cc, height, width, 2, seed)
            return [_check(c["id"], "roi_pool_bwd", gi, ref, bnd)]
    elif k == "dcn_bwd":
        b, cpg, kk, dg, height, width = c["b"], c["cpg"], c["k"], c["dg"], c["h"], c["w"]
        ch, pad = cpg * dg, kk // 2
        pt = height * width
        ldp = (pt + 3) // 4 * 4
        x = torch.randn(b, ch, height, width, generator=g).float().to(dev)
        off = _offsets((b, dg * 2 * kk * kk, height, width), g, dev)
        m = torch.rand(b, dg * kk * kk, height, width, generator=g).float().to(dev) if c["modulated"] else None
        gcols = torch.randn(ch * kk * kk, b * ldp, generator=g).float().to(dev)
        cols = torch.full((ch * kk * kk, b * ldp), float("nan"), device=dev)
        gi0 = torch.randn(x.shape, generator=g).float().to(dev)
        gi = gi0.clone()
        go = torch.full(off.shape, float("nan"), device=dev)
        gm = torch.full(m.shape, float("nan"), device=dev) if m is not None else None
        keep = [(t, t.clone()) for t in (x, off, m, gcols) if t is not None]
        geo = (b, ch, height, width, kk, kk, pad, pad, 1, 1, 1, 1, dg, ldp)

        def call():
            _lib.check(_lib.lib.mega_deform_im2col_kq(_lib.ptr(x), _lib.ptr(off), _lib.ptr(m), *geo, _lib.ptr(cols),
                                                      _lib.stream_ptr()), "kq")
            _lib.check(_lib.lib.mega_deform_col2im_fused(_lib.ptr(gcols), _lib.ptr(x), _lib.ptr(off), _lib.ptr(m),
                                                         *geo, _lib.ptr(gi), _lib.ptr(go), _lib.ptr(gm),
                                                         _lib.stream_ptr()), "col2im")
        launch(call)

        def checks():
            ref, bnd = R.im2col_reference(x, off, m, kk, kk, pad, pad, 1, 1, 1, 1, dg)
            cv = cols.view(ch, kk * kk, b, ldp)
            assert bool(cv[..., pt:].isnan().all()), "%s: wrote into the ldp padding" % c["id"]
            r = [_check(c["id"], "im2col_kq", cv[..., :pt].permute(2, 0, 1, 3).reshape(ref.shape), ref, bnd)]
            refs = R.col2im_reference(gcols, x, off, m, kk, kk, pad, pad, 1, 1, 1, 1, dg, ldp, gi0)
            r.append(_check(c["id"], "dcn_grad_input", gi, *refs[0]))
            r.append(_check(c["id"], "dcn_grad_offset", go, *refs[1]))
            if m is not None:
                r.append(_check(c["id"], "dcn_grad_mask", gm, *refs[2]))
            return r
    else:
        b, cc, p = c["b"], c["c"], c["p"]
        x = torch.randn(b, cc, p, generator=g).float().to(dev)
        seed = torch.randn(cc, generator=g).float().to(dev)
        out = seed.clone()
        keep = [(x, x.clone())]
        launch(lambda: _lib.check(_lib.lib.mega_channel_sum_nchw(_lib.ptr(x), b, cc, p, _lib.ptr(out),
                                                                 _lib.stream_ptr()), "channel_sum"))
        checks = lambda: [_check(c["id"], "channel_sum", out, *R.channel_sum_reference(x, seed))]  # noqa: E731
    fn = calls[0]
    if profile:                # the values are checked in the pytest process: the profiler may have repeated the call
        return _profiled(fn, expected(c)), []
    fn()
    torch.cuda.synchronize()
    for t, before in keep:
        assert torch.equal(_bits(t), _bits(before)), "%s: an input changed" % c["id"]
    return None, checks()


def _key(c):
    return c["id"]


CHILD_CASES = 30           # a process delivers kernel records for a few dozen profiler sessions: several children


def observe_child(out_path, first):
    """runs cases [first, first + CHILD_CASES) under the profiler in this (child) process and writes the kernel
    instantiations each launched and the cases that failed here"""
    dev = torch.device("cuda:0")
    failed = {}
    for c in CASES[first:first + CHILD_CASES]:
        try:
            names, _ = run_case(c, dev, profile=True)
            NAMES[_key(c)] = sorted(names)
        except AssertionError as e:
            failed[_key(c)] = str(e)[:2000]
    with open(out_path, "w") as fh:
        json.dump(dict(names=NAMES, failed=failed), fh)


@pytest.fixture(scope="module")
def observed(cuda_dev, tmp_path_factory):
    """the kernel instantiation each call of the table launches, as torch.profiler sees it in processes of its own"""
    tmp = tmp_path_factory.mktemp("extra_ops_observe")
    env = dict(os.environ,
               PYTHONPATH=os.pathsep.join([TESTS, ROOT, os.path.join(ROOT, "mega.pytorch_b200"), os.path.join(ROOT, "oracle")]
                                          + ([os.environ["PYTHONPATH"]] if os.environ.get("PYTHONPATH") else [])))
    code = "import sys, test_extra_ops_conformance_gpu as t; t.observe_child(sys.argv[1], int(sys.argv[2]))"
    merged = dict(names={}, failed={})
    for first in range(0, len(CASES), CHILD_CASES):
        out = tmp / ("names%d.json" % first)
        args = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code, str(out), str(first)]
        res = subprocess.run(args, env=env, cwd=ROOT, capture_output=True, text=True, timeout=1800)
        assert res.returncode == 0, res.stderr[-4000:]
        part = json.loads(out.read_text())
        merged["names"].update(part["names"])
        merged["failed"].update(part["failed"])
    return merged


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_extra_ops_match_fp64(cuda_dev, observed, case):
    try:
        _, rec = run_case(case, cuda_dev)
    except AssertionError as e:
        raise AssertionError("%s (under the profiler: %s)" % (e, observed["failed"].get(_key(case), "passed"))) \
            from None
    names = set(observed["names"].get(_key(case), ["<no record>"]))
    assert names == expected(case), "%s: launched %s, expected %s" % (case["id"], names, expected(case))
    SEEN.update(names)
    for name, a in rec:
        MEASURED[name] = max(MEASURED.get(name, 0.0), a)


# ------------------------------------------------------------------------------------------------ host-side rejections
@pytest.mark.parametrize("what", ["deform_out_f16", "deform_out_shape", "deform_out_strided", "psroi_out_f64",
                                  "psroi_count_shape"])
def test_outputs_validated_before_launch(cuda_dev, what):
    from mega_core import _C, _lib
    g = torch.Generator().manual_seed(3)
    if what.startswith("deform"):
        x = torch.randn(1, 4, 5, 6, generator=g).to(cuda_dev)
        wt = torch.randn(8, 4, 3, 3, generator=g).to(cuda_dev)
        off = torch.zeros(1, 18, 5, 6, device=cuda_dev)
        out = {"deform_out_f16": torch.full((2, 8, 5, 6), float("nan"), dtype=torch.float16, device=cuda_dev)[:1],
               "deform_out_shape": torch.full((1, 8, 6, 5), float("nan"), device=cuda_dev),
               "deform_out_strided": torch.full((1, 8, 5, 12), float("nan"), device=cuda_dev)[..., ::2]}[what]
        call = lambda: _C.deform_conv_forward(x, wt, off, out, None, None, 3, 3, 1, 1, 1, 1, 1, 1, 1, 1, 64)  # noqa
        guard = out
    else:
        x = torch.randn(1, 9, 6, 6, generator=g).to(cuda_dev)
        rois = torch.tensor([[0, 1.0, 1.0, 10.0, 10.0]], device=cuda_dev)
        out = torch.full((1, 1, 3, 3), float("nan"), device=cuda_dev, dtype=torch.float64 if what == "psroi_out_f64"
                         else torch.float32)
        cnt = torch.full((1, 1, 3, 3) if what == "psroi_out_f64" else (1, 1, 9), float("nan"), device=cuda_dev)
        call = lambda: _C.deform_psroi_pooling_forward(x, rois, None, out, cnt, 1, 0.5, 1, 3, 3, 3, 2, 0.1)  # noqa
        guard = cnt
    before = _bits(guard).clone()
    with pytest.raises(RuntimeError):
        call()
    torch.cuda.synchronize()
    assert torch.equal(_bits(guard), before)
    assert _lib.lib.mega_device_ok() == 1


# ------------------------------------------------------------------------------------------------ coverage gate
def test_zz_every_instantiation_ran(cuda_dev):
    """runs last in this file: all fourteen instantiations, each launched by a case that passed"""
    missing = sorted(set(R.INSTANTIATIONS) - SEEN)
    report = {"A": R.A, "measured_A": MEASURED, "seen": sorted(SEEN), "missing": missing}
    path = os.environ.get("EXTRA_OPS_CONFORMANCE_REPORT")
    if path:
        with open(path, "w") as fh:
            json.dump(report, fh, indent=1)
    print("extra ops conformance:", json.dumps(report))
    assert not missing, "instantiations without a passing case: %s" % missing
