"""CPU half of the conv_gemm conformance suite: the fp64 reference of test_conv_gemm_conformance_gpu.py against torch
convolutions / einsums and a direct loop over the descriptor formula, the 42-entry instantiation table against the kernel
source, the committed case list against the descriptor contract, and the Python restatement of the stream-K split."""
import itertools
import os
import re

import pytest
import torch
import torch.nn.functional as F

from conv_gemm_ref import (GEOMS, GROUPED, MODES, VARIANTS, case_fields, case_problem, chain_rotation,
                           check_case_contract, conv_gemm_ref, cta_first_unit, encoder_grid, epilogue_factors,
                           make_cases, make_sk_cases, mode_bk, sk_geometry, sk_label_holds, unit_owner, variant_of)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNEL_SRC = os.path.join(ROOT, "mega.pytorch_b200", "csrc", "conv_gemm_kernel.cuh")


def _loop_ref(A, B, *, taps, dil, pad, pad_w, stride, k, n_img, out_hw, cout, batch=1, a_c_off=0, a_n_off=0, b_k_off=0,
              b_n_off=0, out_c_off=0, out_n_off=0, res_c_off=0, res_n_off=0, bias_z_off=0, scale=None, bias=None,
              residual=None, relu=0):
    """the header's formula, one tap at a time (no torch convolution)"""
    R, S = taps
    sh, sw = stride
    oh, ow = out_hw
    pw = pad if pad_w is None else pad_w
    outs = []
    for z in range(batch):
        acc = torch.zeros(n_img, oh, ow, cout, dtype=torch.float64)
        for r in range(R):
            for s in range(S):
                hi = torch.arange(oh) * sh + r * dil - pad
                wi = torch.arange(ow) * sw + s * dil - pw
                vh = (hi >= 0) & (hi < A.shape[1])
                vw = (wi >= 0) & (wi < A.shape[2])
                a = A[z * a_n_off:z * a_n_off + n_img][:, hi.clamp(0, A.shape[1] - 1)][:, :, wi.clamp(0, A.shape[2] - 1)]
                a = a[..., z * a_c_off:z * a_c_off + k] * (vh.view(1, -1, 1, 1) & vw.view(1, 1, -1, 1))
                b = B[r * S + s, z * b_n_off:z * b_n_off + cout, z * b_k_off:z * b_k_off + k]
                acc += torch.einsum("nhwc,oc->nhwo", a, b)
        v = acc
        if scale is not None:
            v = v * scale[z * bias_z_off:z * bias_z_off + cout]
        if bias is not None:
            v = v + bias[z * bias_z_off:z * bias_z_off + cout]
        if residual is not None:
            v = v + residual[z * res_n_off:z * res_n_off + n_img, :, :, z * res_c_off:z * res_c_off + cout]
        if relu == 1:
            v = v.clamp_min(0)
        elif relu == 2:
            v = torch.where(v > 0, v, 0.1 * v)
        outs.append(v)
    return outs


def _small(geom, k=8, cout=5):
    """a CPU-sized version of a geometry (same taps / stride / dilation / padding / batching, few channels)"""
    g = dict(geom)
    f = dict(batch=g.get("batch", 1), a_c_off=0, a_n_off=g.get("a_n_off", 0), b_k_off=0, b_n_off=0, out_c_off=0,
             out_n_off=g.get("out_n_off", 0), res_c_off=0, res_n_off=g.get("res_n_off", 0), bias_z_off=0)
    if f["batch"] > 1:
        f.update(a_c_off=k, b_k_off=k, b_n_off=cout, out_c_off=cout, res_c_off=cout, bias_z_off=cout)
    return g, f


GEOM_FORMS = sorted(GEOMS) + ["grouped"] + sorted({c["geom"] for _, c in make_sk_cases()})


@pytest.mark.parametrize("name", GEOM_FORMS)
def test_reference_matches_loop_formula_and_conv2d(name):
    gen = torch.Generator().manual_seed(len(name))
    if name == "grouped":
        geom = dict(GROUPED)
    elif name.startswith("sk_"):
        geom = next(c for _, c in make_sk_cases() if c["geom"] == name)
        geom = {key: geom[key] for key in ("taps", "dil", "pad", "pad_w", "stride", "n_img", "out_hw", "a_hw")}
    else:
        geom = dict(GEOMS[name])
    k, cout = 8, 5
    g, f = _small(geom, k, cout)
    if name == "grouped":
        cout = k = 4
        f = dict(batch=3, a_c_off=4, a_n_off=0, b_k_off=0, b_n_off=4, out_c_off=4, out_n_off=0, res_c_off=4, res_n_off=0,
                 bias_z_off=4)
    bt = f["batch"]
    R, S = g["taps"]
    oh, ow = g["out_hw"]
    A = torch.randn(g["n_img"] + (bt - 1) * f["a_n_off"], g["a_hw"][0], g["a_hw"][1], k + (bt - 1) * f["a_c_off"],
                    generator=gen, dtype=torch.float64)
    B = torch.randn(R * S, cout + (bt - 1) * f["b_n_off"], k + (bt - 1) * f["b_k_off"], generator=gen, dtype=torch.float64)
    if name == "grouped":         # block-diagonal weights over 12 channels, group width 2
        B = torch.zeros(R * S, 12, 4, dtype=torch.float64)
        wl = torch.randn(12, 2, R, S, generator=gen, dtype=torch.float64)
        for co in range(12):
            c0 = (co % 4) // 2 * 2
            B[:, co, c0:c0 + 2] = wl[co].permute(1, 2, 0).reshape(R * S, 2)
    nsb = cout + (bt - 1) * f["bias_z_off"]
    scale, bias = torch.rand(nsb, generator=gen, dtype=torch.float64) + 0.5, torch.randn(nsb, generator=gen, dtype=torch.float64)
    res = torch.randn(g["n_img"] + (bt - 1) * f["res_n_off"], oh, ow, cout + (bt - 1) * f["res_c_off"], generator=gen,
                      dtype=torch.float64)
    kw = dict(taps=g["taps"], dil=g["dil"], pad=g["pad"], pad_w=g["pad_w"], stride=g["stride"], k=k, n_img=g["n_img"],
              out_hw=g["out_hw"], cout=cout, scale=scale, bias=bias, residual=res, **f)
    for relu in (0, 1, 2):
        blocks = conv_gemm_ref(A, B, relu=relu, **kw)
        loops = _loop_ref(A, B, relu=relu, **kw)
        assert len(blocks) == bt
        for (z, v, P, Q), want in zip(blocks, loops):
            assert torch.allclose(v, want, rtol=1e-12, atol=1e-12), (name, z)
            assert (P >= 0).all() and (Q >= v.abs() - 1e-12).all()
    # against F.conv2d directly when the padding is symmetric (P included: the conv of magnitudes)
    if g["pad_w"] in (None, g["pad"]) and bt == 1:
        x = A.permute(0, 3, 1, 2)
        wt = B.reshape(R, S, cout, k).permute(2, 3, 0, 1)
        full = F.conv2d(x, wt, stride=g["stride"], padding=g["pad"], dilation=g["dil"])[:, :, :oh, :ow].permute(0, 2, 3, 1)
        mag = F.conv2d(x.abs(), wt.abs(), stride=g["stride"], padding=g["pad"], dilation=g["dil"])[:, :, :oh, :ow]
        (_, v, P, _), = conv_gemm_ref(A, B, **dict(kw, scale=None, bias=None, residual=None))
        assert torch.allclose(v, full, rtol=1e-12, atol=1e-12)
        assert torch.allclose(P, mag.permute(0, 2, 3, 1), rtol=1e-12, atol=1e-12)
    if name == "grouped":          # the block-diagonal batched layout is a grouped F.conv2d
        x = A.permute(0, 3, 1, 2)
        want = F.conv2d(x, wl, padding=g["pad"], dilation=g["dil"], groups=6).permute(0, 2, 3, 1)
        got = torch.cat([b[1] for b in conv_gemm_ref(A, B, **dict(kw, scale=None, bias=None, residual=None))], 3)
        assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)


def test_reference_matches_the_hand_written_references():
    """the formulas of test_conv_gemm_gpu.py (conv + scale + bias + residual + ReLU, Linear, per-head Q.K^T, P.V' with the
    attention epilogue) at CPU sizes"""
    g = torch.Generator().manual_seed(4)
    d = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    # conv: F.conv2d * scale + bias + res, relu (NCHW)
    n, h, w, cin, cout, ks, dil = 2, 9, 11, 6, 7, 3, 2
    x, wt, scale, bias, res = d(n, cin, h, w), d(cout, cin, ks, ks), d(cout).abs() + 0.5, d(cout), d(n, cout, h, w)
    pad = dil * (ks - 1) // 2
    want = (F.conv2d(x, wt, None, 1, pad, dil) * scale.view(1, -1, 1, 1) + bias.view(1, -1, 1, 1) + res).relu()
    (_, v, _, _), = conv_gemm_ref(x.permute(0, 2, 3, 1), wt.permute(2, 3, 0, 1).reshape(ks * ks, cout, cin), taps=(ks, ks),
                                  dil=dil, pad=pad, k=cin, n_img=n, out_hw=(h, w), cout=cout, scale=scale, bias=bias,
                                  residual=res.permute(0, 2, 3, 1), relu=1)
    assert torch.allclose(v.permute(0, 3, 1, 2), want, rtol=1e-12, atol=1e-12)
    # Linear: x @ w.T + b, relu (ops.linear: an H = 1 image)
    m, kk, nn = 13, 10, 6
    xl, wl, bl = d(m, kk), d(nn, kk), d(nn)
    (_, v, _, _), = conv_gemm_ref(xl.view(1, 1, m, kk), wl.view(1, nn, kk), k=kk, n_img=1, out_hw=(1, m), cout=nn, bias=bl,
                                  relu=1)
    assert torch.allclose(v.view(m, nn), (xl @ wl.t() + bl).relu(), rtol=1e-12, atol=1e-12)
    # per-head Q.K^T through the batch offsets (test_batched_heads)
    nq, mk, heads, dh = 5, 7, 3, 4
    q, kt = d(nq, heads * dh), d(mk, heads * dh)
    want = torch.einsum("ngd,mgd->gnm", q.view(nq, heads, dh), kt.view(mk, heads, dh))
    blocks = conv_gemm_ref(q.view(1, 1, nq, heads * dh), kt.view(1, mk, heads * dh), k=dh, n_img=1, out_hw=(1, nq), cout=mk,
                           batch=heads, a_c_off=dh, b_k_off=dh, out_n_off=1)
    for z, v, _, _ in blocks:
        assert torch.allclose(v.view(nq, mk), want[z], rtol=1e-12, atol=1e-12)
    # P.V'^T + bias + residual with channel-offset batching (test_f16_linear_and_batched_heads)
    mkp = 8
    p, vt, xq, bv = d(heads, nq, mkp), d(heads * dh, mkp), d(nq, heads * dh), d(heads * dh)
    want = torch.einsum("gnm,gdm->ngd", p, vt.view(heads, dh, mkp)).reshape(nq, heads * dh) + bv + xq
    blocks = conv_gemm_ref(p.view(heads, 1, nq, mkp), vt.view(1, heads * dh, mkp), k=mkp, n_img=1, out_hw=(1, nq), cout=dh,
                           batch=heads, a_n_off=1, b_n_off=dh, out_c_off=dh, res_c_off=dh, bias_z_off=dh, bias=bv,
                           residual=xq.view(1, 1, nq, heads * dh))
    got = torch.cat([v.view(nq, dh) for _, v, _, _ in blocks], 1)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------------------------------------ instantiation table
def _launch_mode_source():
    with open(KERNEL_SRC) as fh:
        src = fh.read()
    body = src[src.index("int launch_mode(int block_n"):src.index("#define MEGA_LAUNCH_MODE")]
    return src, body


def test_variant_table_follows_launch_mode():
    src, body = _launch_mode_source()
    assert len(VARIANTS) == 42 and len(set(VARIANTS)) == 42
    grouped = {int(gw) for gw in re.findall(r"case (\d+): return launch\(IntC<64>\(\), IntC<\1>\(\)\)", body)}
    assert grouped == {8, 16, 32}
    every = {int(b) for b in re.findall(r"case (\d+): return launch\(IntC<\1>\(\), IntC<0>\(\)\)", body.split("if constexpr (MODE == kModeTf32 || MODE == kModeF16)")[0])}
    wide = {int(b) for b in re.findall(r"case (\d+): return launch\(IntC<\1>\(\), IntC<0>\(\)\)", body.split("if constexpr (MODE == kModeTf32 || MODE == kModeF16)")[1])}
    assert every == {64, 128} and wide == {32, 96, 160, 192, 256}
    assert "MODE == kModeF16x3 || (MODE == kModeF16 && BN % 64 == 0)" in body     # the out16 instantiations
    want = set()
    for mode in range(4):
        for gw in (0, 8, 16, 32):
            for bn in ((64,) if gw else sorted(every | (wide if mode in (0, 2) else set()))):
                for out16 in (False, True):
                    if not out16 or mode == 3 or (mode == 2 and bn % 64 == 0):
                        want.add((mode, bn, out16, gw))
    assert set(VARIANTS) == want
    counts = {m: sum(v[0] == m for v in VARIANTS) for m in range(4)}
    assert counts == {0: 10, 1: 5, 2: 17, 3: 10}
    # the header: strict modes run block_n 64 / 128, fp16 output needs block_n % 64 == 0, group widths 8..64 at block_n 64
    assert all(v[1] in (64, 128) for v in VARIANTS if v[0] in (1, 3))
    assert all(v[1] % 64 == 0 for v in VARIANTS if v[0] == 2 and v[2])
    assert all(v[1] == 64 for v in VARIANTS if v[3])
    assert variant_of(2, 64, 1, 64) == (2, 64, True, 0)
    # every instantiation's pipeline fits the 227 KB of shared memory (SmemLayout / conv_gemm_stages)
    for mode, bn, _, _ in VARIANTS:
        stages = (4 if bn == 64 else 2) if mode == 1 else (5 if bn == 64 else 4) if mode == 3 else \
            (6 if bn == 32 else 5 if bn == 64 else 4 if bn <= 128 else 3 if bn <= 192 else 2)
        pn = bn if bn <= 128 else (96 if bn == 160 else bn // 2)
        stage = 128 * 128 + pn * 128 + (pn * 128 if mode == 1 else 0)
        total = stages * stage + 2 * 128 * 128 + 4 * 4 * 4096 + 512 + 8 * (128 if bn <= 128 else 256) + 1024
        assert total <= 227 * 1024, (mode, bn, total)
    assert "constexpr int conv_gemm_stages(int mode, int bn)" in src


# ------------------------------------------------------------------------------------------------ the case list
CASES = make_cases()


def test_cases_satisfy_the_descriptor_contract():
    ids = [c["id"] for c in CASES] + [c["id"] for _, c in make_sk_cases()]
    assert len(ids) == len(set(ids))
    for c in CASES + [c for _, c in make_sk_cases()]:
        assert not check_case_contract(c), (c["id"], check_case_contract(c))
        tiles, kb, units = case_problem(c)
        assert tiles <= 65536 and units * 132 < 2 ** 31


def test_cases_cover_every_instantiation_pairwise():
    by_variant = {}
    for c in CASES:
        v = variant_of(c["mode"], c["block_n"], c["out16"], c.get("group_width", 0))
        by_variant.setdefault(v, []).append(c)
    assert set(by_variant) == set(VARIANTS)
    for v, cs in by_variant.items():
        assert {c["stream_k"] for c in cs} == {0, 1}, v
        factors = epilogue_factors(v[0])
        for (na, va), (nb, vb) in itertools.combinations(factors, 2):
            for x, y in itertools.product(va, vb):
                assert any(c[na] == x and c[nb] == y for c in cs), (v, na, x, nb, y)


def test_cases_cover_the_geometry_axes_per_mode():
    for mode in MODES:
        cs = [c for c in CASES if c["mode"] == mode]
        f = [case_fields(c) for c in cs]
        axes = {
            "1x1": any(c["taps"] == (1, 1) for c in cs),
            "3x3": any(c["taps"] == (3, 3) for c in cs),
            "5x5": any(c["taps"] == (5, 5) for c in cs),
            "dil2": any(c["dil"] == 2 and c["stride"] == (1, 1) for c in cs),
            "stride2": any(c["stride"] == (2, 2) and c["dil"] == 1 for c in cs),
            "stride2_dil2": any(c["stride"] == (2, 2) and c["dil"] == 2 for c in cs),
            "pad_w": any(c["pad_w"] is not None and c["pad_w"] != c["pad"] for c in cs),
            "row_skip": any(c["row_skip"] == 2 for c in cs),
            "ragged_tiles": any(c["out_hw"][0] % c["tile"][0] and c["out_hw"][1] % c["tile"][1] for c in cs),
            "n_img": any(c["n_img"] > 1 for c in cs),
            "cout_lt_bn": any(c["cout"] < c["block_n"] for c in cs),
            "batched_all_offsets": any(all(x[key] for key in ("a_c_off", "a_n_off", "b_k_off", "b_n_off", "out_c_off",
                                                               "out_n_off", "res_c_off", "res_n_off", "bias_z_off"))
                                       and x["res_n_off"] != x["out_n_off"] and c["res"] != "none"
                                       for c, x in zip(cs, f)),
        }
        for tile in ((8, 16), (16, 8), (4, 32), (128, 1), (1, 128)):
            axes["tile%dx%d" % tile] = any(c["tile"] == tile for c in cs)
        for cout in (2, 60, 200):
            axes["cout%d" % cout] = any(c["cout"] == cout for c in cs)
        for gw in (8, 16, 32, 64):
            axes["gw%d" % gw] = any(c.get("group_width") == gw for c in cs)
        if mode != 3:        # split-fp16 operands come in whole 32-value groups: precision 3 has no K tail
            axes["k_tail"] = any(c["k"] % mode_bk(mode) for c in cs)
        missing = [a for a, ok in axes.items() if not ok]
        assert not missing, (MODES[mode], missing)


# ------------------------------------------------------------------------------------------------ stream-K geometry
def test_unit_owner_inverts_cta_first_unit():
    for total, grid in ((360, 7), (288, 72), (5120, 120), (5, 3), (1000, 132), (9, 1)):
        for u in range(total):
            c = unit_owner(total, grid, u)
            assert cta_first_unit(total, grid, c) <= u < cta_first_unit(total, grid, c + 1)


def test_sk_cases_have_their_geometry():
    labels = {}
    for label, c in make_sk_cases():
        assert sk_label_holds(label, c), c["id"]
        labels.setdefault(label, set()).add(c["mode"])
    assert labels["a"] == labels["bd"] == labels["c"] == {0, 1, 2, 3}
    assert labels["e"] == labels["f_fires"] == labels["f_stays"] == {2, 3}
    # the concrete numbers behind the labels
    assert encoder_grid(20, 256, 1) == (120, True)
    assert encoder_grid(20, 256, 1, 23) == (20, True) and encoder_grid(20, 256, 1, 24) == (24, False)
    g = sk_geometry(40, 9, 7)
    assert g["span"] and not g["divides"]
    assert sk_geometry(2, 72, 36)["max_parts"] >= 3


def test_chain_rotation_restatement():
    # whole-tile layers advance by the tiles of their last partial wave, stream-K layers by their active CTAs
    assert chain_rotation([(4, 4, 0), (57, 40, 0), (10, 10, 1), (3, 3, 0)], 40) == [0, 4, 21, 31]


def test_stream_k_restatements_follow_the_encoders():
    """the constants and rules that encoder_grid / chain_rotation restate, as they stand in the C++ encoders"""
    csrc = os.path.join(ROOT, "mega.pytorch_b200", "csrc")
    with open(os.path.join(csrc, "conv_gemm.cu")) as fh:
        gemm = re.sub(r"\s+", " ", fh.read())
    with open(os.path.join(csrc, "conv_chain.cu")) as fh:
        chain = re.sub(r"\s+", " ", fh.read())
    with open(KERNEL_SRC) as fh:
        kern = re.sub(r"\s+", " ", fh.read())
    assert "constexpr int kMinUnits = 4;" in gemm
    assert "constexpr int kMaxCtas = 132;" in kern
    for rule in ("long long ctas = p.stream_k ? p.total_units / kMinUnits : tiles;", "if (ctas < 1) ctas = 1;",
                 "if (ctas > g_num_sms) ctas = g_num_sms;", "if (d->max_ctas > 0 && ctas > d->max_ctas) ctas = d->max_ctas;",
                 "if (p.stream_k && p.kb_per_tile >= 256 && tiles <= ctas) {",
                 "const long long aligned = (ctas / tiles) * tiles;", "if (aligned * 100 >= ctas * 85) ctas = aligned;"):
        assert rule in gemm, rule
    for rule in ("return static_cast<int>((static_cast<unsigned>(total) * static_cast<unsigned>(c)) / static_cast<unsigned>(grid));",
                 "int c = static_cast<int>((static_cast<unsigned>(u) * static_cast<unsigned>(grid)) / static_cast<unsigned>(total));"):
        assert rule in kern, rule
    for rule in ("out[l].cta_rot = static_cast<int>(start % grid);",
                 "start += out[l].p.stream_k ? act : (tiles % act == 0 ? act : tiles % act);", "if (ctas > grid) grid = ctas;"):
        assert rule in chain, rule
