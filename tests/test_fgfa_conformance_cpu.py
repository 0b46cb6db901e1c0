"""CPU half of the FGFA / DFF conformance suite: the fp32 geometry restatement of fgfa_ref.py against torch's
F.grid_sample and the oracle's warp, an fp32 emulation of every kernel of csrc/fgfa.cu in the kernels' order that must
lie inside the fp64 interval, deliberate bugs of that emulation the interval must reject, the restatement and the
kernel limits against the source, and the ops wrappers' layout checks (run with the library entries replaced by
recorders, so that no kernel is ever launched on a bad view)."""
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import fgfa_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = {c["id"]: c for c in R.make_cases()}
F32, F16 = np.float32, np.float16
# CPU-sized cases of the table (the emulation is numpy): every aggregate / DFF / pool edge, both production 12 x 20
# windows, and the 600 x 1000 frame
FIXTURES = ["prod_first_12x20", "prod_rot_12x20", "ce1", "ce200", "ce4096", "cf1", "cf100", "cf1030", "L1",
            "L32_key31", "key0", "key_last", "map_2x2", "map_2x9", "map_9x2", "flow_zero", "flow_exact", "flow_far",
            "emb_zero_frame", "emb_zero_key", "emb_tiny", "values_big", "values_sub", "dff_prod_12x20", "dff_c8_2x2",
            "dff_2x9_exact", "dff_9x2_exact", "dff_exact", "dff_zero", "dff_far", "dff_big", "dff_sub", "pool_7x9",
            "pool_8x10", "pool_1x1", "pool_1x9", "pool_9x1", "pool_2x2", "pool_big", "pool_sub", "image_600x1000",
            "image_7x9", "image_8x10", "image_1x1", "image_1x9", "image_9x1", "image_big"]


# ------------------------------------------------------------------------------------------------ fp32 emulation
def _fma(a, b, c):
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(F32)


def _store(v, dtype, mutate):
    """the kernels' output store: fp32 as is, fp16 round-to-nearest (mutation 'rz16': toward zero)"""
    if dtype == "f32":
        return v
    h = v.astype(F16)
    if mutate == "rz16":
        up = np.abs(h.astype(F32)) > np.abs(v)
        h = np.where(up, np.nextafter(h, F16(0)), h)
    return h.astype(F32)


def _geometry(flow, mutate):
    mode = mutate if mutate in ("align_corners", "zeros", "unclamped", "no_fma") else "kernel"
    g = R.Geometry(flow, mode=mode, swap_xy=mutate == "swap_xy")
    return g.idx, g.wts.astype(F32)


def _guarded(m, w):
    """[P, C] map followed by w + 1 NaN rows: a read past the map (an unclamped corner) poisons the result"""
    return np.concatenate([m, np.full((w + 1, m.shape[1]), np.nan, F32)])


def _sample(m, idx, wts):
    """w00 * v00, then three FMAs (the kernel's sample())"""
    acc = (wts[0][:, None] * m[idx[0]]).astype(F32)
    for k in (1, 2, 3):
        acc = _fma(np.broadcast_to(wts[k][:, None], acc.shape), m[idx[k]], acc)
    return acc


def _block_sum(parts):
    """parts [P, per, 256]: per sequential FMAs already applied -> [P, 256]; 5 xor-shuffle levels, 8 warp partials
    summed in order (block_sum)"""
    v = parts
    lane = np.arange(32)
    v = v.reshape(v.shape[0], 8, 32)
    for off in (16, 8, 4, 2, 1):
        v = (v + v[..., lane ^ off]).astype(F32)
    s = np.zeros(v.shape[0], F32)
    for i in range(8):
        s = (s + v[:, i, 0]).astype(F32)
    return s


def _thread_fma(a, b):
    """sum_c a_c b_c per thread: channel tid + j * 256 into thread tid, j ascending -> [P, 256]"""
    p, c = a.shape
    per = (c + 255) // 256
    pa = np.zeros((p, per * 256), F32)
    pb = np.zeros((p, per * 256), F32)
    pa[:, :c], pb[:, :c] = a, b
    acc = np.zeros((p, 256), F32)
    for j in range(per):
        acc = _fma(pa[:, j * 256:(j + 1) * 256], pb[:, j * 256:(j + 1) * 256], acc)
    return acc


def emulate_aggregate(ring, slots, key, flow, cf, ce, dtype, mutate=None):
    """fgfa_aggregate_kernel in fp32: (out [P, cf], weights [L, P]). ring fp32 numpy [S, h, w, ld] (the values the
    kernel reads)"""
    s_, h, w, ld = ring.shape
    L, P = len(slots), h * w
    eps = F32(1e-10)
    flat = [_guarded(ring[s].reshape(P, ld), w) for s in range(s_)]
    geo = [_geometry(flow[slots[f] if mutate == "slot_flow" else f], mutate) for f in range(L)]

    def norm(sq):
        s = _block_sum(sq)
        return (np.sqrt((s + eps).astype(F32)) if mutate == "eps_in_sqrt" else (np.sqrt(s) + eps)).astype(F32)

    if mutate == "key_unwarped":
        ek = flat[slots[key]][:P, cf:cf + ce]
    else:
        ek = _sample(flat[slots[key]][:, cf:cf + ce], *geo[key])
    kn = norm(_thread_fma(ek, ek))
    logit = np.zeros((L, P), F32)
    for f in range(L):
        e = _sample(flat[slots[f]][:, cf:cf + ce], *geo[f])
        dot = _block_sum(_thread_fma(e, ek))
        nn = norm(_thread_fma(e, e))
        logit[f] = ((dot / nn).astype(F32) / kn).astype(F32)
    mx = logit.max(0)
    ex = np.exp((logit - mx).astype(F32)).astype(F32)
    den = np.zeros(P, F32)
    for f in range(L):
        den = (den + ex[f]).astype(F32)
    inv = (F32(1) / den).astype(F32)
    wts = (ex * inv).astype(F32)
    acc = np.zeros((P, cf), F32)
    for f in range(L):
        acc = _fma(np.broadcast_to(wts[f][:, None], acc.shape), _sample(flat[slots[f]][:, :cf], *geo[f]), acc)
    return _store(acc, dtype, mutate), wts


def emulate_dff(key, flow, scale, dtype, mutate=None):
    h, w, c = key.shape
    idx, wts = _geometry(flow, mutate)
    k = key.reshape(h * w, c)
    sc = scale[..., :c].reshape(h * w, c)
    if mutate == "warp_of_product":
        v = _sample(_guarded((k * sc).astype(F32), w), idx, wts)
    else:
        v = (_sample(_guarded(k, w), idx, wts) * sc).astype(F32)
    return _store(v, dtype, mutate)


def _windows(h, w):
    for y in range((h + 1) // 2):
        for x in range((w + 1) // 2):
            yield y, x, [(yy, xx) for yy in range(2 * y, min(2 * y + 2, h)) for xx in range(2 * x, min(2 * x + 2, w))]


def emulate_pool(x, dtype, mutate=None):
    n, h, w, c = x.shape
    out = np.zeros((n, (h + 1) // 2, (w + 1) // 2, c), F32)
    for y, xo, cells in _windows(h, w):
        s = np.zeros((n, c), F32)
        for yy, xx in cells:
            s = (s + x[:, yy, xx]).astype(F32)
        out[:, y, xo] = (s / F32(4 if mutate == "divisor4" else len(cells))).astype(F32)
    return _store(out, dtype, mutate)


def emulate_pool_image(img, dtype, mutate=None):
    _, h, w = img.shape
    out = np.zeros(((h + 1) // 2, (w + 1) // 2, 4), F32)
    for y, xo, cells in _windows(h, w):
        inv = (F32(1) / F32(len(cells))).astype(F32)
        s = np.zeros(3, F32)
        for yy, xx in cells:
            v = img[:, yy, xx]
            s = (s + (v if mutate == "no_255" else (v / F32(255)).astype(F32))).astype(F32)
        out[y, xo, :3] = (s * inv).astype(F32)
    return _store(out, dtype, mutate)


# ------------------------------------------------------------------------------------------------ fixtures
def _as(t, dtype):
    """the values a kernel of element type dtype reads"""
    return t.half().float() if dtype == "f16" else t.float()


def _fixture(cid, dtype):
    """(emulate(mutate) -> list of outputs, list of (ref, bound)) of a case"""
    c = CASES[cid]
    inp = R.build_inputs(c)
    R.check_domain(c, inp)
    if c["kind"] == "agg":
        ring = _as(inp["ring"], dtype)
        out, ob, wt, wb = R.aggregate_reference(ring, inp["slots"], c["key"], inp["flow"], c["cf"], c["ce"])
        emu = lambda m=None: list(emulate_aggregate(ring.numpy(), inp["slots"], c["key"], inp["flow"], c["cf"],
                                                    c["ce"], dtype, m))
        return emu, [(out, ob, dtype, "agg"), (wt, wb, "f32", "weights")]
    if c["kind"] == "dff":
        key = _as(inp["key"][..., c["key_off"]:c["key_off"] + c["c"]], dtype).contiguous()
        scale = _as(inp["scale"], dtype)
        out, ob = R.dff_reference(key, inp["flow"], scale)
        emu = lambda m=None: [emulate_dff(key.numpy(), inp["flow"], scale.numpy(), dtype, m)]
        return emu, [(out, ob, dtype, "dff")]
    if c["kind"] == "pool":
        x = _as(inp["x"][..., :c["c"]], dtype).contiguous()
        out, ob = R.avgpool_reference(x)
        return (lambda m=None: [emulate_pool(x.numpy(), dtype, m)]), [(out, ob, dtype, "pool")]
    img = inp["img"]
    out, ob = R.pool_image_reference(img)
    return (lambda m=None: [emulate_pool_image(img.numpy(), dtype, m)]), [(out, ob, dtype, "pool_image")]


def _inside_all(outs, refs):
    ok = True
    for got, (ref, bound, dt, kind) in zip(outs, refs):
        got = torch.from_numpy(np.ascontiguousarray(got)).reshape(ref.shape)
        ok &= bool(R.inside(got, ref, bound, dt, R.A[kind]).all())
    return ok


@pytest.fixture(scope="module")
def fixtures():
    return {(cid, dt): _fixture(cid, dt) for cid in FIXTURES for dt in CASES[cid]["dtypes"]}


@pytest.mark.parametrize("cid", FIXTURES)
def test_emulation_lies_inside_the_interval(fixtures, cid):
    for dt in CASES[cid]["dtypes"]:
        emu, refs = fixtures[(cid, dt)]
        outs = emu()
        for got, (ref, bound, odt, kind) in zip(outs, refs):
            got = torch.from_numpy(np.ascontiguousarray(got)).reshape(ref.shape)
            ok = R.inside(got, ref, bound, odt, R.A[kind])
            assert bool(ok.all()), "%s %s: %d of %d outside, needed A %.3g" % (
                cid, dt, int((~ok).sum()), ok.numel(), R.needed_a(got, ref, bound, odt))


def test_interval_is_not_vacuous(fixtures):
    """fp32 half-widths are a small fraction of |ref| (median over elements with |ref| > 0): <= 2^-13 for the aggregate
    (a weighted mean of L frames, whose soft-max weights carry the cosine logits' error), <= 2^-15 for its weights,
    <= 2^-19 for the warp-and-scale and the pools"""
    limit = {"agg": 2.0 ** -13, "weights": 2.0 ** -15, "dff": 2.0 ** -19, "pool": 2.0 ** -19, "pool_image": 2.0 ** -19}
    for (cid, dt), (emu, refs) in fixtures.items():
        if dt != "f32":
            continue
        for ref, bound, _, kind in refs:
            live = ref.abs() > 0
            if bool(live.any()):
                rel = (R.half_width(bound, ref, "f32", R.A[kind]) / ref.abs().clamp_min(1e-300))[live]
                assert rel.median().item() <= limit[kind], (cid, kind, rel.median().item())


MUTATIONS = ["align_corners", "zeros", "unclamped", "swap_xy", "no_fma", "key_unwarped", "slot_flow", "eps_in_sqrt",
             "divisor4", "no_255", "warp_of_product", "rz16"]
APPLIES = {"align_corners": ("agg", "dff"), "zeros": ("agg", "dff"), "unclamped": ("agg", "dff"),
           "swap_xy": ("agg", "dff"), "no_fma": ("agg", "dff"), "key_unwarped": ("agg",), "slot_flow": ("agg",),
           "eps_in_sqrt": ("agg",), "divisor4": ("pool",), "no_255": ("pool_image",), "warp_of_product": ("dff",),
           "rz16": ("agg", "dff", "pool", "pool_image")}


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_mutations_are_rejected(fixtures, mutation):
    rejected = []
    for (cid, dt), (emu, refs) in fixtures.items():
        c = CASES[cid]
        if c["kind"] not in APPLIES[mutation] or (mutation == "rz16" and dt != "f16"):
            continue
        if mutation == "slot_flow" and max(R.window(c)) >= c["L"]:
            continue
        if not _inside_all(emu(mutation), refs):
            rejected.append((cid, dt))
    assert rejected, "%s passes the interval on every fixture" % mutation


def test_fixtures_reach_the_edges(fixtures):
    """positions exactly on integer cells, on 0 and on w - 1 unclamped, clamped from both sides, and the one-ulp
    disagreement with F.grid_sample's rounding order"""
    seen = dict(on_int=False, zero=False, last=False, clamp_lo=False, clamp_hi=False, fma_differs=False)
    for cid in FIXTURES:
        c = CASES[cid]
        if c["kind"] not in ("agg", "dff"):
            continue
        inp = R.build_inputs(c)
        flow = inp["flow"]
        for f in (flow if c["kind"] == "agg" else flow[None]):
            xs = np.broadcast_to(np.arange(c["w"])[None, :], f.shape[:2])
            s = (f[..., 0] + xs.astype(F32)).astype(F32)
            g = (s / (F32(c["w"] - 1) * F32(0.5))).astype(F32) - F32(1)
            t = (g + F32(1)).astype(F32)
            raw = ((t.astype(np.float64) * c["w"] - 1.0).astype(F32) * F32(0.5))
            nofma = ((t * F32(c["w"])).astype(F32) - F32(1)).astype(F32) * F32(0.5)
            seen["on_int"] |= bool(((raw == np.floor(raw)) & (raw > 0) & (raw < c["w"] - 1)).any())
            seen["zero"] |= bool((raw == 0).any())
            seen["last"] |= bool((raw == c["w"] - 1).any())
            seen["clamp_lo"] |= bool((raw < 0).any())
            seen["clamp_hi"] |= bool((raw > c["w"] - 1).any())
            seen["fma_differs"] |= bool(((raw != nofma) & (raw > 0) & (raw < c["w"] - 1)).any())
    assert all(seen.values()), seen


def test_zero_flow_is_not_the_identity():
    """get_grid normalises for align_corners=True, grid_sample unnormalises with False: a zero flow samples
    x * w / (w - 1) - 1/2, not x"""
    g = R.Geometry(np.zeros((6, 7, 2), F32))
    xs, x0, lx = g.px
    assert bool((lx != 0).any())
    assert not np.array_equal(x0 + lx, xs.astype(np.float64))


# ------------------------------------------------------------------------------------------------ geometry vs torch
def _get_grid(flow):
    """detector/generalized_rcnn_fgfa.py get_grid in float64: flow [N, 2, h, w] -> grid [N, h, w, 2]"""
    n, _, h, w = flow.shape
    sy, sx = torch.meshgrid(torch.arange(h, dtype=torch.float64), torch.arange(w, dtype=torch.float64), indexing="ij")
    ws = torch.tensor([(w - 1) / 2.0, (h - 1) / 2.0], dtype=torch.float64).view(1, 2, 1, 1)
    return ((flow + torch.stack((sx, sy)).unsqueeze(0)) / ws - 1).permute(0, 2, 3, 1)


@pytest.mark.parametrize("cid", ["flow_exact", "flow_far", "map_2x9", "map_9x2", "prod_rot_12x20", "dff_exact"])
def test_fp64_geometry_matches_grid_sample_and_the_oracle(cid):
    import mega_oracle as mo
    c = CASES[cid]
    inp = R.build_inputs(c)
    flow = inp["flow"] if c["kind"] == "agg" else inp["flow"][None]
    n, h, w = flow.shape[:3]
    g = torch.Generator().manual_seed(5)
    feats = torch.randn(n, 6, h, w, generator=g, dtype=torch.float64)
    fl = torch.from_numpy(np.ascontiguousarray(flow[..., :2])).double().permute(0, 3, 1, 2)
    want = F.grid_sample(feats, _get_grid(fl), mode="bilinear", padding_mode="border", align_corners=False)
    oracle = mo.fgfa_warp(feats, fl)
    geo = R.Geometry(flow, mode="fp64")
    idx, wts = geo.torch("cpu")
    mine = torch.stack([R.sample64(feats[i].permute(1, 2, 0).reshape(h * w, 6), idx[:, i], wts[:, i])
                        for i in range(n)]).view(n, h, w, 6).permute(0, 3, 1, 2)
    assert (mine - want).abs().max().item() < 1e-12
    assert (mine - oracle).abs().max().item() < 1e-12
    # the kernel-order fp32 geometry samples a few fp32 ulps away from the fp64 position (the corners themselves can
    # differ where a position sits on an integer cell)
    kidx, kwts = R.Geometry(flow).torch("cpu")
    kern = torch.stack([R.sample64(feats[i].permute(1, 2, 0).reshape(h * w, 6), kidx[:, i], kwts[:, i])
                        for i in range(n)]).view(n, h, w, 6).permute(0, 3, 1, 2)
    assert (kern - want).abs().max().item() < 1e-4 * feats.abs().max().item()


# ------------------------------------------------------------------------------------------------ restatement vs source
def _src():
    return re.sub(r"\s+", " ", open(os.path.join(ROOT, "mega.pytorch_b200", "csrc", "fgfa.cu")).read())


def test_restatement_and_limits_match_the_source():
    src = _src()
    for cond in (
            "constexpr int kAggThreads = %d;" % R.K_AGG_THREADS,
            "constexpr int kAggMaxFrames = %d;" % R.K_AGG_MAX_FRAMES,
            "MEGA_ARG_CHECK(embed_channels <= 16 * kAggThreads,",
            "MEGA_ARG_CHECK(n_frames > 0 && n_frames <= kAggMaxFrames",
            "const long long cap = 132LL * 16;",
            # flow_corners, as fgfa_ref._axis restates it
            "const float gx = __fadd_rn(__fdiv_rn(__fadd_rn(fx, static_cast<float>(x)), static_cast<float>(w - 1) * "
            "0.5f), -1.0f);",
            "float px = __fmaf_rn(__fadd_rn(gx, 1.0f), static_cast<float>(w), -1.0f) * 0.5f;",
            "px = fminf(fmaxf(px, 0.f), static_cast<float>(w - 1));",
            "const int x1 = min(x0 + 1, w - 1), y1 = min(y0 + 1, h - 1);",
            "const float lx = px - x0f, ly = py - y0f;",
            "c.w00 = (1.f - lx) * (1.f - ly); c.w01 = lx * (1.f - ly); c.w10 = (1.f - lx) * ly; c.w11 = lx * ly;",
            # the sample, the reductions, the soft-max and the sum the interval's chains count
            "return c.w00 * to_f<T>(base[c.o00 + ch]) + c.w01 * to_f<T>(base[c.o01 + ch]) + c.w10 * "
            "to_f<T>(base[c.o10 + ch]) + c.w11 * to_f<T>(base[c.o11 + ch]);",
            "for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);",
            "for (int i = 0; i < kAggThreads / 32; ++i) s += red[i];",
            "kn = sqrtf(block_sum(kn, red)) + 1e-10f;",
            "nn = sqrtf(block_sum(nn, red)) + 1e-10f;",
            "logit[f] = (dot / nn) / kn;",
            "acc += expf(logit[f] - mx) * inv * sample<T>(fbase, corners[f], ch);",
            "const float* f = flow + (static_cast<long long>(tid) * h * w + pix) * flow_ld;",
            "const float v = sample<T>(key, c, ch) * to_f<T>(scale[static_cast<long long>(pix) * scale_ld + ch]);",
            "out[pix * out_ld + c] = from_f<T>(s / static_cast<float>((y1 - y0) * (x1 - x0)));",
            "s += __ldg(img + (static_cast<long long>(c) * height + yy) * width + xx) / 255.0f;",
            "v[c] = s * inv;",
            "__float2half_rn(v)"):
        assert cond in src, cond
    kernels = set(re.findall(r"template <typename T> __global__ void (?:__launch_bounds__\(\w+\) )?(\w+)\(", src))
    assert kernels == set(R.KERNELS), kernels
    assert "use_fast_math" not in open(os.path.join(ROOT, "mega.pytorch_b200", "build.py")).read()


def test_case_table_covers_the_edges():
    cases = list(CASES.values())
    agg = [c for c in cases if c["kind"] == "agg"]
    assert {1, 200, 256, 1000, 4096} <= {c["ce"] for c in agg}
    assert {1, 100, 1030} <= {c["cf"] for c in agg}
    assert {1, 32} <= {c["L"] for c in agg} and max(c["L"] for c in agg) == R.K_AGG_MAX_FRAMES
    assert any(c["key"] == 0 for c in agg if c["L"] > 1) and any(c["key"] == c["L"] - 1 for c in agg if c["L"] > 1)
    maps = {(c["h"], c["w"]) for c in agg}
    assert {(2, 2), (38, 63), (12, 20)} <= maps and any(h == 2 and w > 2 for h, w in maps) and \
        any(w == 2 and h > 2 for h, w in maps)
    prod = [c for c in agg if (c["L"], c["key"], c["cf"], c["ce"], c["ld"]) == (19, 9, 1024, 2048, 3072)]
    assert {"first", "rot"} <= {c["window"] for c in prod}
    assert {"zero", "exact", "far", "randn"} <= {c["flow"] for c in agg}
    assert {"zero_frame", "zero_key", "tiny", "big", "sub"} <= {c["values"] for c in agg}
    dff = [c for c in cases if c["kind"] == "dff"]
    assert any(c["c"] == 1024 and c["key_ld"] == 3072 and c["pad"] > 0 for c in dff)
    # every grid-stride kernel runs at least one case past grid_for's cap
    for kind in ("dff", "pool", "pool_image", "pairs"):
        assert max(R.threads(c) for c in cases if c["kind"] == kind) > R.GRID_CAP * R.BLOCK, kind
    pools = [(c["h"], c["w"]) for c in cases if c["kind"] in ("pool", "pool_image")]
    assert (1, 1) in pools and any(h == 1 and w > 1 for h, w in pools) and any(h % 2 and w % 2 for h, w in pools) \
        and any(h % 2 == 0 and w % 2 == 0 for h, w in pools)
    assert any(c["n"] > 1 for c in cases if c["kind"] == "pool")
    for c in agg:
        if c["values"] in ("randn", "tiny", "zero_frame", "zero_key") and c["h"] * c["w"] <= 64:
            R.check_domain(c, R.build_inputs(c))


# ------------------------------------------------------------------------------------------------ ops layout checks
ENTRIES = ("mega_fgfa_pool_image", "mega_fgfa_build_pairs", "mega_avgpool2_nhwc", "mega_fgfa_aggregate",
           "mega_dff_warp_scale")


@pytest.fixture
def recorded(monkeypatch):
    """ops with every FGFA library entry replaced by a recorder (returns 0) and the CUDA checks switched off"""
    from mega_core.b200 import ops
    calls = []
    for name in ENTRIES:
        monkeypatch.setattr(ops.lib, name, (lambda n: lambda *a: calls.append((n, a)) or 0)(name))
    monkeypatch.setattr(ops, "require_cuda", lambda *t: None)
    monkeypatch.setattr(ops, "stream_ptr", lambda: None)
    return ops, calls


def _agg_args(h=4, w=5, L=3, cf=8, ce=16):
    ring = torch.zeros(L + 1, h, w, cf + ce)
    slots = torch.arange(L, dtype=torch.int32)
    flow = torch.zeros(L, h, w, 4)
    out = torch.zeros(h, w, cf)
    wo = torch.zeros(L, h, w)
    return dict(ring=ring, slots=slots, flow=flow, out=out, weights_out=wo)


def _bad_agg(what):
    a = _agg_args()
    L, h, w = 3, 4, 5
    if what == "agg_ring_cropped_columns":
        a["ring"] = torch.zeros(L + 1, h, w + 2, 24)[:, :, :w]
    elif what == "agg_ring_too_narrow":
        a["ring"] = torch.zeros(L + 1, h, w, 20)
    elif what == "agg_flow_short":
        a["flow"] = torch.zeros(L - 1, h, w, 4)
    elif what == "agg_flow_hw":
        a["flow"] = torch.zeros(L, h, w + 1, 4)
    elif what == "agg_flow_cropped_columns":
        a["flow"] = torch.zeros(L, h, w + 3, 4)[:, :, :w]
    elif what == "agg_flow_frames_not_packed":
        a["flow"] = torch.zeros(L, h + 1, w, 4)[:, :h]
    elif what == "agg_flow_one_channel":
        a["flow"] = torch.zeros(L, h, w, 1)
    elif what == "agg_weights_f16":
        a["weights_out"] = torch.zeros(L, h, w, dtype=torch.float16)
    elif what == "agg_weights_shape":
        a["weights_out"] = torch.zeros(L - 1, h, w)
    elif what == "agg_weights_strided":
        a["weights_out"] = torch.zeros(L, h, w, 2)[..., 0]
    elif what == "agg_out_cropped_columns":
        a["out"] = torch.zeros(h, w + 2, 8)[:, :w]
    elif what == "agg_out_shape":
        a["out"] = torch.zeros(h - 1, w, 8)
    elif what == "agg_out_narrow":
        a["out"] = torch.zeros(h, w, 7)
    elif what == "agg_slots_int64":
        a["slots"] = a["slots"].long()
    return a


AGG_BAD = ["agg_ring_cropped_columns", "agg_ring_too_narrow", "agg_flow_short", "agg_flow_hw",
           "agg_flow_cropped_columns", "agg_flow_frames_not_packed", "agg_flow_one_channel", "agg_weights_f16",
           "agg_weights_shape", "agg_weights_strided", "agg_out_cropped_columns", "agg_out_shape", "agg_out_narrow",
           "agg_slots_int64"]
POOL_BAD = ["pool_x_cropped_columns", "pool_x_images_not_packed", "pool_out_cropped_columns", "pool_out_spatial",
            "pool_out_channels", "pool_x_channel_stride"]
DFF_BAD = ["dff_key_cropped_columns", "dff_flow_cropped_columns", "dff_flow_shape", "dff_scale_cropped_columns",
           "dff_scale_narrow", "dff_out_cropped_columns", "dff_out_shape"]
IMAGE_BAD = ["image_out_strided", "image_out_shape", "image_strided"]
PAIRS_BAD = ["pairs_strided", "pairs_shape", "pairs_slots_count", "pairs_ring_not_dense"]


def _call_bad(ops, what):
    from mega_core._lib import MegaError
    if what.startswith("agg"):
        a = _bad_agg(what)
        fn = lambda: ops.fgfa_aggregate(a["ring"], a["slots"], 1, a["flow"], a["out"], 8, 16, weights_out=a["weights_out"])
    elif what.startswith("pool"):
        x, out = torch.zeros(2, 5, 7, 6), torch.zeros(2, 3, 4, 6)
        if what == "pool_x_cropped_columns":
            x = torch.zeros(2, 5, 9, 6)[:, :, :7]
        elif what == "pool_x_images_not_packed":
            x = torch.zeros(2, 6, 7, 6)[:, :5]
        elif what == "pool_out_cropped_columns":
            out = torch.zeros(2, 3, 5, 6)[:, :, :4]
        elif what == "pool_out_spatial":
            out = torch.zeros(2, 2, 4, 6)
        elif what == "pool_out_channels":
            out = torch.zeros(2, 3, 4, 5)
        else:
            x = torch.zeros(2, 5, 7, 12)[..., ::2]
        fn = lambda: ops.avgpool2_nhwc(x, out)
    elif what.startswith("dff"):
        h, w, c = 4, 5, 16
        key, flow, scale, out = torch.zeros(h, w, c), torch.zeros(h, w, 4), torch.zeros(h, w, c), torch.zeros(h, w, c)
        wide = lambda ch: torch.zeros(h, w + 2, ch)[:, :w]
        if what == "dff_key_cropped_columns":
            key = wide(c)
        elif what == "dff_flow_cropped_columns":
            flow = wide(4)
        elif what == "dff_flow_shape":
            flow = torch.zeros(h, w - 1, 4)
        elif what == "dff_scale_cropped_columns":
            scale = wide(c)
        elif what == "dff_scale_narrow":
            scale = torch.zeros(h, w, c - 8)
        elif what == "dff_out_cropped_columns":
            out = wide(c)
        else:
            out = torch.zeros(h + 1, w, c)
        fn = lambda: ops.dff_warp_scale(key, flow, scale, out)
    elif what.startswith("image"):
        img, out = torch.zeros(1, 3, 7, 9), torch.zeros(4, 5, 4)
        if what == "image_out_strided":
            out = torch.zeros(4, 5, 8)[..., :4]
        elif what == "image_out_shape":
            out = torch.zeros(4, 4, 4)
        else:
            img = torch.zeros(1, 3, 7, 10)[..., :9]
        fn = lambda: ops.fgfa_pool_image(img, out)
    else:
        ring, slots, pairs = torch.zeros(4, 3, 5, 4), torch.arange(3, dtype=torch.int32), torch.zeros(3, 9, 13, 8)
        if what == "pairs_strided":
            pairs = torch.zeros(3, 9, 13, 16)[..., :8]
        elif what == "pairs_shape":
            pairs = torch.zeros(3, 9, 12, 8)
        elif what == "pairs_slots_count":
            slots = torch.arange(2, dtype=torch.int32)
        else:
            ring = torch.zeros(4, 3, 5, 8)[..., :4]
        fn = lambda: ops.fgfa_build_pairs(ring, slots, 1, pairs)
    with pytest.raises(MegaError):
        fn()


@pytest.mark.parametrize("what", AGG_BAD + POOL_BAD + DFF_BAD + IMAGE_BAD + PAIRS_BAD)
def test_ops_rejects_layouts_the_kernels_cannot_read(recorded, what):
    ops, calls = recorded
    _call_bad(ops, what)
    assert not calls, "%s reached %s" % (what, calls[0][0])


def test_ops_passes_good_layouts_with_their_strides(recorded):
    """a channel slice of a wider ring is read at its pixel stride (ring.stride(2)), padded out / scale / key rows at
    theirs; every good call reaches its entry once"""
    ops, calls = recorded
    a = _agg_args()
    ring = torch.zeros(4, 4, 5, 40)[..., 4:28]
    out = torch.zeros(4, 5, 12)[..., :8]
    ops.fgfa_aggregate(ring, a["slots"], 1, a["flow"], out, 8, 16, weights_out=a["weights_out"])
    name, args = calls[-1]
    assert name == "mega_fgfa_aggregate" and args[1] == 4 * 5 * 40 and args[2] == 40 and args[9] == 4 and args[13] == 12
    key = torch.zeros(4, 5, 48)[..., 16:32]
    scale, dout = torch.zeros(4, 5, 24)[..., :16], torch.zeros(4, 5, 20)[..., :16]
    ops.dff_warp_scale(key, torch.zeros(4, 5, 4), scale, dout)
    name, args = calls[-1]
    assert name == "mega_dff_warp_scale" and (args[1], args[2], args[4], args[6], args[10]) == (48, 16, 4, 24, 20)
    ops.avgpool2_nhwc(torch.zeros(2, 5, 7, 12)[..., :6], torch.zeros(2, 3, 4, 10)[..., :6])
    name, args = calls[-1]
    assert name == "mega_avgpool2_nhwc" and (args[5], args[7]) == (12, 10)
    ops.fgfa_pool_image(torch.zeros(1, 3, 7, 9), torch.zeros(4, 5, 4))
    ops.fgfa_build_pairs(torch.zeros(4, 3, 5, 4), torch.arange(3, dtype=torch.int32), 1, torch.zeros(3, 9, 13, 8))
    assert [n for n, _ in calls] == ["mega_fgfa_aggregate", "mega_dff_warp_scale", "mega_avgpool2_nhwc",
                                     "mega_fgfa_pool_image", "mega_fgfa_build_pairs"]
