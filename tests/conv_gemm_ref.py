"""Shared pieces of the conv_gemm conformance suite (test_conv_gemm_conformance_cpu.py / _gpu.py).

- conv_gemm_ref: an fp64 restatement of the mega_conv_gemm_desc contract (include/mega_b200.h), batched offsets included;
- the table of the 42 conv_gemm_kernel instantiations (csrc/conv_gemm_kernel.cuh launch_mode / conv_gemm_stages);
- the committed case list: per instantiation a pairwise covering set of epilogue options over a rotation of geometries;
- the stream-K work split (cta_first_unit / unit_owner and the encoder's grid rule), restated in Python.
"""
import itertools

import torch
import torch.nn.functional as F

MODES = {0: "tf32", 1: "3xtf32", 2: "f16", 3: "3xfp16"}
BLOCK_NS = (32, 64, 96, 128, 160, 192, 256)
GROUP_WIDTHS = (8, 16, 32)      # group widths with their own instantiations; 64 runs the dense block_n 64 kernel
NUM_SMS = 132                   # persistent grid cap of an H100 SXM (kMaxCtas)
COUNTER_INTS = 65536            # tile counters at the head of the stream-K workspace
SLOPE = 0.1                     # LeakyReLU slope of relu == 2


def mode_bk(mode):
    """K-slab of one k-block, in elements"""
    return 64 if mode == 2 else 32


# ------------------------------------------------------------------------------------------------ instantiation table
def _variant_table():
    """(precision, block_n, out16, group_width) of every conv_gemm_kernel instantiation: launch_mode<MODE> instantiates
    the grouped widths 8 / 16 / 32 at block_n 64, block_n 64 / 128 in every mode and 32 / 96 / 160 / 192 / 256 in the
    TF32 and FP16 modes; out16 (fp16 output) exists for precision 2 at block_n % 64 == 0, and (split-fp16 output) for
    every precision-3 instantiation."""
    out = []
    for mode in (0, 1, 2, 3):
        bns = BLOCK_NS if mode in (0, 2) else (64, 128)
        for gw in GROUP_WIDTHS + (0,):
            for bn in ((64,) if gw else bns):
                for out16 in (False, True):
                    if out16 and not (mode == 3 or (mode == 2 and bn % 64 == 0)):
                        continue
                    out.append((mode, bn, out16, gw))
    return out


VARIANTS = _variant_table()


def variant_of(precision, block_n, out_f16, group_width):
    """the instantiation a descriptor launches (conv_gemm.cu: group_width 64 runs the dense issue)"""
    return (precision, block_n, bool(out_f16), 0 if group_width == 64 else group_width)


# ------------------------------------------------------------------------------------------------ fp64 reference
def conv_gemm_ref(A, B, *, taps=(1, 1), dil=1, pad=0, pad_w=None, stride=(1, 1), k, n_img, out_hw, cout, batch=1,
                  a_c_off=0, a_n_off=0, b_k_off=0, b_n_off=0, out_c_off=0, out_n_off=0, res_c_off=0, res_n_off=0,
                  bias_z_off=0, scale=None, bias=None, residual=None, relu=0, acc_scale=1.0):
    """The descriptor's contract in float64:
        out[z*out_n_off + n, h, w, z*out_c_off + co] = act( acc_scale * scale[z*bias_z_off + co]
            * sum_{r,s,ci} A[z*a_n_off + n, h*sh + r*dil - pad, w*sw + s*dil - pad_w, z*a_c_off + ci]
                         * B[r*S + s, z*b_n_off + co, z*b_k_off + ci]
            + bias[z*bias_z_off + co] + residual[z*res_n_off + n, h, w, z*res_c_off + co] )
    with A zero outside its extent. A [a_n, a_h, a_w, a_c], B [taps, b_n, b_k], residual [rn, oh, ow, rc] (the residual
    view's logical coordinates), scale / bias 1-D. Returns a list of (z, ref, P, Q), each [n_img, oh, ow, cout]:
    P = |acc_scale * scale| * conv(|A|, |B|) scales the contraction error, Q = |scaled acc| + |bias| + |residual| the
    epilogue's fp32 rounding."""
    R, S = taps
    sh, sw = stride
    oh, ow = out_hw
    pw = pad if pad_w is None else pad_w
    need_h = (oh - 1) * sh + (R - 1) * dil + 1
    need_w = (ow - 1) * sw + (S - 1) * dil + 1
    blocks = []
    for z in range(batch):
        a = A[z * a_n_off:z * a_n_off + n_img, :, :, z * a_c_off:z * a_c_off + k].double()
        assert a.shape[0] == n_img and a.shape[3] == k, "A does not cover batch entry %d" % z
        b = B[:, z * b_n_off:z * b_n_off + cout, z * b_k_off:z * b_k_off + k].double()
        assert b.shape[2] == k
        if b.shape[1] < cout:       # rows past B's extent read as zeros
            b = torch.cat([b, b.new_zeros(b.shape[0], cout - b.shape[1], k)], 1)
        x = a.permute(0, 3, 1, 2)
        x = F.pad(x, (pw, need_w - pw - x.shape[3], pad, need_h - pad - x.shape[2]))   # negative: crop
        wt = b.reshape(R, S, cout, k).permute(2, 3, 0, 1)
        acc = F.conv2d(x, wt, stride=(sh, sw), dilation=dil).permute(0, 2, 3, 1)
        mag = F.conv2d(x.abs(), wt.abs(), stride=(sh, sw), dilation=dil).permute(0, 2, 3, 1)
        assert acc.shape == (n_img, oh, ow, cout), acc.shape
        s = acc.new_full((cout,), float(acc_scale))
        if scale is not None:
            s = s * scale[z * bias_z_off:z * bias_z_off + cout].double()
        v = acc * s
        P = mag * s.abs()
        Q = v.abs()
        if bias is not None:
            bb = bias[z * bias_z_off:z * bias_z_off + cout].double()
            v = v + bb
            Q = Q + bb.abs()
        if residual is not None:
            r = residual[z * res_n_off:z * res_n_off + n_img, :, :, z * res_c_off:z * res_c_off + cout].double()
            v = v + r
            Q = Q + r.abs()
        if relu == 1:
            v = v.clamp_min(0)
        elif relu == 2:
            v = torch.where(v > 0, v, SLOPE * v)
        blocks.append((z, v, P, Q))
    return blocks


# ------------------------------------------------------------------------------------------------ case list
# Geometries of the variant sweep. a_hw: input map; k: reduction length per tap (a K tail where k is not a multiple of the
# mode's k-block); row_skip 2: the output view skips every other row (out_stride_h).
GEOMS = {
    "g1x1":    dict(taps=(1, 1), dil=1, pad=0, pad_w=None, stride=(1, 1), tile=(8, 16), n_img=2, out_hw=(11, 21),
                    a_hw=(11, 21), k=96, row_skip=1),
    "g3x3d2":  dict(taps=(3, 3), dil=2, pad=2, pad_w=None, stride=(1, 1), tile=(16, 8), n_img=1, out_hw=(19, 13),
                    a_hw=(19, 13), k=64, row_skip=2),
    "g5x5s2":  dict(taps=(5, 5), dil=1, pad=2, pad_w=None, stride=(2, 2), tile=(4, 32), n_img=2, out_hw=(7, 37),
                    a_hw=(14, 74), k=32, row_skip=1),
    "g3x3s2d2": dict(taps=(3, 3), dil=2, pad=2, pad_w=1, stride=(2, 2), tile=(8, 16), n_img=1, out_hw=(9, 17),
                     a_hw=(18, 33), k=64, row_skip=1),
    "gline":   dict(taps=(1, 1), dil=1, pad=0, pad_w=None, stride=(1, 1), tile=(1, 128), n_img=1, out_hw=(1, 300),
                    a_hw=(1, 300), k=160, row_skip=1),
    "gcol":    dict(taps=(3, 1), dil=1, pad=1, pad_w=0, stride=(1, 1), tile=(128, 1), n_img=1, out_hw=(200, 3),
                    a_hw=(200, 3), k=64, row_skip=1),
    "g3x3tail": dict(taps=(3, 3), dil=1, pad=1, pad_w=0, stride=(1, 1), tile=(16, 8), n_img=3, out_hw=(10, 9),
                     a_hw=(10, 9), k=40, row_skip=1),
    # batched launch, every offset non-zero and res_n_off != out_n_off (cout = block_n: channel-offset batching)
    "gbatch":  dict(taps=(3, 3), dil=1, pad=1, pad_w=None, stride=(1, 1), tile=(8, 16), n_img=2, out_hw=(9, 12),
                    a_hw=(9, 12), k=64, row_skip=1, batch=3, a_n_off=1, out_n_off=1, res_n_off=2, a_c_off=64,
                    b_k_off=64),
}
GEOM_ROTATION = ("g1x1", "gbatch", "g3x3d2", "g5x5s2", "g3x3s2d2", "gline", "gcol", "g3x3tail")
# grouped convolution (ResNeXt conv2): 256 channels in the 64-channel batched layout
GROUPED = dict(taps=(3, 3), dil=1, pad=1, pad_w=None, stride=(1, 1), tile=(8, 16), n_img=2, out_hw=(9, 14),
               a_hw=(9, 14), k=64, row_skip=1, channels=256)
COUTS = (None, 2, 60, 200)      # None: cout = block_n


def pairwise_rows(factors):
    """deterministic greedy pairwise covering set over `factors` [(name, values)]: every pair of values of two different
    factors occurs in at least one row"""
    names = [f[0] for f in factors]
    todo = set()
    for (i, (_, vi)), (j, (_, vj)) in itertools.combinations(enumerate(factors), 2):
        for a in vi:
            for b in vj:
                todo.add((i, a, j, b))
    rows = []
    cands = list(itertools.product(*[f[1] for f in factors]))
    while todo:
        best = max(cands, key=lambda r: sum((i, r[i], j, r[j]) in todo
                                            for i, j in itertools.combinations(range(len(r)), 2)))
        for i, j in itertools.combinations(range(len(best)), 2):
            todo.discard((i, best[i], j, best[j]))
        rows.append(dict(zip(names, best)))
    return rows


def epilogue_factors(mode):
    res = ("none", "fp32", "split") if mode == 3 else ("none", "same")
    scale = (False,) if mode == 3 else (False, True)      # precision 3 takes no scale (folded into the packed weights)
    return [("res", res), ("scale", scale), ("bias", (False, True)), ("relu", (0, 1, 2))]


def _round_up(x, m):
    return -(-x // m) * m


def geometry_for(mode, name):
    g = dict(GEOMS[name])
    if mode == 3:
        g["k"] = _round_up(g["k"], 32)      # split-fp16 operands: whole 32-value groups (no K tail in precision 3)
    return g


def make_cases():
    """the committed sweep: per instantiation one row per pairwise combination of the epilogue options (alternating
    stream-K off / on, varying max_ctas), geometries rotating per mode; grouped instantiations run the grouped layout,
    and every dense block_n 64 instantiation also runs a group-width-64 launch"""
    cases = []
    queue = {m: [] for m in MODES}
    for vi, (mode, bn, out16, gw) in enumerate(VARIANTS):
        rows = pairwise_rows(epilogue_factors(mode))
        extra = [dict(rows[0], grouped=64)] if (gw == 0 and bn == 64) else []
        for ri, opts in enumerate(rows + extra):
            sk = (ri + vi) % 2
            c = dict(mode=mode, block_n=bn, out16=out16, stream_k=sk, max_ctas=(0, 5, 13)[(ri + vi) % 3] if sk else 0,
                     res=opts["res"], scale=opts["scale"], bias=opts["bias"], relu=opts["relu"], seed=1000 * vi + ri)
            grouped = gw or opts.get("grouped", 0)
            if grouped:
                g = dict(GROUPED)
                c.update(geom="grouped", group_width=grouped, cout=64, **g)
            else:
                if not queue[mode]:
                    queue[mode] = list(GEOM_ROTATION)
                # the batched geometry checks res_n_off against out_n_off: give it a row with a residual
                pick = 1 if (queue[mode][0] == "gbatch" and opts["res"] == "none" and len(queue[mode]) > 1) else 0
                name = queue[mode].pop(pick)
                g = geometry_for(mode, name)
                cout = COUTS[(ri + vi) % len(COUTS)] or bn
                if name == "gbatch":
                    cout = bn
                    g.update(b_n_off=bn, out_c_off=bn, res_c_off=bn, bias_z_off=bn)
                c.update(geom=name, group_width=0, cout=cout, **g)
            c["id"] = "%s-bn%d-%s-gw%d-sk%d-%s-%s%s%s-relu%d-%s-co%d" % (
                MODES[mode], bn, "o16" if out16 else "o32", gw, sk, c["geom"], "res_" + c["res"],
                "-scale" if c["scale"] else "", "-bias" if c["bias"] else "", c["relu"], "mc%d" % c["max_ctas"], c["cout"])
            cases.append(c)
    return cases


def case_fields(c):
    """descriptor-level fields of a case (batch / offsets default to the plain launch)"""
    f = dict(batch=1, a_c_off=0, a_n_off=0, b_k_off=0, b_n_off=0, out_c_off=0, out_n_off=0, res_c_off=0, res_n_off=0,
             bias_z_off=0)
    for key in f:
        if key in c:
            f[key] = c[key]
    if c.get("group_width"):
        z = 64
        f.update(batch=c["channels"] // z, a_c_off=z, b_n_off=z, out_c_off=z, res_c_off=z, bias_z_off=z)
    return f


def operand_extents(c):
    """(a_n, a_h, a_w, a_c), (taps, b_n, b_k), output logical (on, oh, ow, oc), residual logical (rn, rc) of a case;
    split-fp16 outputs / residuals cover whole 32-value groups"""
    f = case_fields(c)
    R, S = c["taps"]
    k, cout, bt = c["k"], c["cout"], f["batch"]
    oh, ow = c["out_hw"]
    a = (c["n_img"] + (bt - 1) * f["a_n_off"], c["a_hw"][0], c["a_hw"][1],
         c["channels"] if c.get("group_width") else k + (bt - 1) * f["a_c_off"])
    b = (R * S, c["channels"] if c.get("group_width") else cout + (bt - 1) * f["b_n_off"],
         64 if c.get("group_width") else k + (bt - 1) * f["b_k_off"])
    out_split = c["mode"] == 3 and c["out16"]
    oc = cout + (bt - 1) * f["out_c_off"]
    if out_split:
        oc = _round_up(oc, 32)
    o = (c["n_img"] + (bt - 1) * f["out_n_off"], oh, ow, oc)
    rc = cout + (bt - 1) * f["res_c_off"]
    if c["res"] == "split":
        rc = _round_up(rc, 32)
    r = (c["n_img"] + (bt - 1) * f["res_n_off"], rc)
    return a, b, o, r


def check_case_contract(c):
    """the ops.conv_gemm asserts and the encoder's documented constraints for a case; returns a list of violations"""
    bad = []
    mode, bn, out16 = c["mode"], c["block_n"], c["out16"]
    f = case_fields(c)
    (a_n, a_h, a_w, a_c), (taps, b_n, b_k), (on, oh, ow, oc), (rn, rc) = operand_extents(c)
    th, tw = c["tile"]
    sh, sw = c["stride"]
    if th * tw != 128 or (tw - 1) * sw + 1 > 256 or (th - 1) * sh + 1 > 256:
        bad.append("tile")
    if variant_of(mode, bn, out16, c.get("group_width", 0)) not in VARIANTS:
        bad.append("no instantiation")
    esz = 2 if mode == 2 else 4
    if (a_c * esz) % 16 or (b_k * esz) % 16:
        bad.append("operand rows not 16-byte multiples")
    if f["out_c_off"] and c["cout"] != bn:
        bad.append("channel-offset batching needs cout == block_n")
    bk = mode_bk(mode)
    kk = _round_up(c["k"], bk)
    # the last k-block of a K tail reads up to kk channels: they must run past the tensor (zero fill), not into data
    if kk != c["k"] and (f["batch"] > 1 or a_c != c["k"] or b_k != c["k"]):
        bad.append("K tail reads live channels")
    if mode in (1, 3) and bn not in (64, 128):
        bad.append("strict block_n")
    if mode == 3:
        if a_c % 32 or b_k % 32 or c["k"] % 32 or f["a_c_off"] % 32 or f["b_k_off"] % 32:
            bad.append("split-fp16 operand channels")
        if c["scale"]:
            bad.append("precision 3 takes no scale")
        if out16 and (f["out_c_off"] % 32 or (c["cout"] % 32 and f["batch"] != 1)):
            bad.append("split-fp16 output channels")
        if c["res"] == "split" and (f["res_c_off"] % 32 or (c["cout"] % 32 and f["batch"] != 1)):
            bad.append("split-fp16 residual channels")
    if c.get("group_width"):
        if not (bn == 64 and c["cout"] == 64 and c["k"] == 64 and c["channels"] % 64 == 0):
            bad.append("group layout")
    # every batch entry stays inside A / B (the reference and the kernel then read the same values)
    if f["batch"] > 1 and not c.get("group_width"):
        if (f["batch"] - 1) * f["a_c_off"] + c["k"] > a_c or (f["batch"] - 1) * f["b_k_off"] + c["k"] > b_k:
            bad.append("batch entry outside the operands")
    return bad


def case_problem(c):
    """(tiles, kb_per_tile, total_units) of a case as encode_conv_gemm_problem counts them"""
    f = case_fields(c)
    th, tw = c["tile"]
    oh, ow = c["out_hw"]
    m_tiles = c["n_img"] * -(-oh // th) * -(-ow // tw)
    n_tiles = -(-c["cout"] // c["block_n"])
    kb = c["taps"][0] * c["taps"][1] * -(-c["k"] // mode_bk(c["mode"]))
    tiles = f["batch"] * m_tiles * n_tiles
    return tiles, kb, tiles * kb


# ------------------------------------------------------------------------------------------------ stream-K geometry
def cta_first_unit(total, grid, c):
    return ((total * c) & 0xFFFFFFFF) // grid


def unit_owner(total, grid, u):
    c = ((u * grid) & 0xFFFFFFFF) // total
    if c >= grid:
        c = grid - 1
    while c + 1 < grid and cta_first_unit(total, grid, c + 1) <= u:
        c += 1
    while c > 0 and cta_first_unit(total, grid, c) > u:
        c -= 1
    return c


def encoder_grid(tiles, kb_per_tile, stream_k, max_ctas=0, num_sms=NUM_SMS):
    """the persistent grid encode_conv_gemm_problem picks; also whether the aligned-grid rule changed it"""
    units = tiles * kb_per_tile
    ctas = units // 4 if stream_k else tiles
    ctas = max(ctas, 1)
    ctas = min(ctas, num_sms)
    if max_ctas > 0:
        ctas = min(ctas, max_ctas)
    aligned_fired = False
    if stream_k and kb_per_tile >= 256 and tiles <= ctas:
        aligned = (ctas // tiles) * tiles
        if aligned * 100 >= ctas * 85:
            aligned_fired = aligned != ctas
            ctas = aligned
    return ctas, aligned_fired


def sk_geometry(tiles, kb_per_tile, grid):
    """facts about the stream-K split of `tiles` x `kb_per_tile` units over `grid` CTAs"""
    total = tiles * kb_per_tile
    max_parts = max(unit_owner(total, grid, t * kb_per_tile + kb_per_tile - 1) - unit_owner(total, grid, t * kb_per_tile) + 1
                    for t in range(tiles))
    span = False          # a CTA whose range starts inside a tile, covers >= 1 whole tile and ends inside another
    for c in range(grid):
        u0, u1 = cta_first_unit(total, grid, c), cta_first_unit(total, grid, c + 1)
        if u1 <= u0:
            continue
        first_partial = u0 % kb_per_tile != 0
        last_partial = u1 % kb_per_tile != 0
        whole = (u1 // kb_per_tile) - (-(-u0 // kb_per_tile))
        if first_partial and last_partial and whole >= 1:
            span = True
    return dict(grid=grid, max_parts=max_parts, span=span, divides=total % grid == 0)


# (label, mode, spec): stream-K scheduling cases; spec is a case dict without the epilogue options
def _sk_spec(mode, geom, **kw):
    c = dict(mode=mode, out16=False, stream_k=1, res="same" if mode != 3 else "fp32", scale=mode != 3, bias=True, relu=1,
             group_width=0, row_skip=1)
    c.update(geom)
    c.update(kw)
    return c


def make_sk_cases():
    out = []
    for mode in (0, 1, 2, 3):
        bk = mode_bk(mode)
        deep = dict(taps=(3, 3), dil=1, pad=1, pad_w=None, stride=(1, 1), tile=(8, 16), n_img=1, out_hw=(16, 16),
                    a_hw=(16, 16), k=4 * bk, geom="sk_deep")
        many = dict(taps=(3, 3), dil=1, pad=1, pad_w=None, stride=(1, 1), tile=(8, 16), n_img=2, out_hw=(40, 32),
                    a_hw=(40, 32), k=bk, geom="sk_many")
        out.append(("a", _sk_spec(mode, deep, block_n=64, cout=64, max_ctas=0, seed=10 + mode)))
        out.append(("bd", _sk_spec(mode, many, block_n=64, cout=128, max_ctas=7, seed=20 + mode)))
        out.append(("c", _sk_spec(mode, many, block_n=64, cout=128, max_ctas=1, seed=30 + mode)))
    for mode in (2, 3):
        # a Linear with a 256-k-block reduction over 5 x 4 = 20 tiles: the aligned-grid rule
        line = dict(taps=(1, 1), dil=1, pad=0, pad_w=None, stride=(1, 1), tile=(1, 128), n_img=1, out_hw=(1, 640),
                    a_hw=(1, 640), k=256 * mode_bk(mode), geom="sk_line")
        out.append(("e", _sk_spec(mode, line, block_n=64, cout=256, max_ctas=0, seed=40 + mode)))
        out.append(("f_fires", _sk_spec(mode, line, block_n=64, cout=256, max_ctas=23, seed=50 + mode)))
        out.append(("f_stays", _sk_spec(mode, line, block_n=64, cout=256, max_ctas=24, seed=60 + mode)))
    for label, c in out:
        c["id"] = "%s-%s-mc%d" % (label, MODES[c["mode"]], c["max_ctas"])
    return out


def sk_label_holds(label, c):
    tiles, kb, _ = case_problem(c)
    grid, fired = encoder_grid(tiles, kb, 1, c["max_ctas"])
    g = sk_geometry(tiles, kb, grid)
    if label == "a":
        return g["max_parts"] >= 3
    if label == "bd":
        return g["span"] and not g["divides"]
    if label == "c":
        return grid == 1
    if label in ("e", "f_fires"):
        return kb >= 256 and fired
    if label == "f_stays":
        _, fired_below = encoder_grid(tiles, kb, 1, c["max_ctas"] - 1)
        return kb >= 256 and not fired and fired_below
    raise KeyError(label)


def chain_rotation(layers, grid):
    """cta_rot of every layer of a depth-2 chain (mega_conv_chain_encode2): layers = [(tiles, active_ctas, stream_k)]"""
    rots, start = [], 0
    for tiles, act, sk in layers:
        rots.append(start % grid)
        start += act if sk else (act if tiles % act == 0 else tiles % act)
    return rots
