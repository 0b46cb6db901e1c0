"""Shared pieces of the relation soft-max conformance suite (test_relation_softmax_conformance_cpu.py / _gpu.py).

- reference / prob_interval: an fp64 restatement of the mega_relation_softmax* contract (include/mega_b200.h) and a
  per-element interval that bounds what an fp32 kernel may return;
- dispatch: which kernel a call reaches (csrc/relation.cu relation_softmax_impl / relation_softmax_pe_impl);
- the committed case table: the engines' attention geometries (MEGA G / L0 / L1 / L2, RDN) and odd small shapes, with
  key counts, padded query rows, boxes, logits and weights placed where the kernels can go wrong.

Error model (interval propagation; first-order errors do not survive log(relu(.) + 1e-6) near its kink). With
a_e = 100 delta_c / dim_k the sin / cos argument of feature e and kappa_c the condition of delta_c on the kernel's fp32
box arithmetic (widths, centres, the difference of centres, the divide; 5 for the size ratios):
    db    = sum_e |Wg[g,e]| (A_ARG 2^-24 (|a_e| + kappa_c 100 / dim_k) + A_SFU 2^-21)
            + A_ACC 2^-24 (sum_e |Wg[g,e] emb_e| + |bg[g]|)
    beta  in [log(max(b - db, 0) + 1e-6), log(max(b + db, 0) + 1e-6)]  widened by A_LOG 2^-21 + 2^-24 (|beta| + 2 |s x|)
    p_hi  = e^{L_hi,m} / (e^{L_hi,m} + sum_{j != m} e^{L_lo,j})        (p_lo the mirror image, both shifted by max L)
    slack = A_EXP 2^-22 p (1 + |L_m - max L|) + output rounding (fp32 2^-24 p; fp16 2^-11 p + 2^-25;
            split-fp16 2^-23 p + 2^-25) + 2^-125 (a flushed exp)
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "oracle") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
import mega_oracle  # noqa: E402

GROUPS = 16
SCALE = 0.125                  # 1 / sqrt(64): the engines' soft-max scale (a power of two: s * x is exact)
FORMATS = ("f32", "f16", "split")
# constants of the error model (calibration: test_relation_softmax_conformance_gpu.py)
CONSTS = dict(A_ARG=2.0, A_SFU=2.0, A_ACC=16.0, A_LOG=1.0, A_EXP=2.0)

# ------------------------------------------------------------------------------------------------ dispatch
PAIRS = (
    ("plain_softmax_kernel", False),
    ("relation_softmax_kernel<true>", True),
    ("relation_softmax_kernel<false>", True),
    ("relation_softmax_kernel<false>", False),
    ("relation_softmax_pe_kernel<true>", True),
    ("relation_softmax_pe_kernel<false>", True),
    ("relation_softmax_mma_kernel<true>", True),
)
COMBOS = tuple((k, pe, f) for k, pe in PAIRS for f in FORMATS)


def dispatch(boxes, host_w, ldm, simt):
    """(kernel, position term) a call reaches. Without boxes: the one-warp-per-row kernel up to 1024 keys, else the
    two-pass CTA kernel. Device weights: the shared-memory-weight kernel, logits staged in shared memory up to 1024 keys.
    Host weights (kernel parameters): the tensor-core bias up to 1024 keys unless MEGA_B200_SOFTMAX_SIMT=1 selects the
    FFMA kernel; above 1024 keys always the global two-pass FFMA kernel."""
    if not boxes:
        return ("plain_softmax_kernel" if ldm <= 1024 else "relation_softmax_kernel<false>", False)
    stage = "true" if ldm <= 1024 else "false"
    if not host_w:
        return ("relation_softmax_kernel<%s>" % stage, True)
    if ldm > 1024:
        return ("relation_softmax_pe_kernel<false>", True)
    return ("relation_softmax_pe_kernel<true>" if simt else "relation_softmax_mma_kernel<true>", True)


# ------------------------------------------------------------------------------------------------ fp64 reference
def dim_mat_fp32():
    """the divisors 1000^(k/8) the engine passes (engine.py _Att / _alloc_attention), fp32"""
    return torch.full((8,), 1000.0).pow(8.0 / 64 * torch.arange(0, 8, dtype=torch.float32)).contiguous()


def _kappa(q, k):
    """[r, m, 4]: condition of the four log-ratios on the kernel's fp32 box arithmetic, in units of 2^-24"""
    def geo(b):
        w, h = b[:, 2] - b[:, 0] + 1, b[:, 3] - b[:, 1] + 1
        return w, h, 0.5 * (b[:, 0] + b[:, 2]), 0.5 * (b[:, 1] + b[:, 3])
    qw, qh, qcx, qcy = geo(q)
    _, _, kcx, kcy = geo(k)
    out = []
    for qc, kc, qs in ((qcx, kcx, qw), (qcy, kcy, qh)):
        u = (qc[:, None] - kc[None, :]).abs() / qs[:, None]
        out.append(((qc.abs()[:, None] + kc.abs()[None, :]) / qs[:, None] + 5 * u + 2e-3) / (u + 1e-3))
    five = torch.full_like(out[0], 5.0)
    return torch.stack(out + [five, five], 2)


def reference(x, m_valid, scale=SCALE, boxes_q=None, boxes_k=None, wg=None, bg=None, dim_mat=None, rows=32):
    """fp64 pieces of the contract over the valid keys, on x's device. x: fp32 logits [16, N, >= m_valid]. Returns a dict
    of [16, N, m_valid] tensors: sx = scale * x and, with boxes, b (the position bias before ReLU) and the three
    constant-free parts of its error bound (arg, sfu, acc). The embedding comes from mega_oracle.position_embedding
    on fp64 boxes with the given fp32 divisors, evaluated `rows` query rows at a time."""
    dev = x.device
    n = x.shape[1]
    sx = scale * x[:, :, :m_valid].double()
    out = dict(sx=sx, pe=boxes_q is not None, m_valid=m_valid)
    if boxes_q is None or m_valid == 0:
        return out
    W = wg.to(dev).double().view(GROUPS, 64)
    B = bg.to(dev).double().view(GROUPS, 1, 1)
    dm = dim_mat.to(dev)
    inv100 = 100.0 / dm.double()                                            # [8]
    Wsc = (W.abs().view(GROUPS, 4, 2, 8)).sum(2)                            # |W_sin| + |W_cos| per (coord, k)
    k = boxes_k[:m_valid].to(dev).double()
    b = torch.empty(GROUPS, n, m_valid, dtype=torch.float64, device=dev)
    arg, acc = torch.empty_like(b), torch.empty_like(b)
    for r0 in range(0, n, rows):
        q = boxes_q[r0:r0 + rows].to(dev).double()
        emb = mega_oracle.position_embedding(q, k, dim_mat=dm)              # [64, r, m]
        pm = mega_oracle.position_matrix(q, k)                              # [r, m, 4]
        a = pm.unsqueeze(3) * inv100                                        # [r, m, 4, 8] sin / cos arguments
        t = a.abs() + _kappa(q, k).unsqueeze(3) * inv100
        b[:, r0:r0 + rows] = torch.einsum("ge,erm->grm", W, emb) + B
        arg[:, r0:r0 + rows] = torch.einsum("gck,rmck->grm", Wsc, t)
        acc[:, r0:r0 + rows] = torch.einsum("ge,erm->grm", W.abs(), emb.abs()) + B.abs()
    out.update(b=b, arg=arg * 2.0 ** -24, acc=acc * 2.0 ** -24, sfu=W.abs().sum(1).view(GROUPS, 1, 1) * 2.0 ** -21)
    return out


def _log_bias(b):
    return torch.log(b.clamp_min(0) + 1e-6)


def prob_interval(ref, fmt, consts=CONSTS):
    """(p, lo, hi) [16, N, m_valid]: the fp64 probabilities and the interval an fp32 kernel's `fmt` output must lie in"""
    c = consts
    sx = ref["sx"]
    if ref["pe"] and ref["m_valid"] > 0:
        db = c["A_ARG"] * ref["arg"] + c["A_SFU"] * ref["sfu"] + c["A_ACC"] * ref["acc"]
        b = ref["b"]
        beta, beta_lo, beta_hi = _log_bias(b), _log_bias(b - db), _log_bias(b + db)
        wl = c["A_LOG"] * 2.0 ** -21 + 2.0 ** -24 * (torch.maximum(beta_lo.abs(), beta_hi.abs()) + 2 * sx.abs())
        L, L_lo, L_hi = beta + sx, beta_lo + sx - wl, beta_hi + sx + wl
    else:
        wl = 2.0 ** -24 * 2 * sx.abs()
        L, L_lo, L_hi = sx, sx - wl, sx + wl
    if L.shape[-1] == 0:
        return L, L, L
    p = torch.softmax(L, dim=-1)
    M = L_hi.amax(-1, keepdim=True)
    e_lo, e_hi = torch.exp(L_lo - M), torch.exp(L_hi - M)
    s_lo, s_hi = e_lo.sum(-1, keepdim=True), e_hi.sum(-1, keepdim=True)
    p_hi = e_hi / (e_hi + (s_lo - e_lo).clamp_min(0))
    p_lo = e_lo / (e_lo + (s_hi - e_hi).clamp_min(0))
    slack = c["A_EXP"] * 2.0 ** -22 * p_hi * (1 + (L - L.amax(-1, keepdim=True)).abs()) + 2.0 ** -125
    if fmt == "f16":
        slack = slack + 2.0 ** -11 * p_hi + 2.0 ** -25
    elif fmt == "split":
        slack = slack + 2.0 ** -23 * p_hi + 2.0 ** -25
    else:
        slack = slack + 2.0 ** -24 * p_hi
    return p, p_lo - slack, p_hi + slack


def interval_check(got, ref, fmt, consts=CONSTS):
    """boolean [16, N, m_valid]: got (the valid-key part of an output) inside its interval"""
    _, lo, hi = prob_interval(ref, fmt, consts)
    g = got.double()
    return (g >= lo) & (g <= hi)


def needed_constants(got, ref, fmt, consts=CONSTS, steps=8):
    """for each constant, the smallest value (others as given, bisected to 2^-steps of it) the output still passes with:
    what the measurement asks of that constant"""
    out = {}
    keys = list(consts) if ref["pe"] else ["A_EXP"]
    for name in keys:
        lo_t, hi_t = 0.0, 1.0
        if bool(interval_check(got, ref, fmt, dict(consts, **{name: 0.0})).all()):
            out[name] = 0.0
            continue
        for _ in range(steps):
            mid = 0.5 * (lo_t + hi_t)
            if bool(interval_check(got, ref, fmt, dict(consts, **{name: mid * consts[name]})).all()):
                hi_t = mid
            else:
                lo_t = mid
        out[name] = hi_t * consts[name]
    return out


# ------------------------------------------------------------------------------------------------ case table
def _boxes(n, g, style, w=1000.0, h=600.0):
    xy = torch.rand(n, 2, generator=g) * torch.tensor([w * 0.9, h * 0.9])
    wh = torch.rand(n, 2, generator=g) * 256.0 + 4.0
    b = torch.cat([xy, xy + wh], 1)
    b[:, 0::2].clamp_(0, w - 1)
    b[:, 1::2].clamp_(0, h - 1)
    if style == "edge" and n >= 8:
        i = torch.arange(n)
        b[i % 8 == 1, 2] = b[i % 8 == 1, 0]                                  # width 1
        b[i % 8 == 1, 3] = b[i % 8 == 1, 1]                                  # height 1
        b[i % 8 == 3] = torch.tensor([0.0, 0.0, 0.0, 0.0])                   # 1 x 1 in a corner: |dx / w| ~ 1e3
        b[i % 8 == 5] = torch.tensor([0.0, 0.0, w - 1, h - 1])               # whole image: width ratio ~1e3
        b[i % 8 == 6, 2] = b[i % 8 == 6, 0] + 0.5                            # sub-pixel
    return b


def build_inputs(c):
    """CPU tensors of case `c`: logits x [16, N, ldm] (padded keys hold 123), boxes, Wg [16, 64], bg [16], divisors"""
    g = torch.Generator().manual_seed(c["seed"])
    n, ldm, mk = c["n"], c["ldm"], c["keys"]
    x = torch.randn(GROUPS, n, ldm, generator=g) * {"normal": 8.0, "wide": 400.0}[c["logits"]]
    if c["logits"] == "wide":
        x[:, 0, :] *= 0.02
        x[:, 0, min(3, ldm - 1)] = 3000.0                                  # row 0: one dominant key
    x[:, :, mk:] = 123.0
    inp = dict(x=x.contiguous(), dim_mat=dim_mat_fp32())
    if not c["boxes"]:
        return inp
    bq = _boxes(n, g, c["box"])
    bk = _boxes(max(mk, 1), g, c["box"])                                     # (a key tensor even for 0 valid keys)
    if c["box"] == "edge":
        nn_ = min(n, mk) // 4
        bk[:nn_] = bq[:nn_]                                                  # identical query and key: argument -690 rad
    wg = torch.randn(GROUPS, 64, generator=g) * 0.02                         # the reference initialises Wg with std 0.01
    bg = torch.rand(GROUPS, generator=g) * 0.8 + 0.2
    bg[12] = 0.0                                                             # straddles the kink
    bg[15] = -10.0                                                           # entirely below the ReLU
    if mk:
        e0 = mega_oracle.position_embedding(bq[:1].double(), bk[:2].double(), dim_mat=inp["dim_mat"])[:, 0]   # [64, <= 2]
        for h, j in ((13, 0), (14, 1)):                                      # exactly at the kink for one pair
            bg[h] = float(-(wg[h].double() @ e0[:, min(j, e0.shape[1] - 1)]))
    inp.update(boxes_q=bq.contiguous(), boxes_k=bk.contiguous(), wg=wg.contiguous(), bg=bg.contiguous())
    return inp


def _case(cid, n, ldm, keys, *, boxes=True, host_w=True, simt=False, m=None, m_dev=True, n_valid=None, logits="normal",
          box="random", seed):
    """keys: rows of key boxes / valid logit columns built; m: the key count passed (default keys; through the device
    pointer when m_dev, which the kernel clamps to ldm, else as m_host)"""
    m = keys if m is None else m
    c = dict(id=cid, n=n, ldm=ldm, keys=keys, boxes=boxes, host_w=host_w and boxes, simt=simt, m=m, m_dev=m_dev,
             n_valid=n_valid, logits=logits, box=box, seed=seed)
    c["m_valid"] = min(m, ldm)
    assert keys >= c["m_valid"] and keys <= ldm, cid
    c["kernel"], c["pe"] = dispatch(boxes, c["host_w"], ldm, simt)
    return c


def make_cases():
    """the committed case table (fixed seeds: every case is reproducible)"""
    C = []
    add = lambda *a, **k: C.append(_case(*a, **k))
    # MEGA global stage G: 2175 query rows x 750 keys, no position term (plain kernel)
    add("mega_g_2175x768", 2175, 768, 750, boxes=False, seed=11)
    # MEGA local stage 0: 675 x 3776, 1875 + memory keys from the device, key-frame padding rows (FFMA two-pass kernel)
    add("mega_l0_675x3776", 675, 3776, 3137, n_valid=(287, 300), logits="wide", box="edge", seed=12)
    # MEGA local stages 1 / 2 (tensor-core bias)
    add("mega_l1_675x768", 675, 768, 700, n_valid=(150, 300), box="edge", seed=13)
    add("mega_l2_300x768", 300, 768, 768, m=767, m_dev=False, logits="wide", seed=14)
    # RDN: advanced stage 555 x 2784 (2775 refs), base stages 300 x 2784, distilled 300 x 576
    add("rdn_adv_555x2784", 555, 2784, 2775, m_dev=False, box="edge", seed=15)
    add("rdn_base_300x2784_nv_all", 300, 2784, 2775, n_valid=(300, 300), seed=16)
    add("rdn_att3_300x576", 300, 576, 555, n_valid=(0, 300), seed=17)
    add("rdn_att3_300x576_nv", 300, 576, 555, n_valid=(211, 300), logits="wide", box="edge", seed=18)
    # odd small shapes
    add("pe_9x1500x1504_m_ldm", 9, 1504, 1504, m_dev=False, box="edge", seed=19)
    add("pe_9x1504_m_over", 9, 1504, 1504, m=5000, box="edge", seed=20)
    add("mma_37x203x224", 37, 224, 203, box="edge", logits="wide", seed=21)
    add("mma_37x224_m0", 37, 224, 0, m_dev=False, seed=22)
    add("mma_37x224_m1", 37, 224, 1, seed=23)
    add("pe_9x1504_m0", 9, 1504, 0, seed=24)
    add("pe_9x1504_m31", 9, 1504, 31, m_dev=False, seed=25)
    # device weights (shared-memory weight kernel)
    add("devw_37x203x224", 37, 224, 203, host_w=False, box="edge", seed=31)
    add("devw_37x224_m33", 37, 224, 33, host_w=False, m_dev=False, n_valid=(20, 30), seed=32)
    add("devw_37x224_m_over", 37, 224, 224, host_w=False, m=999, logits="wide", seed=33)
    add("devw_9x1500x1504", 9, 1504, 1500, host_w=False, box="edge", seed=34)
    add("devw_200x3776_m_ldm", 200, 3776, 3776, host_w=False, m_dev=False, logits="wide", seed=35)
    add("devw_9x1504_m0", 9, 1504, 0, host_w=False, seed=36)
    # no position term
    add("plain_37x224_m0", 37, 224, 0, boxes=False, m_dev=False, seed=41)
    add("plain_37x224_m1", 37, 224, 1, boxes=False, seed=42)
    add("plain_37x224_m31_nv0", 37, 224, 31, boxes=False, m_dev=False, n_valid=(0, 20), seed=43)
    add("plain_37x224_m_over", 37, 224, 224, boxes=False, m=300, logits="wide", seed=44)
    add("plain_1024_m1023", 40, 1024, 1023, boxes=False, m_dev=False, seed=45)
    add("nope_9x1500x1504", 9, 1504, 1500, boxes=False, logits="wide", seed=46)
    add("nope_300x2784_m33", 300, 2784, 33, boxes=False, n_valid=(100, 300), seed=47)
    add("nope_9x1504_m0", 9, 1504, 0, boxes=False, seed=48)
    add("nope_200x3776_m_ldm", 200, 3776, 3776, boxes=False, m_dev=False, seed=49)
    # MEGA_B200_SOFTMAX_SIMT=1 (FFMA kernels with the weights in the kernel parameters)
    add("simt_37x203x224", 37, 224, 203, simt=True, box="edge", logits="wide", seed=51)
    add("simt_675x768", 675, 768, 750, simt=True, n_valid=(150, 300), seed=52)
    add("simt_37x224_m0", 37, 224, 0, simt=True, m_dev=False, seed=53)
    add("simt_37x224_m_over", 37, 224, 224, simt=True, m=300, seed=54)
    add("simt_9x1500x1504", 9, 1504, 1500, simt=True, box="edge", seed=55)
    return C


def live_rows(c):
    """query rows the kernel computes (rows in [n_valid, n_valid_off) are padding it skips)"""
    rows = torch.ones(c["n"], dtype=torch.bool)
    if c["n_valid"] is not None:
        nv, off = c["n_valid"]
        rows[nv:off] = False
    return rows
