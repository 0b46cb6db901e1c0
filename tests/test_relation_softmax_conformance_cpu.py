"""CPU half of the relation soft-max conformance suite: the fp64 reference and interval of
test_relation_softmax_conformance_gpu.py against the reference model's own fp32 forward (mega_oracle, as the GPU parity
tests build it), the sharpness of the interval, mutations of that forward it must reject, and the restated dispatch
rule against the kernel source."""
import os
import re

import pytest
import torch

from relation_softmax_ref import (COMBOS, CONSTS, FORMATS, GROUPS, PAIRS, SCALE, build_inputs, dispatch,
                                  interval_check, live_rows, make_cases, mega_oracle, prob_interval, reference)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = {c["id"]: c for c in make_cases()}
# CPU-sized cases of the table: the tensor-core, shared-memory-weight and plain geometries with edge boxes and wide logits
FIXTURES = ["mma_37x203x224", "devw_37x203x224", "simt_37x203x224", "devw_37x224_m33", "plain_37x224_m_over"]


def _pm(bq, bk, plus=1.0):
    """position_matrix with the box-width offset as a parameter (plus=1 is mega_oracle.position_matrix)"""
    def geo(b):
        return (b[:, 2] - b[:, 0] + plus, b[:, 3] - b[:, 1] + plus, 0.5 * (b[:, 0] + b[:, 2]), 0.5 * (b[:, 1] + b[:, 3]))
    qw, qh, qcx, qcy = geo(bq)
    kw, kh, kcx, kcy = geo(bk)
    dx = (((qcx[:, None] - kcx[None, :]) / qw[:, None]).abs() + 1e-3).log()
    dy = (((qcy[:, None] - kcy[None, :]) / qh[:, None]).abs() + 1e-3).log()
    return torch.stack([dx, dy, (qw[:, None] / kw[None, :]).log(), (qh[:, None] / kh[None, :]).log()], 2)


def fp32_forward(c, inp, *, mutate=None):
    """the reference model's forward in fp32 (mega_oracle's embedding, Wg projection, ReLU, log(. + 1e-6), soft-max over
    the valid keys), written as the kernels' contract output [16, N, ldm]; `mutate` names a deliberate bug"""
    x, n, ldm, mv = inp["x"], c["n"], c["ldm"], c["m_valid"]
    if mutate == "m_valid_off_by_one":
        mv = mv - 1 if mv > 1 else mv + 1
    out = torch.zeros(GROUPS, n, ldm)
    if mv == 0:
        return out
    aff = x[:, :, :mv] * SCALE
    if c["boxes"]:
        bq, bk, wg, bg = inp["boxes_q"], inp["boxes_k"][:mv], inp["wg"], inp["bg"]
        if mutate == "key_boxes_off_by_one_row":
            bk = inp["boxes_k"][1:mv + 1] if inp["boxes_k"].shape[0] > mv else torch.roll(bk, 1, 0)
        if mutate == "heads_swapped":
            wg, bg = wg[[1, 0] + list(range(2, GROUPS))], bg[[1, 0] + list(range(2, GROUPS))]
        if mutate == "width_without_plus_one":
            pm = _pm(bq, bk, plus=0.0)
            div = pm.unsqueeze(3) * 100.0 / inp["dim_mat"].view(1, 1, 1, -1)
            pe = torch.cat([div.sin(), div.cos()], 3).reshape(bq.shape[0], bk.shape[0], 64).permute(2, 0, 1)
        else:
            pe = mega_oracle.position_embedding(bq, bk)                                     # [64, n, mv]
        w = torch.relu(torch.einsum("ge,enm->gnm", wg, pe) + bg.view(GROUPS, 1, 1))
        eps = 0.0 if mutate == "no_1e-6" else 1e-6
        aff = (w + eps).log() + aff
    p = torch.softmax(aff, dim=2)
    if mutate == "top_key_dropped":
        j = p[0, 0].argmax()
        rest = 1.0 - p[0, 0, j]
        p[0, 0, j] = 0.0
        p[0, 0] /= rest
    out[:, :, :mv] = p
    return out


def _ref(c, inp):
    return reference(inp["x"], c["m_valid"], SCALE, inp.get("boxes_q"), inp.get("boxes_k"), inp.get("wg"),
                     inp.get("bg"), inp["dim_mat"])


def _passes(c, inp, ref, got, fmt="f32"):
    live = live_rows(c)
    mv = c["m_valid"]
    ok = interval_check(got[:, :, :mv], ref, fmt)[:, live]
    return bool(ok.all()) and bool((got[:, live, mv:] == 0).all())


@pytest.fixture(scope="module")
def fixtures():
    out = {}
    for cid in FIXTURES:
        c = CASES[cid]
        inp = build_inputs(c)
        out[cid] = (c, inp, _ref(c, inp))
    return out


def test_position_matrix_restatement_is_the_oracle():
    c = CASES["mma_37x203x224"]
    inp = build_inputs(c)
    assert torch.equal(_pm(inp["boxes_q"], inp["boxes_k"]), mega_oracle.position_matrix(inp["boxes_q"], inp["boxes_k"]))


def test_dim_mat_argument_matches_the_oracle_default():
    c = CASES["mma_37x203x224"]
    inp = build_inputs(c)
    bq, bk = inp["boxes_q"][:5].double(), inp["boxes_k"][:7].double()
    assert torch.equal(mega_oracle.position_embedding(bq, bk), mega_oracle.position_embedding(bq, bk, dim_mat=inp["dim_mat"]))


@pytest.mark.parametrize("cid", FIXTURES)
@pytest.mark.parametrize("fmt", FORMATS)
def test_fp32_oracle_forward_passes_the_bound(fixtures, cid, fmt):
    c, inp, ref = fixtures[cid]
    got = fp32_forward(c, inp)
    if fmt == "f16":
        got = got.half().float()
    elif fmt == "split":
        hi = got.half()
        got = hi.float() + (got - hi.float()).half().float()
    assert _passes(c, inp, ref, got, fmt)


def test_fp64_probabilities_inside_their_interval(fixtures):
    for c, inp, ref in fixtures.values():
        for fmt in FORMATS:
            p, lo, hi = prob_interval(ref, fmt)
            assert bool(((lo <= p) & (p <= hi)).all()), (c["id"], fmt)
            if c["m_valid"]:
                assert torch.allclose(p.sum(-1), torch.ones(()).double(), atol=1e-12)


def test_bound_is_sharp(fixtures):
    """on well-conditioned elements (b - db > 1e-4) the interval's relative width has a median <= 4e-4. Most of the width
    is the fp32 rounding of sin / cos arguments of up to ~700 rad (2^-24 |a_e| ~ 4e-5 rad each), summed over the 64
    features without cancellation; the mutation tests below show it still rejects the bugs it is meant to catch."""
    widths = []
    for c, inp, ref in fixtures.values():
        if not ref["pe"] or not c["m_valid"]:
            continue
        db = CONSTS["A_ARG"] * ref["arg"] + CONSTS["A_SFU"] * ref["sfu"] + CONSTS["A_ACC"] * ref["acc"]
        p, lo, hi = prob_interval(ref, "f32")
        well = (ref["b"] - db > 1e-4) & (p > 1e-30)
        widths.append(((hi - lo) / p)[well])
    w = torch.cat(widths)
    assert w.numel() > 10000
    assert w.median().item() <= 4e-4, w.median().item()


MUTATIONS = ["top_key_dropped", "key_boxes_off_by_one_row", "heads_swapped", "m_valid_off_by_one",
             "width_without_plus_one", "no_1e-6"]


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_mutations_are_rejected(fixtures, mutation):
    """every fixture with a position term (and, for the key-count / dropped-key bugs, every fixture) rejects the bug"""
    tried = 0
    for c, inp, ref in fixtures.values():
        if mutation not in ("top_key_dropped", "m_valid_off_by_one") and not c["boxes"]:
            continue
        got = fp32_forward(c, inp, mutate=mutation)
        assert not _passes(c, inp, ref, got), "%s: %s passes the bound" % (c["id"], mutation)
        tried += 1
    assert tried >= 3


def test_case_table_covers_every_combination():
    cases = list(CASES.values())
    assert len(COMBOS) == 21 and len(set(PAIRS)) == 7
    for c in cases:
        assert (c["kernel"], c["pe"]) == dispatch(c["boxes"], c["host_w"], c["ldm"], c["simt"])
        assert c["ldm"] % 32 == 0 and c["m_valid"] <= c["keys"] <= c["ldm"]
    covered = {(c["kernel"], c["pe"], f) for c in cases for f in FORMATS}
    assert covered == set(COMBOS)
    # the edges the table promises
    mvs = {(c["m_valid"], c["m_dev"]) for c in cases}
    for m in (0, 1, 31, 33):
        assert any(mv == m for mv, _ in mvs), m
    assert any(c["m_valid"] == c["ldm"] - 1 for c in cases) and any(c["m_valid"] == c["ldm"] and not c["m_dev"] for c in cases)
    assert any(c["m_dev"] and c["m"] > c["ldm"] for c in cases)
    assert any(c["m_dev"] and 0 < c["m"] < c["ldm"] - 31 for c in cases)                       # ragged device count
    nvs = [c["n_valid"] for c in cases if c["n_valid"]]
    assert any(nv == 0 for nv, _ in nvs) and any(0 < nv < off for nv, off in nvs) and any(nv >= off for nv, off in nvs)
    geoms = {(c["n"], c["ldm"]) for c in cases}
    for gm in ((2175, 768), (675, 3776), (675, 768), (300, 768), (555, 2784), (300, 2784), (300, 576), (9, 1504),
               (37, 224)):
        assert gm in geoms, gm


def test_dispatch_restatement_matches_the_source():
    """the kernels relation.cu launches are exactly the seven of the table"""
    src = open(os.path.join(ROOT, "mega.pytorch_b200", "csrc", "relation.cu")).read()
    launched = set(re.findall(r"(\w+softmax\w*kernel(?:<(?:true|false)>)?)<<<", src))
    assert launched == {k for k, _ in PAIRS}, launched
    assert "use_mma > 1" not in src
