"""Query rows at and past the key count the host-weight soft-max can stage in the shared memory of its 2-CTA cluster
(ops.RELATION_PE_MAX_KEYS, csrc/relation.cu kPairMaxLdm): at the limit the cluster kernel runs; past it ops.relation_softmax
takes the device-weight entry points (the same bits as calling them directly), and the host-weight C entry points reject
the call without touching the logits."""
import pytest
import torch

from relation_softmax_ref import GROUPS, SCALE, _case, build_inputs

pytestmark = pytest.mark.gpu


def _setup(dev, n, ldm, keys, seed):
    inp = build_inputs(_case("wide", n, ldm, keys, seed=seed))
    s = inp["x"].to(dev).contiguous()
    kw = dict(m_host=keys, boxes_q=inp["boxes_q"].to(dev), boxes_k=inp["boxes_k"].to(dev))
    host_w = (inp["wg"], inp["bg"], inp["dim_mat"])
    dev_w = dict(wg=inp["wg"].to(dev), bg=inp["bg"].to(dev), dim_mat=inp["dim_mat"].to(dev))
    return s, kw, host_w, dev_w


def _check_probs(p, keys):
    assert bool(torch.isfinite(p).all())
    assert bool((p[..., keys:] == 0).all())
    assert torch.allclose(p[..., :keys].double().sum(-1), torch.ones((), dtype=torch.float64), atol=1e-4)


@pytest.mark.parametrize("fmt", ["f32", "split"])
def test_at_the_limit_the_cluster_kernel_runs(cuda_dev, fmt):
    from mega_core.b200 import ops
    n, ldm, keys = 3, ops.RELATION_PE_MAX_KEYS, ops.RELATION_PE_MAX_KEYS - 7
    s, kw, host_w, _ = _setup(cuda_dev, n, ldm, keys, seed=61)
    p = ops.mark_split16(torch.zeros(GROUPS, n, ldm, device=cuda_dev)) if fmt == "split" else None
    ops.relation_softmax(s, n, ldm, SCALE, probs_f16=p, host_w=host_w, **kw)
    torch.cuda.synchronize()
    _check_probs(s if p is None else ops.split16_decode(p), keys)


@pytest.mark.parametrize("fmt", ["f32", "split"])
def test_past_the_limit_rows_take_the_device_weight_kernel(cuda_dev, fmt):
    from mega_core.b200 import ops
    n, ldm, keys = 3, ops.RELATION_PE_MAX_KEYS + 32, ops.RELATION_PE_MAX_KEYS + 20
    s, kw, host_w, dev_w = _setup(cuda_dev, n, ldm, keys, seed=62)
    outs = []
    for hw in (host_w, None):
        x = s.clone()
        p = ops.mark_split16(torch.zeros(GROUPS, n, ldm, device=cuda_dev)) if fmt == "split" else None
        ops.relation_softmax(x, n, ldm, SCALE, probs_f16=p, host_w=hw, **dev_w, **kw)
        torch.cuda.synchronize()
        outs.append(x if p is None else p)
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32))
    _check_probs(outs[0] if fmt == "f32" else ops.split16_decode(outs[0]), keys)


def test_host_weight_entry_rejects_rows_past_the_limit(cuda_dev):
    from mega_core._lib import MegaError, check, lib, ptr, stream_ptr
    from mega_core.b200 import ops
    n, ldm, keys = 2, ops.RELATION_PE_MAX_KEYS + 32, ops.RELATION_PE_MAX_KEYS + 32
    s, kw, host_w, _ = _setup(cuda_dev, n, ldm, keys, seed=63)
    before = s.clone()
    wg, bg, dm = host_w
    with pytest.raises(MegaError):
        check(lib.mega_relation_softmax_pe(ptr(s), None, n, ldm, ptr(kw["boxes_q"]), ptr(kw["boxes_k"]), ptr(wg), ptr(bg),
                                           ptr(dm), None, keys, None, 0, SCALE, stream_ptr()), "relation_softmax_pe")
    torch.cuda.synchronize()
    assert torch.equal(s.view(torch.int32), before.view(torch.int32))
    assert lib.mega_device_ok() == 1
