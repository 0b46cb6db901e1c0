"""GPU diagnostic: engine (TF32 kernels) and engine with the fp32 GEMM shadow vs the reference fixture /
the oracle, at several probe points. Writes gpurun_out/diag_parity.json."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "mega.pytorch_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import mega_oracle as mo  # noqa: E402
from fp32_shadow import fp32_shadow  # noqa: E402
from mega_core.b200 import engine, synth  # noqa: E402

dev = torch.device("cuda:0")
gold = torch.load(os.path.join(ROOT, "tests", "golden", "mega_r101_192x320.pt"))
h, w, total = gold["h"], gold["w"], gold["total"]
sd = synth.make_state_dict(gold["arch"], seed=gold["seed"])
frames = [synth.synthetic_frame(i, h, w) for i in range(total)]
dframes = [f.to(dev) for f in frames]
gpf = gold["globals_per_frame"]
orc = mo.MegaOracle(sd, mo.Cfg(cuda_nms_semantics=True), record=True)
traces = []
for t in range(3):
    infos = {"frame_category": 0 if t == 0 else 1, "ref_l": frames[1:13] if t == 0 else [frames[min(t + 12, total - 1)]],
             "ref_g": [frames[j] for j in gpf[t]]}
    orc.forward(frames[t], infos)
    traces.append({k: v.clone() for k, v in orc.trace.items()})


def match(a, b, tol=0.75):
    d = (a[:, None, :] - b[None, :, :]).abs().amax(2)
    val, idx = d.min(0)
    idx[val > tol] = -1
    return idx


def run(label, ctx, precision="tf32"):
    out = []
    with ctx:
        eng = engine.MegaEngine(sd, engine.EngineConfig(precision=precision), device=dev)
        for t in range(3):
            if t == 0:
                eng.start_video(dframes[0], dframes[1:13], [dframes[j] for j in gpf[0]], w, h)
            else:
                eng.step(dframes[min(t + 12, total - 1)], dframes[gpf[t][0]], w, h)
            torch.cuda.synchronize()
            tr = traces[t]
            k = int(eng.cur_cnt.view(-1)[0].item())
            props = eng.Bq0[:k].cpu()
            idx = match(props, tr["proposals"])
            m = idx >= 0
            kslot = list(eng.win_slots)[eng.cfg.key_frame_location]
            xfc = eng.win_x[kslot * eng.KP: kslot * eng.KP + k].cpu()
            pred = eng.last_pred[:k].cpu()
            x4 = eng.X4[:k].cpu()
            rec = {"frame": t, "k": k, "k_ref": int(tr["proposals"].shape[0]), "matched": m.float().mean().item(),
                   "prop_maxdiff_matched": (props[idx[m]] - tr["proposals"][m]).abs().max().item(),
                   "x_key_fc_err": (xfc[idx[m]] - tr["x_key_fc"][m]).abs().max().item(),
                   "x_key_fc_rms": tr["x_key_fc"].pow(2).mean().sqrt().item(),
                   "x_final_err": (x4[idx[m]] - tr["x_final"][m]).abs().max().item(),
                   "x_final_rms": tr["x_final"].pow(2).mean().sqrt().item(),
                   "logits_err": (pred[idx[m], :31] - tr["class_logits"][m]).abs().max().item(),
                   "logits_rms": tr["class_logits"].pow(2).mean().sqrt().item()}
            out.append(rec)
            print(label, rec)
    return out


import contextlib  # noqa: E402
from mega_core.b200 import ops  # noqa: E402
import fp32_shadow as _fs  # noqa: E402


def per_gemm_audit():
    """strict mode: run every conv_gemm of two frames twice -- wgmma 3xTF32 and the fp64 shadow on the SAME
    inputs -- and report the worst relative error with the call's signature"""
    worst = []
    real = ops.conv_gemm

    def audited(a, w, out, **kw):
        res = kw.get("residual")
        res_copy = res.clone() if res is not None else None
        real(a, w, out, **kw)
        got = out.clone()
        if res is not None and res.data_ptr() == out.data_ptr():
            kw = dict(kw)
            kw["residual"] = res_copy
        ref = torch.zeros_like(out)
        ref.copy_(got)
        _fs._shadow_conv_gemm(a, w, ref, **kw)
        cout = kw.get("cout") or w.shape[1]
        if kw.get("out_c_off"):
            width = cout + (kw.get("batch", 1) - 1) * kw["out_c_off"]
        else:
            width = cout
        d = (got[..., :width] - ref[..., :width]).abs().max().item()
        r = ref[..., :width].pow(2).mean().sqrt().item()
        worst.append((d / max(r, 1e-20), tuple(a.shape), tuple(w.shape), {k: v for k, v in kw.items()
                                                                            if k in ("taps", "dil", "batch", "k", "cout", "block_n")}))
        out.copy_(got)
        return out

    ops.conv_gemm = audited
    try:
        eng = engine.MegaEngine(sd, engine.EngineConfig(precision="fp32x3"), device=dev)
        eng.start_video(dframes[0], dframes[1:13], [dframes[j] for j in gpf[0]], w, h)
        eng.step(dframes[13], dframes[gpf[1][0]], w, h)
        torch.cuda.synchronize()
    finally:
        ops.conv_gemm = real
    worst.sort(key=lambda t: -t[0])
    for t in worst[:12]:
        print("AUDIT", "%.3e" % t[0], t[1], t[2], t[3])
    return [[t[0], str(t[1]), str(t[2]), str(t[3])] for t in worst[:12]]

audit = per_gemm_audit()
res = {"gemm_audit_fp32x3": audit, "fp32x3": run("fp32x3", contextlib.nullcontext(), "fp32x3"), "tf32": run("tf32", contextlib.nullcontext()),
       "fp32_shadow": run("fp32", fp32_shadow())}
os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
json.dump(res, open(os.path.join(ROOT, "gpurun_out", "diag_parity.json"), "w"), indent=1)
