"""Helpers shared by the DyMN test files: synthetic inputs, the BatchNorm calibration and the training step of the fp64
oracle (oracle/net_oracle.py), the engine's training step, and the per-tensor comparison of a step's gradients with the
oracle's under the bounds of each GEMM route."""
import contextlib

import torch
import torch.nn.functional as Fn

from oracle import net_oracle
from tests.util import build_model, report

WIDTH = {"dymn04": 0.4, "dymn10": 1.0}

# route -> (gemm, dyn_tma_min_rps) and the bounds on every gradient tensor: (relative L2, relative error of the norm) for
# the attention-logit layers (`*.residuals.0.*`) and for all other tensors, and the logits' max-abs error
TRAIN_ROUTES = {"simt": ("simt", None), "auto_tma": ("auto", 0), "auto_reg": ("auto", 10 ** 9)}
BOUNDS = {"simt": dict(res=(2e-2, 1e-2), other=(1e-2, 2e-3), logits=5e-5),
          "auto_tma": dict(res=(0.25, 0.2), other=(0.15, 3e-2), logits=5e-4),
          "auto_reg": dict(res=(0.25, 0.2), other=(0.15, 3e-2), logits=5e-4)}


def conv_ps(x, w, k, s):
    """x [B, F, T, C], w [B, k*k, C] -> per-sample depthwise conv (DynamicConv's per-sample tables), NHWC out"""
    B, F, T, C = x.shape
    wc = w.permute(0, 2, 1).reshape(B * C, 1, k, k)
    y = Fn.conv2d(x.permute(0, 3, 1, 2).reshape(1, B * C, F, T), wc, None, s, (k - 1) // 2, 1, B * C)
    return y.view(B, C, y.shape[2], y.shape[3]).permute(0, 2, 3, 1)


def train_inputs(B, frames):
    """(spec [B, 1, 128, frames] fp32 CPU, labels [B, 527]) from the seeds of tests/golden/make_golden.py"""
    from efficientat_b200.synth import synth_labels, synth_waveform
    spec = synth_waveform(B, 128 * frames, seed=21, std=0.7).view(B, 1, 128, frames)
    return spec, synth_labels(B, 527, seed=5)


def temperature(tag):
    return float(build_model(tag).layers[0].depth_conv.temperature)


def calibrate(sd, spec, width, temp):
    """the running statistics of one training-mode oracle pass with momentum 1 over spec (as tests/golden/make_golden.py
    calibrates the golden state): on these clips the eval network then does not saturate.  Runs in spec's dtype and
    device; sd is not changed"""
    cal = {k: v.clone() for k, v in sd.items()}
    mom = net_oracle.BN_MOM
    try:
        net_oracle.BN_MOM = 1.0
        with torch.no_grad():
            net_oracle.dymn_forward(cal, spec, width_mult=width, training=True, temperature=temp)
    finally:
        net_oracle.BN_MOM = mom
    return {k: v for k, v in cal.items() if k.endswith(("running_mean", "running_var"))}


@contextlib.contextmanager
def exact_fp32():
    """plain fp32 in cuDNN convolutions and cuBLAS matmuls (no TF32): the reference's own arithmetic"""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def oracle_step(tag, temp, spec, y, device="cpu", with_eval=True, dtype=torch.float64):
    """oracle training step (autograd) on device: loss, logits, gradients, BatchNorm buffers after the step; with
    with_eval the eval logits under buffers calibrated on spec.  Results on the CPU.  dtype float64: the reference every
    engine result is checked against; float32 (under exact_fp32): plain fp32 torch, whose distance from float64 measures
    how much this state and batch amplify fp32 rounding"""
    model = build_model(tag)
    params = {k for k, _ in model.named_parameters()}
    sd0 = {k: (v.to(dtype) if v.is_floating_point() else v).to(device).clone() for k, v in model.state_dict().items()}
    x = spec.to(dtype).to(device)
    out = {}
    if with_eval:
        cal = calibrate(sd0, x, WIDTH[tag], temp)
        with torch.no_grad():
            ev, _ = net_oracle.dymn_forward({**sd0, **cal}, x, width_mult=WIDTH[tag], temperature=temp)
        out.update(eval_logits=ev.cpu(), cal={k: v.cpu() for k, v in cal.items()})
    sd = {k: v.clone() for k, v in sd0.items()}
    for k in params:
        sd[k].requires_grad_(True)
    logits, _ = net_oracle.dymn_forward(sd, x, width_mult=WIDTH[tag], training=True, temperature=temp)
    loss = Fn.binary_cross_entropy_with_logits(logits, y.to(dtype).to(device))
    loss.backward()
    out.update(loss=loss.item(), logits=logits.detach().double().cpu(),
               grads={k: sd[k].grad.detach().double().cpu() for k in params},
               buffers={k: v.detach().double().cpu() for k, v in sd.items() if k.endswith(("running_mean", "running_var"))})
    return out


def engine_step(tag, precision, gemm, spec, y, dyn_tma_min_rps=None):
    """one training step of the engine, dropout off -> (model with .grad set, loss, logits fp64 CPU)"""
    model = build_model(tag, precision=precision).cuda().train()
    eng = model.engine()
    eng.gemm_impl = gemm
    if dyn_tma_min_rps is not None:
        eng.dyn_tma_min_rps = dyn_tma_min_rps
    model.classifier[4].p = 0.0
    eng.dropout_p = 0.0
    logits, _ = model(spec.cuda())
    loss = Fn.binary_cross_entropy_with_logits(logits, y.cuda())
    loss.backward()
    return model, loss.item(), logits.detach().double().cpu()


def grads_of(model):
    return {n: p.grad.detach().double().cpu() for n, p in model.named_parameters()}


def grad_errors(grads, ref):
    """per-tensor relative L2 of every gradient against the oracle; tensors whose fp64 gradient is analytically zero
    (BatchNorm biases whose constant shift the next training-mode BatchNorm removes: below 1e-9 of the whole gradient's
    norm) are measured against the whole gradient's norm instead"""
    total = torch.sqrt(sum((g * g).sum() for g in ref["grads"].values())).item()
    rel, zero, norm = {}, {}, {}
    for n, g in grads.items():
        r = ref["grads"][n]
        e = (g - r).norm().item()
        if r.norm().item() <= 1e-9 * total:
            zero[n] = e / total
        else:
            rel[n] = e / r.norm().item()
            norm[n] = abs(g.norm().item() - r.norm().item()) / r.norm().item()
    return rel, zero, norm


# Caps on the bounds that plain fp32's own error widens (check_train_step with fp32 runs): a gradient that is zeroed or
# unrelated to the right one is >= 1 relative L2 off, and a logit read for the wrong sample is off by O(0.1-1)
CAP_REL, CAP_LOGITS = 0.5, 3e-2


def _step_errors(loss, logits, grads, buffers, ref):
    rel, zero, norm = grad_errors(grads, ref)
    berr = max(((buffers[k].double().cpu() - v).abs().max().item() / max(1.0, v.abs().max().item()))
               for k, v in ref["buffers"].items())
    return dict(loss=abs(loss - ref["loss"]), logits=(logits - ref["logits"]).abs().amax(1), rel=rel, zero=zero,
                norm=norm, buffers=berr)


def _fp32_errors(runs, ref):
    """per quantity, the larger error of the plain fp32 runs (each sums in its own order, and one order can be 50x
    luckier than another on a tensor); the norm's conditioning is the tensor's relative L2, which bounds it"""
    es = [_step_errors(r["loss"], r["logits"], r["grads"], r["buffers"], ref) for r in runs]
    z = {q: max(e[q] for e in es) for q in ("loss", "buffers")}
    z["logits"] = torch.stack([e["logits"] for e in es]).amax(0)
    z["rel"] = {n: max(e["rel"].get(n, 0.0) for e in es) for n in es[0]["rel"]}
    return z


def step_bounds(route, ref, fp32=(), k=0.0):
    """the bounds check_train_step applies: BOUNDS[route] (the logits' per sample), each raised by k times plain fp32's
    own error on the same quantity when fp32 runs are given, and then capped at CAP_REL / CAP_LOGITS.  -> dict(rel={name:
    (relative L2, norm)}, logits [B], loss, buffers, capped=[names])"""
    z = _fp32_errors(fp32, ref) if fp32 else dict(loss=0.0, logits=torch.zeros(ref["logits"].shape[0],
                                                                                dtype=torch.float64), rel={}, buffers=0.0)
    bd = BOUNDS[route]
    out = dict(rel={}, capped=[], loss=1e-5 * max(1.0, abs(ref["loss"])) + k * z["loss"],
               buffers=1e-5 + k * z["buffers"], logits=bd["logits"] + k * z["logits"], z=z)
    for n, r in ref["grads"].items():
        brel, bnorm = bd["res" if ".residuals." in n else "other"]
        zn = k * z["rel"].get(n, 0.0)
        if fp32 and max(brel, bnorm) + zn > CAP_REL:
            out["capped"].append(n)
        out["rel"][n] = (min(brel + zn, CAP_REL), min(bnorm + zn, CAP_REL)) if fp32 else (brel, bnorm)
    if fp32:
        out["logits"] = out["logits"].clamp(max=CAP_LOGITS)
    return out


def defect_margin(bounds, grads, logits, ref):
    """how far a planted defect's step lies outside the bounds: the largest of relative L2 / bound over the gradient
    tensors and |logit error| / bound over the samples -> (margin, where, the largest over the gradient tensors alone)"""
    e = _step_errors(ref["loss"], logits, grads, ref["buffers"], ref)
    g = max((v / bounds["rel"][n][0], n) for n, v in e["rel"].items())
    r = e["logits"] / bounds["logits"]
    return max(g, (r.max().item(), f"logits of sample {r.argmax().item()}")) + (g[0],)


def check_train_step(what, route, model, loss, logits, ref, fp32=(), k=0.0):
    """loss, logits (per sample), every BatchNorm running statistic and every gradient tensor of an engine step against
    the oracle's, under step_bounds(route, ref, fp32, k): where this state amplifies rounding, fp32 itself cannot meet a
    bound set on better-conditioned clips"""
    e = _step_errors(loss, logits, grads_of(model), model.state_dict(), ref)
    bnd = step_bounds(route, ref, fp32, k)
    z = bnd["z"]
    rel, norm = e["rel"], e["norm"]
    res_rel = max(v for n, v in rel.items() if ".residuals." in n)
    oth_rel = max(v for n, v in rel.items() if ".residuals." not in n)
    worst_oth = max((v, n) for n, v in rel.items() if ".residuals." not in n)[1]
    report(f"[parity] {what} route={route}: loss {e['loss']:.2e}, logits {e['logits'].max().item():.2e}, "
           f"grad rel-L2 max {oth_rel:.2e} ({worst_oth}), attention-logit layers {res_rel:.2e}, "
           f"analytically-zero tensors {max(e['zero'].values(), default=0.0):.2e} of the gradient norm ({len(e['zero'])}), "
           f"BatchNorm buffers {e['buffers']:.2e}; grad-norm rel err max {max(v for n, v in norm.items() if '.residuals.' not in n):.2e}"
           f" (attention-logit layers {max(v for n, v in norm.items() if '.residuals.' in n):.2e})")
    if fp32:
        zr = z["rel"]
        worst = max((max(v / bnd["rel"][n][0], norm[n] / bnd["rel"][n][1]), n) for n, v in rel.items())
        report(f"[parity] {what} route={route}, plain fp32 torch for comparison: loss {z['loss']:.2e}, logits "
               f"{z['logits'].max().item():.2e}, grad rel-L2 max {max(v for n, v in zr.items() if '.residuals.' not in n):.2e}, "
               f"attention-logit layers {max(v for n, v in zr.items() if '.residuals.' in n):.2e}, BatchNorm buffers "
               f"{z['buffers']:.2e}; worst error/bound: gradients {worst[0]:.3f} ({worst[1]}), logits "
               f"{(e['logits'] / bnd['logits']).max().item():.3f}; {len(bnd['capped'])} tensors at the {CAP_REL} cap"
               + (f" ({', '.join(bnd['capped'])})" if 0 < len(bnd["capped"]) <= len(rel) // 2 else "")
               + (f" (all but {', '.join(n for n in rel if n not in bnd['capped'])})"
                  if len(bnd["capped"]) > len(rel) // 2 else ""))
    assert e["loss"] < bnd["loss"], (loss, ref["loss"])
    assert bool((e["logits"] < bnd["logits"]).all()), e["logits"].max().item()
    assert e["buffers"] < bnd["buffers"], e["buffers"]                  # running statistics, relative to max(1, |value|)
    bad = []
    for n, v in rel.items():
        brel, bnorm = bnd["rel"][n]
        if v > brel or norm[n] > bnorm:
            bad.append(f"{n}: relative L2 {v:.2e} (bound {brel:.1e}), norm {norm[n]:.2e} (bound {bnorm:.1e})")
    assert not bad, "\n".join(bad)
    assert max(e["zero"].values(), default=0.0) < 1e-7
