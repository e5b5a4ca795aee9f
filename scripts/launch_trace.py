#!/usr/bin/env python
"""Launch-by-launch trace of the host engines, without a GPU:

    python scripts/launch_trace.py [--root TREE] > trace.txt

The engines (efficientat_b200/engine.py, engine_dymn.py) never read device memory on the host, so they run on CPU tensors
against a library that only records its calls.  Each line is one C-ABI launch: the entry point, its scalar arguments,
and each pointer as `0` (null), the parameter or buffer it points into (`+bytes` past its start), `grad:<parameter>`
inside the gradient arena, or `*` for any other tensor.  `--root` imports the package from another tree, so a refactor
of the engines can be checked by diffing its trace against its parent's:

    git worktree add ../parent HEAD~1
    python scripts/launch_trace.py --root ../parent > old.txt; python scripts/launch_trace.py > new.txt; diff old.txt new.txt

The host-only planners (eat_pw_bwd_plan, eat_pw_proj_bwd_plan) run in the tree's libeat_b200.so when it is built (it
loads without a GPU), and otherwise accept every shape; compare two trees with the same library state."""
import argparse
import ctypes
import os
import sys
import types

import torch

PLANNERS = ("pw_bwd_plan", "pw_proj_bwd_plan")
B, F, T = 3, 128, 96
LENGTHS = [96, 50, 17]
# the engine attributes the tests flip away from their defaults
SWITCHES = (("gemm_impl", "simt"), ("pw_impl", "tc"), ("se_fused", False), ("dgrad_bnred", True), ("dw_bwd_fused", False),
            ("expand_bwd_fused", False), ("proj_bwd_fused", False), ("stem_bwd_fused", False))


class Recorder:
    """stands in for the ctypes library: each call is kept as (entry point, raw arguments)"""

    def __init__(self, protos, real):
        self.protos, self.real, self.calls = protos, real, []

    def __getattr__(self, name):
        if name in PLANNERS:
            return getattr(self.real, name) if self.real is not None else (lambda *args: None)
        argtypes = self.protos["eat_" + name][1]

        def call(*args):
            assert len(args) == len(argtypes), f"{name}: {len(args)} arguments, the header declares {len(argtypes)}"
            self.calls.append((name, args))
        return call


class Resolver:
    """pointer -> name of the parameter, buffer or gradient view it points into"""

    def __init__(self, model, grads=None):
        self.spans = []
        for name, t in list(model.named_parameters()) + list(model.named_buffers()):
            self._add(t, name)
        names = {id(p): n for n, p in model.named_parameters()}
        for p, g in (grads or {}).items():
            if id(p) in names:
                self._add(g, "grad:" + names[id(p)])

    def _add(self, t, name):
        if t.numel():
            self.spans.append((t.data_ptr(), t.data_ptr() + t.numel() * t.element_size(), name))

    def __call__(self, ptr):
        if ptr == 0:
            return "0"
        for lo, hi, name in self.spans:
            if lo <= ptr < hi:
                return name if ptr == lo else f"{name}+{ptr - lo}"
        return "*"


def emit(out, calls, protos, resolve):
    for name, args in calls:
        words = [name]
        for a, ty in zip(args, protos["eat_" + name][1]):
            if a is STREAM:
                words.append("st")
            elif ty is ctypes.c_void_p:
                words.append(resolve(int(a)))
            else:
                words.append(repr(a))
        out.write(" ".join(words) + "\n")
    calls.clear()


STREAM = object()


def models(pkg):
    from_mn = pkg.models.mn.model.get_model
    from_dy = pkg.models.dymn.model.get_model
    yield "mn04", lambda p: from_mn(width_mult=0.4, precision=p, verbose=False)
    yield "mn10", lambda p: from_mn(width_mult=1.0, precision=p, verbose=False)
    yield "mn10-dilated", lambda p: from_mn(width_mult=1.0, dilated=True, precision=p, verbose=False)
    yield "mn04-mha", lambda p: from_mn(width_mult=0.4, head_type="multihead_attention_pooling", precision=p, verbose=False)
    for k in (1, 2, 3, 4):
        yield f"dymn04-k{k}", lambda p, k=k: from_dy(width_mult=0.4, dyrelu_k=k, precision=p, verbose=False)
    yield "dymn10-replace_se", lambda p: from_dy(width_mult=1.0, use_dy_blocks="replace_se", precision=p, verbose=False)


def trace_model(out, rec, protos, engine_cls, make, precision):
    torch.manual_seed(0)
    model = make(precision)
    x = torch.randn(B, 1, F, T)
    params = list(model.parameters())

    def engine(**attrs):
        eng = engine_cls(model)
        for k, v in attrs.items():
            setattr(eng, k, v)
        return eng

    def case(title, fn):
        out.write(f"# {title}\n")
        grads = fn()
        emit(out, rec.calls, protos, Resolver(model, grads))

    def train_step(eng, fmaps=False, frozen=False, **bwd):
        def run():
            logits, feat, S = eng._forward_train(x, frozen=frozen, fmaps=fmaps)
            emit(out, rec.calls, protos, Resolver(model))
            dlogits = torch.randn_like(logits)
            if fmaps:
                maps = S["fmaps"]
                dfm = [None] * len(maps)
                for i in (5, len(maps) - 1):
                    dfm[i] = torch.randn_like(maps[i]).permute(0, 3, 1, 2)
                bwd.update(dembed=torch.randn_like(feat), dfmaps=dfm)
            return eng._backward(S, bwd.pop("dlogits", dlogits), **bwd)
        return run

    def eval_fwd(eng, *args, **kw):
        return lambda: eng._forward_eval(x, *args, **kw) and None

    model.eval()
    case("eval", eval_fwd(engine()))
    case("eval lengths", eval_fwd(engine(), lengths=LENGTHS))
    case("eval return_fmaps", eval_fwd(engine(), True))
    case("frozen input_grad wanted=[]", train_step(engine(), frozen=True, input_grad=True, wanted=[]))
    case("frozen input_grad wanted=params[::3]", train_step(engine(), frozen=True, input_grad=True, wanted=params[::3]))
    model.train()
    case("train", train_step(engine()))
    case("train dembed dfmaps", train_step(engine(), fmaps=True))
    case("train dembed dfmaps, no dlogits", train_step(engine(), fmaps=True, dlogits=None))
    for k, v in SWITCHES:
        case(f"train {k}={v}", train_step(engine(**{k: v})))
    model.eval()
    case("eval gemm_impl=simt", eval_fwd(engine(gemm_impl="simt")))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                    help="tree to import efficientat_b200 from (default: this one)")
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import efficientat_b200.models.dymn.model  # noqa: F401
    import efficientat_b200.models.mn.model  # noqa: F401
    from efficientat_b200 import _lib, engine, engine_dymn
    pkg = sys.modules["efficientat_b200"]
    assert os.path.dirname(pkg.__file__) == os.path.join(os.path.abspath(args.root), "efficientat_b200"), pkg.__file__

    protos = _lib.parse_header()
    real = _lib.lib() if os.path.exists(_lib.LIB_PATH) else None
    rec = Recorder(protos, real)
    for mod in (engine, engine_dymn):
        mod.lib = lambda: rec
        mod._stream = lambda: STREAM
    # the SE-fused reduce sizes its slices from the SM count (H100 SXM: 132)
    torch.cuda.get_device_properties = lambda dev: types.SimpleNamespace(multi_processor_count=132)

    out = sys.stdout
    out.write(f"# planners: {'libeat_b200.so' if real is not None else 'accept every shape'}\n")
    for name, make in models(pkg):
        cls = engine_dymn.DyMNEngine if name.startswith("dymn") else engine.MNEngine
        for precision in ("fp32", "bf16"):
            out.write(f"## {name} {precision}\n")
            trace_model(out, rec, protos, cls, make, precision)


if __name__ == "__main__":
    main()
