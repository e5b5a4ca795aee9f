"""torch.autograd glue: one Function for the whole network, so that the reference's training loop
(`loss.backward()`, ex_audioset.py:197) drives the hand-written backward chain in efficientat_b200.engine unchanged.
Parameter gradients come back as views of one flat fp32 arena.

The same Function carries gradients to the input spectrogram (saliency maps, adversarial evaluation, a frozen tagger
used as a loss): in train() on batch statistics, in eval() on the running statistics (engine._forward_train(frozen=True)).
Only the gradients autograd asks for are computed: with every parameter frozen, no weight-gradient pass runs."""
import torch


class _MNFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, engine, frozen, x, *params):
        logits, feat, saved = engine._forward_train(x, frozen=frozen)
        ctx.engine = engine
        ctx.saved = saved
        ctx.mark_non_differentiable(feat)
        return logits, feat

    @staticmethod
    def backward(ctx, dlogits, _dfeat):
        input_grad = ctx.needs_input_grad[2]
        params = ctx.engine.param_list()
        if input_grad:
            if torch.is_grad_enabled():
                raise NotImplementedError("double backward (create_graph=True) through efficientat_b200 models is not "
                                          "implemented: the backward kernels build no graph")
            wanted = [p for p, need in zip(params, ctx.needs_input_grad[3:]) if need]
            grads = ctx.engine._backward(ctx.saved, dlogits, input_grad=True, wanted=wanted)
        else:
            grads = ctx.engine._backward(ctx.saved, dlogits)
        ctx.saved = None
        out = [grads[p] if p.requires_grad else None for p in params]
        return (None, None, grads["x"] if input_grad else None) + tuple(out)


def mn_train_forward(engine, x, needs_grad):
    if not needs_grad:
        logits, feat, _ = engine._forward_train(x)
        return logits, feat
    return _MNFn.apply(engine, False, x, *engine.param_list())


def mn_eval_grad_forward(engine, x):
    """eval() with an input that requires grad: the saving forward on running statistics, no dropout, no buffer update"""
    return _MNFn.apply(engine, True, x, *engine.param_list())
