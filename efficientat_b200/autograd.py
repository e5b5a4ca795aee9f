"""torch.autograd glue: one Function for the whole network, so that the reference's training loop
(`loss.backward()`, ex_audioset.py:197) drives the hand-written backward chain in efficientat_b200.engine unchanged.
Parameter gradients come back as views of one flat fp32 arena.

The same Function carries gradients to the input spectrogram (saliency maps, adversarial evaluation, a frozen tagger
used as a loss): in train() on batch statistics, in eval() on the running statistics (engine._forward_train(frozen=True)).
Only the gradients autograd asks for are computed: with every parameter frozen, no weight-gradient pass runs.

Every output the reference's autograd can use is differentiable: the logits, the embedding (`features`, the global
average of the last conv's output) and, in train() with return_fmaps=True, the 17 feature maps (stem, 15 blocks, last
conv) as [B, C, F, T] views of the engine's NHWC storage.  An output the loss does not use gets no gradient (None) and
no backward work: with the embedding alone, the classifier's parameters are not part of the graph and get None."""
import torch


class _MNFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, engine, frozen, want_fmaps, x, *params):
        logits, feat, saved = engine._forward_train(x, frozen=frozen, fmaps=want_fmaps)
        ctx.set_materialize_grads(False)
        ctx.engine = engine
        ctx.saved = saved
        fmaps = [_nchw(t) for t in saved["fmaps"]] if want_fmaps else []
        # the block outputs are the next block's saved input: an in-place edit of a returned map raises at backward()
        ctx.save_for_backward(*fmaps)
        return (logits, feat, *fmaps)

    @staticmethod
    def backward(ctx, dlogits, dfeat, *dfmaps):
        ctx.saved_tensors                           # the version check of the returned maps
        input_grad = ctx.needs_input_grad[3]
        engine = ctx.engine
        params = engine.param_list()
        kw = dict(dembed=dfeat, dfmaps=list(dfmaps) if dfmaps else None)
        if input_grad:
            if torch.is_grad_enabled():
                raise NotImplementedError("double backward (create_graph=True) through efficientat_b200 models is not "
                                          "implemented: the backward kernels build no graph")
            wanted = [p for p, need in zip(params, ctx.needs_input_grad[4:]) if need]
            grads = engine._backward(ctx.saved, dlogits, input_grad=True, wanted=wanted, **kw)
        else:
            grads = engine._backward(ctx.saved, dlogits, **kw)
        ctx.saved = None
        # without a logits gradient the classifier is not part of the graph
        off_graph = set() if dlogits is not None else {id(p) for p in engine.model.classifier.parameters()}
        out = [grads[p] if p.requires_grad and id(p) not in off_graph else None for p in params]
        return (None, None, None, grads["x"] if input_grad else None) + tuple(out)


def _nchw(t):
    """NHWC storage [B, F, T, C] -> the reference's [B, C, F, T] layout, as a view"""
    return t.permute(0, 3, 1, 2)


def mn_train_forward(engine, x, needs_grad):
    if not needs_grad:
        logits, feat, _ = engine._forward_train(x)
        return logits, feat
    logits, feat = _MNFn.apply(engine, False, False, x, *engine.param_list())
    return logits, feat


def mn_train_forward_fmaps(engine, x, needs_grad):
    """train() with return_fmaps=True -> (logits, features, [17 maps]); a graph through all of them when needs_grad"""
    if not needs_grad:
        logits, feat, saved = engine._forward_train(x, fmaps=True)
        return logits, feat, [_nchw(t) for t in saved["fmaps"]]
    out = _MNFn.apply(engine, False, True, x, *engine.param_list())
    return out[0], out[1], list(out[2:])


def mn_eval_grad_forward(engine, x):
    """eval() with an input that requires grad: the saving forward on running statistics, no dropout, no buffer update"""
    logits, feat = _MNFn.apply(engine, True, False, x, *engine.param_list())
    return logits, feat
