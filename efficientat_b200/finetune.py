"""Device-resident fine-tuning step: the body of the training loops of the reference's downstream scripts
(ex_esc50.py:96-126, ex_dcase20.py:98-131, ex_fsd50k.py:97-125, ex_openmic.py:97-127) as a chain of this package's
kernels, on the flat parameter arena, Adam launch, gradient buckets and CUDA-graph capture of `AudioSetTrainer`.

    loss="ce"          ESC-50 / DCASE20: softmax cross-entropy (eat_ce_loss).  y is either int class indices [B]
                       (DCASE20) or probability rows [B, C] (ESC-50: one-hot, or blended by waveform mixing).
                       mixstyle_p > 0 (DCASE20): MixStyle on the log-mel, then an un-mixed CE; otherwise, when
                       mixup_alpha is set, mixup on the log-mel and the blended CE.  MixStyle excludes mixup, as in
                       ex_dcase20.py:104-116.
    loss="bce"         FSD50K: mixup-blended BCE-with-logits over all B*C elements (eat_bce_kd_loss, no teacher).
    loss="bce_masked"  OpenMIC: y [B, 2C] = targets | mask; targets binarised before the blend, the mask applied per row
                       (eat_bce_masked_loss), mean over all B*C elements.

Mixup and MixStyle draw on the host from the same generators, in the same order, as the scripts do (mel jitter, then
`helpers.utils.mixup` / `helpers.utils.mixstyle`), and launch outside the captured graph.  `step` does not synchronise
with the host and returns the loss as a 0-dim fp64 device tensor.

    tr = FineTuneTrainer(model, mel, loss="ce", lr=6e-5, mixup_alpha=0.3, schedule=exp_warmup_linear_down(...),
                         cuda_graph=True)
    for epoch in range(n_epochs):
        tr.set_epoch(epoch)
        for x, f, y in dl:
            loss = tr.step(x.cuda(non_blocking=True), y.cuda(non_blocking=True))
"""
import torch

from ._lib import lib
from .helpers.utils import mixstyle
from .helpers.utils import mixup as draw_mixup
from .train import AudioSetTrainer, _stream

LOSSES = ("ce", "bce", "bce_masked")


class FineTuneTrainer(AudioSetTrainer):
    def __init__(self, model, mel, loss="ce", lr=8e-4, mixup_alpha=0.3, mixstyle_p=0.0, mixstyle_alpha=0.4,
                 weight_decay=0.0, adamw=False, betas=(0.9, 0.999), eps=1e-8, process_group=None, cuda_graph=False,
                 schedule=None, grad_buckets=3):
        if loss not in LOSSES:
            raise ValueError(f"FineTuneTrainer: loss must be one of {LOSSES}, got {loss!r}")
        if mixstyle_p and loss != "ce":
            raise ValueError("FineTuneTrainer: MixStyle is part of the cross-entropy (DCASE20) step only")
        super().__init__(model, mel, lr=lr, kd_lambda=1.0, mixup_alpha=mixup_alpha, weight_decay=weight_decay,
                         adamw=adamw, betas=betas, eps=eps, process_group=process_group, cuda_graph=cuda_graph,
                         schedule=schedule, grad_buckets=grad_buckets)
        self.loss = loss
        self.mixstyle_p, self.mixstyle_alpha = mixstyle_p, mixstyle_alpha

    def set_epoch(self, epoch):
        """start of epoch `epoch`: learning rate of the LambdaLR schedule only.  The fine-tuning scripts never call
        `update_params`: a DyMN keeps the temperature it was built with (`pretrain_final_temp`)."""
        self.epoch = int(epoch)

    def _check_y(self, y, B, dev):
        if y.device != dev:
            raise RuntimeError(f"y must be on {dev}, got {y.device}")
        if y.shape[0] != B:
            raise ValueError(f"y must have B = {B} rows, got {tuple(y.shape)}")
        if self.loss == "ce" and y.dim() == 1:
            if y.is_floating_point():
                raise ValueError("class-index targets must be an integer tensor")
            return y.to(torch.int32).contiguous()
        if y.dim() != 2:
            raise ValueError(f"y must be [B, C] (or [B] class indices for loss='ce'), got {tuple(y.shape)}")
        if self.loss == "bce_masked" and y.shape[1] % 2:
            raise ValueError(f"loss='bce_masked' takes y = [B, 2C] (targets | mask), got {tuple(y.shape)}")
        return y.to(torch.float32).contiguous()

    def forward_backward(self, wave, y, teacher=None, perm=None, lam=None, teacher_known=None):
        """-> (loss fp64 device scalar, flat gradient arena)"""
        L = lib()
        st = _stream()
        B = wave.shape[0]
        spec = self.mel(wave.reshape(B, -1))                       # [B, n_mels, T]
        dev = spec.device
        y = self._check_y(y, B, dev)
        perm_d = lam_d = None
        if self.loss == "ce" and self.mixstyle_p > 0:              # ex_dcase20.py:104-107
            spec = mixstyle(spec.unsqueeze(1), self.mixstyle_p, self.mixstyle_alpha).squeeze(1)
        elif self.mixup_alpha or perm is not None:
            if perm is None:
                perm, lam = draw_mixup(B, self.mixup_alpha)
            perm_d = perm.to(dtype=torch.int32).to(device=dev, non_blocking=True)
            lam_d = lam.to(dtype=torch.float32).to(device=dev, non_blocking=True)
            mixed = torch.empty_like(spec)
            L.mixup(spec.data_ptr(), perm_d.data_ptr(), lam_d.data_ptr(), mixed.data_ptr(), B,
                    spec.shape[1] * spec.shape[2], st)
            spec = mixed
        if self.cuda_graph:
            return self._graph_fwd_bwd(spec, y, None, perm_d, lam_d, None)
        return self._core(spec.unsqueeze(1), y, None, perm_d, lam_d, None)

    def _loss(self, logits, y, teacher, perm_d, lam_d, known):
        B, C = logits.shape
        dlogits = torch.empty_like(logits)
        loss = torch.zeros((), device=logits.device, dtype=torch.float64)
        perm_p = perm_d.data_ptr() if perm_d is not None else 0
        lam_p = lam_d.data_ptr() if lam_d is not None else 0
        if self.loss == "ce":
            index = y.dim() == 1
            if not index and y.shape[1] != C:
                raise ValueError(f"y has {y.shape[1]} classes, the model {C}")
            lib().ce_loss(logits.data_ptr(), y.data_ptr() if index else 0, 0 if index else y.data_ptr(), perm_p, lam_p,
                          B, C, dlogits.data_ptr(), loss.data_ptr(), _stream())
        elif self.loss == "bce":
            if y.shape[1] != C:
                raise ValueError(f"y has {y.shape[1]} classes, the model {C}")
            lib().bce_kd_loss(logits.data_ptr(), y.data_ptr(), 0, 0, perm_p, lam_p, 1.0, B, C, dlogits.data_ptr(),
                              loss.data_ptr(), _stream())
        else:
            if y.shape[1] != 2 * C:
                raise ValueError(f"y must be [B, 2 * {C}] (targets | mask), got {tuple(y.shape)}")
            lib().bce_masked_loss(logits.data_ptr(), y.data_ptr(), 2 * C, y[:, C:].data_ptr(), 2 * C, perm_p, lam_p,
                                  B, C, dlogits.data_ptr(), loss.data_ptr(), _stream())
        return loss, dlogits

    def _graph_key(self, spec, y, teacher, perm_d, known):
        return super()._graph_key(spec, y, teacher, perm_d, known) + (self.loss, y.dtype)

    def step(self, wave, y, perm=None, lam=None):
        """one optimiser step on a batch: wave [B, N] (or [B, 1, N]) and y as described for `loss`; perm/lam
        optionally replace the mixup draw.  -> the loss, a 0-dim fp64 device tensor"""
        return super().step(wave, y, None, perm, lam, None)
