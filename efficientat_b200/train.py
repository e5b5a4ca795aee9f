"""Device-resident AudioSet training step: the body of the reference's loop, ex_audioset.py:135-199
(mel -> mixup -> model -> hard-label + distillation BCE -> backward -> Adam), as a chain of this
package's kernels with one optional NCCL all-reduce of the flat gradient arena (the data-parallel
semantics of ex_pl_audioset.py:287-293: replicas, per-replica BatchNorm, gradient mean).

No host synchronisation happens inside `step`; the loss comes back as a device tensor.

With `cuda_graph=True` the ~440 launches of forward + loss + backward are captured once per input shape into a
CUDA graph and replayed; only the mel front end, the mixup kernel (their per-step random scalars come from the
host RNG, as in the reference), the all-reduce and the Adam kernel stay eager.  Enqueueing a step then costs the
host ~1 ms instead of ~45 ms, which is what keeps the GPU busy at small per-GPU batches."""
import torch

from . import parallel
from ._lib import lib
from .helpers.utils import mixup as draw_mixup
from .models.common import head_dropout


def _stream():
    return torch.cuda.current_stream().cuda_stream


class HostPrefetcher:
    """Double-buffered host -> device feed for the training loop (the role of the reference's pinned-memory DataLoader,
    ex_audioset.py:104-110): batch i+1 is copied from pinned host memory on a side stream while step i runs.

        pf = HostPrefetcher(device)
        pf.submit(0, first_batch)
        for i, nxt in enumerate(batches[1:] + [None]):
            if nxt is not None: pf.submit((i + 1) % 2, nxt)
            wave, y, teacher = pf.get(i % 2)
            loss = trainer.step(wave, y, teacher)
            pf.release(i % 2)
    """

    def __init__(self, device, slots=2):
        self.device = torch.device(device)
        self.stream = torch.cuda.Stream(self.device)
        self.bufs = [None] * slots
        self.ready = [torch.cuda.Event() for _ in range(slots)]
        self.free = [torch.cuda.Event() for _ in range(slots)]
        for e in self.free:
            e.record(torch.cuda.current_stream(self.device))

    def submit(self, slot, host_tensors):
        """enqueue the copy of one batch (a tuple of pinned CPU tensors) into slot `slot`"""
        if self.bufs[slot] is None or any(b.shape != h.shape or b.dtype != h.dtype for b, h in zip(self.bufs[slot], host_tensors)):
            self.bufs[slot] = tuple(torch.empty(h.shape, dtype=h.dtype, device=self.device) for h in host_tensors)
        with torch.cuda.stream(self.stream):
            self.stream.wait_event(self.free[slot])          # the step that read this slot two batches ago is done
            for b, h in zip(self.bufs[slot], host_tensors):
                b.copy_(h, non_blocking=True)
            self.ready[slot].record(self.stream)

    def get(self, slot):
        torch.cuda.current_stream(self.device).wait_event(self.ready[slot])
        return self.bufs[slot]

    def release(self, slot):
        self.free[slot].record(torch.cuda.current_stream(self.device))


class LossReader:
    """Pipelined device -> host read-back of per-step results (the loss), for loops that log every step.

    The reference's loop calls `.item()` three times per step (ex_audioset.py:192-194): the host then waits for the
    device after EVERY step, and the device idles while the host enqueues the next one.  Here `push(t)` enqueues an
    asynchronous copy of the small device tensor into a pinned host slot behind the step that produced it, and `pop()`
    returns the OLDEST outstanding value, waiting only for that step's event.  Popping one step behind keeps the host a
    step ahead of the device; every step's value still reaches the host, in order.

        rd = LossReader(device)
        for i, batch in enumerate(batches):
            rd.push(trainer.step(*batch))
            if i: log(rd.pop())          # loss of step i-1, step i is already queued
        log(rd.pop())
    """

    def __init__(self, device, depth=2):
        self.device = torch.device(device)
        self.depth = int(depth)
        self.slots = [None] * self.depth
        self.events = [torch.cuda.Event() for _ in range(self.depth)]
        self.head = 0                    # next slot to write
        self.pending = 0

    def push(self, t):
        if self.pending == self.depth:
            raise RuntimeError("LossReader: all slots are outstanding; pop() before the next push()")
        if not t.is_cuda:
            raise RuntimeError("LossReader.push expects a CUDA tensor")
        k = self.head
        if self.slots[k] is None or self.slots[k].shape != t.shape or self.slots[k].dtype != t.dtype:
            self.slots[k] = torch.empty(t.shape, dtype=t.dtype, device="cpu").pin_memory()
        with torch.cuda.device(self.device):
            self.slots[k].copy_(t.detach(), non_blocking=True)       # stream-ordered behind the producing step
            self.events[k].record(torch.cuda.current_stream(self.device))
        self.head = (k + 1) % self.depth
        self.pending += 1

    def pop(self):
        if self.pending == 0:
            raise RuntimeError("LossReader.pop without an outstanding push")
        k = (self.head - self.pending) % self.depth
        self.events[k].synchronize()
        self.pending -= 1
        return self.slots[k].clone()


class AudioSetTrainer:
    """The body of the reference's training loop (ex_audioset.py:120-201) on device-resident tensors.

    lr schedule: `schedule` is the reference's epoch -> factor lambda (helpers/utils.py:56-84, built by
    `exp_warmup_linear_down`); the learning rate of epoch e is `lr * schedule(e)`, which is what
    `LambdaLR` + one `scheduler.step()` per epoch give (ex_audioset.py:95-97,201).  `set_epoch(e)` also forwards to
    `model.update_params(e)` (DyMN temperature schedule, ex_audioset.py:132-133)."""

    def __init__(self, model, mel, lr=8e-4, kd_lambda=0.1, mixup_alpha=0.3, weight_decay=0.0, adamw=False,
                 betas=(0.9, 0.999), eps=1e-8, process_group=None, cuda_graph=False, schedule=None, grad_buckets=3,
                 augment=None):
        if not 0.0 <= kd_lambda <= 1.0:
            raise AssertionError("Lambda for Knowledge Distillation must be between 0 and 1.")     # ex_audioset.py:100
        self.model, self.mel = model, mel
        self.augment = augment                  # augment.WaveAugment: gain / roll / waveform mixing before the mel
        self.engine = model.engine()
        self.lr, self.kd_lambda, self.mixup_alpha = lr, kd_lambda, mixup_alpha
        self.weight_decay, self.adamw, self.betas, self.eps = weight_decay, adamw, betas, eps
        self.schedule = schedule
        self.epoch = 0
        self.pg = process_group
        self.world = 1
        if torch.distributed.is_available() and torch.distributed.is_initialized():
            self.world = torch.distributed.get_world_size(process_group)
        self._flatten()
        # world > 1: the gradient all-reduce is cut into buckets that start on a side stream while backward is still
        # running (parallel.GradBucketer); grad_buckets = 0 keeps one all-reduce after backward
        self.bucketer = None
        if self.world > 1 and grad_buckets and grad_buckets > 0:
            self.bucketer = parallel.GradBucketer([p.numel() for p in self.engine.param_list()], grad_buckets, process_group)
        self.steps = 0
        self.cuda_graph = cuda_graph
        self._graphs = {}

    # ------------------------------------------------------------------ schedule
    def current_lr(self):
        return self.lr * (self.schedule(self.epoch) if self.schedule is not None else 1.0)

    def set_epoch(self, epoch):
        """start of epoch `epoch`: learning rate of the LambdaLR schedule + DyMN temperature update"""
        self.epoch = int(epoch)
        if hasattr(self.model, "update_params"):
            import contextlib
            import io
            with contextlib.redirect_stdout(io.StringIO()):          # the reference prints one line per DynamicConv
                self.model.update_params(self.epoch)

    def _flatten(self):
        """Re-point every parameter into one contiguous fp32 arena (order = model.parameters()), so the
        optimiser is one kernel and the gradient all-reduce one collective.  state_dict()/load_state_dict()
        keep working (they copy in place).  With world > 1 the replicas start from rank 0's parameters AND
        buffers (DistributedDataParallel's constructor broadcast; ex_pl_audioset.py:287-293)."""
        params = self.engine.param_list()
        dev = params[0].device
        for p in params:
            if p.device != dev or p.dtype != torch.float32:
                raise RuntimeError("AudioSetTrainer: all parameters must be fp32 tensors on one CUDA device "
                                   f"(got {p.dtype} on {p.device}); call model.to(device) first")
        if dev.type != "cuda":
            raise RuntimeError("AudioSetTrainer: the model must be on a CUDA device (no CPU fallback)")
        n = sum(p.numel() for p in params)
        flat = torch.empty(n, device=dev, dtype=torch.float32)
        off = 0
        for p in params:
            k = p.numel()
            flat[off:off + k].copy_(p.data.reshape(-1))
            p.data = flat[off:off + k].view(p.shape)
            off += k
        self.flat_p = flat
        self.exp_avg = torch.zeros_like(flat)
        self.exp_avg_sq = torch.zeros_like(flat)
        if self.world > 1:
            parallel.broadcast_from_rank0_(self.flat_p, group=self.pg)
            for b in self.model.buffers():
                parallel.broadcast_from_rank0_(b, group=self.pg)

    # ------------------------------------------------------------------ one step
    @staticmethod
    def _check_targets(t, B, name, dev):
        if t is None:
            return None
        if t.dim() != 2 or t.shape[0] != B:
            raise ValueError(f"{name} must have shape [B, num_classes] with B = {B}, got {tuple(t.shape)}")
        if t.device != dev:
            raise RuntimeError(f"{name} must be on {dev}, got {t.device}")
        return t.to(torch.float32).contiguous()

    def forward_backward(self, wave, y, teacher=None, perm=None, lam=None, teacher_known=None, draws=None):
        """-> (loss_acc fp64[2] device = weighted label / distillation losses, flat gradient arena).
        teacher_known: optional [B] bool/float, False/0 for clips without teacher predictions (their distillation
        loss is zeroed, ex_audioset.py:166-178).  With `augment`, see `step` for `wave`, `y` and `draws`."""
        L = lib()
        st = _stream()
        if self.augment is not None:
            wave, y = self.augment(wave, y, draws)
        B = wave.shape[0]
        spec = self.mel(wave.reshape(B, -1))                       # [B, n_mels, T]
        dev = spec.device
        y = self._check_targets(y, B, "y", dev)
        teacher = self._check_targets(teacher, B, "teacher", dev)
        if teacher is not None and teacher.shape != y.shape:
            raise ValueError(f"teacher {tuple(teacher.shape)} and y {tuple(y.shape)} must have the same shape")
        if teacher_known is not None:
            if teacher is None:
                raise ValueError("teacher_known given without teacher predictions")
            teacher_known = teacher_known.to(device=dev, dtype=torch.float32).contiguous().view(B)
        if self.kd_lambda <= 0:                                    # ex_audioset.py:159,183: no distillation term at all
            teacher = teacher_known = None
        if self.mixup_alpha and perm is None:
            perm, lam = draw_mixup(B, self.mixup_alpha)
        if perm is not None:
            perm_d = perm.to(dtype=torch.int32).to(device=dev, non_blocking=True)
            lam_d = lam.to(dtype=torch.float32).to(device=dev, non_blocking=True)
            mixed = torch.empty_like(spec)
            L.mixup(spec.data_ptr(), perm_d.data_ptr(), lam_d.data_ptr(), mixed.data_ptr(), B,
                    spec.shape[1] * spec.shape[2], st)
            spec = mixed
        else:
            perm_d = lam_d = None
        if self.cuda_graph:
            return self._graph_fwd_bwd(spec, y, teacher, perm_d, lam_d, teacher_known)
        return self._core(spec.unsqueeze(1), y, teacher, perm_d, lam_d, teacher_known)

    def _core(self, spec4, y, teacher, perm_d, lam_d, known=None):
        """model forward + loss + backward on device tensors -> (loss_acc, flat gradient arena)"""
        logits, _, saved = self.engine._forward_train(spec4)
        loss_acc, dlogits = self._loss(logits, y, teacher, perm_d, lam_d, known)
        if self.bucketer is not None:
            grads = self.engine._backward(saved, dlogits, on_ready=self.bucketer.ready)
            self.bucketer.finish(grads[None])                     # joins the side stream: the arena is reduced (sum)
        else:
            grads = self.engine._backward(saved, dlogits)
        return loss_acc, grads[None]

    def _loss(self, logits, y, teacher, perm_d, lam_d, known):
        """-> (loss_acc, dlogits): the loss of the step and its gradient w.r.t. the logits, on the device"""
        B = logits.shape[0]
        dlogits = torch.empty_like(logits)
        loss_acc = torch.zeros(2, device=logits.device, dtype=torch.float64)
        # without a teacher the label loss carries weight 1 (ex_audioset.py:182-183)
        lib().bce_kd_loss(logits.data_ptr(), y.data_ptr(), teacher.data_ptr() if teacher is not None else 0,
                          known.data_ptr() if known is not None else 0,
                          perm_d.data_ptr() if perm_d is not None else 0, lam_d.data_ptr() if lam_d is not None else 0,
                          self.kd_lambda, B, logits.shape[1], dlogits.data_ptr(), loss_acc.data_ptr(), _stream())
        return loss_acc, dlogits

    def _graph_key(self, spec, y, teacher, perm_d, known):
        """everything a captured graph bakes in: shapes, optional-operand presence and the host scalars passed by value
        (loss weight, dropout rate, BatchNorm momentum / eps, DynamicConv temperatures)"""
        bn = next((m for m in self.model.modules() if isinstance(m, torch.nn.BatchNorm2d)), None)
        return (tuple(spec.shape), tuple(y.shape), teacher is not None, perm_d is not None, known is not None,
                float(self.kd_lambda), head_dropout(self.model),
                (float(bn.momentum), float(bn.eps)) if bn is not None else None,
                tuple(float(getattr(m, "temperature", 0.0)) for m in self.model.modules() if hasattr(m, "temperature")))

    def _graph_fwd_bwd(self, spec, y, teacher, perm_d, lam_d, known=None):
        key = self._graph_key(spec, y, teacher, perm_d, known)
        g = self._graphs.get(key)
        if g is None:
            g = self._capture(spec, y, teacher, perm_d, lam_d, known)
            self._graphs = {key: g}             # one live graph (a new shape / scalar replaces it)
        g["spec"].copy_(spec.unsqueeze(1), non_blocking=True)
        g["y"].copy_(y, non_blocking=True)
        if teacher is not None:
            g["teacher"].copy_(teacher, non_blocking=True)
        if known is not None:
            g["known"].copy_(known, non_blocking=True)
        if perm_d is not None:
            g["perm"].copy_(perm_d, non_blocking=True)
            g["lam"].copy_(lam_d, non_blocking=True)
        g["graph"].replay()
        return g["loss"], g["grads"]

    def _capture(self, spec, y, teacher, perm_d, lam_d, known=None):
        dev = spec.device
        st = {"spec": spec.unsqueeze(1).clone(), "y": y.clone(),
              "teacher": teacher.clone() if teacher is not None else None,
              "known": known.clone() if known is not None else None,
              "perm": perm_d.clone() if perm_d is not None else None,
              "lam": lam_d.clone() if lam_d is not None else None}
        # eager warm-up on a side stream (allocator / one-time attribute calls); BatchNorm buffers are restored
        # afterwards so the warm-up does not count as training steps
        saved_buffers = [b.detach().clone() for b in self.model.buffers()]
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                self._core(st["spec"], st["y"], st["teacher"], st["perm"], st["lam"], st["known"])
        torch.cuda.current_stream().wait_stream(side)
        with torch.no_grad():
            for b, sb in zip(self.model.buffers(), saved_buffers):
                b.copy_(sb)
        graph = torch.cuda.CUDAGraph()
        # thread-local capture mode: the NCCL watchdog thread may touch the CUDA API while this thread captures
        with torch.cuda.graph(graph, capture_error_mode="thread_local" if self.world > 1 else "global"):
            loss_acc, flat_g = self._core(st["spec"], st["y"], st["teacher"], st["perm"], st["lam"], st["known"])
        st.update(graph=graph, loss=loss_acc, grads=flat_g)
        return st

    def close(self):
        """Drop the captured CUDA graph(s).  With world > 1 the graph holds NCCL kernels of the process group's
        communicator: destroy the graph BEFORE `torch.distributed.destroy_process_group()`, which otherwise waits for it
        forever (observed with NCCL 2.28)."""
        self._graphs = {}
        import gc
        gc.collect()
        if self.flat_p.is_cuda:
            torch.cuda.synchronize(self.flat_p.device)

    def step(self, wave, y, teacher=None, perm=None, lam=None, teacher_known=None, draws=None):
        """one optimiser step.  With `augment` (augment.WaveAugment), gain, roll and waveform mixing run first, on
        the device: with its store, `wave` is the batch's [B] dataset indices (CPU) and `y` None; without one, `wave`
        and `y` are the batch that is augmented.  `teacher` / `teacher_known` belong to the primary items (the
        reference looks the teacher up by the primary index, audioset.py:96-100).  `draws` optionally replaces the
        augmentation's host draw.  -> the loss, as `forward_backward`."""
        self.model.train()
        self.mel.train()
        self.engine.dropout_p = head_dropout(self.model)             # read at call time, not at engine construction
        with torch.cuda.device(self.flat_p.device):
            loss_acc, flat_g = self.forward_backward(wave, y, teacher, perm, lam, teacher_known, draws)
            if self.world > 1 and self.bucketer is None:
                torch.distributed.all_reduce(flat_g, group=self.pg)        # one collective per step (sum)
            self.steps += 1
            lib().adam_step(self.flat_p.data_ptr(), flat_g.data_ptr(), self.exp_avg.data_ptr(),
                            self.exp_avg_sq.data_ptr(), flat_g.numel(), self.current_lr(), self.betas[0], self.betas[1],
                            self.eps, self.weight_decay, 1 if self.adamw else 0, self.steps, 1.0 / self.world, _stream())
        return loss_acc
