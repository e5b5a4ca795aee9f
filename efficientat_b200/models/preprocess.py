"""Drop-in for the reference's models/preprocess.py: AugmentMelSTFT backed by one fused CUDA kernel.

Same constructor, buffers, RNG side effects and output as reference models/preprocess.py:6-67;
the seven library calls of its forward (:41-65) are one launch of eat_mel_fwd (csrc/mel.cu).
A waveform that requires grad gets its gradient from eat_mel_bwd, with the filterbank and masks of the forward call.
"""
import ctypes
import math

import torch
import torch.nn as nn

from .._lib import check_module_tensors, lib
from ..packed import as_int_list, check_lengths
from .filterbank import kaldi_mel_banks, to_bands


class _AxisMasking(nn.Module):
    """torchaudio.transforms.{Frequency,Time}Masking(param, iid_masks=True) on [B, F, T]
    (models/preprocess.py:31-38, applied :61-63 in training only): one band per example, width ~ U[0, param),
    start ~ U[0, size - width), filled with 0.0, drawn with torch.rand on the spectrogram's DEVICE generator.
    This is the behaviour of torchaudio >= 2.1 (`mask_along_axis_iid` over all leading dimensions), i.e. of the
    installed 2.11 that serves as the oracle here.  The reference's requirements.txt pins torchaudio 0.13, where
    iid masking required a 4-D input and a 3-D spectrogram got ONE mask shared by the batch from the CPU generator;
    that older behaviour is NOT reproduced.  Both scripts' defaults are freqm = timem = 0 (ex_audioset.py:380-381),
    for which the module is an Identity and no random number is drawn."""

    def __init__(self, mask_param, axis):
        super().__init__()
        self.mask_param = mask_param
        self.axis = axis      # 1 = frequency, 2 = time

    def extra_repr(self):
        return f"mask_param={self.mask_param}, axis={self.axis}, iid_masks=True"

    def draw(self, spec):
        b, size = spec.shape[0], spec.shape[self.axis]
        value = torch.rand(b, device=spec.device) * self.mask_param
        min_value = torch.rand(b, device=spec.device) * (size - value)
        start = min_value.long()
        end = min_value.long() + value.long()
        return start.int(), end.int()


class AugmentMelSTFT(nn.Module):
    def __init__(self, n_mels=128, sr=32000, win_length=800, hopsize=320, n_fft=1024, freqm=48, timem=192,
                 fmin=0.0, fmax=None, fmin_aug_range=10, fmax_aug_range=2000):
        super().__init__()
        self.win_length = win_length
        self.n_mels = n_mels
        self.n_fft = n_fft
        self.sr = sr
        self.fmin = fmin
        if fmax is None:
            fmax = sr // 2 - fmax_aug_range // 2
            print(f"Warning: FMAX is None setting to {fmax} ")
        self.fmax = fmax
        self.hopsize = hopsize
        self.register_buffer("window", torch.hann_window(win_length, periodic=False), persistent=False)
        assert fmin_aug_range >= 1, f"fmin_aug_range={fmin_aug_range} should be >=1; 1 means no augmentation"
        assert fmax_aug_range >= 1, f"fmax_aug_range={fmax_aug_range} should be >=1; 1 means no augmentation"
        self.fmin_aug_range = fmin_aug_range
        self.fmax_aug_range = fmax_aug_range
        self.register_buffer("preemphasis_coefficient", torch.as_tensor([[[-.97, 1]]]), persistent=False)
        self.freqm = nn.Identity() if freqm == 0 else _AxisMasking(freqm, 1)
        self.timem = nn.Identity() if timem == 0 else _AxisMasking(timem, 2)
        # FFT twiddles in fp64 -> fp32, with M = n_fft / 2: exp(-2 pi i m / M), m < M, then exp(-2 pi i k / n_fft), k < M.
        # The kernel takes n_fft in {256, 512, 1024, 2048, 4096}; any other value raises EatError at the first forward.
        half = n_fft // 2
        m = torch.arange(half, dtype=torch.float64)
        tw = torch.cat([torch.stack([torch.cos(2 * math.pi * m / half), -torch.sin(2 * math.pi * m / half)], 1),
                        torch.stack([torch.cos(2 * math.pi * m / n_fft), -torch.sin(2 * math.pi * m / n_fft)], 1)])
        self.register_buffer("_twiddle", tw.float().contiguous(), persistent=False)
        self._fb_cache = {}
        self._preemph = 0.97      # value of preemphasis_coefficient[0,0,0] negated (preprocess.py:30)

    def _filterbank(self, fmin, fmax, device):
        key = (float(fmin), float(fmax), str(device))
        hit = self._fb_cache.get(key)
        if hit is None:
            start, length, taps = to_bands(kaldi_mel_banks(self.n_mels, self.n_fft, self.sr, fmin, fmax))
            hit = (start.to(device), length.to(device), taps.to(device).contiguous(), taps.shape[0])
            if len(self._fb_cache) > 4096:
                self._fb_cache.clear()
            self._fb_cache[key] = hit
        return hit

    def _device_filterbank(self, fmin, fmax, device, private=False):
        """private: a filterbank of this call's own, kept for its backward (the shared buffer is rebuilt every call)"""
        cap = self.n_fft // 2 + 1
        buf = None if private else getattr(self, "_fb_dev", None)
        if buf is None or buf[0].device != device:
            buf = (torch.empty(self.n_mels, dtype=torch.int32, device=device),
                   torch.empty(self.n_mels, dtype=torch.int32, device=device),
                   torch.empty(cap, self.n_mels, dtype=torch.float32, device=device))
            if not private:
                self._fb_dev = buf
        lib().mel_filterbank(self.n_mels, self.n_fft, float(self.sr), float(fmin), float(fmax), buf[0].data_ptr(),
                             buf[1].data_ptr(), buf[2].data_ptr(), cap, torch.cuda.current_stream().cuda_stream)
        return buf[0], buf[1], buf[2], cap

    def forward(self, x, lengths=None):
        """x [B, N] -> log-mel [B, n_mels, 1 + (N - 1) // hopsize].

        lengths (eval only): each clip's sample count, a sequence of ints or a CPU integer tensor of length B, each
        between n_fft // 2 + 2 (the shortest waveform the call accepts) and N.  Clip b's frames t < num_frames(lengths)[b]
        then equal this module on x[b:b+1, :lengths[b]] alone (pre-emphasis and reflect padding end at the clip's own
        last sample); later frames are 0.0; samples at or past lengths[b] are never read.  The two torch.randint draws
        of every call happen once per call, not once per clip."""
        if not x.is_cuda:
            raise RuntimeError("efficientat_b200.AugmentMelSTFT runs on CUDA (sm_90a) only; got a CPU tensor")
        if x.dim() != 2:
            raise ValueError(f"expected waveform of shape [B, N], got {tuple(x.shape)}")
        if lengths is not None:
            if self.training:
                raise NotImplementedError("lengths: per-clip lengths are supported in eval() only")
            if x.requires_grad:
                raise NotImplementedError("lengths: per-clip lengths are not supported for a waveform that requires grad")
            lengths = check_lengths(lengths, x.shape[0], self.n_fft // 2 + 2, x.shape[1])
        check_module_tensors(self, x.device, "AugmentMelSTFT")
        with torch.cuda.device(x.device):
            if lengths is not None:
                n_valid = torch.tensor(lengths, dtype=torch.int32).to(x.device)
                return self._forward(x.float().contiguous(), n_valid=n_valid)
            if torch.is_grad_enabled() and x.requires_grad:
                return _MelFn.apply(self, x)
            return self._forward(x.float().contiguous())

    def num_frames(self, lengths):
        """each clip's frame count for sample counts `lengths`: 1 + (n - 1) // hopsize, the `lengths` the models take"""
        return [1 + (n - 1) // self.hopsize for n in as_int_list(lengths)]

    def _forward(self, x, saved=None, n_valid=None):
        """saved: a dict that receives the filterbank and masks of this call, for eat_mel_bwd.
        n_valid: int32 [B] on the device, each clip's sample count (eval only)"""
        # the reference draws both randints on every call, eval included (preprocess.py:45-46)
        fmin = self.fmin + torch.randint(self.fmin_aug_range, (1,)).item()
        fmax = self.fmax + self.fmax_aug_range // 2 - torch.randint(self.fmax_aug_range, (1,)).item()
        if not self.training:
            fmin, fmax = self.fmin, self.fmax
        if self.training and (self.fmin_aug_range > 1 or self.fmax_aug_range > 1):
            # jittered filterbank: build it on the device, no host work or copy in the step
            start, length, taps, max_len = self._device_filterbank(fmin, fmax, x.device, private=saved is not None)
        else:
            start, length, taps, max_len = self._filterbank(fmin, fmax, x.device)
        b, n = x.shape
        t = 1 + (n - 1) // self.hopsize
        out = torch.empty(b, self.n_mels, t, device=x.device, dtype=torch.float32)
        if n_valid is not None:
            lib().mel_fwd_len(x.data_ptr(), b, n, self.window.data_ptr(), self.win_length, self.hopsize, self.n_fft,
                              self._twiddle.data_ptr(), start.data_ptr(), length.data_ptr(), taps.data_ptr(), max_len,
                              self.n_mels, self._preemph, out.data_ptr(), n_valid.data_ptr(),
                              torch.cuda.current_stream().cuda_stream)
            return out
        lib().mel_fwd(x.data_ptr(), b, n, self.window.data_ptr(), self.win_length, self.hopsize, self.n_fft,
                      self._twiddle.data_ptr(), start.data_ptr(), length.data_ptr(), taps.data_ptr(), max_len,
                      self.n_mels, self._preemph, out.data_ptr(),
                      torch.cuda.current_stream().cuda_stream)
        if self.training:
            fm = self.freqm.draw(out) if isinstance(self.freqm, _AxisMasking) else None
            tm = self.timem.draw(out) if isinstance(self.timem, _AxisMasking) else None
            if fm is not None or tm is not None:
                z = torch.zeros(b, dtype=torch.int32, device=x.device)
                fs, fe = fm if fm is not None else (z, z)
                ts, te = tm if tm is not None else (z, z)
                # masks are applied in the log domain before the affine, i.e. value (0 + 4.5) / 5 = 0.9
                lib().mel_mask(out.data_ptr(), b, self.n_mels, t, fs.data_ptr(), fe.data_ptr(), ts.data_ptr(),
                               te.data_ptr(), 0.9, torch.cuda.current_stream().cuda_stream)
                if saved is not None:
                    saved["masks"] = (fs, fe, ts, te)
        if saved is not None:
            saved.update(fb=(start, length, taps, max_len))
        return out

    def _backward(self, x, dspec, saved):
        b, n = x.shape
        start, length, taps, max_len = saved["fb"]
        masks = saved.get("masks")
        L = lib()
        st = torch.cuda.current_stream().cuda_stream
        need = ctypes.c_longlong()
        L.mel_bwd_workspace(b, n, self.hopsize, self.n_fft, ctypes.addressof(need))
        work = torch.empty(need.value, device=x.device, dtype=torch.float32)
        dx = torch.empty_like(x)
        L.mel_bwd(dspec.data_ptr(), x.data_ptr(), b, n, self.window.data_ptr(), self.win_length, self.hopsize, self.n_fft,
                  self._twiddle.data_ptr(), start.data_ptr(), length.data_ptr(), taps.data_ptr(), max_len, self.n_mels,
                  self._preemph, *([m.data_ptr() for m in masks] if masks is not None else [0, 0, 0, 0]),
                  work.data_ptr(), work.numel(), dx.data_ptr(), st)
        return dx


class _MelFn(torch.autograd.Function):
    """waveform -> log-mel with the waveform's gradient from eat_mel_bwd (fp32; the frame spectra are recomputed)"""

    @staticmethod
    def forward(ctx, module, x):
        x = x.detach().float().contiguous()
        saved = {}
        out = module._forward(x, saved)
        ctx.module, ctx.x, ctx.saved = module, x, saved
        return out

    @staticmethod
    def backward(ctx, dspec):
        if torch.is_grad_enabled():
            raise NotImplementedError("double backward (create_graph=True) through AugmentMelSTFT is not implemented")
        with torch.cuda.device(ctx.x.device):
            dx = ctx.module._backward(ctx.x, dspec.float().contiguous(), ctx.saved)
        ctx.x = ctx.saved = None
        return None, dx
