"""Windowed audio tagging (the reference's windowed_inference.py:12-127, class EATagger) with the windows BATCHED.

The reference walks the recording window by window: one mel call, one model call, one device -> host copy and one
host argsort per window (windowed_inference.py:100-120).  Here all windows of a recording (in chunks of `max_batch`)
go through ONE mel launch and ONE forward at batch = number of windows, sigmoid and top-k run on the device, and the
result comes back in a single copy.  Same constructor, same `tag_audio_window` signature, same result structure:

    [{'start': s, 'end': s, 'tags': [{'tag': name, 'probability': p} x 10]} per window]

Differences, both deliberate: there is no CPU path (this package has none), and the CUDA run is fp32 (the reference
wraps its CUDA loop in `autocast`, i.e. fp16 convolutions; this package's kernels ignore autocast).
"""
import numpy as np
import torch

from .helpers.utils import NAME_TO_WIDTH, load_labels
from .models.preprocess import AugmentMelSTFT
from .resample import Resample


def window_plan(n_samples, window, hop):
    """-> (n_windows, padded length) as windowed_inference.py:95-97 computes them (the last window is zero padded).  One
    deliberate difference: a recording shorter than `window - hop` samples still gets ONE zero-padded window, where the
    reference's formula yields zero (or a negative number of) windows and an empty result."""
    if window <= 0 or hop <= 0:
        raise ValueError("window_size and hop_length must be positive")
    n_windows = int(np.ceil((n_samples - window) / hop)) + 1
    if n_windows < 1:
        n_windows = 1
    return n_windows, n_windows * hop + window


class EATagger:
    def __init__(self, model_name=None, ensemble=None, device="cuda", sample_rate=32000, window_size=800, hop_size=320,
                 n_mels=128, labels=None, max_batch=256):
        if not str(device).startswith("cuda") or not torch.cuda.is_available():
            raise RuntimeError("efficientat_b200.windowed.EATagger runs on CUDA (sm_90a) only; there is no CPU path")
        self.device = torch.device(device if ":" in str(device) else "cuda:%d" % torch.cuda.current_device())
        self.sample_rate, self.window_size, self.hop_size, self.n_mels = sample_rate, window_size, hop_size, n_mels
        self.max_batch = int(max_batch)
        if ensemble is not None:
            from .models.ensemble import get_ensemble_model
            self.model = get_ensemble_model(ensemble)
        elif model_name is not None:
            if model_name.startswith("dymn"):
                from .models.dymn.model import get_model
            else:
                from .models.mn.model import get_model
            self.model = get_model(width_mult=NAME_TO_WIDTH(model_name), pretrained_name=model_name)
        else:
            raise ValueError("Please provide a model name or an ensemble of models")
        self.model.to(self.device).eval()
        self.mel = AugmentMelSTFT(n_mels=n_mels, sr=sample_rate, win_length=window_size, hopsize=hop_size)
        self.mel.to(self.device).eval()
        self.labels = list(labels) if labels is not None else load_labels()[0]
        self._resamplers = {}                                               # native rate -> Resample, built on first use

    # ------------------------------------------------------------------ device part
    @torch.no_grad()
    def window_probabilities(self, waveform, window_size=20.0, hop_length=10.0, sr=None):
        """waveform: 1-D (or [1, N]) float tensor / array at `sample_rate` -> (probabilities [n_windows, classes] on the
        device, window start samples, window length in samples).  sr: the waveform's own rate when it is not
        `sample_rate`; the whole recording is then resampled on the device once (efficientat_b200.resample, the semantics
        of scipy.signal.resample_poly) and windowed after, as librosa.core.load resamples the file before the reference
        cuts its windows."""
        w = torch.as_tensor(waveform, dtype=torch.float32).reshape(1, -1).to(self.device)
        if sr is not None and int(sr) != self.sample_rate:
            rs = self._resamplers.get(int(sr))
            if rs is None:
                rs = self._resamplers[int(sr)] = Resample(int(sr), self.sample_rate).to(self.device)
            w = rs(w)
        win, hop = int(window_size * self.sample_rate), int(hop_length * self.sample_rate)
        n_windows, padded = window_plan(w.shape[1], win, hop)
        w = torch.nn.functional.pad(w, (0, max(padded - w.shape[1], 0)))
        frames = w[0].unfold(0, win, hop)[:n_windows]                     # [n_windows, win] overlapping view
        probs = []
        for s in range(0, n_windows, self.max_batch):
            chunk = frames[s:s + self.max_batch].contiguous()
            spec = self.mel(chunk)                                          # one launch for the whole chunk
            logits = self.model(spec.unsqueeze(1))[0]
            probs.append(torch.sigmoid(logits.float().reshape(chunk.shape[0], -1)))
        return torch.cat(probs), [i * hop for i in range(n_windows)], win

    def tag_waveform(self, waveform, window_size=20.0, hop_length=10.0, top_k=10, sr=None):
        """sr: the waveform's rate when it is not `sample_rate` (see window_probabilities); the window times are in
        seconds either way"""
        probs, starts, win = self.window_probabilities(waveform, window_size, hop_length, sr=sr)
        k = min(top_k, probs.shape[1])
        p, idx = torch.topk(probs, k, dim=1)                                # descending, as argsort(preds)[::-1][:k]
        p, idx = p.cpu().numpy(), idx.cpu().numpy()                         # the recording's only device -> host copies
        name = (lambda c: self.labels[c]) if len(self.labels) > int(idx.max(initial=0)) else (lambda c: str(c))
        return [{"start": s / self.sample_rate, "end": (s + win) / self.sample_rate,
                 "tags": [{"tag": name(int(c)), "probability": float(q)} for c, q in zip(idx[i], p[i])]}
                for i, s in enumerate(starts)]

    # ------------------------------------------------------------------ the reference's entry point
    def tag_audio_window(self, audio_path, window_size=20.0, hop_length=10.0):
        """windowed_inference.py:73-127.  Decoding is the caller's library, as in the reference: `librosa.core.load`."""
        try:
            import librosa
        except ImportError as e:
            raise ImportError("tag_audio_window decodes with librosa.core.load like the reference; without librosa, load "
                              "the file yourself and call tag_waveform(samples, ...)") from e
        waveform, _ = librosa.core.load(audio_path, sr=self.sample_rate, mono=True)
        return self.tag_waveform(waveform, window_size, hop_length)
