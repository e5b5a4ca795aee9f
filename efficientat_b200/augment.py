"""Waveform augmentation of the training datasets on the device: gain, roll and waveform mixing, the `--gain_augment`,
`--roll` and `--wavmix` of the reference's scripts (ex_esc50.py:64-66, ex_dcase20.py:65-67, ex_fsd50k.py:64-66,
ex_openmic.py:64-66, ex_audioset.py:73-74).  In the reference they run in the `Dataset`, item by item, on the CPU:

    gain   pydub_augment / gain_augment_func: g = torch.randint(2G) - G dB, x *= 10^(g/20); no draw when G == 0
    roll   PreprocessDataset(get_roll_func()): s = np.random.random_integers(-R, R), out[n] = x[(n - s) mod N]
    wavmix MixupDataset: with probability `rate` a partner idx2 = torch.randint(len(dataset)) with its own gain and
           roll, l = max(l, 1 - l) with l ~ np.random.beta(beta, beta), x = l (x1 - mean x1) + (1 - l)(x2 - mean x2),
           x -= mean x, and the labels blended with l

`WaveAugment.draw` makes these draws on the host, from the global torch and numpy generators in the order a
`num_workers=0` DataLoader over the reference's wrapped dataset makes them (it differs between datasets, KINDS).
The kernels of csrc/wave_aug.cu apply them: `eat_wave_aug` writes the augmented batch that the mel front end reads,
`eat_label_mix` the matching labels.

Two sources feed the same kernel:
  store  `source` [S, N] fp32 on the device holds the un-augmented training clips (decoded once, e.g. from the
         reference's `get_training_set(roll=False, wavmix=False, gain_augment=0)`) and `labels` their targets; a step
         then takes the batch's dataset indices, and a partner is drawn from the whole set, as in the reference.
  batch  without a store, a step's own `wave` [B, N] and `y` are the source: the partner is another item of the
         SAME BATCH (torch.randint(B)), not of the dataset.  This deviates from the reference, and is what fits data
         that is too large to hold on the device (AudioSet).
"""
import numpy as np
import torch

from ._lib import lib

# order of the draws of one item: "g" gain, "r" roll, "c" the mixing coin, "m" the partner (index, its own gain and
# roll, then the beta draw)
KINDS = {
    "esc50": "c" + "gr" + "m",        # esc50.py:56-69 (gain in AudioSetDataset.__getitem__, roll in PreprocessDataset)
    "fsd50k": "c" + "gr" + "m",       # fsd50k.py:79-92
    "audioset": "c" + "gr" + "m",     # audioset.py:75-88
    "openmic": "gr" + "c" + "m",      # openmic.py:73-95: the primary item is read before the coin
    "dcase20": "rg" + "c" + "m",      # dcase20.py:99-118, 123-129: roll wraps the base set, gain wraps the roll
}
DCASE20_CLASSES = 10                  # dcase20.py:92, MixupDataset(num_classes=10)

LABEL_PLAIN, LABEL_ONEHOT, LABEL_OPENMIC = 0, 1, 2          # EAT_LABEL_* of include/eat_b200.h
_INT32_MAX = 2 ** 31 - 1


def _stream():
    return torch.cuda.current_stream().cuda_stream


class WaveAugment:
    """Gain, roll and waveform mixing of dataset `kind` (one of KINDS), applied inside the trainers' step
    (`AudioSetTrainer(..., augment=...)`, `FineTuneTrainer(..., augment=...)`) before the mel.

    gain_augment  G: an integer gain in [-G, G-1] dB per item (0: none, and no draw)
    roll          a circular shift in [-shift_range, shift_range] samples per item
    wavmix        mix with a partner item with probability `rate`, weight max(l, 1 - l) for l ~ Beta(beta, beta)
    source        optional store [S, N] fp32 CUDA tensor of un-augmented clips, with `labels` [S, C] fp32 rows (for
                  "dcase20": [S] integer class indices).  `source` is read, never written, and must not change while
                  this object uses it: its per-clip sums are taken once, here.
    """

    def __init__(self, kind, gain_augment=0, roll=False, wavmix=False, shift_range=4000, rate=0.5, beta=2,
                 source=None, labels=None):
        if kind not in KINDS:
            raise ValueError(f"WaveAugment: kind must be one of {tuple(KINDS)}, got {kind!r}")
        if int(gain_augment) != gain_augment or gain_augment < 0:
            raise ValueError(f"WaveAugment: gain_augment must be a non-negative integer, got {gain_augment!r}")
        if int(shift_range) != shift_range or not 0 <= shift_range <= _INT32_MAX // 2:
            raise ValueError(f"WaveAugment: shift_range must be a non-negative integer, got {shift_range!r}")
        if not beta > 0:
            raise ValueError(f"WaveAugment: beta must be positive, got {beta!r}")
        self.kind, self.order = kind, KINDS[kind]
        self.gain_augment, self.roll, self.wavmix = int(gain_augment), bool(roll), bool(wavmix)
        self.shift_range, self.rate, self.beta = int(shift_range), float(rate), beta
        self.source = self.labels = self.sums = None
        if source is not None:
            self._set_store(source, labels)
        elif labels is not None:
            raise ValueError("WaveAugment: labels given without a source")

    def _set_store(self, source, labels):
        if not (source.is_cuda and source.dtype == torch.float32 and source.dim() == 2 and source.is_contiguous()):
            raise ValueError("WaveAugment: source must be a contiguous [S, N] fp32 CUDA tensor, got "
                             f"{source.dtype} {tuple(source.shape)} on {source.device}")
        S, N = source.shape
        if S < 1 or N < 1:
            raise ValueError(f"WaveAugment: source must hold at least one sample, got {tuple(source.shape)}")
        if labels is None or labels.device != source.device or labels.shape[0] != S:
            raise ValueError(f"WaveAugment: labels must be a tensor on {source.device} with S = {S} rows")
        self.source = source
        self.labels = self._check_labels(labels)
        self.sums = torch.empty(S, device=source.device, dtype=torch.float64)
        with torch.cuda.device(source.device):
            lib().clip_sum(source.data_ptr(), S, N, self.sums.data_ptr(), _stream())

    def _check_labels(self, y):
        if self.kind == "dcase20":
            if y.dim() != 1 or y.is_floating_point():
                raise ValueError(f"WaveAugment('dcase20'): labels are [S] integer class indices, got {y.dtype} "
                                 f"{tuple(y.shape)}")
            return y.to(torch.int32).contiguous()
        if y.dim() != 2 or not y.is_floating_point():
            raise ValueError(f"WaveAugment({self.kind!r}): labels are [S, C] float rows, got {y.dtype} {tuple(y.shape)}")
        if self.kind == "openmic" and y.shape[1] % 2:
            raise ValueError(f"WaveAugment('openmic'): labels are [S, 2C] (scores | mask), got {tuple(y.shape)}")
        return y.to(torch.float32).contiguous()

    # ------------------------------------------------------------------ host draws
    def _item(self):
        """gain (dB) and shift of one item, drawn in this dataset's order"""
        g = s = 0
        for op in self.order:
            if op == "g" and self.gain_augment:
                g = torch.randint(self.gain_augment * 2, (1,)).item() - self.gain_augment
            elif op == "r" and self.roll:
                # np.random.random_integers(-R, R) is randint(-R, R + 1) (same stream), without its deprecation warning
                s = int(np.random.randint(-self.shift_range, self.shift_range + 1))
        return g, s

    def draw(self, indices, n_items):
        """The draws of one batch: `indices` [B] are the items' dataset indices (or batch positions without a store),
        partners are drawn from range(n_items).  Consumes torch's and numpy's global generators exactly as the
        reference's wrapped dataset does for these items, in order.  -> dict of CPU tensors [B]: idx1, idx2 (-1: not
        mixed), shift1, shift2, gain1, gain2 (int64; gains in dB), lam (fp64; 1 where not mixed)."""
        idx1 = torch.as_tensor(indices, dtype=torch.int64).reshape(-1)
        B = idx1.numel()
        d = {"idx1": idx1, "idx2": torch.full((B,), -1, dtype=torch.int64),
             "shift1": torch.zeros(B, dtype=torch.int64), "shift2": torch.zeros(B, dtype=torch.int64),
             "gain1": torch.zeros(B, dtype=torch.int64), "gain2": torch.zeros(B, dtype=torch.int64),
             "lam": torch.ones(B, dtype=torch.float64)}
        for b in range(B):
            coin = False
            for op in self.order:
                if op == "c":
                    coin = self.wavmix and bool(torch.rand(1) < self.rate)
                elif op == "g":                      # "gr" / "rg": the item's two draws, in the dataset's order
                    d["gain1"][b], d["shift1"][b] = self._item()
                elif op == "m" and coin:
                    d["idx2"][b] = torch.randint(n_items, (1,)).item()
                    d["gain2"][b], d["shift2"][b] = self._item()
                    l = np.random.beta(self.beta, self.beta)
                    d["lam"][b] = max(l, 1. - l)
        return d

    # ------------------------------------------------------------------ device
    def check_draws(self, d, B, S):
        """the draws of a B-item batch over S source clips, as `draw` returns them (or given by the caller)"""
        for k in ("idx1", "idx2", "shift1", "shift2", "gain1", "gain2", "lam"):
            if k not in d or torch.as_tensor(d[k]).shape != (B,):
                raise ValueError(f"WaveAugment: draws[{k!r}] must be a [{B}] tensor")
        idx1, idx2 = torch.as_tensor(d["idx1"]), torch.as_tensor(d["idx2"])
        if bool(((idx1 < 0) | (idx1 >= S)).any()) or bool(((idx2 < -1) | (idx2 >= S)).any()):
            raise ValueError(f"WaveAugment: idx1 must lie in [0, {S}) and idx2 in [-1, {S})")
        for k in ("shift1", "shift2"):
            if bool((torch.as_tensor(d[k]).abs() > self.shift_range).any()):
                raise ValueError(f"WaveAugment: {k} must lie in [-{self.shift_range}, {self.shift_range}]")
        lam = torch.as_tensor(d["lam"], dtype=torch.float64)
        gains = torch.cat([torch.as_tensor(d["gain1"]), torch.as_tensor(d["gain2"])]).double()
        if not bool(((lam >= 0) & (lam <= 1)).all()) or not bool(torch.isfinite(gains).all()) or bool((gains.abs() > 200).any()):
            raise ValueError("WaveAugment: lam must lie in [0, 1] and gains in [-200, 200] dB")

    def __call__(self, wave, y, draws=None):
        """-> (augmented waveforms [B, N] fp32, labels) on the device, launched on the current stream.

        store:  `wave` is the [B] dataset indices (CPU integers) and `y` must be None; labels come from the store.
        batch:  `wave` [B, N] (or [B, 1, N]) fp32 CUDA waveforms and `y` their labels ([B, C], or [B] class indices
                for "dcase20").
        `draws` (optional): the dict `draw` returns, to replace the draw.  The labels are fp32 [B, C] blended rows,
        except for "dcase20" without wavmix, whose class indices pass through."""
        if self.source is not None:
            if y is not None:
                raise ValueError("WaveAugment: with a store the step takes dataset indices and no y")
            idx = torch.as_tensor(wave)
            if idx.is_floating_point() or idx.dim() != 1 or idx.is_cuda:
                raise ValueError("WaveAugment: with a store the step takes [B] CPU integer dataset indices")
            src, labels, sums = self.source, self.labels, self.sums
            S = src.shape[0]
            B = idx.numel()
            if draws is None:
                draws = self.draw(idx, S)
            elif not torch.equal(torch.as_tensor(draws["idx1"]).reshape(-1), idx.to(torch.int64)):
                raise ValueError("WaveAugment: draws['idx1'] must equal the step's dataset indices")
        else:
            if not (wave.is_cuda and wave.dtype == torch.float32):
                raise ValueError(f"WaveAugment: wave must be an fp32 CUDA tensor, got {wave.dtype} on {wave.device}")
            B = wave.shape[0]
            src = wave.reshape(B, -1).contiguous()
            S = B
            if y is None or y.shape[0] != B or y.device != src.device:
                raise ValueError(f"WaveAugment: y must be a tensor on {src.device} with B = {B} rows")
            labels = self._check_labels(y)
            if draws is None:
                draws = self.draw(range(B), B)
            sums = None
        self.check_draws(draws, B, S)
        dev = src.device
        N = src.shape[1]
        ints = torch.stack([torch.as_tensor(draws[k], dtype=torch.int64) for k in ("idx1", "idx2", "shift1", "shift2")])
        gains = 10.0 ** (torch.stack([torch.as_tensor(draws[k], dtype=torch.float64) for k in ("gain1", "gain2")]) / 20.0)
        floats = torch.cat([gains, torch.as_tensor(draws["lam"], dtype=torch.float64)[None]])
        di = ints.to(torch.int32).to(dev, non_blocking=True)
        df = floats.to(torch.float32).to(dev, non_blocking=True)
        L, st = lib(), _stream()
        mixed = bool((torch.as_tensor(draws["idx2"]) >= 0).any())
        if mixed and sums is None:
            sums = torch.empty(S, device=dev, dtype=torch.float64)
            L.clip_sum(src.data_ptr(), S, N, sums.data_ptr(), st)
        out = torch.empty(B, N, device=dev, dtype=torch.float32)
        L.wave_aug(src.data_ptr(), sums.data_ptr() if sums is not None else 0, S, N, di[0].data_ptr(), di[1].data_ptr(),
                   di[2].data_ptr(), di[3].data_ptr(), df[0].data_ptr(), df[1].data_ptr(), df[2].data_ptr(),
                   out.data_ptr(), B, st)
        if self.kind == "dcase20" and not self.wavmix:        # dcase20.py: index targets unless wavmix one-hots them
            return out, labels.index_select(0, di[0].long())
        C = DCASE20_CLASSES if self.kind == "dcase20" else labels.shape[1]
        rule = LABEL_ONEHOT if self.kind == "dcase20" else LABEL_OPENMIC if self.kind == "openmic" else LABEL_PLAIN
        y_out = torch.empty(B, C, device=dev, dtype=torch.float32)
        L.label_mix(rule, labels.data_ptr() if rule != LABEL_ONEHOT else 0, labels.data_ptr() if rule == LABEL_ONEHOT else 0,
                    S, C, di[0].data_ptr(), di[1].data_ptr(), df[2].data_ptr(), B, y_out.data_ptr(), st)
        return out, y_out
