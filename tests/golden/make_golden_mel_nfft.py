"""Generate tests/golden/mel_nfft.npz by running the UNMODIFIED reference AugmentMelSTFT at every n_fft the fused
mel kernel supports (256, 512, 1024, 2048, 4096).

Run where a checkout of the original project exists (read-only), named by $EAT_REFERENCE_DIR:
    EAT_REFERENCE_DIR=<checkout> python tests/golden/make_golden_mel_nfft.py
tests/test_gpu_mel_nfft.py only reads the .npz file.  Inputs come from efficientat_b200.synth (seeded), so the GPU test
regenerates identical waveforms without the reference.

Per size, in eval mode: 1 s of noise (B = 2) and one ragged length (T not a multiple of a CTA's frames), plus the
reference's own fp32 error against the fp64 oracle on two 10 s noise clips at the same geometry (the bound of the GPU
test where the 5e-5 absolute bound is out of reach for an fp32 FFT).
"""
import contextlib
import io
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
REF = os.environ["EAT_REFERENCE_DIR"]
sys.path.insert(0, REPO)
from efficientat_b200.synth import synth_waveform  # noqa: E402
from oracle import mel_oracle  # noqa: E402

sys.path.insert(0, REF)
with contextlib.redirect_stdout(io.StringIO()):
    from models.preprocess import AugmentMelSTFT as RefMel  # noqa: E402

import warnings  # noqa: E402
warnings.filterwarnings("ignore")
torch.set_num_threads(8)

# (n_fft, win_length, hopsize, n_mels, sr) per supported FFT size; the GPU test reads them from the file
GEOMS = [(256, 256, 80, 64, 32000), (512, 400, 160, 128, 16000), (1024, 640, 160, 96, 16000),
         (2048, 800, 320, 256, 32000), (4096, 4096, 1024, 128, 32000)]


def main():
    res = {}
    for n_fft, win, hop, n_mels, sr in GEOMS:
        with contextlib.redirect_stdout(io.StringIO()):
            mel = RefMel(n_mels=n_mels, sr=sr, win_length=win, hopsize=hop, n_fft=n_fft)
        mel.eval()
        with torch.no_grad():
            y = mel(synth_waveform(2, sr, seed=31))
            n_rag = 5000 + n_fft - 1
            y_rag = mel(synth_waveform(1, n_rag, seed=32))
            x10 = synth_waveform(2, 10 * sr, seed=4)
            y10 = mel(x10)
        truth = mel_oracle.mel_forward(x10, n_mels=n_mels, sr=sr, win_length=win, hopsize=hop, n_fft=n_fft,
                                       fmax=float(sr // 2 - 1000), dtype=torch.float64)
        ref_err = (y10.double() - truth).abs().max().item()
        res[f"geom_{n_fft}"] = np.array([n_fft, win, hop, n_mels, sr])
        res[f"y_noise_{n_fft}"] = y.numpy()
        res[f"n_ragged_{n_fft}"] = np.array(n_rag)
        res[f"y_ragged_{n_fft}"] = y_rag.numpy()
        res[f"ref_err_10s_{n_fft}"] = np.array(ref_err)
        print("mel_nfft", n_fft, y.shape, y_rag.shape, "reference fp32 error on 10 s noise", ref_err)
    np.savez_compressed(os.path.join(HERE, "mel_nfft.npz"), **res)


if __name__ == "__main__":
    main()
