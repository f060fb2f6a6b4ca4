"""Drop-in for `MelFilter` of vietTTS/nat/dsp.py:104-128.

MelFilter(sample_rate, n_fft, n_mels, fmin, fmax)(y): y f32 [B,S] in [-1,1) ->
log-mel f32 [B,S/256,80].  The filterbank is the librosa-compatible Slaney bank
(viettts_b200.weights.mel_filterbank); the STFT + filterbank + log run in the
sm_90a melspec kernel."""
from __future__ import annotations

import numpy as np

from .. import config
from ..engine import get_engine
from ..weights import mel_filterbank


class MelFilter:
    def __init__(self, sample_rate: int, n_fft: int, n_mels: int, fmin=0.0, fmax=8000, engine=None):
        if (n_fft, n_mels) != (config.N_FFT, config.MEL_DIM):
            raise ValueError(f"the melspec kernel is specialised on n_fft={config.N_FFT}, n_mels={config.MEL_DIM}")
        self.melfb = mel_filterbank(sample_rate, n_fft, n_mels, fmin, fmax)
        self.n_fft = n_fft
        self._engine = engine

    def __call__(self, y) -> np.ndarray:
        y = np.asarray(y, dtype=np.float32)
        assert len(y.shape) == 2          # dsp.py:118
        eng = self._engine or get_engine()
        eng.load_mel_filterbank(self.melfb)
        return eng.melspec(y)
