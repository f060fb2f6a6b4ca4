"""Drop-in for vietTTS/hifigan/mel2wave.py:20-41.

Same name, argument and return conventions as the reference: `mel2wave(mel)`
takes an array-like f32 [B,T,80] (B=1 from the CLI), reads the generator config
and the Haiku-layout checkpoint from the same cwd-relative paths, and returns a
numpy float32 waveform, squeezed ([256*T] for B=1), in (-1,1).  Differences: the
forward runs on the sm_90a kernels, and the parsed checkpoint is cached per
(path, mtime, size) instead of being re-read on every call."""
from __future__ import annotations

import json
import os

import numpy as np

from .. import config
from ..engine import get_engine
from ..weights import load_pickle

CONFIG_FILE = config.HIFIGAN_CONFIG_FILE   # "assets/hifigan/config.json"   (mel2wave.py:21)
CKPT_FILE = config.HIFIGAN_CKPT            # FLAGS.ckpt_dir / "hk_hifi.pickle" (mel2wave.py:35)


def _file_key(path):
    st = os.stat(path)
    return (str(path), st.st_mtime_ns, st.st_size)


def load_generator(engine=None, config_file=None, ckpt_file=None):
    engine = engine or get_engine()
    config_file = config_file or CONFIG_FILE
    ckpt_file = ckpt_file or CKPT_FILE
    key = (_file_key(config_file), _file_key(ckpt_file))
    if engine._hifigan_key != key:
        with open(config_file) as f:
            config.check_hifigan_config(json.loads(f.read()))
        engine.load_hifigan(load_pickle(ckpt_file), key=key)
    return engine


def mel2wave(mel):
    engine = load_generator()
    mel = np.asarray(mel, dtype=np.float32)
    if mel.ndim == 2:
        mel = mel[None]
    wav = engine.mel2wave(mel)
    return np.squeeze(wav)
