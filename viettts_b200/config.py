"""Constants of the hot path, mirrored from the reference.

Sources (all in /root/reference):
  * vietTTS/nat/config.py:8-59          (FLAGS: dims, dsp constants, alphabet)
  * assets/hifigan/config.json:2-28     (generator hyper-parameters)

The CUDA library is specialised on these values (see csrc/vtts_config.h); the
Python side validates any user-supplied config.json against them and raises if
they differ, instead of silently running a different model.
"""
from __future__ import annotations

from pathlib import Path

# ---- vietTTS/nat/config.py:43-47 (dsp) ------------------------------------
MEL_DIM = 80
N_FFT = 1024
HOP = N_FFT // 4            # 256, mel2wave total upsampling 8*8*2*2
SAMPLE_RATE = 16000
FMIN = 0.0
FMAX = 8000.0

# ---- vietTTS/nat/config.py:11-17 (model dims) ------------------------------
VOCAB_SIZE = 256
DURATION_LSTM_DIM = 256
ACOUSTIC_ENCODER_DIM = 256   # BiLSTM -> 2*256 = 512 conditioning channels
ACOUSTIC_DECODER_DIM = 512
POSTNET_DIM = 512
PRENET_DIM = 256             # hk.Linear(256) x2, vietTTS/nat/model.py:88-89
ENC_OUT_DIM = 2 * ACOUSTIC_ENCODER_DIM

# ---- vietTTS/nat/config.py:25-40 (alphabet) --------------------------------
SPECIAL_PHONEMES = ["sil", "sp", "spn", " "]
SIL_INDEX = 0
WORD_END_INDEX = 3
N_NORMAL_PHONEMES = 89       # len(FLAGS._normal_phonemes)
ALPHABET_SIZE = len(SPECIAL_PHONEMES) + N_NORMAL_PHONEMES  # 93
# the 89 letters of FLAGS._normal_phonemes, in the reference's order (token id = 4 + position)
NORMAL_PHONEMES = list(
    "abcdeghiklmnopqrstuvxy"
    "àáâãèéêìíòóôõùúýăđĩũơư"
    "ạảấầẩẫậắằẳẵặẹẻẽếềểễệỉịọỏốồổỗộớờởỡợụủứừửữựỳỵỷỹ"
)
assert len(NORMAL_PHONEMES) == N_NORMAL_PHONEMES
PHONEMES = SPECIAL_PHONEMES + NORMAL_PHONEMES   # data_loader.py:11-13 load_phonemes_set()

# ---- assets/hifigan/config.json --------------------------------------------
HIFIGAN = dict(
    resblock="1",
    upsample_rates=[8, 8, 2, 2],
    upsample_kernel_sizes=[16, 16, 4, 4],
    upsample_initial_channel=512,
    resblock_kernel_sizes=[3, 7, 11],
    resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]],
    num_mels=80,
    hop_size=256,
    sampling_rate=16000,
)
HIFIGAN_KEYS_CHECKED = tuple(HIFIGAN.keys())

# default checkpoint locations, cwd-relative exactly like the reference
# (vietTTS/hifigan/mel2wave.py:21, vietTTS/hifigan/config.py:6, vietTTS/nat/config.py:58)
HIFIGAN_CONFIG_FILE = Path("assets/hifigan/config.json")
HIFIGAN_CKPT = Path("assets/infore/hifigan/hk_hifi.pickle")
ACOUSTIC_CKPT = Path("assets/infore/nat/acoustic_latest_ckpt.pickle")
DURATION_CKPT = Path("assets/infore/nat/duration_latest_ckpt.pickle")   # text2mel.py:27
LEXICON_FILE = Path("train_data/lexicon.txt")                           # text2mel.py:86 (FLAGS.data_dir / "lexicon.txt")

# analytical work figures (SURVEY.md §8d / BASELINE.md §3) used by bench.py
HIFIGAN_MAC_PER_FRAME = 307_052_544
HIFIGAN_FLOP_PER_FRAME = 2 * HIFIGAN_MAC_PER_FRAME
HIFIGAN_IO_BYTES_PER_FRAME = (80 + 256) * 4
HIFIGAN_PARAMS = 13_926_017


def check_hifigan_config(cfg: dict) -> None:
    """Raise ValueError if a config.json describes a generator other than the
    one the kernels are specialised on."""
    for k in HIFIGAN_KEYS_CHECKED:
        if k in cfg and cfg[k] != HIFIGAN[k]:
            raise ValueError(
                f"hifigan config key {k!r}={cfg[k]!r} differs from the value the "
                f"sm_90a kernels are specialised on ({HIFIGAN[k]!r})"
            )
