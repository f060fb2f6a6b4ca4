"""CPU oracle for the vietTTS hot path.  TEST INFRASTRUCTURE -- NOT PRODUCT CODE.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline /
`--impl reference` legs may import this package, and there only as the checker
(or the timed CPU baseline), never as the thing shipped.  Nothing under
`viettts_b200/` imports it; the product path fails loudly when the CUDA library
is missing.

What each module restates (file:line into the reference tree, NTT123/vietTTS):

  hifigan_oracle.py  vietTTS/hifigan/model.py:8-125 (Generator, ResBlock1, get_padding)
                     PINNED: checked against the reference's own importable torch
                     implementation vietTTS/hifigan/torch_model.py:156-209 through the
                     reference's own converter convert_torch_model_to_haiku.py:27-62
                     (tests/golden/make_golden.py, fixtures in tests/golden/).
  nat_oracle.py      vietTTS/nat/model.py:9-47,76-144 and nat/text2mel.py:61-82; also the callers of the
                     path: DurationModel (model.py:49-70), the text2mel duration fix-ups
                     (text2mel.py:85-103), the teacher-forced pass with zoneout
                     (model.py:146-169) and the GTA forward (gta.py:28-41).
                     PINNED TO THE REFERENCE'S OWN SOURCE (wiring), third-party primitives restated:
                     jax / dm-haiku cannot be installed on either box
                     and the reference's tests hold no golden vectors for this path, so the golden
                     vectors come from EXECUTING the unmodified vietTTS/nat/{model,text2mel,gta}.py with
                     numpy stand-ins for the jax / haiku API surface they touch (tests/refshim,
                     tests/golden/make_nat_golden.py -> tests/golden/nat_ref_*.npz, including the masks
                     the reference draws from the checkpoint rng).  tests/test_reference_goldens.py holds
                     this restatement to those vectors at float64 (<= 3e-5), i.e. the concat orders,
                     BN-before-tanh, residuals, ResetCore mask, zoneout tree order, seconds->frames and
                     the Haiku parameter names are pinned.  What stays a restatement is the third-party
                     primitives inside the shim (hk.LSTM, hk.Conv1D, hk.BatchNorm, jax.nn.*, threefry):
                     each is cross-checked against torch's independent operator
                     (tests/test_oracle_crosschecks.py) and the rng against Random123 / JAX-documented
                     known answers (tests/test_refshim_rng.py).
  mel_oracle.py      vietTTS/nat/dsp.py:11-25,65-128 (rolling_window, batched_stft,
                     MelFilter).  Pinned the same way: the reference's dsp.py runs unmodified on the
                     shim (numpy fft, librosa.filters.mel restated from its published algorithm) and
                     tests/test_reference_goldens.py compares; additionally cross-checked against
                     torch.stft and torchaudio's Slaney filterbank (independent implementations).
"""
