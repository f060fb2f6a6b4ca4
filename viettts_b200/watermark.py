"""Watermark detection from the command line (`python -m viettts_b200.watermark detect --key K [--key ...] FILE.wav ...`).

Reads each WAV file the synthesizer writes (16-bit PCM, or 8-bit G.711 mu-law or A-law from --encoding, expanded on the
device by Engine.decode; any rate the resampler reaches from 16 kHz), scores it against every key on the device
(Engine.detect_watermark) and prints one line per file and key: the score z, the offset in
16 kHz samples where the file's first sample sits in the mark's 4.096 s period, and the verdict.  Search mode (the
default) finds the mark wherever a crop starts and calls z >= 6.5 marked; `--aligned` scores only offset 0, for files
that start where the mark started, and calls z >= 5 marked.  For audio without the key either verdict is wrong with
probability at most 7e-7 or 3.7e-6 per file and key.  Exits 0 when every file carries at least one of the keys, 1 when
one does not, 2 on a usage error.
"""
from __future__ import annotations

import argparse
from pathlib import Path


def main(argv=None) -> int:
    parser = argparse.ArgumentParser(prog="python -m viettts_b200.watermark", description=__doc__.split("\n\n")[0])
    sub = parser.add_subparsers(dest="cmd", required=True)
    det = sub.add_parser("detect", help="score WAV files against one or more keys")
    det.add_argument("--key", action="append", required=True, help="a key in [0, 2^64) (repeat for several keys)")
    det.add_argument("--aligned", action="store_true", help="score offset 0 only (threshold 5 instead of 6.5)")
    det.add_argument("files", nargs="+", type=Path, metavar="FILE.wav")
    args = parser.parse_args(argv)

    from .engine import get_engine, watermark_keys
    from .synthesizer import read_wav_codes
    try:
        keys = watermark_keys(args.key)
    except ValueError as e:
        parser.error(f"--key: {e}")
    eng = get_engine()
    all_marked = True
    for fn in args.files:
        try:
            codes, rate, encoding = read_wav_codes(fn)
        except (OSError, ValueError):
            parser.error(f"{fn}: not a mono 16-bit PCM, mu-law or A-law WAV file")
        wav = eng.decode(codes, encoding)
        r = eng.detect_watermark(wav, keys, rate=rate, search=not args.aligned)
        for k, z, off, hit in zip(keys, r.z, r.offset, r.detected):
            print(f"{fn}\tkey={int(k)}\tz={float(z):.2f}\toffset={int(off)}\t{'marked' if hit else 'not marked'}")
        all_marked &= bool(r.detected.any())
    return 0 if all_marked else 1


if __name__ == "__main__":
    raise SystemExit(main())
