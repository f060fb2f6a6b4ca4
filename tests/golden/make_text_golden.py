"""Generates tests/golden/text_frontend.json + tests/golden/lexicon_small.txt from the REFERENCE's own text
front end (needs a reference checkout named by VIETTTS_REFERENCE; the outputs are committed).

The reference modules cannot be imported (synthesizer.py parses argv at import, nat/config.py and text2mel.py
import jax/haiku), so the three pure-Python functions are lifted out of their source files with `ast` and
executed unchanged against a FLAGS namespace built from nat/config.py's own class body:
  nat_normalize_text   vietTTS/synthesizer.py:21-32
  load_lexicon         vietTTS/nat/text2mel.py:16-19
  text2tokens          vietTTS/nat/text2mel.py:37-58   (+ load_phonemes_set, data_loader.py:11-13)
"""
import ast
import json
import os
import re
import unicodedata
from argparse import Namespace
from pathlib import Path

REF = Path(os.environ.get("VIETTTS_REFERENCE", "vietTTS-reference"))   # a checkout of NTT123/vietTTS
OUT = Path(__file__).resolve().parent


def lift(path, names):
    src = path.read_text()
    tree = ast.parse(src)
    return "\n\n".join(ast.get_source_segment(src, n) for n in tree.body
                       if isinstance(n, (ast.FunctionDef, ast.ClassDef)) and n.name in names)


def main():
    ns = {"Namespace": Namespace, "Path": Path, "re": re, "unicodedata": unicodedata}
    exec(lift(REF / "vietTTS/nat/config.py", {"FLAGS"}), ns)
    exec(lift(REF / "vietTTS/nat/data_loader.py", {"load_phonemes_set"}), ns)
    exec(lift(REF / "vietTTS/nat/text2mel.py", {"load_lexicon", "text2tokens"}), ns)
    exec(lift(REF / "vietTTS/synthesizer.py", {"nat_normalize_text"}), ns)

    texts = [
        "Xin chào, tôi là trợ lý ảo.",
        "hôm nay trời đẹp quá! bạn có khỏe không?",
        'anh ấy nói: "đi thôi"... rồi đi mất',
        "  nhiều   khoảng trắng ,,, và dấu câu ;;; lạ !?  ",
        "dòng một\ndòng hai\n\ndòng ba.",
        "từlạkhôngcótrongtừđiển và z w f j",
        "từlạkhôngcótrongtừđiển và q-x 42",
        "sil sp spn",
        "ＡＢＣ ｆｕｌｌｗｉｄｔｈ １２３",
        "",
        "một . , : hai",
    ]
    full = ns["load_lexicon"](str(REF / "assets/infore/lexicon.txt"))
    words = set()
    norm = []
    for t in texts:
        n = ns["nat_normalize_text"](t)
        norm.append(n)
        words.update(n.split())
    # small lexicon: the entries the samples hit, minus a few deliberately left out to exercise the
    # letter-by-letter branch
    drop = {"khỏe", "mất"}
    lex_lines = [f"{w}\t{full[w]}" for w in sorted(words) if w in full and w not in drop]
    (OUT / "lexicon_small.txt").write_text("\n".join(lex_lines) + "\n")
    cases = []
    for t, n in zip(texts, norm):
        try:
            cases.append(dict(text=t, normalized=n, tokens=ns["text2tokens"](n, str(OUT / "lexicon_small.txt"))))
        except ValueError:   # a lexicon entry whose phoneme is outside the alphabet: the reference raises
            cases.append(dict(text=t, normalized=n, error="ValueError"))
    (OUT / "text_frontend.json").write_text(json.dumps(dict(
        phonemes=ns["load_phonemes_set"](), sil_index=ns["FLAGS"].sil_index, word_end_index=ns["FLAGS"].word_end_index,
        cases=cases), ensure_ascii=False, indent=1))
    print(f"{len(cases)} cases, {len(lex_lines)} lexicon entries")


if __name__ == "__main__":
    main()
