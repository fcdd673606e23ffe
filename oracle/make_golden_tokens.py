"""Token ids of the reference's own CLIP tokenizer (utils/clip_tokenizer.py) on 300 generated texts — mixed case, digits,
punctuation, apostrophe forms, runs of spaces, accented and non-Latin characters, emoji, html entities — stored with the
texts in tests/golden/clip_tokens_random.json for tests/test_oracle_cpu.py.

TEST INFRASTRUCTURE: imports the reference checkout (REF below), which needs its tokenizer's dependencies (ftfy, regex).

    python oracle/make_golden_tokens.py
"""
import importlib.util
import json
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
REF = Path("/root/reference")
WORDS = ["person", "Ferrari", "F40", "don't", "it's", "we'll", "I'M", "dog's", "naïve", "café", "Zürich", "北京", "мотоцикл", "🚗", "😀",
         "&amp;", "&lt;b&gt;", "3.14", "1080p", "a", "THE", "x-ray", "e-mail", "#tag", "@home", "100%", "(red)", "white/blue", "...",
         "  ", "\t", "van", "ladder", "night-time", "ＦＵＬＬ", "ﬁre", "o'clock", "10:30", "$5", "état", "straße"]


def random_texts(n=300, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        k = int(rng.integers(1, 9))
        out.append(" ".join(WORDS[int(i)] for i in rng.integers(0, len(WORDS), k)))
    return out


def main():
    spec = importlib.util.spec_from_file_location("_ref_clip_tokenizer", REF / "utils" / "clip_tokenizer.py")
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    rt = ref.SimpleTokenizer()
    pairs = [[t, rt.encode(t)] for t in random_texts()]
    with open(ROOT / "tests" / "golden" / "clip_tokens_random.json", "w", encoding="utf-8") as f:
        json.dump(pairs, f, ensure_ascii=False)


if __name__ == "__main__":
    main()
