"""Generates tests/golden/normalize_text_golden.json from the reference's own function
(`contriever/src/normalize_text.py::normalize` of the reference checkout named by REFERENCE_ROOT); the fixture it
writes is what the tests read, so the tests need no reference checkout.

  REFERENCE_ROOT=<reference checkout> python tests/golden/make_normalize_golden.py
"""
import importlib.util
import json
import os
import random

REL = "contriever/src/normalize_text.py"
HERE = os.path.dirname(os.path.abspath(__file__))


def main():
    spec = importlib.util.spec_from_file_location("ref_normalize_text", os.path.join(os.environ["REFERENCE_ROOT"], REL))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    # (1) every code point the reference changes, as {codepoint: replacement}
    changed = {}
    for cp in range(0x110000):
        if 0xD800 <= cp <= 0xDFFF:
            continue
        out = mod.normalize(chr(cp))
        if out != chr(cp):
            changed[str(cp)] = out
    # (2) strings: hand-picked interactions plus seeded random mixtures of affected and ordinary characters
    rng = random.Random(20260924)
    pool = [chr(int(c)) for c in changed] + list("abc XYZ 019 . , ' \" - / \t\n\r") + ["é", "ﬁ", "Ａ", "中", " . . . ", ". . ."]
    strings = ["", "plain ascii question?", "who wrote “the road” — and when…", "a\r\nb\x0bc\x0cd\x85e",
               "x . . . y", " . . .  . . . ", "… . . . …", "soft\xadhyphen", "1⁄2 − 3∕ 4", "it’s 5′ 10″",
               " .\x01 . . "]
    for _ in range(200):
        strings.append("".join(rng.choice(pool) for _ in range(rng.randint(1, 40))))
    cases = [[s, mod.normalize(s)] for s in strings]
    with open(os.path.join(HERE, "normalize_text_golden.json"), "w", encoding="utf-8") as f:
        json.dump({"source": REL, "changed_codepoints": changed, "cases": cases}, f, ensure_ascii=True, indent=0)
    print(f"{len(changed)} changed code points, {len(cases)} string cases")


if __name__ == "__main__":
    main()
