#!/usr/bin/env python
"""Extracts the reference's known-answer vectors for the logexp helpers temporal RDO uses into
tests/golden/logexp_kats.json (run by hand: `python tests/golden/make_logexp_kats.py RAV1E_CHECKOUT`).

Source (xiph/rav1e @ 564ae3b): src/util/logexp.rs:292-302, `blog64_vectors` and `bexp64_vectors`.
bexp64 rows are [input, expected, tolerance]: 0 means exact, otherwise |got - expected| < tolerance, as
the reference asserts.  The Rust test code is parsed textually; nothing is executed.
"""
import json
import os
import re
import sys

REF = os.path.join(sys.argv[1] if len(sys.argv) > 1 else "rav1e", "src")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "logexp_kats.json")
NUM = r"(0x[0-9a-fA-F]+|\d+)"


def main():
    lx = open(os.path.join(REF, "util", "logexp.rs")).read()
    lx = lx[lx.index("fn blog64_vectors"):lx.index("fn blog64_bexp64_round_trip")]
    out = {
        "source": "xiph/rav1e @ 564ae3b src/util/logexp.rs:292-302, extracted by tests/golden/make_logexp_kats.py",
        "blog64": [[int(a, 0), int(b, 0)] for a, b in re.findall(r"blog64\(" + NUM + r"\)\s*==\s*" + NUM, lx)],
        "bexp64": [[int(a, 0), int(b, 0), 0] for a, b in re.findall(r"assert!\(bexp64\(" + NUM + r"\)\s*==\s*" + NUM, lx)]
        + [[int(a, 0), int(b, 0), int(t)] for a, b, t in
           re.findall(r"\(bexp64\(" + NUM + r"\)\s*-\s*" + NUM + r"\)\.abs\(\)\s*<\s*(\d+)", lx)],
    }
    assert len(out["blog64"]) == 2 and len(out["bexp64"]) == 2, out
    with open(OUT, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
