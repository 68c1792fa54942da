#!/usr/bin/env python
"""Extracts what segmentation needs from the reference into tests/golden/segmentation_kats.json (run by
hand: `python tests/golden/make_segmentation_kats.py RAV1E_CHECKOUT`).

Source (xiph/rav1e @ 564ae3b):
- src/quantize/tables.rs: `ac_qlookup_Q3_raw`, `ac_qlookup_10_Q3_raw`, `ac_qlookup_12_Q3_raw` (256 entries
  each), the AC quantizer tables `ac_q` / `select_ac_qi` index at 8, 10 and 12 bit;
- src/util/kmeans.rs:108-122: the reference's k-means tests `three_means` and `four_means` as
  [data, expected centroids].
The Rust source is parsed textually; nothing is executed.
"""
import json
import os
import re
import sys

REF = os.path.join(sys.argv[1] if len(sys.argv) > 1 else "rav1e", "src")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "segmentation_kats.json")


def table(src, name):
    body = src[src.index(f"const {name}: [u16; QINDEX_RANGE] = ["):]
    body = body[body.index("[", body.index("=")) + 1:body.index("];")]
    return [int(v) for v in re.findall(r"\d+", body)]


def main():
    tb = open(os.path.join(REF, "quantize", "tables.rs")).read()
    km = open(os.path.join(REF, "util", "kmeans.rs")).read()
    km = km[km.index("mod test"):]
    kats = []
    for data, want in re.findall(r"let mut data = \[([-\d,\s]+)\];.*?assert_eq!\(centroids, \[([-\d,\s]+)\]\)", km, re.S):
        kats.append([[int(v) for v in data.split(",") if v.strip()], [int(v) for v in want.split(",") if v.strip()]])
    out = {
        "source": "xiph/rav1e @ 564ae3b src/quantize/tables.rs (ac_qlookup_*_Q3_raw) and src/util/kmeans.rs:108-122, "
                  "extracted by tests/golden/make_segmentation_kats.py",
        "ac_qlookup_Q3": {str(bd): table(tb, name) for bd, name in
                          ((8, "ac_qlookup_Q3_raw"), (10, "ac_qlookup_10_Q3_raw"), (12, "ac_qlookup_12_Q3_raw"))},
        "kmeans": kats,
    }
    assert all(len(t) == 256 for t in out["ac_qlookup_Q3"].values()), out
    assert [len(k[1]) for k in kats] == [3, 4], kats
    with open(OUT, "w") as f:
        json.dump(out, f)
        f.write("\n")
    print("wrote", OUT)


if __name__ == "__main__":
    main()
