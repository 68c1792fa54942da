#!/usr/bin/env python
"""Extracts what the coefficient rate needs from the reference into tests/golden/coeff_cdf_kats.json (run by
hand: `python tests/golden/make_coeff_cdf_kats.py RAV1E_CHECKOUT`).

Source (xiph/rav1e @ 564ae3b):
- src/token_cdfs.rs: the default coefficient CDFs of the four q contexts (`av1_default_*_cdfs`, selected by
  CDFContext::new, context/cdf_context.rs:103-108 and :152-168);
- src/entropymode.rs: the default tx-type CDFs (`default_{intra,inter}_tx_*_cdf`, cdf_context.rs:124-128);
- sha256 digests of the context and tx-set tables (context/transform_unit.rs:36-58, :272-310, :316-508, and
  the `skip_contexts` / `dc_sign_contexts` tables of get_txb_ctx, context/block_unit.rs:450-498), each as
  the little-endian int32 bytes of its values in row-major order.
The CDFs are stored in b200_coeff_cdfs field order (include/b200rdo.h), converted as util/cdf.rs:10-25 does:
each listed value v becomes 32768 - v, and the last slot (the adaptation count) is 0.
The Rust source is parsed textually; nothing is executed.
"""
import hashlib
import json
import os
import re
import struct
import sys

REF = os.path.join(sys.argv[1] if len(sys.argv) > 1 else "rav1e", "src")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "coeff_cdf_kats.json")

# b200_coeff_cdfs fields: (name, dims without the q context, N) -> reference table
TOKEN_FIELDS = [("txb_skip", (5, 13), 2, "av1_default_txb_skip_cdfs"),
                ("dc_sign", (2, 3), 2, "av1_default_dc_sign_cdfs"),
                ("eob_extra", (5, 2, 9), 2, "av1_default_eob_extra_cdfs"),
                ("eob_flag16", (2, 2), 5, "av1_default_eob_multi16_cdfs"),
                ("eob_flag32", (2, 2), 6, "av1_default_eob_multi32_cdfs"),
                ("eob_flag64", (2, 2), 7, "av1_default_eob_multi64_cdfs"),
                ("eob_flag128", (2, 2), 8, "av1_default_eob_multi128_cdfs"),
                ("eob_flag256", (2, 2), 9, "av1_default_eob_multi256_cdfs"),
                ("eob_flag512", (2, 2), 10, "av1_default_eob_multi512_cdfs"),
                ("eob_flag1024", (2, 2), 11, "av1_default_eob_multi1024_cdfs"),
                ("coeff_base_eob", (5, 2, 4), 3, "av1_default_coeff_base_eob_multi_cdfs"),
                ("coeff_base", (5, 2, 42), 4, "av1_default_coeff_base_multi_cdfs"),
                ("coeff_br", (5, 2, 21), 4, "av1_default_coeff_lps_multi_cdfs")]
TX_FIELDS = [("intra_tx_1", (4, 13), 7, "default_intra_tx_1_cdf"),
             ("intra_tx_2", (4, 13), 5, "default_intra_tx_2_cdf"),
             ("inter_tx_1", (4,), 16, "default_inter_tx_1_cdf"),
             ("inter_tx_2", (4,), 12, "default_inter_tx_2_cdf"),
             ("inter_tx_3", (4,), 2, "default_inter_tx_3_cdf")]


def prod(t):
    n = 1
    for v in t:
        n *= v
    return n


def cdf_values(src, name):
    """The listed values of `pub static NAME ... = cdf_Nd([...]);`, products such as `128 * 125` evaluated."""
    body = src[src.index(f"pub static {name}:"):]
    body = body[re.search(r"=\s*cdf", body).start():]
    body = body[body.index("(") + 1:body.index("]);")]
    return [eval(e) for e in re.findall(r"\d+(?:\s*\*\s*\d+)?", body)]  # noqa: S307 - digits and '*' only


def to_icdf(vals, nsym):
    out = []
    for i in range(0, len(vals), nsym - 1):
        out += [32768 - v for v in vals[i:i + nsym - 1]] + [0]
    return out


def static_values(src, name, consts=None):
    body = src[src.index(f"static {name}:"):]
    body = body[body.index("=") + 1:]
    body = re.sub(r"//[^\n]*", "", body[:body.index(";")])
    consts = consts or {}
    toks = re.findall(r"-?\d+|[A-Z_][A-Z0-9_]*", body.split("[", 1)[1] if body.lstrip().startswith("[") else body)
    return [int(t) if re.fullmatch(r"-?\d+", t) else consts[t] for t in toks]


def const_values(src, name):
    body = src[src.index(f"const {name}:"):]
    body = body[body.index("=") + 1:]
    body = re.sub(r"//[^\n]*", "", body[:body.index(";")])
    return [int(v) for v in re.findall(r"\d+", body)]


def digest(vals):
    return hashlib.sha256(struct.pack("<%di" % len(vals), *vals)).hexdigest()


def main():
    tok = open(os.path.join(REF, "token_cdfs.rs")).read()
    em = open(os.path.join(REF, "entropymode.rs")).read()
    tu = open(os.path.join(REF, "context", "transform_unit.rs")).read()
    bu = open(os.path.join(REF, "context", "block_unit.rs")).read()
    tx_part = []
    for _, dims, n, ref in TX_FIELDS:
        vals = cdf_values(em, ref)
        assert len(vals) == prod(dims) * (n - 1), (ref, len(vals))
        tx_part += to_icdf(vals, n)
    snapshots = []
    for q in range(4):
        flat = []
        for field, dims, n, ref in TOKEN_FIELDS:
            vals = cdf_values(tok, ref)
            per_q = prod(dims) * (n - 1)
            assert len(vals) == 4 * per_q, (ref, len(vals))
            flat += to_icdf(vals[q * per_q:(q + 1) * per_q], n)
        snapshots.append(flat + tx_part)
    assert all(len(s) == 3930 for s in snapshots)

    classes = {"TX_CLASS_2D": 0, "TX_CLASS_HORIZ": 1, "TX_CLASS_VERT": 2}
    nz = {"NZ_MAP_CTX_0": 26, "NZ_MAP_CTX_5": 31, "NZ_MAP_CTX_10": 36}
    assert "const NZ_MAP_CTX_0: usize = SIG_COEF_CONTEXTS_2D;" in tu and "SIG_COEF_CONTEXTS_2D: usize = 26;" in tu
    tables = {
        "num_tx_set": static_values(tu, "num_tx_set"),
        "av1_tx_used": static_values(tu, "av1_tx_used"),
        "av1_tx_ind": static_values(tu, "av1_tx_ind"),
        "tx_type_to_class": static_values(tu, "tx_type_to_class", classes),
        "eob_to_pos_small": static_values(tu, "eob_to_pos_small"),
        "eob_to_pos_large": static_values(tu, "eob_to_pos_large"),
        "k_eob_group_start": static_values(tu, "k_eob_group_start"),
        "k_eob_offset_bits": static_values(tu, "k_eob_offset_bits"),
        "av1_nz_map_ctx_offset": static_values(tu, "av1_nz_map_ctx_offset"),
        "nz_map_ctx_offset_1d": static_values(tu, "nz_map_ctx_offset_1d", nz),
        "skip_contexts": const_values(bu, "skip_contexts"),
        "dc_sign_contexts": const_values(bu, "dc_sign_contexts"),
    }
    want_len = {"num_tx_set": 6, "av1_tx_used": 96, "av1_tx_ind": 96, "tx_type_to_class": 16, "eob_to_pos_small": 33,
                "eob_to_pos_large": 17, "k_eob_group_start": 12, "k_eob_offset_bits": 12,
                "av1_nz_map_ctx_offset": 19 * 25, "nz_map_ctx_offset_1d": 32, "skip_contexts": 25,
                "dc_sign_contexts": 65}
    for k, v in tables.items():
        assert len(v) == want_len[k], (k, len(v))
    out = {
        "source": "xiph/rav1e @ 564ae3b src/token_cdfs.rs, src/entropymode.rs, src/context/transform_unit.rs and "
                  "src/context/block_unit.rs, extracted by tests/golden/make_coeff_cdf_kats.py",
        "fields": [[f, list(d), n] for f, d, n, _ in TOKEN_FIELDS + TX_FIELDS],
        "default_cdfs": snapshots,
        "table_digests": {k: {"n": len(v), "sha256": digest(v)} for k, v in tables.items()},
    }
    with open(OUT, "w") as f:
        json.dump(out, f)
        f.write("\n")
    print("wrote", OUT)


if __name__ == "__main__":
    main()
