"""Segmentation in the oracle (oracle/segmentation.c): the k-means against the reference's own tests
(util/kmeans.rs:108-122), and segmentation_optimize (segmentation.rs:23-160) with update_threshold, get_qidx
and select_segment (segmentation.rs:163-196) with spatiotemporal_scale (rdo.rs:464-504) against an
independent Python restatement.  The restatement sorts with sorted(), runs the k-means on upper / lower
bounds and prefix sums instead of the reference's incremental walks, and uses Python integers with the
release build's wraps made explicit.  blog32_q11 is test_oracle_temporal_rdo's Python restatement; bexp64 /
blog64 are the oracle's, pinned there by the reference's known answers.
The case builders here are shared with tests/test_segmentation_gpu.py and bench_kernels.py."""
import bisect
import ctypes as C
import json
import os

import numpy as np
import pytest

from rav1e_b200.backend import SEGMENT_ITEM_DTYPE, SEGMENTATION_DTYPE
from tests import oracle_lib as O
from tests.test_oracle_temporal_rdo import T as temporal_lib
from tests.test_oracle_temporal_rdo import py_blog32_q11

GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                                     "segmentation_kats.json")))
AC_Q = {int(bd): np.array(t, np.uint16) for bd, t in GOLDEN["ac_qlookup_Q3"].items()}
DS_MAX = (1 << 28) - 1
# BlockSize::width() / height() by discriminant (partition.rs:130-153)
BW = [4, 4, 8, 8, 8, 16, 16, 16, 32, 32, 32, 64, 64, 64, 128, 128, 4, 16, 8, 32, 16, 64]
BH = [4, 8, 4, 8, 16, 8, 16, 32, 16, 32, 64, 32, 64, 128, 64, 128, 16, 4, 32, 8, 64, 16]


def L():
    l = temporal_lib()
    vp, sz, i32 = C.c_void_p, C.c_size_t, C.c_int
    l.orc_kmeans_i16.restype, l.orc_kmeans_i16.argtypes = None, [vp, sz, i32, vp]
    l.orc_select_qi.restype, l.orc_select_qi.argtypes = i32, [C.c_int64, vp]
    l.orc_segmentation_optimize.restype = i32
    l.orc_segmentation_optimize.argtypes = [vp, sz, i32, i32, vp, i32, vp, vp]
    l.orc_select_segment.restype = None
    l.orc_select_segment.argtypes = [vp, sz, vp, vp, sz, sz, i32, i32, vp, vp, vp]
    return l


# ---------------------------------------------------------------- Python restatement
def wrap(v, bits):
    m = 1 << bits
    v &= m - 1
    return v - m if v >= m >> 1 else v


def tdiv(a, b):
    """Rust's `/` on signed integers: truncation toward zero"""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def py_kmeans(data, K, trace=None):
    """kmeans::<i16, K> (kmeans.rs:11-66) on sorted `data`: after scan(), high[i] is the upper bound of
    threshold i, low[i + 1] its lower bound, and sum[i] the prefix-sum difference between them"""
    n = len(data)
    P = [0]
    for v in data:
        P.append(P[-1] + v)
    means = [data[(i * (n - 1)) // (K - 1)] for i in range(K)]
    high, low = [0] * K, [0] * K
    high[K - 1] = n
    for _ in range(2 * n.bit_length()):
        for i in range(K - 1):
            t = (means[i + 1] + means[i] + 1) >> 1
            high[i] = bisect.bisect_right(data, t)
            low[i + 1] = bisect.bisect_left(data, t)
        changed = False
        for i in range(K):
            count = high[i] - low[i]
            if count == 0:
                continue
            new = wrap(tdiv(P[high[i]] - P[low[i]] + (count >> 1), count), 16)
            if trace is not None and count > 0 and not data[low[i]] <= new <= data[high[i] - 1]:
                trace.add("mean_outside_cluster")
            changed |= new != means[i]
            means[i] = new
        if not changed:
            break
    return means


def py_select_qi(q, table):
    """select_qi (quantize/mod.rs:52-77); the i32 products wrap"""
    t = [int(v) for v in table]
    if q < t[0]:
        return 0
    if q >= t[255]:
        return 255
    qi = bisect.bisect_left(t, q)
    if t[qi] == q:
        return qi
    return qi - 1 if wrap(q * q, 32) < wrap(t[qi - 1] * t[qi], 32) else qi


def ds_new(num, den):
    raw = min((num << 14) + den // 2, (1 << 64) - 1) // den
    return raw if raw <= DS_MAX else DS_MAX


def py_update_threshold(st, base, table):
    """SegmentationState::update_threshold (encoder.rs:566-580): ac_q(base, data as i8, bd)"""
    ac = lambda d: int(table[min(max(base + d, 0), 255)])
    real = [ac(wrap(st["data"][i][0], 8)) for i in range(st["max_segment"] + 1)]
    st["threshold"] = [0] * 7
    for i in range(st["max_segment"]):
        st["threshold"][i] = ds_new(ac(0) ** 2, real[i + 1] * real[i])


def default_state():
    return {"enabled": 0, "update_data": 0, "update_map": 0, "preskip": 0, "last_active_segid": 0,
            "min_segment": 0, "max_segment": 0, "features": [[0] * 8 for _ in range(8)],
            "data": [[0] * 8 for _ in range(8)], "threshold": [0] * 7}


def py_optimize(scores, base, table, update_data, prev=None, trace=None):
    """segmentation_optimize (segmentation.rs:23-74) from get_initial_segmentation's state; then get_qidx"""
    st = json.loads(json.dumps(prev)) if prev is not None else default_state()
    st.update(enabled=1, update_map=1, update_data=int(update_data), status=0)
    lower = 1 - base
    if not update_data:
        cand = [i for i in range(8) if st["features"][i][0] and st["data"][i][0] >= lower]
        if not cand:
            st["status"] = 1
        else:
            st["min_segment"] = cand[0]
            if st["max_segment"] > 7:
                st["status"] = 2
            else:
                py_update_threshold(st, base, table)
    else:
        logs = sorted(wrap(py_blog32_q11(int(s)) - (14 << 11), 16) for s in scores)
        cs = [py_kmeans(logs, K, trace) for K in range(8, 2, -1)]

        def var(c):
            delta = [c[j] - c[j + 1] for j in range(len(c) - 1)]
            mean = tdiv(sum(delta), len(delta))
            return sum((d - mean) ** 2 for d in delta)

        v = [var(c) for c in cs]
        position = max(p for p in range(6) if v[p] == min(v))
        if trace is not None and v.count(min(v)) > 1:
            trace.add("variance_tie")
        lq = L().orc_blog64(int(table[base]))
        deltas = []
        for c in reversed(cs[position]):
            q = L().orc_bexp64(wrap(lq - (c << 45), 64))
            deltas.append(max(py_select_qi(q, table), 1) - base)
        st["min_segment"], st["max_segment"] = 0, len(deltas) - 1
        for s, d in enumerate(deltas):
            st["features"][s][0] = 1
            st["data"][s][0] = max(d, lower)
            if trace is not None and not -128 <= st["data"][s][0] <= 127:
                trace.add("i8_wrap")
        py_update_threshold(st, base, table)
        st["preskip"], st["last_active_segid"] = 0, 0
        for i in range(8):
            for j in range(8):
                if st["features"][i][j]:
                    st["last_active_segid"] = i
                    if j >= 5:
                        st["preskip"] = 1
    st["qidx"] = [min(max(wrap(base + st["data"][i][0], 16), 0), 255) if st["features"][i][0] else base
                  for i in range(8)]
    if trace is not None and any(a < b for a, b in zip(st["threshold"][:st["max_segment"]],
                                                       st["threshold"][1:st["max_segment"]])):
        trace.add("non_monotone")
    return st


def py_partition_point(thr, s):
    """threshold.partition_point(|&t| s < t) in Rust 1.83's binary_search_by probe order"""
    size, base = 7, 0
    while size > 1:
        half = size // 2
        mid = base + half
        base = mid if s < thr[mid] else base
        size -= half
    return base + (1 if s < thr[base] else 0)


def py_scale(scales, activity, w_imp, h_imp, x, y, bsize, scales_off):
    """spatiotemporal_scale (rdo.rs:464-504); the u64 sum wraps"""
    if scales_off:
        return 1 << 14
    x0, y0 = (x >> 2) >> 1, (y >> 2) >> 1
    x1, y1 = min(x0 + max(BW[bsize] >> 3, 1), w_imp), min(y0 + max(BH[bsize] >> 3, 1), h_imp)
    den = ((x1 - x0) * (y1 - y0)) << 14
    tot = 0
    for r in range(y0, y1):
        for c in range(x0, x0 + min(x1 - x0, 16)):
            a = 1 << 14 if activity is None else int(activity[r * w_imp + c])
            tot += int(scales[r * w_imp + c]) * a
    return ((tot % (1 << 64) + (den >> 1)) // den) & 0xFFFFFFFF


def py_select(items, scales, activity, w_imp, h_imp, scales_off, level, st):
    out, sc = [], []
    for x, y, bs, skip in items:
        if st["status"] or bs >= 22 or x < 0 or y < 0 or x % 4 or y % 4 or x >> 3 >= w_imp or y >> 3 >= h_imp:
            out.append((255, 255))
            sc.append(0xFFFFFFFF)
            continue
        s = py_scale(scales, activity, w_imp, h_imp, x, y, bs, scales_off)
        sc.append(s)
        if skip:
            out.append((0, 0))
        elif level == 3:
            out.append((st["min_segment"], st["max_segment"]))
        else:
            sidx = max(py_partition_point(st["threshold"], s), st["min_segment"])
            out.append((sidx, min(st["max_segment"], sidx + 1)) if level == 2 else (sidx, sidx))
    return out, sc


# ---------------------------------------------------------------- records and cases
def to_record(st):
    r = np.zeros(1, SEGMENTATION_DTYPE)
    for k in ("enabled", "update_data", "update_map", "preskip", "last_active_segid", "min_segment", "max_segment"):
        r[k] = st[k]
    r["features"][0] = st["features"]
    r["data"][0] = st["data"]
    r["threshold"][0] = st["threshold"]
    if "qidx" in st:
        r["qidx"][0] = st["qidx"]
        r["status"] = st["status"]
    return r


def from_record(r):
    r = r.reshape(-1)[0]
    st = {k: int(r[k]) for k in ("enabled", "update_data", "update_map", "preskip", "last_active_segid",
                                 "min_segment", "max_segment", "status")}
    st["features"] = r["features"].astype(int).tolist()
    st["data"] = r["data"].astype(int).tolist()
    st["threshold"] = r["threshold"].astype(int).tolist()
    st["qidx"] = r["qidx"].astype(int).tolist()
    return st


def _lognormal(rng, n, sigma=1.0, centre=1 << 14):
    return np.clip(np.rint(centre * np.exp(rng.normal(0, sigma, n))), 1, DS_MAX).astype(np.uint32)


def score_maps():
    """(name, scores, w_imp, h_imp)"""
    rng = np.random.default_rng(7)
    maps = [("1080p", _lognormal(rng, 240 * 135), 240, 135),
            ("odd_37x23", _lognormal(rng, 37 * 23, 2.0), 37, 23),
            ("n1", np.array([5000], np.uint32), 1, 1),
            ("n2", np.array([300, 90000], np.uint32), 2, 1),
            ("n3", np.array([16384, 7, 1 << 20], np.uint32), 1, 3),
            ("constant", np.full(40 * 30, 20000, np.uint32), 40, 30)]
    bi = np.where(rng.random(64 * 36) < 0.5, 1 << 11, 1 << 17).astype(np.uint32)
    maps.append(("bimodal", (bi + rng.integers(0, 64, bi.size)).astype(np.uint32), 64, 36))
    ext = rng.choice(np.array([1, DS_MAX, 16384], np.uint32), 50 * 20)
    maps.append(("extremes", ext, 50, 20))
    # clusters of equal negative log values: the rounded mean of such a cluster lies above every member
    neg = np.repeat(np.array([900, 3000, 9000, 16384, 60000], np.uint32), [7, 5, 9, 4, 6])
    maps.append(("equal_negatives", rng.permutation(neg), 31, 1))
    maps.append(("high_scales", rng.choice(np.array([DS_MAX, DS_MAX >> 3, 1 << 14, 1 << 10], np.uint32), 30 * 17),
                 30, 17))
    return maps


def prev_states():
    """previous states for update_data 0, by name"""
    s = default_state()
    for i, d in enumerate([-40, -12, 0, 9, 30]):
        s["features"][i][0], s["data"][i][0] = 1, d
    s["max_segment"], s["min_segment"] = 4, 0
    wide = json.loads(json.dumps(s))
    wide["data"][0][0], wide["data"][4][0] = -200, 150  # ac_q(.., data as i8): both wrap
    stale = json.loads(json.dumps(s))
    stale["features"][7][6], stale["data"][7][0] = 1, 77  # a feature past k: last_active_segid / preskip
    stale["max_segment"] = 7
    no_alt = default_state()
    no_alt["max_segment"] = 3
    bad_max = json.loads(json.dumps(s))
    bad_max["max_segment"] = 9
    return {"five": s, "wide": wide, "stale": stale, "no_alt_q": no_alt, "bad_max_segment": bad_max}


def optimize_cases():
    """(name, scores, w_imp, h_imp, base_q_idx, bit_depth, update_data, prev name or None)"""
    maps = score_maps()
    out = []
    for name, sc, w, h in maps:
        for base, bd in ((100, 8), (0, 10), (1, 12), (255, 8), (200, 12)):
            out.append((f"{name}-q{base}-{bd}bit", sc, w, h, base, bd, 1, None))
    sc1080 = maps[0][1]
    out.append(("1080p-stale-prev", sc1080, 240, 135, 120, 10, 1, "stale"))
    for pname in ("five", "wide", "stale", "no_alt_q", "bad_max_segment"):
        for base in (0, 1, 60, 255):
            out.append((f"keep-{pname}-q{base}", None, 240, 135, base, 8, 0, pname))
    out.append(("keep-default-panics", None, 4, 4, 90, 10, 0, None))
    return out


def oracle_optimize(scores, w, h, base, bd, update_data, prev):
    l = L()
    out = np.zeros(1, SEGMENTATION_DTYPE)
    sc = np.ascontiguousarray(scores if scores is not None else np.zeros(w * h), np.uint32)
    p = None if prev is None else to_record(prev)
    st = l.orc_segmentation_optimize(O.ptr(sc), sc.size, base, bd, O.ptr(AC_Q[bd]), update_data,
                                     None if p is None else O.ptr(p), O.ptr(out))
    assert st == int(out["status"][0])
    return out


def block_items(w, h, rng=None, skip_frac=0.25):
    """every BlockSize at interior, right-edge and bottom-edge positions (and the corner) of a w x h frame in
    luma px, with invalid items mixed in"""
    rng = rng or np.random.default_rng(3)
    it = []
    for bs in range(22):
        bw, bh = BW[bs], BH[bs]
        xs = {0, max(0, (w // 2) // bw * bw), max(0, (w - 4) // 4 * 4), max(0, (w - bw) // 4 * 4)}
        ys = {0, max(0, (h // 2) // bh * bh), max(0, (h - 4) // 4 * 4), max(0, (h - bh) // 4 * 4)}
        for x in sorted(xs):
            for y in sorted(ys):
                it.append((x, y, bs, int(rng.random() < skip_frac)))
    it += [(0, 0, 22, 0), (-4, 0, 3, 0), (2, 0, 3, 0), (0, 6, 3, 0), (w + 8, 0, 3, 0), (0, h + 8, 3, 0)]
    a = np.zeros(len(it), SEGMENT_ITEM_DTYPE)
    for k, (x, y, bs, sk) in enumerate(it):
        a[k] = (x, y, bs, sk, (0, 0))
    return a


def scale_maps(w_imp, h_imp, seed=5):
    rng = np.random.default_rng(seed)
    d = _lognormal(rng, w_imp * h_imp, 1.5)
    a = np.clip(np.rint((1 << 14) * np.exp(rng.normal(0, 0.5, w_imp * h_imp))), 1, DS_MAX).astype(np.uint32)
    return d, a


def oracle_select(items, scales, activity, w_imp, h_imp, scales_off, level, rec):
    l = L()
    sidx = np.zeros((len(items), 2), np.uint8)
    scale = np.zeros(len(items), np.uint32)
    l.orc_select_segment(O.ptr(items), len(items), None if scales is None else O.ptr(scales),
                         None if activity is None else O.ptr(activity), w_imp, h_imp, scales_off, level, O.ptr(rec),
                         O.ptr(sidx), O.ptr(scale))
    return sidx, scale


# ---------------------------------------------------------------- tests
def test_fixture_tables():
    for bd, t in AC_Q.items():
        assert t.shape == (256,) and t[0] > 0 and (np.diff(t.astype(int)) > 0).all(), bd
    assert sorted(AC_Q) == [8, 10, 12]


@pytest.mark.parametrize("kat", range(2))
def test_kmeans_reference_kats(kat):
    data, want = GOLDEN["kmeans"][kat]
    a = np.array(sorted(data), np.int16)
    got = np.zeros(8, np.int16)
    L().orc_kmeans_i16(O.ptr(a), a.size, len(want), O.ptr(got))
    assert got[:len(want)].tolist() == want
    assert py_kmeans(sorted(data), len(want)) == want


def test_kmeans_walks_equal_bounds():
    """the oracle's incremental scan == the Python bound / prefix-sum form on random sorted data"""
    rng = np.random.default_rng(11)
    for n in (1, 2, 3, 5, 17, 200, 3000):
        for lo, hi in ((-20, 20), (-30000, 30000), (-3, 0)):
            a = np.sort(rng.integers(lo, hi, n)).astype(np.int16)
            for K in range(2, 9):
                got = np.zeros(8, np.int16)
                L().orc_kmeans_i16(O.ptr(a), n, K, O.ptr(got))
                assert got[:K].tolist() == py_kmeans(a.tolist(), K), (n, lo, K)


def test_select_qi():
    for bd, t in AC_Q.items():
        for q in [0, 1, 3, 4, 5] + [int(v) + d for v in t[::7] for d in (-1, 0, 1)] + [int(t[255]), 1 << 40]:
            assert L().orc_select_qi(q, O.ptr(t)) == py_select_qi(q, t), (bd, q)


CASES = optimize_cases()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_optimize_matches_restatement(case):
    name, scores, w, h, base, bd, upd, pname = case
    prev = None if pname is None else prev_states()[pname]
    got = from_record(oracle_optimize(scores, w, h, base, bd, upd, prev))
    want = py_optimize(scores, base, AC_Q[bd], upd, prev)
    assert got == want


def test_optimize_cases_reach_the_hard_paths():
    """the fixtures above reach each trap the restatement must get right"""
    seen = set()
    for name, scores, w, h, base, bd, upd, pname in CASES:
        prev = None if pname is None else prev_states()[pname]
        st = py_optimize(scores, base, AC_Q[bd], upd, prev, trace=seen)
        seen.add(f"status{st['status']}")
        if upd and st["max_segment"] < 7:
            seen.add("k_below_8")
    for want in ("mean_outside_cluster", "variance_tie", "i8_wrap", "non_monotone", "status0", "status1",
                 "status2", "k_below_8"):
        assert want in seen, (want, seen)


def select_cases():
    """(name, record case, level, scales_off, with activity)"""
    idx = {c[0]: i for i, c in enumerate(CASES)}
    out = []
    for name in ("1080p-q100-8bit", "1080p-q0-10bit", "odd_37x23-q100-8bit", "n2-q200-12bit", "keep-five-q60"):
        for level in (1, 2, 3):
            out.append((f"{name}-L{level}", idx[name], level, 0, True))
    out.append(("no-activity", 0, 2, 0, False))
    out.append(("scales-off", 0, 1, 1, True))
    for level in (1, 2):
        out.append((f"non-monotone-L{level}", idx["extremes-q100-8bit"], level, 0, True))
    out.append(("panicked-record", idx["keep-default-panics"], 2, 0, True))
    return out


SELECT = select_cases()


def select_inputs(ci, with_activity):
    name, scores, w, h, base, bd, upd, pname = CASES[ci]
    prev = None if pname is None else prev_states()[pname]
    rec = oracle_optimize(scores, w, h, base, bd, upd, prev)
    W, H = 8 * w - 3, 8 * h - 5  # a frame whose importance grid is w x h, neither side a multiple of 8
    items = block_items(W, H)
    d, a = scale_maps(w, h)
    return rec, items, d, (a if with_activity else None), w, h


@pytest.mark.parametrize("case", SELECT, ids=[c[0] for c in SELECT])
def test_select_segment_matches_restatement(case):
    name, ci, level, off, act = case
    rec, items, d, a, w, h = select_inputs(ci, act)
    sidx, scale = oracle_select(items, d, a, w, h, off, level, rec)
    want, want_scale = py_select([tuple(int(v) for v in (r["x"], r["y"], r["bsize"], r["skip"])) for r in items],
                                 d, a, w, h, off, level, from_record(rec))
    assert [tuple(v) for v in sidx.tolist()] == want
    assert scale.tolist() == want_scale
    if name.startswith("non-monotone"):
        seen = set()
        py_optimize(CASES[ci][1], CASES[ci][4], AC_Q[CASES[ci][5]], 1, trace=seen)
        assert "non_monotone" in seen
