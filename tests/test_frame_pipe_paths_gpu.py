"""The frame pipe (csrc/frame_pipe.cu: b200_frame_pipe_create / _push / _set_lists / _push_packed) on every path,
bit exact against an oracle chain built from the CPU oracle:
- the expanded lists (centre + 8 * offset, wrapped to i16 like the device) through O.fullpel_candidates; the
  first minimum in list order wins, an all-empty list gives MotionSearchResult::empty();
- the residual against the reference displaced by the SAD winner (Rust's truncating mv / 8; zero motion for an
  empty winner or a pipe without a SAD leg), O.forward_transform_batch, the inter quantize chain;
- for packed pushes q[b][scan[:eob[b]]] block after block.

1. every transform the pipe accepts: all 19 sizes (block = transform), a 2-D, a V_* and an H_* type (the three
   scan classes) at every size up to 16, DCT_DCT and IDTX at the 32-point sizes, the 64-point sizes raw and
   quantized, 8 / 10 / 12 bit across the set; an ME-only pipe of 128x128 blocks;
2. geometry: partial blocks dropped, frames that are not a multiple of 8 with candidates on the mv-range limits,
   8-bit frames with an odd pixel count and HBD frames whose staging prefix is odd (the staging alignment), a
   non-dense host frame;
3. lists: SAD only, SATD only, both, neither; 1 and 200 per block; offsets at -128 / 127; centres absent, multiples
   of 8, odd with negative parts, near +-32767 (whole lists wrap out of range); a window hint below the reach;
4. every input copy path: the one-copy packet and its partial forms, separate buffers, resident lists, per-push
   lists that replace resident ones;
5. every output copy path, with sentinel guards around each host region;
6. 1080p: 8040 blocks of 16x16 with 64 + 8 lists (the eob scan carries between 1024-block chunks, the offset
   expansion grid-strides) and 130560 blocks of 4x4 (the packing grid-strides); packed capacity below the total;
7. asynchronous contexts, one host thread each, push and push_packed interleaved, against a synchronous run;
8. rejected calls return B200_ERR_ARG and launch nothing;
9. examples/stream_frames.cpp on the device: block 0 of its last frame against the oracle."""
import concurrent.futures as cf
import ctypes as C
import re
import subprocess

import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests import oracle_lib as O
from tests.test_oracle_quantize import L as OL
from tests.test_oracle_quantize import chain as oracle_chain

pytestmark = pytest.mark.gpu

THREADS = O.host_threads()
ME = B.ME_RESULT_DTYPE
EMPTY_COST, EMPTY_SAD = (1 << 64) - 1, (1 << 32) - 1   # MotionSearchResult::empty() (me.rs:111-116)
SENTINEL = 0xA5                                        # every host byte the pipe must not write
GUARD = 64                                             # sentinel bytes around each host output region
OUT_KEYS = ("best_sad", "best_satd", "coeffs", "eob", "tx_dist")


@pytest.fixture(scope="module")
def c():
    ctx = B.Context(0)
    yield ctx
    ctx.close()


# ------------------------------------------------------------------ configuration, frames, lists

class Cfg:
    """One b200_frame_pipe_cfg, and the block grid the pipe derives from it."""

    def __init__(self, W, H, block=(16, 16), bd=8, ns=8, nt=4, lam=900, hint=0, ts=-1, tt=0, quant=False):
        self.W, self.H, self.bd = W, H, bd
        self.bw, self.bh = block
        self.ns, self.nt, self.lam, self.hint = ns, nt, lam, hint
        self.ts, self.tt = ts, tt
        self.dcq, self.acq = (88 << (bd - 8), 72 << (bd - 8)) if quant and ts >= 0 else (0, 0)
        self.quant = self.acq != 0
        self.pad = G.min_pad(W, H, *block)       # the smallest border every accepted footprint fits in
        self.dtype = np.uint8 if bd == 8 else np.uint16
        self.ct = np.int16 if bd == 8 else np.int32
        self.blocks = G.grid_blocks(W, H, *block)
        self.nb = len(self.blocks)
        # coefficients per block in the output: raw = w * h, quantized = the coded area (<= 32x32)
        self.ncoef = 0 if ts < 0 else OL().orc_coded_tx_area(ts) if self.quant else self.bw * self.bh

    def pipe(self, ctx):
        p = B.FramePipe(ctx, self.W, self.H, self.pad, (self.bw, self.bh), self.lam, self.ns, self.nt, self.hint,
                        tx_size=self.ts, tx_type=self.tt, dc_quant=self.dcq, ac_quant=self.acq, bit_depth=self.bd)
        assert p.nblocks == self.nb
        return p


def frames(cfg, n, seed):
    """n frames of one low-pass scene under a steady pan (SAD surfaces with real minima)."""
    return [G.make_planes(cfg.W, cfg.H, 0, cfg.dtype, seed=seed, bit_depth=cfg.bd, shift=(2 * f - 4, 3 - f))[0]
            for f in range(n)]


def offsets(rng, nb, per, reach):
    return None if per == 0 else rng.integers(-reach, reach + 1, (nb, per, 2)).astype(np.int8)


def centres(kind, nb, rng):
    if kind is None:
        return None
    if kind == "mult8":
        return (rng.integers(-6, 7, (nb, 2)) * 8).astype(np.int16)
    if kind == "int8":   # 128 px away, so that offset -128 (even blocks) or 127 (odd blocks) brings a candidate home
        c = np.full((nb, 2), 1024)
        c[1::2] = -1016
        return c.astype(np.int16)
    c = rng.integers(-40, 41, (nb, 2)) * 2 + 1               # odd: never a multiple of 8, both signs
    if kind == "wrap":                                       # centre + 8 * offset wraps in i16: out of range
        c[0::3] = 32767 - rng.integers(0, 8, c[0::3].shape)
        c[1::3] = -32768 + rng.integers(0, 8, c[1::3].shape)
    return c.astype(np.int16)


# ------------------------------------------------------------------ the oracle chain

def scan_order(ts, tt):
    scan = np.zeros(OL().orc_coded_tx_area(ts), np.uint16)
    OL().orc_scan_order(ts, tt, scan.ctypes.data, None)
    return scan


def expand(offs, cen, nb):
    per = offs.shape[1]
    cands = np.zeros(nb * per, B.CAND_DTYPE)
    cands["block"] = np.repeat(np.arange(nb, dtype=np.uint32), per)
    base = np.zeros((nb, 2), np.int32) if cen is None else cen.astype(np.int32)
    mv = (base[:, None, :] + 8 * offs.astype(np.int32)).astype(np.int16).reshape(-1, 2)   # i16 wrap
    cands["mv_row"], cands["mv_col"] = mv[:, 0], mv[:, 1]
    return cands


def winners(ocur, oref, blocks, bw, bh, lam, offs, cen, satd):
    nb, per = len(blocks), offs.shape[1]
    cands = expand(offs, cen, nb)
    sad, cost = O.fullpel_candidates(ocur, oref, blocks, cands, bw, bh, satd, lam, threads=THREADS)
    k = np.arange(nb) * per + cost.reshape(nb, per).argmin(axis=1)     # the first minimum in list order
    live = cost[k] != EMPTY_COST
    out = np.zeros(nb, ME)
    out["cost"] = cost[k]
    out["sad"] = np.where(live, sad[k], EMPTY_SAD)
    out["mv_row"] = np.where(live, cands["mv_row"][k], 0)
    out["mv_col"] = np.where(live, cands["mv_col"][k], 0)
    return out


def trunc8(v):
    v = v.astype(np.int64)
    return np.sign(v) * (np.abs(v) // 8)                     # Rust's i16 `/ 8`, not Python's `//`


def residuals(ocur, oref, blocks, bw, bh, best):
    nb, pad = len(blocks), ocur.pad
    dx = dy = np.zeros(nb, np.int64)
    if best is not None:
        live = best["cost"] != EMPTY_COST
        dx, dy = np.where(live, trunc8(best["mv_col"]), 0), np.where(live, trunc8(best["mv_row"]), 0)
    ys = blocks["y"].astype(np.int64)[:, None] + pad + np.arange(bh)
    xs = blocks["x"].astype(np.int64)[:, None] + pad + np.arange(bw)
    cur = ocur.data[ys[:, :, None], xs[:, None, :]].astype(np.int32)
    ref = oref.data[(ys + dy[:, None])[:, :, None], (xs + dx[:, None])[:, None, :]]
    return (cur - ref).astype(np.int16)


def oracle_planes(W, H, pad, dtype, cur, ref):
    ocur, oref = O.Plane(W, H, pad, dtype), O.Plane(W, H, pad, dtype)
    ocur.fill_from(cur)
    oref.fill_from(ref)
    return ocur, oref


def expect(cfg, cur, ref, so, to, cen):
    """Everything one push of `cur` (previous frame `ref`) with these lists returns."""
    ocur, oref = oracle_planes(cfg.W, cfg.H, cfg.pad, cfg.dtype, cur, ref)
    args = (ocur, oref, cfg.blocks, cfg.bw, cfg.bh, cfg.lam)
    e = {k: None for k in OUT_KEYS + ("packed",)}
    if cfg.ns:
        e["best_sad"] = winners(*args, so, cen, False)
    if cfg.nt:
        e["best_satd"] = winners(*args, to, cen, True)
    if cfg.ts >= 0:
        coef = O.forward_transform_batch(residuals(ocur, oref, cfg.blocks, cfg.bw, cfg.bh, e["best_sad"]),
                                         cfg.ts, cfg.tt, cfg.bd, threads=THREADS)
        e["coeffs"] = coef
        if cfg.quant:
            q, _, eob, dist = oracle_chain(coef, cfg.ts, cfg.tt, cfg.dcq, cfg.acq, False, threads=THREADS)
            scan = scan_order(cfg.ts, cfg.tt)
            e.update(coeffs=q, eob=eob, tx_dist=dist, packed=q[:, scan][np.arange(len(scan)) < eob[:, None]])
    return e


def assert_outputs(want, got, what=""):
    """Every output in `got` (None: not asked for) equals the oracle's."""
    for k in OUT_KEYS:
        if got.get(k) is not None and want[k] is not None:
            np.testing.assert_array_equal(got[k].reshape(want[k].shape), want[k], err_msg=f"{what} {k}")


# ------------------------------------------------------------------ host buffers

def pinned(nbytes):
    import torch
    return torch.empty(max(nbytes, 1), dtype=torch.uint8).pin_memory().numpy()


class Arena:
    """Host bytes filled with SENTINEL, carved into output regions at chosen offsets.  check(): every byte outside
    the regions the pipe owns still holds SENTINEL, and every region expected to come back zero is zero."""

    def __init__(self, nbytes, pin=False):
        self.buf = pinned(nbytes) if pin else np.empty(nbytes, np.uint8)
        self.buf[:] = SENTINEL
        self.owned = np.zeros(nbytes, bool)
        self.zero = []
        self.off = GUARD

    def take(self, count, dtype, skip=0, owned=True):
        dt = np.dtype(dtype)
        o = self.off + skip
        n = count * dt.itemsize
        assert o + n + GUARD <= len(self.buf)
        self.owned[o:o + n] = owned
        self.off = o + n
        return self.buf[o:o + n].view(dt)

    def take_zero(self, nbytes):
        self.zero.append((self.off, nbytes))
        self.take(nbytes, np.uint8)

    def check(self, what=""):
        bad = np.nonzero(self.buf[~self.owned] != SENTINEL)[0]
        assert len(bad) == 0, f"{what}: {len(bad)} bytes written outside the outputs"
        for o, n in self.zero:
            assert (self.buf[o:o + n] == 0).all(), f"{what}: alignment gap not zero"


def arena_bytes(cfg, extra=0):
    return 2 * cfg.nb * 16 + cfg.nb * cfg.ncoef * 4 + cfg.nb * 10 + 16 * GUARD + extra


def separate_outputs(cfg, arena):
    """All five outputs, GUARD bytes apart; those of a leg the pipe does not have must stay untouched."""
    return dict(best_sad=arena.take(cfg.nb, ME, GUARD, owned=cfg.ns > 0),
                best_satd=arena.take(cfg.nb, ME, GUARD, owned=cfg.nt > 0),
                coeffs=arena.take(cfg.nb * max(cfg.ncoef, 1), cfg.ct, GUARD, owned=cfg.ts >= 0),
                eob=arena.take(cfg.nb, np.uint16, GUARD, owned=cfg.quant),
                tx_dist=arena.take(cfg.nb, np.uint64, GUARD, owned=cfg.quant))


def packed_buffer(cfg, cap, pin=False):
    buf = pinned((cap + GUARD) * np.dtype(cfg.ct).itemsize) if pin else np.empty((cap + GUARD) * 4, np.uint8)
    buf[:] = SENTINEL
    return buf[:(cap + GUARD) * np.dtype(cfg.ct).itemsize].view(cfg.ct)


def push_packed(cfg, pipe, frame, cap=None, pin=False):
    """push_packed with every output guarded; returns (total, outputs, arena, packed buffer, capacity)."""
    cap = cfg.nb * cfg.ncoef if cap is None else cap
    a = Arena(arena_bytes(cfg), pin)
    o = separate_outputs(cfg, a)
    del o["coeffs"]
    buf = packed_buffer(cfg, cap, pin)
    total = pipe.push_packed(frame, packed=buf[:cap] if cap else None, **o)
    return total, o, a, buf, cap


def check_packed(want, total, o, a, buf, cap, what=""):
    assert_outputs(want, o, what)
    a.check(what)
    assert total == len(want["packed"]), what
    k = min(total, cap)
    np.testing.assert_array_equal(buf[:k], want["packed"][:k], err_msg=what)
    assert (buf[k:].view(np.uint8) == SENTINEL).all(), f"{what}: packed written beyond min(total, capacity)"


def addr(a):
    return None if a is None else a.ctypes.data


def push_at(pipe, frame, stride, so, to, cen, out):
    """b200_frame_pipe_push on raw host addresses (ints or None)."""
    pipe.ctx.check(pipe.ctx.L.b200_frame_pipe_push(pipe.h, frame, stride, so, to, cen,
                                                   *[addr(out.get(k)) for k in OUT_KEYS]))


class Packet:
    """[frame | sad offsets | satd offsets | centres] with the first `k` inputs directly behind the frame in one host
    buffer (one copy) and the rest in buffers of their own."""

    def __init__(self, frame, lists, k):
        inside = [a for a in lists[:k] if a is not None]
        self.buf = np.concatenate([frame.view(np.uint8).reshape(-1)] + [a.view(np.uint8).reshape(-1) for a in inside])
        self.frame, self.stride = self.buf.ctypes.data, frame.shape[1] * frame.itemsize
        off, self.lists = frame.nbytes, []
        for i, a in enumerate(lists):
            if a is not None and i < k:
                self.lists.append(self.buf.ctypes.data + off)
                off += a.nbytes
            else:
                self.lists.append(addr(a))


# ------------------------------------------------------------------ 1. every transform

TWO_D = [1, 2, 3, 4, 5, 6, 7, 8, 9]            # ADST_DCT .. IDTX: the default scan


def tx_cases():
    out = []
    for ts, (w, h) in enumerate(O.TX_SIZES):
        if max(w, h) <= 16:   # a 2-D type, a V_* (row scan) and an H_* (column scan)
            types = [(TWO_D[ts % len(TWO_D)], ts % 2 == 0), (10 + 2 * (ts % 3), True), (11 + 2 * (ts % 3), ts % 2 == 1)]
        elif max(w, h) == 32:
            types = [(0, True), (9, False)]
        else:                 # 64-point: 32x32 coded area, log_tx_scale 2 (64x64) or 1
            types = [(0, False), (0, True)]
        out += [(ts, tt, q) for tt, q in types]
    return [(ts, tt, (8, 10, 12)[k % 3], q) for k, (ts, tt, q) in enumerate(out)]


TX_CASES = tx_cases()


@pytest.mark.parametrize("ts,tt,bd,quant", TX_CASES,
                         ids=[f"{O.TX_SIZES[ts][0]}x{O.TX_SIZES[ts][1]}-{O.TX_TYPE_NAMES[tt]}-{bd}bit-"
                              f"{'quant' if q else 'raw'}" for ts, tt, bd, q in TX_CASES])
def test_every_transform(c, ts, tt, bd, quant):
    assert O.valid_txfm(ts, tt)
    cfg = Cfg(192, 128, O.TX_SIZES[ts], bd, ns=6, nt=3, hint=24, ts=ts, tt=tt, quant=quant)
    fr = frames(cfg, 3, seed=ts * 17 + tt)
    rng = np.random.default_rng(ts * 31 + tt)
    so, to, cen = offsets(rng, cfg.nb, 6, 20), offsets(rng, cfg.nb, 3, 20), centres("mult8", cfg.nb, rng)
    dense = cfg.pipe(c)
    dense.push(fr[0])
    wants = []
    for f in (1, 2):
        want = expect(cfg, fr[f], fr[f - 1], so, to, cen)
        a = Arena(arena_bytes(cfg))
        o = separate_outputs(cfg, a)
        dense.push(fr[f], so, to, cen, **o)
        assert_outputs(want, o, f"frame {f}")
        a.check(f"frame {f}")
        wants.append(want)
    dense.close()
    if quant:   # the packed output follows the scan of this (size, type)
        packed = cfg.pipe(c)
        packed.set_lists(so, to, cen)
        assert packed.push_packed(fr[0]) == 0
        for f in (1, 2):
            check_packed(wants[f - 1], *push_packed(cfg, packed, fr[f]), what=f"packed frame {f}")
        assert any(len(w["packed"]) for w in wants)
        packed.close()


def test_me_only_pipe_of_128x128_blocks(c):
    """tx_size < 0: winners only; a coefficient, eob or tx_dist buffer passed anyway is never written."""
    cfg = Cfg(384, 256, (128, 128), 8, ns=16, nt=8, hint=48)
    fr = frames(cfg, 3, seed=3)
    rng = np.random.default_rng(3)
    so, to = offsets(rng, cfg.nb, 16, 40), offsets(rng, cfg.nb, 8, 40)
    pipe = cfg.pipe(c)
    pipe.push(fr[0])
    for f in (1, 2):
        want = expect(cfg, fr[f], fr[f - 1], so, to, None)
        a = Arena(arena_bytes(cfg, 4096))
        o = separate_outputs(cfg, a)
        pipe.push(fr[f], so, to, None, **o)
        assert_outputs(want, o)
        a.check()
    pipe.close()


# ------------------------------------------------------------------ 2. geometry

def border_lists(cfg, rng):
    """SAD list: the candidates ON the block's x_max and y_max limits; SATD list: one full pel BEYOND them.  Those
    limits depend on w_in_b / h_in_b, which round the frame up to 8 pixels.  Blocks whose limits int8 offsets do not
    reach get random offsets instead."""
    so, to = rng.integers(-8, 9, (2, cfg.nb, 2, 2))
    lim = np.array([G.mv_range(cfg.W, cfg.H, int(b["x"]), int(b["y"]), cfg.bw, cfg.bh) for b in cfg.blocks]) // 8
    nx, ny = lim[:, 1] < 127, lim[:, 3] < 127
    so[nx, 0, 0], so[nx, 0, 1] = 0, lim[nx, 1]
    so[ny, 1, 0], so[ny, 1, 1] = lim[ny, 3], 0
    to[nx, 0, 0], to[nx, 0, 1] = 0, lim[nx, 1] + 1
    to[ny, 1, 0], to[ny, 1, 1] = lim[ny, 3] + 1, 0
    return so.astype(np.int8), to.astype(np.int8), nx & ny


GEOMETRY = [
    # id, W, H, block, bit depth, centres, resident lists, strided host frame
    ("partial_blocks", 200, 120, (16, 16), 8, "mult8", False, False),
    ("not_multiple_of_8", 203, 118, (8, 8), 10, None, False, False),
    ("odd_area_8bit", 333, 185, (16, 16), 8, "odd", False, False),
    ("odd_area_8bit_resident", 333, 185, (16, 16), 8, "odd", True, False),
    ("odd_prefix_10bit", 333, 185, (16, 16), 10, "odd", False, False),
    ("odd_prefix_12bit_resident", 333, 185, (16, 16), 12, "odd", True, False),
    ("strided_frame", 200, 120, (16, 16), 12, "mult8", False, True),
    ("strided_odd_area_8bit", 333, 185, (16, 16), 8, "odd", False, True),
]


@pytest.mark.parametrize("name,W,H,block,bd,cen_kind,resident,strided", GEOMETRY, ids=[g[0] for g in GEOMETRY])
def test_geometry(c, name, W, H, block, bd, cen_kind, resident, strided):
    ts = {(16, 16): 2, (8, 8): 1}[block]
    border = name == "not_multiple_of_8"
    cfg = Cfg(W, H, block, bd, ns=2 if border else 12, nt=2 if border else 5, hint=0 if border else 32, ts=ts,
              quant=True)
    assert cfg.nb == (W // block[0]) * (H // block[1])
    if name.startswith("odd_area"):
        assert (W * H) % 2 == 1                       # the offsets follow an odd number of frame bytes
    if name.startswith("odd_prefix"):
        assert (W * H + cfg.nb * (cfg.ns + cfg.nt)) % 2 == 1 and cen_kind   # 2-aligned but not 4-aligned centres
    rng = np.random.default_rng(W + H + bd)
    if border:
        so, to, both = border_lists(cfg, rng)
        assert both.any()
    else:
        so, to = offsets(rng, cfg.nb, cfg.ns, 40), offsets(rng, cfg.nb, cfg.nt, 40)
    cen = centres(cen_kind, cfg.nb, rng)
    fr = frames(cfg, 3, seed=W * H + bd)
    if strided:     # views into wider arrays: the pitched copy
        wide = [np.zeros((H, W + 13), cfg.dtype) for _ in fr]
        for w, f in zip(wide, fr):
            w[:, 5:5 + W] = f
        send = [w[:, 5:5 + W] for w in wide]
        assert send[0].strides[0] != W * send[0].itemsize
    else:
        send = fr
    pipe = cfg.pipe(c)
    if resident:
        pipe.set_lists(so, to, cen)
    pipe.push(send[0])
    for f in (1, 2):
        want = expect(cfg, fr[f], fr[f - 1], so, to, cen)
        if border:   # on-limit candidates are accepted, beyond-limit ones are not
            assert (want["best_sad"]["cost"][both] != EMPTY_COST).all()
            assert (want["best_satd"]["cost"][both] == EMPTY_COST).all()
        a = Arena(arena_bytes(cfg))
        o = separate_outputs(cfg, a)
        if resident:
            pipe.push(send[f], None, None, None, **o)
        else:
            pipe.push(send[f], so, to, cen, **o)
        assert_outputs(want, o, f"frame {f}")
        a.check(f"frame {f}")
    pipe.close()


# ------------------------------------------------------------------ 3. lists

LIST_CASES = [
    # id, sad per block, satd per block, centres, offset reach (or "int8" for -128 / 127), window hint, bit depth
    ("sad_only", 8, 0, None, 40, 48, 8),
    ("satd_only", 0, 8, None, 40, 48, 10),
    ("both", 8, 4, "mult8", 40, 48, 8),
    ("neither", 0, 0, None, 0, 0, 8),
    ("one_per_block", 1, 1, "odd", 40, 48, 8),
    ("200_per_block", 200, 200, "mult8", 40, 48, 8),
    ("offsets_at_int8_limits", 16, 8, "int8", "int8", 0, 8),
    ("centres_odd_negative", 16, 8, "odd", 40, 48, 10),
    ("centres_wrap_i16", 16, 8, "wrap", 40, 48, 8),
    ("hint_below_reach", 16, 8, "mult8", 40, 8, 8),
]


@pytest.mark.parametrize("name,ns,nt,cen_kind,reach,hint,bd", LIST_CASES, ids=[l[0] for l in LIST_CASES])
def test_lists(c, name, ns, nt, cen_kind, reach, hint, bd):
    """Dense pushes with per-push lists, and packed pushes with the same lists resident.  A leg with no list writes
    no winners; without a SAD leg the transform runs at zero motion."""
    cfg = Cfg(256, 144, (16, 16), bd, ns=ns, nt=nt, hint=hint, ts=2, quant=True)
    rng = np.random.default_rng(ns * 7 + nt)
    if reach == "int8":
        so, to = offsets(rng, cfg.nb, ns, 20), offsets(rng, cfg.nb, nt, 20)
        for o in (so, to):
            o[:, 0], o[:, 1], o[:, 2], o[:, 3] = (-128, 127), (127, -128), (-128, -128), (127, 127)
    else:
        so, to = offsets(rng, cfg.nb, ns, reach), offsets(rng, cfg.nb, nt, reach)
    cen = centres(cen_kind, cfg.nb, rng)
    fr = frames(cfg, 3, seed=ns + nt + bd)
    dense, packed = cfg.pipe(c), cfg.pipe(c)
    packed.set_lists(so, to, cen)
    dense.push(fr[0])
    assert packed.push_packed(fr[0]) == 0
    for f in (1, 2):
        want = expect(cfg, fr[f], fr[f - 1], so, to, cen)
        if name == "centres_wrap_i16":   # the lists of every third block wrap to far out of range in each direction
            assert (want["best_sad"]["cost"][0::3] == EMPTY_COST).all()
            assert (want["best_sad"]["cost"][1::3] == EMPTY_COST).all()
            assert (want["best_satd"]["cost"][2::3] != EMPTY_COST).any()
        if name in ("centres_odd_negative", "one_per_block"):   # truncating and flooring / 8 differ on these
            mv = want["best_sad"]["mv_col"]
            assert ((mv < 0) & (mv % 8 != 0) & (want["best_sad"]["cost"] != EMPTY_COST)).any()
        if reach == "int8":   # most winners are the candidate an extreme offset brought back to (0, 0)
            assert ((want["best_sad"]["mv_row"] == 0) & (want["best_sad"]["mv_col"] == 0)).mean() > 0.5
        a = Arena(arena_bytes(cfg))
        o = separate_outputs(cfg, a)
        dense.push(fr[f], so, to, cen, **o)
        assert_outputs(want, o, f"frame {f}")
        a.check(f"frame {f}")
        check_packed(want, *push_packed(cfg, packed, fr[f]), what=f"packed frame {f}")
    dense.close()
    packed.close()


# ------------------------------------------------------------------ 4. input copy paths

INPUT_PATHS = ["packet_all", "packet_frame_sad", "packet_no_centres", "separate", "resident"]


@pytest.mark.parametrize("bd", [8, 10])
def test_input_copy_paths_agree(c, bd):
    """The same frames and lists through every way of sending them: identical results, equal to the oracle.  At
    333x185 the 8-bit frame has an odd byte count and the HBD staging prefix is 2 but not 4 bytes long."""
    cfg = Cfg(333, 185, (16, 16), bd, ns=12, nt=5, hint=32, ts=2, quant=True)
    rng = np.random.default_rng(50 + bd)
    lists = (offsets(rng, cfg.nb, 12, 40), offsets(rng, cfg.nb, 5, 40), centres("odd", cfg.nb, rng))
    fr = frames(cfg, 3, seed=60 + bd)
    pipes = {p: cfg.pipe(c) for p in INPUT_PATHS}
    pipes["resident"].set_lists(*lists)
    for f in range(3):
        want = expect(cfg, fr[f], fr[f - 1], *lists) if f else None
        for path, pipe in pipes.items():
            a = Arena(arena_bytes(cfg))
            o = separate_outputs(cfg, a)
            if path.startswith("packet"):
                pk = Packet(fr[f], lists, {"packet_all": 3, "packet_frame_sad": 1, "packet_no_centres": 2}[path])
                push_at(pipe, pk.frame, pk.stride, *pk.lists, o)
            elif path == "separate":
                pipe.push(fr[f], *lists, **o)
            else:
                pipe.push(fr[f], None, None, None, **o)
            if f:
                assert_outputs(want, o, f"{path} frame {f}")
                a.check(f"{path} frame {f}")
            else:
                assert (a.buf == SENTINEL).all(), "the first push writes no outputs"
    for pipe in pipes.values():
        pipe.close()


def test_per_push_lists_replace_resident_ones(c):
    """set_lists(A); a push with lists B searches B and drops A; a push without lists is then refused (and neither
    launches nor consumes the frame); set_lists(A) again restores A."""
    cfg = Cfg(240, 160, (16, 16), 8, ns=10, nt=4, hint=32, ts=2, quant=True)
    rng = np.random.default_rng(70)
    A = (offsets(rng, cfg.nb, 10, 30), offsets(rng, cfg.nb, 4, 30), centres("mult8", cfg.nb, rng))
    Bl = (offsets(rng, cfg.nb, 10, 30), offsets(rng, cfg.nb, 4, 30), None)
    fr = frames(cfg, 4, seed=70)
    pipe = cfg.pipe(c)
    pipe.set_lists(*A)
    pipe.push(fr[0])
    for f, lists, per_push in ((1, A, False), (2, Bl, True), (3, A, False)):
        if f == 3:   # B replaced A: nothing is resident any more
            before = c.launches
            with pytest.raises(B.B200Error) as e:
                pipe.push(fr[f])
            assert e.value.status == B.ERR_ARG and c.launches == before
            with pytest.raises(B.B200Error) as e:
                pipe.push_packed(fr[f])
            assert e.value.status == B.ERR_ARG and c.launches == before
            pipe.set_lists(*A)
        want = expect(cfg, fr[f], fr[f - 1], *lists)
        o = separate_outputs(cfg, Arena(arena_bytes(cfg)))
        pipe.push(fr[f], *(lists if per_push else (None, None, None)), **o)
        assert_outputs(want, o, f"frame {f}")
    pipe.close()


# ------------------------------------------------------------------ 5. output copy paths

def out_forms(cfg):
    """(name, arena builder) pairs: each builder carves the outputs of one push and returns them."""
    nb, n = cfg.nb, cfg.nb * cfg.ncoef
    gap = -(2 * nb) % 8

    def one_block(a):          # [best_sad | best_satd | coeffs | eob | gap | tx_dist]: one copy, the gap zeroed
        o = dict(best_sad=a.take(nb, ME), best_satd=a.take(nb, ME), coeffs=a.take(n, cfg.ct), eob=a.take(nb, np.uint16))
        a.take_zero(gap)
        o["tx_dist"] = a.take(nb, np.uint64)
        return o

    def best_best2_coef(a):    # the bench's result block; eob and tx_dist elsewhere
        o = dict(best_sad=a.take(nb, ME), best_satd=a.take(nb, ME), coeffs=a.take(n, cfg.ct))
        o.update(eob=a.take(nb, np.uint16, GUARD + 2), tx_dist=a.take(nb, np.uint64, GUARD))
        return o

    def eob_not_dist(a):       # eob travels with the block, tx_dist 8 bytes past its aligned place
        o = dict(best_sad=a.take(nb, ME), best_satd=a.take(nb, ME), coeffs=a.take(n, cfg.ct), eob=a.take(nb, np.uint16))
        o["tx_dist"] = a.take(nb, np.uint64, gap + 8)
        return o

    def raw_block(a):          # a raw pipe's one-copy block; eob / tx_dist buffers behind it are never written
        o = dict(best_sad=a.take(nb, ME), best_satd=a.take(nb, ME), coeffs=a.take(n, cfg.ct))
        o.update(eob=a.take(nb, np.uint16, owned=False), tx_dist=a.take(nb, np.uint64, gap, owned=False))
        return o

    def alone(key, count, dtype):
        return lambda a: {key: a.take(count, dtype)}

    forms = [("one_block", one_block), ("best_best2_coef", best_best2_coef), ("eob_not_dist", eob_not_dist),
             ("eob_alone", alone("eob", nb, np.uint16)), ("tx_dist_alone", alone("tx_dist", nb, np.uint64))]
    if not cfg.quant:
        forms = [("raw_block_with_eob_behind", raw_block)]
    return forms + [("best_sad_alone", alone("best_sad", nb, ME)), ("best_satd_alone", alone("best_satd", nb, ME)),
                    ("coeffs_alone", alone("coeffs", n, cfg.ct))]


@pytest.mark.parametrize("bd,quant", [(8, True), (10, True), (8, False), (12, False)])
def test_output_copy_paths(c, bd, quant):
    """One push per host layout (117 blocks: eob ends 6 bytes short of tx_dist's 8-byte alignment): the outputs equal
    the oracle, and no byte outside them (nor any eob / tx_dist of a raw pipe) is written."""
    cfg = Cfg(208, 144, (16, 16), bd, ns=8, nt=4, hint=32, ts=2, quant=quant)
    assert cfg.nb == 117 and (2 * cfg.nb) % 8 == 2
    rng = np.random.default_rng(80 + bd)
    so, to, cen = offsets(rng, cfg.nb, 8, 40), offsets(rng, cfg.nb, 4, 40), centres("mult8", cfg.nb, rng)
    forms = out_forms(cfg)
    fr = frames(cfg, len(forms) + 1, seed=90 + bd)
    pipe = cfg.pipe(c)
    pipe.push(fr[0])
    for f, (name, build) in enumerate(forms, 1):
        want = expect(cfg, fr[f], fr[f - 1], so, to, cen)
        a = Arena(arena_bytes(cfg))
        o = build(a)
        push_at(pipe, fr[f].ctypes.data, fr[f].strides[0], addr(so), addr(to), addr(cen), o)
        assert_outputs(want, o, name)
        a.check(name)
    pipe.close()


# ------------------------------------------------------------------ 6. block counts at scale

def test_1080p_16x16_bench_lists(c):
    """8040 blocks: the eob scan walks eight 1024-block chunks, 578880 candidates outrun one grid of the offset
    expansion.  Packed pushes with a full, a short and no buffer, and a dense push in between."""
    cfg = Cfg(1920, 1080, (16, 16), 8, ns=64, nt=8, lam=6400, hint=64, ts=2, quant=True)
    assert cfg.nb == 8040
    rng = np.random.default_rng(1080)
    so, to = offsets(rng, cfg.nb, 64, 64), offsets(rng, cfg.nb, 8, 2)
    fr = frames(cfg, 5, seed=1080)
    pipe = cfg.pipe(c)
    pipe.set_lists(so, to)
    assert pipe.push_packed(fr[0]) == 0
    for f in range(1, 5):
        want = expect(cfg, fr[f], fr[f - 1], so, to, None)
        total = len(want["packed"])
        assert total > 0
        if f == 3:
            a = Arena(arena_bytes(cfg))
            o = separate_outputs(cfg, a)
            pipe.push(fr[f], None, None, None, **o)
            assert_outputs(want, o, "dense")
            a.check("dense")
            continue
        cap = {1: None, 2: total * 3 // 5, 4: 0}[f]
        check_packed(want, *push_packed(cfg, pipe, fr[f], cap), what=f"frame {f} capacity {cap}")
    pipe.close()


def test_4x4_blocks_over_1080p(c):
    """130560 4x4 blocks: the packing's warps and the eob scan's 1024-block chunks both loop many times."""
    cfg = Cfg(1920, 1088, (4, 4), 8, ns=2, nt=1, lam=300, ts=0, quant=True)
    assert cfg.nb == 130560
    rng = np.random.default_rng(44)
    so, to = offsets(rng, cfg.nb, 2, 6), offsets(rng, cfg.nb, 1, 6)
    fr = frames(cfg, 3, seed=44)
    pipe = cfg.pipe(c)
    pipe.set_lists(so, to)
    assert pipe.push_packed(fr[0]) == 0
    want = expect(cfg, fr[1], fr[0], so, to, None)
    check_packed(want, *push_packed(cfg, pipe, fr[1]), what="packed")
    want = expect(cfg, fr[2], fr[1], so, to, None)
    a = Arena(arena_bytes(cfg))
    o = separate_outputs(cfg, a)
    pipe.push(fr[2], so, to, None, **o)
    assert_outputs(want, o, "dense")
    a.check("dense")
    pipe.close()


# ------------------------------------------------------------------ 7. asynchronous contexts

ASYNC_BDS = [8, 10, 8, 12]


def drive(ctx, cfg, lists, fr, pin):
    """What the bench does per context: resident lists, then push_packed and push alternately, one frame each."""
    pipe = cfg.pipe(ctx)
    pipe.set_lists(*lists)
    res = []
    for f, frame in enumerate(fr):
        if f % 2 == 0:
            res.append(("packed",) + push_packed(cfg, pipe, frame, pin=pin))
        else:
            a = Arena(arena_bytes(cfg), pin)
            o = dict(best_sad=a.take(cfg.nb, ME), best_satd=a.take(cfg.nb, ME),
                     coeffs=a.take(cfg.nb * cfg.ncoef, cfg.ct), eob=a.take(cfg.nb, np.uint16))
            a.take_zero(-(2 * cfg.nb) % 8)
            o["tx_dist"] = a.take(cfg.nb, np.uint64)
            pipe.push(frame, None, None, None, **o)
            res.append(("dense", o, a))
    ctx.synchronize()
    pipe.close()
    return res


def test_async_contexts_on_host_threads(c):
    cfgs = [Cfg(256, 144, (16, 16), bd, ns=12, nt=4, hint=32, ts=2, quant=True) for bd in ASYNC_BDS]
    lists, frs = [], []
    for k, cfg in enumerate(cfgs):
        rng = np.random.default_rng(200 + k)
        lists.append((offsets(rng, cfg.nb, 12, 40), offsets(rng, cfg.nb, 4, 40), centres("odd", cfg.nb, rng)))
        host = frames(cfg, 6, seed=300 + k)
        frs.append([pinned(f.nbytes).view(cfg.dtype).reshape(f.shape) for f in host])
        for dst, src in zip(frs[-1], host):
            dst[:] = src
    ctxs = [B.Context(0) for _ in cfgs]
    for x in ctxs:
        x.set_async(True)
    with cf.ThreadPoolExecutor(len(cfgs)) as pool:
        got = list(pool.map(lambda k: drive(ctxs[k], cfgs[k], lists[k], frs[k], True), range(len(cfgs))))
    for x in ctxs:
        x.close()
    for k, cfg in enumerate(cfgs):
        sync = drive(c, cfg, lists[k], frs[k], False)
        assert got[k][0][1] == 0 and sync[0][1] == 0          # the first push only uploads
        for f in range(1, 6):
            what = f"context {k} frame {f}"
            a, s = got[k][f], sync[f]
            if a[0] == "packed":     # (kind, total, outputs, arena, packed buffer, capacity)
                assert a[1] == s[1], what
                np.testing.assert_array_equal(a[4][:a[1]], s[4][:s[1]], err_msg=what)
                outs = (a[2], s[2])
            else:                    # (kind, outputs, arena)
                outs = (a[1], s[1])
            for key in outs[0]:
                np.testing.assert_array_equal(outs[0][key], outs[1][key], err_msg=f"{what} {key}: async != sync")
            # and both equal the oracle searching frame f against frame f - 1
            want = expect(cfg, frs[k][f], frs[k][f - 1], *lists[k])
            if a[0] == "packed":
                check_packed(want, *a[1:], what=what)
            else:
                assert_outputs(want, a[1], what)
                a[2].check(what)


# ------------------------------------------------------------------ 8. rejected calls

def create_status(c, **fields):
    cfg = B.FramePipeCfg(128, 64, 32, 1, 8, 16, 16, 900, 4, 2, 0, 2, 0, 88, 72)
    for k, v in fields.items():
        setattr(cfg, k, v)
    h = C.c_void_p()
    st = c.L.b200_frame_pipe_create(c.h, C.byref(cfg), C.byref(h))
    return st, h


def test_rejected_calls_launch_nothing(c):
    def rejected(call):
        before = c.launches
        with pytest.raises(B.B200Error) as e:
            call()
        assert e.value.status == B.ERR_ARG
        assert c.launches == before

    cfg_raw = Cfg(128, 64, (16, 16), 8, ns=4, nt=2, ts=2, quant=False)
    cfg_q = Cfg(128, 64, (16, 16), 8, ns=4, nt=2, ts=2, quant=True)
    rng = np.random.default_rng(9)
    so, to = offsets(rng, cfg_q.nb, 4, 20), offsets(rng, cfg_q.nb, 2, 20)
    fr = frames(cfg_q, 3, seed=9)
    raw, q = cfg_raw.pipe(c), cfg_q.pipe(c)
    raw.set_lists(so, to)
    rejected(lambda: raw.push_packed(fr[0]))                 # nothing to pack: a raw pipe
    rejected(lambda: q.push_packed(fr[0]))                   # no resident lists
    q.set_lists(so, to)
    n = C.c_size_t(0)
    rejected(lambda: c.check(c.L.b200_frame_pipe_push_packed(q.h, fr[0].ctypes.data, fr[0].strides[0], None, None,
                                                             None, None, None, 10, C.byref(n))))
    q.close()
    q = cfg_q.pipe(c)                                        # lists per push, none resident
    q.push(fr[0])
    rejected(lambda: q.push(fr[1]))
    # the refused push consumed nothing: the next one still searches fr[1] against fr[0]
    o = separate_outputs(cfg_q, Arena(arena_bytes(cfg_q)))
    q.push(fr[1], so, to, None, **o)
    assert_outputs(expect(cfg_q, fr[1], fr[0], so, to, None), o)
    raw.close()
    q.close()
    for what, fields in [("8x8 transform on 16x16 blocks", dict(tx_size=1)),
                         ("8x16 transform on 16x8 blocks", dict(block_h=8, tx_size=7)),
                         ("invalid type for 32x32", dict(block_w=32, block_h=32, tx_size=3, tx_type=1)),
                         ("bpp 1 at 10 bit", dict(bit_depth=10)),
                         ("bpp 2 at 8 bit", dict(bpp=2)),
                         ("dc_quant 0", dict(dc_quant=0)),
                         ("ac_quant 65536", dict(ac_quant=65536)),
                         ("dc_quant 65536", dict(dc_quant=65536))]:
        before = c.launches
        st, h = create_status(c, **fields)
        assert st == B.ERR_ARG and h.value is None, what
        assert c.launches == before
    for what, fields in [("the reference configuration", {}), ("raw coefficients", dict(dc_quant=0, ac_quant=0)),
                         ("no transform: nothing to quantize", dict(tx_size=-1, dc_quant=0)),
                         ("largest step sizes", dict(dc_quant=65535, ac_quant=65535))]:
        st, h = create_status(c, **fields)
        assert st == B.OK and h.value, what
        c.L.b200_frame_pipe_destroy(h)


# ------------------------------------------------------------------ 9. the example

def xorshift(n, rng_range, seed=12345):
    """examples/stream_frames.cpp's stand-in search pattern: the first n values of its xorshift stream."""
    out = []
    for _ in range(n):
        seed = (seed ^ (seed << 13)) & 0xFFFFFFFF
        seed ^= seed >> 17
        seed = (seed ^ (seed << 5)) & 0xFFFFFFFF
        out.append(seed % (2 * rng_range + 1) - rng_range)
    return out


def example_frame(f, W=1920, H=1080):
    y, x = np.mgrid[0:H, 0:W]
    return (128 + 60 * (((x + f) >> 5) & 1) + ((y >> 4) & 15)).astype(np.uint8)


def test_stream_frames_example_matches_the_oracle(tmp_path):
    from tests.test_examples import build
    exe = build(tmp_path)
    r = subprocess.run([exe, "3"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    m = re.search(r"^3 frames in [0-9.]+ s: .* block 0 of the last frame: mv \((-?\d+), (-?\d+)\) sad (\d+) eob (\d+)$",
                  r.stdout, re.M)
    assert m, r.stdout
    # block 0 (at 0, 0) of frame 2 against frame 1, its 64 SAD candidates = the first 128 values of the stream
    so = np.array(xorshift(128, 64), np.int8).reshape(1, 64, 2)
    ocur, oref = oracle_planes(1920, 1080, 96, np.uint8, example_frame(2), example_frame(1))
    blocks = G.grid_blocks(16, 16, 16, 16)
    best = winners(ocur, oref, blocks, 16, 16, 6400, so, None, False)
    coef = O.forward_transform_batch(residuals(ocur, oref, blocks, 16, 16, best), 2, 0, 8)
    _, _, eob, _ = oracle_chain(coef, 2, 0, 88, 100, False)
    assert tuple(int(v) for v in m.groups()) == (int(best[0]["mv_row"]), int(best[0]["mv_col"]), int(best[0]["sad"]),
                                                 int(eob[0]))
