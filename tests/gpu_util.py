"""Helpers shared by the `-m gpu` parity tests: same seeded inputs to the CUDA path (through
the C ABI) and to the oracle."""
import numpy as np

from rav1e_b200 import backend as B
from tests import oracle_lib as O

_CTX = None


def ctx():
    global _CTX
    if _CTX is None:
        # kernels go to torch's current stream: the tests fill torch tensors (torch.zeros, .cuda())
        # on that stream and the ctx's own stream is non-blocking, so sharing one stream is what
        # orders "fill, then launch" (the ordering contract stated in include/b200rdo.h)
        _CTX = B.Context(0, use_torch_stream=True)
    return _CTX


def to_dev(a):
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.uint8).reshape(-1)).cuda()


def from_dev(t, dtype):
    return t.cpu().numpy().view(dtype)


def dev_empty(nbytes):
    import torch
    return torch.empty(max(nbytes, 1), dtype=torch.uint8, device="cuda")


def make_planes(width, height, pad, dtype=np.uint8, seed=0, bit_depth=8, smooth=True, shift=None):
    """`ref` = (optionally low-passed) noise, `cur` = ref displaced per-frame + noise, so that
    SAD surfaces have real minima (SURVEY §8d).  Returns numpy images (visible area)."""
    rng = np.random.default_rng(seed)
    maxv = (1 << bit_depth) - 1
    base = rng.integers(0, maxv + 1, (height + 64, width + 64)).astype(np.float64)
    if smooth:
        k = np.ones(5) / 5.0
        base = np.apply_along_axis(lambda r: np.convolve(r, k, mode="same"), 1, base)
        base = np.apply_along_axis(lambda c: np.convolve(c, k, mode="same"), 0, base)
        base = (base - base.min()) / (base.max() - base.min()) * maxv
    dx, dy = shift if shift is not None else (3, -2)
    ref = base[32:32 + height, 32:32 + width]
    cur = base[32 + dy:32 + dy + height, 32 + dx:32 + dx + width] + rng.normal(0, 2, (height, width))
    # C-contiguous: callers hand .ctypes.data / .strides[0] to the C ABI
    ref = np.ascontiguousarray(np.clip(np.rint(ref), 0, maxv).astype(dtype))
    cur = np.ascontiguousarray(np.clip(np.rint(cur), 0, maxv).astype(dtype))
    return cur, ref


def both_planes(img, pad):
    """(oracle Plane, device b200_plane) of the same image, edges replicated into `pad`."""
    op = O.Plane(img.shape[1], img.shape[0], pad, dtype=img.dtype)
    op.fill_from(img)
    dp = ctx().plane_from_host(img, pad)
    return op, dp


def grid_blocks(width, height, bw, bh):
    xs = np.arange(0, width - bw + 1, bw)
    ys = np.arange(0, height - bh + 1, bh)
    b = np.zeros(len(xs) * len(ys), B.BLOCK_DTYPE)
    b["x"] = np.tile(xs, len(ys))
    b["y"] = np.repeat(ys, len(xs))
    return b


def zorder_blocks(width, height, bw, bh, sb=64):
    """Blocks of a bw x bh grid in the order rav1e walks them: superblocks in raster order, and
    inside a superblock the partition (Z) order of the quadtree, down to the block size."""
    def z(x0, y0, size_w, size_h):
        if size_w <= bw and size_h <= bh:
            return [(x0, y0)]
        hw, hh = max(size_w // 2, bw), max(size_h // 2, bh)
        out = []
        for dy in range(0, size_h, hh):
            for dx in range(0, size_w, hw):
                out += z(x0 + dx, y0 + dy, hw, hh)
        return out
    pos = []
    for sy in range(0, height, sb):
        for sx in range(0, width, sb):
            pos += [(x, y) for x, y in z(sx, sy, sb, sb) if x + bw <= width and y + bh <= height]
    b = np.zeros(len(pos), B.BLOCK_DTYPE)
    b["x"] = [p[0] for p in pos]
    b["y"] = [p[1] for p in pos]
    return b


def mv_range(width, height, x, y, bw, bh):
    """get_mv_range (me.rs:339-362) of the block at luma (x, y), in 1/8 pel:
    (x_min, x_max, y_min, y_max).  w_in_b / h_in_b round the frame up to 8 pixels."""
    w_in_b, h_in_b = 2 * ((width + 7) >> 3), 2 * ((height + 7) >> 3)
    bx, by = x // 4, y // 4
    x_min = -bx * 32 - (128 + 8 * bw)
    x_max = (w_in_b - bx - bw // 4) * 32 + 128 + 8 * bw
    y_min = -by * 32 - (128 + 8 * bh)
    y_max = (h_in_b - by - bh // 4) * 32 + 128 + 8 * bh
    return max(x_min, -(1 << 14) + 1), min(x_max, (1 << 14) - 1), max(y_min, -(1 << 14) + 1), min(y_max, (1 << 14) - 1)


def min_pad(width, height, bw, bh):
    """The smallest border that keeps every footprint get_mv_range accepts readable.  The right-most
    footprint ends at 4 * w_in_b + 16 + bw (the 8-aligned width, not `width`); likewise for y."""
    w8, h8 = 8 * ((width + 7) >> 3), 8 * ((height + 7) >> 3)
    return max(w8 - width + 16 + bw, h8 - height + 16 + bh)


def border_cands(blocks, width, height, bw, bh, reach=None):
    """For every block: the mvs exactly on each get_mv_range limit and on each corner, then one
    eighth-pel and one full-pel beyond each limit (out of range: empty results).  With `reach`
    (pixels), limits farther than that from the block are left out (a window hint must cover
    every candidate)."""
    rows = []
    for k, b in enumerate(blocks):
        x_min, x_max, y_min, y_max = mv_range(width, height, int(b["x"]), int(b["y"]), bw, bh)
        mvs = [(0, x_min), (0, x_max), (y_min, 0), (y_max, 0),
               (y_min, x_min), (y_min, x_max), (y_max, x_min), (y_max, x_max)]
        for d in (1, 8):
            mvs += [(0, x_min - d), (0, x_max + d), (y_min - d, 0), (y_max + d, 0), (y_max + d, x_max + d)]
        if reach is not None:
            mvs = [m for m in mvs if abs(m[0]) <= 8 * reach and abs(m[1]) <= 8 * reach]
        rows += [(k, r, c) for r, c in mvs]
    c = np.zeros(len(rows), B.CAND_DTYPE)
    c["block"] = [r[0] for r in rows]
    c["mv_row"] = [r[1] for r in rows]
    c["mv_col"] = [r[2] for r in rows]
    return c


def merge_lists(nblocks, *lists):
    """Concatenate per-block candidate lists (each sorted by block or not) into one list grouped
    by block, keeping each list's order and the lists' order inside a block.  Returns (cands, offs)."""
    c = np.concatenate(lists)
    c = c[np.argsort(c["block"], kind="stable")]
    offs = np.zeros(nblocks + 1, np.uint32)
    offs[1:] = np.cumsum(np.bincount(c["block"], minlength=nblocks))
    return np.ascontiguousarray(c), offs


class ViewPlane:
    """A caller-built b200_plane over a device buffer this object owns: any element stride, pixel
    (0,0) `offset` bytes past a 128-byte boundary, `alloc` set to the buffer or NULL.  `full` is
    the padded image ((height + 2 pad) x (width + 2 pad)); the buffer has slack all around."""

    def __init__(self, full, pad, stride, offset, with_alloc=True):
        import torch
        full = np.ascontiguousarray(full)
        rows, cols = full.shape
        bpp = full.itemsize
        assert stride >= cols
        before = pad * (stride + 1) * bpp     # bytes from pixel (-pad, -pad) to pixel (0, 0)
        lead = (before + 64 + 127) // 128 * 128 + offset - before   # bytes before pixel (-pad, -pad)
        nbytes = lead + rows * stride * bpp + 256
        host = np.zeros(nbytes, np.uint8)
        body = np.zeros((rows, stride), full.dtype)
        body[:, :cols] = full
        host[lead:lead + body.nbytes] = body.view(np.uint8).reshape(-1)
        self.buf = torch.from_numpy(host).cuda()
        base = self.buf.data_ptr()
        assert base % 256 == 0
        self.plane = B.Plane()
        self.plane.data = base + lead + before
        self.plane.stride = stride
        self.plane.width, self.plane.height = cols - 2 * pad, rows - 2 * pad
        self.plane.pad, self.plane.bpp = pad, bpp
        self.plane.alloc = base if with_alloc else None


def profiled_kernels(fn, prefix="me_"):
    """Run `fn` under torch.profiler and return the kernels whose names start with `prefix` (by
    default the motion-estimation kernels) in launch order, as `name<template args>` (e.g.
    `me_cand_group_u8<16, 16, false>`).  Fails when the profiler saw no device activity at all: an
    empty list must mean "no such kernel ran"."""
    import re
    import time
    import torch
    from torch.profiler import ProfilerActivity, profile
    # A session now and then delivers no device activity at all (not even the marker kernel):
    # such a record is incomplete, and the call (which only writes its outputs) runs again.
    for attempt in range(6):
        time.sleep(0.1 * attempt)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            torch.zeros(1, device="cuda").add_(1)    # one kernel the profiler must see
            fn()
            torch.cuda.synchronize()
        dev = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        if dev:
            break
    assert dev, "torch.profiler recorded no CUDA kernels on this machine: kernel routing cannot be checked"
    names = []
    for n in dev:
        m = re.search(r"\b(" + prefix + r"\w+(?:<[^()]*>)?)\(", n)
        if m:
            names.append(m.group(1))
    return names


def random_cands(nblocks, per_block, max_px, seed=2, fullpel=True, jitter=True):
    """Grouped-by-block candidate list + CSR offsets.  per_block may vary +-50% per block."""
    rng = np.random.default_rng(seed)
    if jitter:
        counts = rng.integers(max(per_block // 2, 0), per_block * 3 // 2 + 1, nblocks)
    else:
        counts = np.full(nblocks, per_block)
    offs = np.zeros(nblocks + 1, np.uint32)
    offs[1:] = np.cumsum(counts)
    n = int(offs[-1])
    c = np.zeros(n, B.CAND_DTYPE)
    c["block"] = np.repeat(np.arange(nblocks, dtype=np.uint32), counts)
    mv = rng.integers(-max_px, max_px + 1, (n, 2))
    if fullpel:
        mv = mv * 8
    else:
        mv = mv * 8 + rng.integers(-7, 8, (n, 2))   # fullpel offset is still mv/8 (trunc)
    c["mv_row"] = mv[:, 0]
    c["mv_col"] = mv[:, 1]
    return c, offs
