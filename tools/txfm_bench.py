#!/usr/bin/env python3
"""Time the fused residual + forward transform leg on its own (b200_fwd_txfm_residual_multi_dev).

The default line is bench.py's transform leg: 32 resident 1080p 8-bit frame pairs in one launch, one
16x16 DCT_DCT of each 16x16 block's residual against the reference displaced by its full-pel winner
(winners uniform in +-64 px, as bench.py's candidates are).  Three more lines run the same shapes at 10 bit
(u16 planes, i32 coefficients) and with 32x32 and 8x8 blocks.  Each line is one JSON object: ms per launch
(median of several CUDA-event windows after warm-up), the algorithmic bytes of a launch and the rate they
give against the H100 SXM data sheet's 3.35 TB/s, with the card's name and power limit read in the same run.

    python tools/txfm_bench.py [--out profiles/fwd_txfm_h100.jsonl] [--launches 50] [--windows 7]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

W, H, PAD = 1920, 1080, 96     # bench.py's frames
FRAMES = 32                    # bench.py's frame pairs per GPU, all in one launch
MV_RANGE_PX = 64
HBM_BPS = 3.35e12              # H100 SXM data sheet
TX_SIZE = {8: 1, 16: 2, 32: 3}  # TX_8X8, TX_16X16, TX_32X32


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.splitlines()[0]
    name, power = (s.strip() for s in q.split(","))
    return name, power


def run(ctx, B, torch, bd, n, launches, windows):
    bpp = 1 if bd == 8 else 2
    px = np.uint8 if bd == 8 else np.uint16
    rng = np.random.default_rng(bd * 100 + n)
    planes = []
    for f in range(FRAMES):
        pair = []
        for _ in range(2):
            img = rng.integers(0, 1 << bd, (H + 2 * PAD, W + 2 * PAD)).astype(px)
            p = B.Plane()
            ctx.check(ctx.L.b200_plane_alloc(ctx.h, W + 2 * PAD, H + 2 * PAD, 0, bpp, C.byref(p)))
            ctx.check(ctx.L.b200_plane_upload(ctx.h, C.byref(p), img.ctypes.data, img.strides[0]))
            q = B.Plane()
            q.data = p.data + (PAD * p.stride + PAD) * bpp
            q.stride, q.width, q.height, q.pad, q.bpp, q.alloc = p.stride, W, H, PAD, bpp, None
            pair.append((p, q))
        planes.append(pair)
    xs, ys = np.arange(0, W - n + 1, n), np.arange(0, H - n + 1, n)
    blocks = np.zeros(len(xs) * len(ys), B.BLOCK_DTYPE)
    blocks["x"], blocks["y"] = np.tile(xs, len(ys)), np.repeat(ys, len(xs))
    nb = len(blocks)
    total = FRAMES * nb
    mv = np.zeros(total, B.ME_RESULT_DTYPE)
    mv["mv_row"] = rng.integers(-MV_RANGE_PX, MV_RANGE_PX + 1, total) * 8
    mv["mv_col"] = rng.integers(-MV_RANGE_PX, MV_RANGE_PX + 1, total) * 8
    mv["cost"] = rng.integers(0, 1 << 40, total)
    d_blocks = torch.from_numpy(np.tile(blocks, FRAMES).view(np.uint8)).cuda()
    d_mv = torch.from_numpy(mv.view(np.uint8)).cuda()
    coef_bytes = 2 if bd == 8 else 4
    d_coef = torch.empty(total * n * n * coef_bytes, dtype=torch.uint8, device="cuda")
    ends = [(i + 1) * nb for i in range(FRAMES)]
    pairs = B.PlanePairs([pl[0][1] for pl in planes], [pl[1][1] for pl in planes], ends, ends)
    stream = torch.cuda.current_stream()

    def launch():
        ctx.fwd_txfm_residual_multi_dev(pairs, d_blocks, total, d_mv, d_coef, TX_SIZE[n], 0, bd)

    for _ in range(20):
        launch()
    torch.cuda.synchronize()
    times = []
    for _ in range(windows):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(launches):
            launch()
        e1.record(stream)
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / launches)
    for pl in planes:
        for p, _ in pl:
            ctx.check(ctx.L.b200_plane_free(ctx.h, C.byref(p)))
    ms = float(np.median(times))
    # cur and reference pixels, the block record, the winner and the coefficients of every block
    alg = total * (2 * n * n * bpp + 4 + 16 + n * n * coef_bytes)
    return {"leg": "residual+fwd_txfm", "tx": f"{n}x{n} DCT_DCT", "bit_depth": bd, "frame_pairs": FRAMES,
            "blocks": total, "ms_per_launch": ms, "ms_spread": [float(min(times)), float(max(times))],
            "windows": windows, "launches_per_window": launches, "algorithmic_bytes": alg,
            "gb_per_s": alg / (ms * 1e-3) / 1e9, "frac_of_3_35_tb_s": alg / (ms * 1e-3) / HBM_BPS}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", help="append the JSON lines to this file as well")
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--windows", type=int, default=7)
    args = ap.parse_args()
    import torch
    from rav1e_b200 import backend as B
    if not torch.cuda.is_available():
        sys.exit("txfm_bench: no CUDA device")
    torch.cuda.set_device(0)
    ctx = B.Context(0, use_torch_stream=True)
    name, power = card()
    lines = []
    for bd, n in ((8, 16), (10, 16), (8, 32), (8, 8)):
        r = run(ctx, B, torch, bd, n, args.launches, args.windows)
        r.update({"gpu": name, "power_limit": power, "lib": os.path.basename(B.LIB_PATH)})
        print(json.dumps(r), flush=True)
        lines.append(r)
    if args.out:
        with open(args.out, "a") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
