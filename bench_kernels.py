#!/usr/bin/env python
"""bench_kernels.py — per-kernel throughput and roofline for every row of SURVEY §8(a), on the
BASELINE configs that are not the headline one (configs[2..4] shapes).  Not the driver's
contract (that is bench.py); this fills BASELINE.md §5's per-kernel table.

Each leg: device-resident inputs, >=3 warm-up launches, CUDA events on the launching stream,
algorithmic bytes per unit from SURVEY §8(d).  Prints one JSON line per leg.
"""
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from rav1e_b200 import backend as B  # noqa: E402
from tests import oracle_lib as O  # noqa: E402  (CPU baseline column only)

PEAK, PEAK_SOURCE = 3350.0, "H100 SXM data sheet 3.35 TB/s"
if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")):
    PEAK = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    PEAK_SOURCE = "measured (MEASURED_PEAKS.json hbm_gbs)"
TX_SIZES = [(4, 4), (8, 8), (16, 16), (32, 32), (64, 64), (4, 8), (8, 4), (8, 16), (16, 8), (16, 32),
            (32, 16), (32, 64), (64, 32), (4, 16), (16, 4), (8, 32), (32, 8), (16, 64), (64, 16)]


def timed(fn, reps=20, warm=3):
    """ms per launch, CUDA events.  The GPU idles (and clocks down) while a CPU-port leg runs between two GPU legs:
    warm up until at least 3 launches AND 3 ms of back-to-back work have gone by."""
    import time
    t0, k = time.perf_counter(), 0
    while k < warm or time.perf_counter() - t0 < 3e-3:
        fn()
        k += 1
        if k % 8 == 0:
            torch.cuda.synchronize()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def cpu_rate(fn, units):
    """units/s of the oracle (all usable host threads) on the same inputs: ~0.5 s of work."""
    import time
    fn()
    t0, reps = time.perf_counter(), 0
    while time.perf_counter() - t0 < 0.5:
        fn()
        reps += 1
    return units * reps / (time.perf_counter() - t0)


def card():
    """name and power limit of cuda:0, read now (nvidia-smi's row with the same PCI bus id)"""
    import subprocess
    props = torch.cuda.get_device_properties(0)
    d = {"device": props.name, "power_limit_w": None}
    try:
        rows = subprocess.run(["nvidia-smi", "--query-gpu=pci.bus_id,name,power.limit", "--format=csv,noheader,nounits"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError):
        return d
    bus = getattr(props, "pci_bus_id", None)
    for r in rows:
        f = [x.strip() for x in r.split(",")]
        if len(f) == 3 and (len(rows) == 1 or (bus is not None and int(f[0].split(":")[1], 16) == bus)):
            d["nvidia_smi_name"] = f[1]
            try:
                d["power_limit_w"] = float(f[2])
            except ValueError:
                pass
    return d


def emit(name, units, unit_name, ms, bytes_per_unit, note="", cpu=None, extra=None, cpu_threads=None):
    gbs = units * bytes_per_unit / (ms * 1e-3) / 1e9
    d = {"kernel": name, "units_per_launch": units, "unit": unit_name, "launch_ms": ms,
         "units_per_s": units / (ms * 1e-3), "algorithmic_bytes_per_unit": bytes_per_unit,
         "algorithmic_GBps": gbs, "frac_of_hbm_peak": gbs / PEAK, "peak_source": PEAK_SOURCE, "note": note}
    d.update(extra or {})
    if cpu is not None:
        d["cpu_port_units_per_s"] = cpu
        d["cpu_threads"] = cpu_threads if cpu_threads is not None else O.host_threads()
        d["gpu_over_cpu"] = d["units_per_s"] / cpu
    print(json.dumps(d))


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).cuda()


def grid_blocks(w, h, bw, bh):
    xs, ys = np.arange(0, w - bw + 1, bw), np.arange(0, h - bh + 1, bh)
    b = np.zeros(len(xs) * len(ys), B.BLOCK_DTYPE)
    b["x"], b["y"] = np.tile(xs, len(ys)), np.repeat(ys, len(xs))
    return b


def host_diamond(ctx, cur, ref, d_blocks, nb, start, p, mode, allow_hp):
    """subpel_diamond_search (me.rs:1311-1383) as a caller without b200_subpel_search_dev runs it: the four
    diamond points of every block still searching go through one b200_me_subpel_candidates_dev launch per
    step, and the per-block first minimum comes back to the host, which moves the centres or halves the
    radii.  Returns the final results and the number of steps."""
    pattern = np.array([(1, 0), (0, 1), (-1, 0), (0, -1)])
    res = start.copy()
    radius = np.full(nb, 2)
    end = 0 if allow_hp else 1
    active = np.ones(nb, bool)
    d_best = torch.empty(nb * 16, dtype=torch.uint8, device="cuda")
    steps = 0
    while active.any():
        idx = np.nonzero(active)[0]
        sh = radius[idx][:, None]
        rows = res["mv_row"][idx].astype(np.int64)[:, None] + (pattern[None, :, 0] << sh)
        cols = res["mv_col"][idx].astype(np.int64)[:, None] + (pattern[None, :, 1] << sh)
        cands = np.zeros(4 * len(idx), B.CAND_DTYPE)
        cands["block"] = np.repeat(idx, 4)
        cands["mv_row"] = ((rows.reshape(-1) + 32768) % 65536 - 32768).astype(np.int16)
        cands["mv_col"] = ((cols.reshape(-1) + 32768) % 65536 - 32768).astype(np.int16)
        counts = np.zeros(nb, np.int64)
        counts[idx] = 4
        offs = np.zeros(nb + 1, np.uint32)
        offs[1:] = np.cumsum(counts)
        ctx.me_subpel_candidates_dev(cur, ref, d_blocks, nb, dev(cands), len(cands), p, mode, dev(offs), None, None,
                                     None, d_best)
        best = d_best.cpu().numpy().view(B.ME_RESULT_DTYPE)[idx]
        better = best["cost"] < res["cost"][idx]
        res[idx[better]] = best[better]
        stay = idx[~better]
        active[stay[radius[stay] == end]] = False
        radius[stay[radius[stay] != end]] -= 1
        steps += 1
    return res, steps


def subpel_sizes(ctx):
    """b200_subpel_search_dev (diamond search + SATD + the winner's DCT_DCT) on a 1080p pair at sizes with a
    side of 64, a control (8x8) and a size below 8 (4x8), 8 and 10 bit, next to the host-driven loop over
    b200_me_subpel_candidates_dev + b200_mc_blocks_dev + b200_fwd_txfm_pred_dev that computes the same."""
    import time
    from scipy.ndimage import uniform_filter
    rng = np.random.default_rng(12)
    W, H, PAD = 1920, 1080, 160
    base = uniform_filter(rng.integers(0, 256, (H + 64, W + 64)).astype(np.float32), 7)
    base = (base - base.min()) / (base.max() - base.min())
    for bd in (8, 10):
        maxv = (1 << bd) - 1
        dtype = np.uint8 if bd == 8 else np.uint16
        ref_img = np.rint(base[32:32 + H, 32:32 + W] * maxv).astype(dtype)
        # the current frame: the reference moved by (+5.5, -3) px, plus noise
        mov = (base[29:29 + H, 37:37 + W] + base[29:29 + H, 38:38 + W]) / 2 * maxv
        cur_img = np.clip(np.rint(mov + rng.normal(0, 1.5 * (maxv / 255), (H, W))), 0, maxv).astype(dtype)
        cur, ref = ctx.plane_from_host(cur_img, PAD), ctx.plane_from_host(ref_img, PAD)
        for (w, h) in ((64, 64), (64, 32), (16, 64), (8, 8), (4, 8)):
            ts = TX_SIZES.index((w, h))
            blocks = grid_blocks(W, H, w, h)
            nb = len(blocks)
            d_blocks = dev(blocks)
            lam = 1200 << (bd - 8)
            p = B.me_params(w, h, W, H, lam, use_satd=True, bit_depth=bd)
            # full-pel starts around the true vector, SATD-scored on the device (the rescore of me.rs:596-616)
            st = np.zeros(nb, B.CAND_DTYPE)
            st["block"] = np.arange(nb)
            st["mv_row"] = (-3 + rng.integers(-1, 2, nb)) * 8
            st["mv_col"] = (5 + rng.integers(0, 2, nb)) * 8
            d_sad = torch.empty(nb * 4, dtype=torch.uint8, device="cuda")
            d_cost = torch.empty(nb * 8, dtype=torch.uint8, device="cuda")
            ctx.me_candidates_dev(cur, ref, d_blocks, nb, dev(st), nb, p, None, None, d_sad, d_cost)
            start = np.zeros(nb, B.ME_RESULT_DTYPE)
            start["sad"] = d_sad.cpu().numpy().view(np.uint32)
            start["cost"] = d_cost.cpu().numpy().view(np.uint64)
            start["mv_row"], start["mv_col"] = st["mv_row"], st["mv_col"]
            d_start = dev(start)
            d_best = torch.empty(nb * 16, dtype=torch.uint8, device="cuda")
            ct = torch.int16 if bd == 8 else torch.int32
            d_coef = torch.empty(nb * w * h, dtype=ct, device="cuda")
            ms = timed(lambda: ctx.subpel_search_dev(cur, ref, d_blocks, nb, d_start, p, d_best, 0, ts, 0, None, d_coef),
                       reps=10)
            fused = d_best.cpu().numpy().view(B.ME_RESULT_DTYPE)
            fused_coef = d_coef.cpu().numpy()
            # the host-driven loop: same starts, same results
            d_pred = torch.empty(nb * w * h * (1 if bd == 8 else 2), dtype=torch.uint8, device="cuda")
            d_coef2 = torch.empty(nb * w * h, dtype=ct, device="cuda")

            def host_chain():
                res, steps = host_diamond(ctx, cur, ref, d_blocks, nb, start, p, 0, False)
                mvs = np.stack([res["mv_row"], res["mv_col"]], 1).astype(np.int16)
                ctx.mc_blocks_dev(ref, d_blocks, dev(mvs), nb, w, h, 0, 0, bd, 0, 0, 0, d_pred)
                ctx.fwd_txfm_pred_dev(cur, d_pred, d_blocks, nb, d_coef2, ts, 0, bd)
                torch.cuda.synchronize()
                return res, steps
            host_chain()
            reps, t0 = 0, time.perf_counter()
            while reps < 3 or time.perf_counter() - t0 < 1.0:
                res, steps = host_chain()
                reps += 1
            host_ms = (time.perf_counter() - t0) * 1e3 / reps
            same = bool(all((res[f] == fused[f]).all() for f in ("cost", "sad", "mv_row", "mv_col"))
                        and (d_coef2.cpu().numpy() == fused_coef).all())
            assert same, f"{w}x{h} {bd}-bit: the host-driven loop and b200_subpel_search_dev disagree"
            moved = int(((fused["mv_row"] != start["mv_row"]) | (fused["mv_col"] != start["mv_col"])).sum())
            bpp = 1 if bd == 8 else 2
            emit(f"subpel_search_dev {w}x{h} {bd}-bit (diamond + SATD + DCT_DCT, fused)", nb, "blocks", ms,
                 (w + 7) * (h + 7) * bpp, "1080p, one launch; bytes: one source footprint per block (lower bound: "
                 "every diamond point re-reads its footprint)",
                 extra={"w": w, "h": h, "bit_depth": bd, "blocks_moved": moved,
                        "library": os.path.basename(B.LIB_PATH)})
            emit(f"host-driven diamond {w}x{h} {bd}-bit (me_subpel_candidates_dev per step + mc_blocks + "
                 "fwd_txfm_pred)", nb, "blocks", host_ms, (w + 7) * (h + 7) * bpp,
                 "same starts and results as the fused leg; launch_ms = whole loop by host clock, "
                 "one device round trip per step", extra={"w": w, "h": h, "bit_depth": bd, "steps": steps,
                                                          "same_results": same,
                                                          "fused_speedup": host_ms / ms})
        ctx.plane_free(cur)
        ctx.plane_free(ref)


def intra_screen(ctx):
    """b200_intra_mode_screen_dev over every block of a 1080p frame (one launch per size), 8 and 10 bit,
    num_modes_rdo 3, next to the same items through b200_get_intra_edges_dev + b200_predict_intra_dev.
    That pair is a lower bound for the composition a caller has without the fused call: it writes the 12
    predictions per block to HBM and stops there, because the library has no SATD against packed
    predictions.  The fused results are checked against the CPU oracle on a sample of blocks."""
    from scipy.ndimage import uniform_filter
    from tests.test_oracle_intra_edges import BSIZES
    from tests.test_oracle_intra_screen import intra_mode_screen
    rng = np.random.default_rng(21)
    W, H, PAD, NM = 1920, 1080, 96, 3
    base = uniform_filter(rng.integers(0, 256, (H, W)).astype(np.float32), 5)
    base = (base - base.min()) / (base.max() - base.min())
    angle = {1: 90, 2: 180, 3: 45, 4: 135, 5: 113, 6: 157, 7: 203, 8: 67}
    for bd in (8, 10):
        maxv = (1 << bd) - 1
        dtype = np.uint8 if bd == 8 else np.uint16
        rec_img = np.rint(base * maxv).astype(dtype)
        src_img = np.clip(np.rint(base * maxv + rng.normal(0, 2 * (maxv / 255), (H, W))), 0, maxv).astype(dtype)
        rec, src = ctx.plane_from_host(rec_img, PAD), ctx.plane_from_host(src_img, PAD)
        orec, osrc = O.Plane(W, H, PAD, dtype), O.Plane(W, H, PAD, dtype)
        orec.fill_from(rec_img)
        osrc.fill_from(src_img)
        for (w, h) in ((4, 4), (8, 8), (16, 16), (16, 8), (32, 32), (64, 64)):
            xs, ys = np.arange(0, W, w), np.arange(0, H, h)          # the last row overhangs 1080
            nb = len(xs) * len(ys)
            items = np.zeros(nb, B.INTRA_SCREEN_ITEM_DTYPE)
            items["x"], items["y"] = np.tile(xs, len(ys)), np.repeat(ys, len(xs))
            items["bsize"] = BSIZES.index((w, h))
            items["ief"] = 0
            items["modes"] = rng.permuted(np.tile(np.arange(13, dtype=np.uint8), (nb, 1)), axis=1)
            d_items = dev(items)
            d_satd = torch.empty(nb * 13 * 4, dtype=torch.uint8, device="cuda")
            d_modes = torch.empty(nb * 13, dtype=torch.uint8, device="cuda")
            rect = (0, 0, W, H)
            ms = timed(lambda: ctx.intra_mode_screen_dev(rec, src, rect, bd, NM, d_items, nb, d_satd, d_modes))
            satd = d_satd.cpu().numpy().view(np.uint32).reshape(nb, 13)
            modes = d_modes.cpu().numpy().reshape(nb, 13)
            sample = rng.choice(nb, min(nb, 2000), replace=False)
            want_satd, want_modes = intra_mode_screen(orec, osrc, rect, bd, NM, items[sample])
            same = bool((satd[sample] == want_satd).all() and (modes[sample] == want_modes).all())
            assert same, f"{w}x{h} {bd}-bit: b200_intra_mode_screen_dev disagrees with the oracle"
            cpu = cpu_rate(lambda: intra_mode_screen(orec, osrc, rect, bd, NM, items), nb)
            # the two-launch lower bound: one edge buffer per block, the 12 screened predictions per block
            eit = np.zeros(nb, B.EDGE_ITEM_DTYPE)
            eit["po_x"], eit["po_y"] = items["x"], items["y"]
            eit["part_x"], eit["part_y"] = items["x"] >> 2, items["y"] >> 2
            eit["bsize"], eit["tx_size"], eit["mode"], eit["enable_ief"] = items["bsize"], TX_SIZES.index((w, h)), 255, 1
            d_eit = dev(eit)
            d_edges = torch.empty(nb * 257 * rec_img.itemsize, dtype=torch.uint8, device="cuda")
            d_lens = torch.empty(nb * 2, dtype=torch.uint8, device="cuda")
            ctx.get_intra_edges_dev(rec, rect, 0, 0, bd, d_eit, nb, d_edges, d_lens)
            lens = d_lens.cpu().numpy().reshape(nb, 2)
            k = 13 - NM // 2
            lm = items["modes"][:, NM // 2:].reshape(-1).astype(np.int64)
            bx, by = np.repeat(items["x"], k), np.repeat(items["y"], k)
            variant = np.where((bx == 0) & (by == 0), 0, np.where(by == 0, 1, np.where(bx == 0, 2, 3)))
            mode = np.where(lm == 12, np.array([0, 2, 1, 12])[variant], lm)
            pit = np.zeros(nb * k, B.INTRA_ITEM_DTYPE)
            pit["edge"] = np.repeat(np.arange(nb), k)
            pit["x"], pit["y"] = bx, by
            pit["angle"] = [angle.get(int(m), 0) for m in mode]
            pit["mode"], pit["variant"] = mode, variant
            pit["ief"] = np.where((lm >= 1) & (lm <= 8), 0, -1)
            pit["left_len"], pit["above_len"] = np.repeat(lens[:, 0], k), np.repeat(lens[:, 1], k)
            d_pit = dev(pit)
            d_pred = torch.empty(nb * k * w * h * rec_img.itemsize, dtype=torch.uint8, device="cuda")

            def two_launch():
                ctx.get_intra_edges_dev(rec, rect, 0, 0, bd, d_eit, nb, d_edges, d_lens)
                ctx.predict_intra_dev(d_edges, d_pit, nb * k, None, w, h, bd, W, H, d_pred)
            ms2 = timed(two_launch)
            bpp = rec_img.itemsize
            nbytes = (2 * (w + h) + 1) * bpp + w * h * bpp + 13 * 4 + 13
            emit(f"intra_mode_screen_dev {w}x{h} {bd}-bit (edges + 12 predictions + SATD + tail sort, fused)", nb,
                 "blocks", ms, nbytes, "1080p, num_modes_rdo 3, one launch; bytes: edge reads + source block + "
                 "13 SATDs and 13 modes out", cpu=cpu,
                 extra={"w": w, "h": h, "bit_depth": bd, "ms_per_frame": ms, "oracle_sample": len(sample),
                        "same_as_oracle": same, "library": os.path.basename(B.LIB_PATH)})
            emit(f"get_intra_edges_dev + predict_intra_dev {w}x{h} {bd}-bit (lower bound of the unfused "
                 "composition)", nb, "blocks", ms2, nbytes + 257 * bpp + k * w * h * bpp,
                 "same items; edges + the 12 predictions written to HBM, no SATD (the library has no SATD over "
                 "packed predictions), so a lower bound for today's composition",
                 extra={"w": w, "h": h, "bit_depth": bd, "ms_per_frame": ms2, "fused_speedup": ms2 / ms})
        ctx.plane_free(rec)
        ctx.plane_free(src)


def cfl_alpha(ctx):
    """b200_cfl_alpha_dev over every chroma-carrying block of each cfl_allowed size of a 1080p 4:2:0 frame (one
    call per size, tx_size = the size's largest luma tx), and one call with all sizes mixed, 8 and 10 bit.  Next
    to it, the same blocks through b200_pred_cfl_ac_dev + b200_get_intra_edges_dev (both planes) +
    b200_predict_intra_dev with 33 items per (block, plane): a lower bound for the composition a caller has
    without the fused call, since it writes every prediction to HBM and computes no SSE and no decision.  A
    sample of every timed fused call is checked against the CPU oracle."""
    from scipy.ndimage import uniform_filter
    from tests.test_oracle_cfl_alpha import CFL_ITEM_DTYPE, Frame, cfl_alpha as orc_cfl_alpha, grid_items, valid
    from tests.test_oracle_intra_edges import BSIZES
    rng = np.random.default_rng(23)
    W, H, PAD = 1920, 1080, 96
    cw, ch = W // 2, H // 2

    def smooth(w, h):
        b = uniform_filter(rng.integers(0, 256, (h, w)).astype(np.float32), 5)
        return (b - b.min()) / (b.max() - b.min())
    luma, cb, cr = smooth(W + 32, H + 32), smooth(cw, ch), smooth(cw, ch)
    for bd in (8, 10):
        maxv = (1 << bd) - 1
        dtype = np.uint8 if bd == 8 else np.uint16
        bpp = np.dtype(dtype).itemsize
        q = [np.rint(p * maxv).astype(dtype) for p in (luma, cb, cr)]
        srcs = [q[0]] + [np.clip(np.rint(p * maxv + rng.normal(0, 3 * maxv / 255, p.shape)), 0, maxv).astype(dtype)
                         for p in (cb, cr)]
        F = Frame(q, srcs, 1, 1, W, H, bd)
        rec = [ctx.plane_from_host(p.view(), PAD) for p in F.rec]
        src = [ctx.plane_from_host(p.view(), PAD) for p in F.src]
        rect = (0, 0, W, H)
        per_size = {}
        for bs in range(10):
            items = grid_items(rng, rect, [bs], tx_random=False)
            keep = np.array([valid(F, rect, int(i["x"]), int(i["y"]), bs, int(i["tx_size"])) for i in items])
            per_size[bs] = items[keep]
        mixed = np.concatenate([per_size[bs] for bs in range(10)])
        mixed = mixed[rng.permutation(len(mixed))]
        for bs in list(range(10)) + ["mixed"]:
            items = mixed if bs == "mixed" else per_size[bs]
            label = "mixed sizes" if bs == "mixed" else "%dx%d" % BSIZES[bs]
            nb = len(items)
            d_items = dev(items)
            d_alpha = torch.empty(nb * 2, dtype=torch.uint8, device="cuda")
            d_sse = torch.empty(nb * 66 * 8, dtype=torch.uint8, device="cuda")
            ms = timed(lambda: ctx.cfl_alpha_dev(rec, src, 1, 1, rect, W, H, bd, d_items, nb, d_alpha, d_sse))
            alpha = d_alpha.cpu().numpy().view(np.int8).reshape(nb, 2)
            sse = d_sse.cpu().numpy().view(np.uint64).reshape(nb, 2, 33)
            sample = rng.choice(nb, min(nb, 2000), replace=False)
            want_alpha, want_sse = orc_cfl_alpha(F, rect, items[sample])
            same = bool((alpha[sample] == want_alpha).all() and (sse[sample] == want_sse).all())
            assert same, f"{label} {bd}-bit: b200_cfl_alpha_dev disagrees with the oracle"
            cpu = cpu_rate(lambda: orc_cfl_alpha(F, rect, items, threads=O.host_threads()), nb)
            bw = np.array([BSIZES[b][0] for b in items["bsize"]])
            bh = np.array([BSIZES[b][1] for b in items["bsize"]])
            tw, th = np.maximum(bw // 2, 4), np.maximum(bh // 2, 4)
            # bytes per block: the luma footprint, two edge buffers, two source blocks, the 2 + 66 * 8 outputs
            nbytes = float(np.mean((tw * th * 4 + 2 * (2 * (tw + th) + 1) + 2 * tw * th) * bpp + 2 + 66 * 8))
            extra = {"block": label, "bit_depth": bd, "ms_per_call": ms, "oracle_sample": len(sample),
                     "same_as_oracle": same, "alphas_evaluated_mean": float((sse != np.uint64(2**64 - 1)).sum() / nb / 2),
                     "library": os.path.basename(B.LIB_PATH)}
            emit(f"cfl_alpha_dev {label} {bd}-bit 4:2:0 (luma AC + 2 x (edges + 33 CfL predictions + SSE) + early "
                 "exit, fused)", nb, "blocks", ms, nbytes, "1080p 4:2:0, every chroma-carrying block, tx = largest "
                 "luma tx, one call; bytes: luma footprint + 2 edges + 2 source blocks + outputs", cpu=cpu, extra=extra)
            if bs == "mixed":
                continue
            # the lower bound: AC, edges of both planes, 33 predictions per (block, plane) written to HBM
            w, h = int(tw[0]), int(th[0])
            blocks = np.zeros(nb, B.BLOCK_DTYPE)
            blocks["x"], blocks["y"] = items["x"] - 4 * (bw == 4), items["y"] - 4 * (bh == 4)   # sub8x8_offset
            d_blocks = dev(blocks)
            d_ac = torch.empty(nb * w * h * 2, dtype=torch.uint8, device="cuda")
            eit = np.zeros(nb, B.EDGE_ITEM_DTYPE)
            eit["po_x"], eit["po_y"] = (items["x"] >> 3) << 2, (items["y"] >> 3) << 2
            eit["part_x"], eit["part_y"] = items["x"] >> 2, items["y"] >> 2
            eit["bsize"], eit["tx_size"], eit["mode"] = bs, TX_SIZES.index((w, h)), 13
            d_eit = dev(eit)
            ebytes = nb * 257 * bpp
            d_edges = torch.empty(2 * ebytes, dtype=torch.uint8, device="cuda")
            d_lens = torch.empty(2 * nb * 2, dtype=torch.uint8, device="cuda")
            crect = (0, 0, cw, ch)
            for p in (0, 1):
                ctx.get_intra_edges_dev(rec[1 + p], crect, 1, 1, bd, d_eit, nb, d_edges[p * ebytes:],
                                        d_lens[p * nb * 2:])
            lens = d_lens.cpu().numpy().reshape(2, nb, 2)
            pit = np.zeros((2, nb, 33), B.INTRA_ITEM_DTYPE)
            al = np.arange(-16, 17)
            px, py = eit["po_x"][None, :, None], eit["po_y"][None, :, None]
            pit["edge"] = np.arange(2)[:, None, None] * nb + np.arange(nb)[None, :, None]
            pit["ac"] = np.arange(nb)[None, :, None]
            pit["x"], pit["y"] = px, py
            pit["angle"], pit["mode"] = al[None, None, :], np.where(al == 0, 0, 13)[None, None, :]
            pit["variant"] = np.where((px == 0) & (py == 0), 0, np.where(py == 0, 1, np.where(px == 0, 2, 3)))
            pit["ief"] = -1
            pit["left_len"], pit["above_len"] = lens[:, :, 0][:, :, None], lens[:, :, 1][:, :, None]
            d_pit = dev(pit.reshape(-1))
            d_pred = torch.empty(2 * nb * 33 * w * h * bpp, dtype=torch.uint8, device="cuda")

            def composed():
                ctx.pred_cfl_ac_dev(rec[0], d_blocks, nb, w, h, 0, 0, 1, 1, d_ac)
                for p in (0, 1):
                    ctx.get_intra_edges_dev(rec[1 + p], crect, 1, 1, bd, d_eit, nb, d_edges[p * ebytes:],
                                            d_lens[p * nb * 2:])
                ctx.predict_intra_dev(d_edges, d_pit, 2 * nb * 33, d_ac, w, h, bd, cw, ch, d_pred)
            ms2 = timed(composed)
            emit(f"pred_cfl_ac_dev + get_intra_edges_dev x2 + predict_intra_dev x66 {label} {bd}-bit 4:2:0 (lower "
                 "bound of the unfused composition)", nb, "blocks", ms2, nbytes + 66 * w * h * bpp,
                 "same blocks; the 66 predictions per block written to HBM, no SSE and no decision (the library has "
                 "no SSE over packed predictions), so a lower bound for today's composition",
                 extra={"block": label, "bit_depth": bd, "ms_per_call": ms2, "fused_speedup": ms2 / ms})
        for p in rec + src:
            ctx.plane_free(p)


def inter_screen(ctx):
    """b200_inter_mode_screen_dev over every block of a 1080p frame (one call per size), 8 and 10 bit, on
    lists from the mode-list model (rdo.rs:1158-1318) for two references, one forward and one backward, with
    include_near_mvs off as at speed 6.  Beside it, the same entries through what a caller has without the
    fused call: b200_mc_blocks_dev put for the single entries (one launch per reference), prep of both
    references and b200_mc_avg_dev for the compound ones.  That path writes every prediction to HBM and
    computes no SATD, so it is a lower bound.  The fused results are checked against the CPU oracle on a
    sample of blocks."""
    from scipy.ndimage import uniform_filter
    from tests.test_oracle_intra_edges import BSIZES
    from tests.test_oracle_inter_screen import ENTRIES, build_mode_list, host_plane, inter_mode_screen, origins
    rng = np.random.default_rng(23)
    W, H, SPAD, RPAD = 1920, 1080, 64, 128
    base = uniform_filter(rng.integers(0, 256, (H + 64, W + 64)).astype(np.float32), 9)
    base = (base - base.min()) / (base.max() - base.min())
    dy, dx = -2, 5                     # cur = ref0 moved by (dx, dy); ref1 moved the other way
    z = (0, 0)
    for bd in (8, 10):
        maxv = (1 << bd) - 1
        dtype = np.uint8 if bd == 8 else np.uint16
        img = lambda oy, ox: np.ascontiguousarray(np.rint(base[32 + oy:32 + oy + H, 32 + ox:32 + ox + W] * maxv)
                                                  .astype(dtype))
        ref0_img, ref1_img = img(0, 0), img(-2 * dy, -2 * dx)
        src_img = np.clip(img(dy, dx).astype(np.float64) + rng.normal(0, 2 * maxv / 255, (H, W)), 0, maxv).astype(dtype)
        src, refs = ctx.plane_from_host(src_img, SPAD), [ctx.plane_from_host(r, RPAD) for r in (ref0_img, ref1_img)]
        osrc, orefs = host_plane(src_img, SPAD), [host_plane(r, RPAD) for r in (ref0_img, ref1_img)]
        xo, yo = origins(bd)
        for (w, h) in ((4, 4), (8, 8), (16, 8), (16, 16), (32, 32), (64, 64)):
            xs, ys = np.arange(0, W, w), np.arange(0, H, h)
            nb = len(xs) * len(ys)
            items = np.zeros(nb, B.INTER_SCREEN_ITEM_DTYPE)
            items["x"], items["y"] = np.tile(xs, len(ys)), np.repeat(ys, len(xs))
            items["bsize"] = BSIZES.index((w, h))
            # per block: two-entry stacks and ME vectors near the true motion (1/8 pel), one compound entry
            true = [(-8 * dy, -8 * dx), (8 * dy, 8 * dx)]
            jit = rng.integers(-12, 13, (nb, 8, 2))
            refs_a = np.full((nb, ENTRIES, 2), 0, np.uint8)
            mvs_a = np.zeros((nb, ENTRIES, 2, 2), np.int16)
            ns = np.zeros(nb, np.uint8)
            for b in range(nb):
                v = [tuple(int(t) for t in np.add(true[k % 2], jit[b, k])) for k in range(8)]
                lst = build_mode_list(w, h, [[(v[0], z), (v[2], z)], [(v[1], z), (v[3], z)]], [v[4], v[5]], False,
                                      True, 0, 1, [(v[6], v[7])])
                ns[b] = len(lst)
                for k, (_, r, mv) in enumerate(lst):
                    refs_a[b, k] = (r[0], 0xFF if r[1] is None else r[1])
                    mvs_a[b, k] = mv
            items["n"] = ns
            items["cands"]["ref"] = refs_a
            items["cands"]["mv"] = mvs_a
            d_items = dev(items)
            d_satd = torch.empty(nb * ENTRIES * 4, dtype=torch.uint8, device="cuda")
            d_order = torch.empty(nb * ENTRIES, dtype=torch.uint8, device="cuda")
            rect = (0, 0, W, H)
            ms = timed(lambda: ctx.inter_mode_screen_dev(src, rect, refs, xo, yo, 0, bd, d_items, nb, d_satd, d_order))
            satd = d_satd.cpu().numpy().view(np.uint32).reshape(nb, ENTRIES)
            order = d_order.cpu().numpy().reshape(nb, ENTRIES)
            sample = rng.choice(nb, min(nb, 2000), replace=False)
            want_satd, want_order = inter_mode_screen(osrc, rect, orefs, xo, yo, 0, bd, items[sample])
            same = bool((satd[sample] == want_satd).all() and (order[sample] == want_order).all())
            assert same, f"{w}x{h} {bd}-bit: b200_inter_mode_screen_dev disagrees with the oracle"
            cpu_items = items[sample]
            cpu = cpu_rate(lambda: inter_mode_screen(osrc, rect, orefs, xo, yo, 0, bd, cpu_items,
                                                     threads=O.host_threads()), len(cpu_items))
            # the unfused lower bound: every entry's prediction through the MC launches, written to HBM
            n_ent = int(ns.sum())
            bi = np.repeat(np.arange(nb), ns)
            ki = np.concatenate([np.arange(k) for k in ns])
            e_refs, e_mvs = refs_a[bi, ki], mvs_a[bi, ki]
            single = e_refs[:, 1] == 0xFF
            blk = np.zeros(n_ent, B.BLOCK_DTYPE)
            blk["x"], blk["y"] = items["x"][bi], items["y"][bi]
            bpp = src_img.itemsize
            groups = []
            for r in (0, 1):
                m = single & (e_refs[:, 0] == r)
                groups.append((refs[r], dev(blk[m]), dev(e_mvs[m, 0].copy()), int(m.sum()), 0))
            comp = ~single
            nc = int(comp.sum())
            d_cb = dev(blk[comp])
            groups.append((refs[0], d_cb, dev(e_mvs[comp, 0].copy()), nc, 1))
            groups.append((refs[1], d_cb, dev(e_mvs[comp, 1].copy()), nc, 1))
            d_out = [torch.empty(max(g[3], 1) * w * h * (bpp if g[4] == 0 else 2), dtype=torch.uint8, device="cuda")
                     for g in groups]
            d_avg = torch.empty(max(nc, 1) * w * h * bpp, dtype=torch.uint8, device="cuda")

            def unfused():
                for g, o in zip(groups, d_out):
                    if g[3]:
                        ctx.mc_blocks_dev(g[0], g[1], g[2], g[3], w, h, 0, 0, bd, 0, 0, g[4], o)
                if nc:
                    ctx.mc_avg_dev(d_out[2], d_out[3], d_avg, nc, w, h, bd)
            ms2 = timed(unfused)
            per_block = n_ent / nb
            ncomp = nc / nb
            fp = (w + 7) * (h + 7) * bpp
            nbytes = 248 + w * h * bpp + (per_block + ncomp) * fp + ENTRIES * 5
            emit(f"inter_mode_screen_dev {w}x{h} {bd}-bit (single + compound predictions + SATD + stable sort, fused)",
                 nb, "blocks", ms, nbytes, "1080p, two references, speed-6 lists from the mode-list model; one call "
                 "(bucketing + 3 size-class launches); bytes: item + source block + footprints + 20 SATDs / order out",
                 cpu=cpu, extra={"w": w, "h": h, "bit_depth": bd, "ms_per_frame": ms, "entries_per_block": per_block,
                                 "compound_per_block": ncomp, "oracle_sample": len(sample), "same_as_oracle": same,
                                 "cpu_port_sample_blocks": len(cpu_items), "library": os.path.basename(B.LIB_PATH)})
            emit(f"mc_blocks_dev put + prep x2 + mc_avg_dev {w}x{h} {bd}-bit (lower bound of the unfused composition)",
                 nb, "blocks", ms2, nbytes + (per_block * w * h + ncomp * (4 * w * h)) * bpp,
                 "same entries; predictions written to HBM and no SATD or sort (the library has no SATD over packed "
                 "predictions), so a lower bound for today's composition",
                 extra={"w": w, "h": h, "bit_depth": bd, "ms_per_frame": ms2, "fused_speedup": ms2 / ms})
        for p in [src] + refs:
            ctx.plane_free(p)


def cdef_rdo(ctx):
    """b200_cdef_rdo_dev over whole 1080p 4:2:0 frames: 8 and 10 bit, cdef_bits 0 and 3, areas of 1x1 and 2x2
    superblocks (trimmed at the frame's edge), 30 % of the 8x8 blocks skipped, the winner's pixels written.  The
    fused results are checked against the CPU oracle on the same frame.  Beside it, what a caller can launch
    today: b200_cdef_find_dir_dev once, then per index the CDEF filter for three planes, b200_cdef_dist_dev over
    the luma 8x8 blocks and b200_weighted_sse_dev over the chroma blocks.  That chain takes no decision, filters
    with frame-relative edges (so its output is not the reference's) and has no cost or argmin: a lower bound."""
    from tests.test_oracle_cdef_rdo import DEFAULT_STRENGTHS, cdef_rdo as orc_cdef_rdo, make_frame
    rng = np.random.default_rng(31)
    W, H, PAD = 1920, 1080, 8
    sbw, sbh = 30, 17
    w8, h8 = W // 8, (H + 7) // 8
    for bd in (8, 10):
        rec, src = make_frame(rng, W, H, "420", bd)
        skip8 = (rng.random((h8, w8)) < 0.3).astype(np.uint8)
        bpp = rec[0].itemsize
        d_rec = [ctx.plane_from_host(r, PAD) for r in rec]
        d_src = [ctx.plane_from_host(s, PAD) for s in src]
        d_out = [ctx.plane_from_host(r, PAD) for r in rec]
        d_skip = dev(skip8)
        for cdef_bits in (0, 3):
            n_idx = 1 << cdef_bits
            for a in (1, 2):
                areas = [(x, y, min(a, sbw - x), min(a, sbh - y)) for y in range(0, sbh, a) for x in range(0, sbw, a)]
                n = len(areas)
                d_err = torch.empty(n * 16 * 8 * 8, dtype=torch.uint8, device="cuda")
                d_cost = torch.empty(n * 16 * 8 * 8, dtype=torch.uint8, device="cuda")
                d_best = torch.empty(n * 16, dtype=torch.uint8, device="cuda")
                ys, us = DEFAULT_STRENGTHS, DEFAULT_STRENGTHS[::-1]

                def fused():
                    ctx.cdef_rdo_dev(d_rec, d_src, d_out, 1, 1, W, H, bd, 5, cdef_bits, ys, us, d_skip, None,
                                     (16384, 16384, 16384), 1000.0, areas, None, d_err, d_cost, d_best)
                ms = timed(fused, reps=10)
                want_out = [r.copy() for r in rec]
                err, cost, best = orc_cdef_rdo(rec, src, want_out, 1, 1, W, H, bd, 5, cdef_bits, ys, us, skip8, None,
                                               (16384,) * 3, 1000.0, areas)
                got_best = d_best.cpu().numpy().view(np.int8)
                got_err = d_err.cpu().numpy().view(np.uint64).reshape(n * 16, 8)
                inside = np.zeros(n * 16, bool)      # slots of superblocks inside their area; the rest are not written
                for k, (_, _, aw, ah) in enumerate(areas):
                    for y in range(ah):
                        inside[k * 16 + y * 4:k * 16 + y * 4 + aw] = True
                dec = inside & (best[:n * 16] >= 0)
                same = bool((got_best[inside] == best[:n * 16][inside]).all()
                            and (got_err[dec, :n_idx] == err[:n * 16][dec, :n_idx]).all())
                for p in range(3):
                    got = np.empty_like(rec[p])
                    ctx.check(ctx.L.b200_plane_download(ctx.h, C.byref(d_out[p]), got.ctypes.data, got.strides[0]))
                    same = same and bool((got == want_out[p]).all())
                assert same, f"{bd}-bit cdef_bits {cdef_bits} {a}x{a}: b200_cdef_rdo_dev disagrees with the oracle"
                nsb = sbw * sbh
                tile = (68 * 68 + 2 * 36 * 36) * bpp
                nbytes = tile + 2 * (64 * 64 + 2 * 32 * 32) * bpp + 64 + n_idx * 16 + 1
                emit(f"cdef_rdo_dev {bd}-bit cdef_bits {cdef_bits} {a}x{a} areas (filter + dist + cost + argmin, fused)",
                     nsb, "superblocks", ms, nbytes,
                     "1080p 4:2:0, 30 % skipped 8x8 blocks, winner written; bytes per superblock: rec tiles with halo "
                     "+ src + out + skip flags + err/cost/best",
                     extra={"bit_depth": bd, "cdef_bits": cdef_bits, "area_sb": a, "areas": n, "ms_per_frame": ms,
                            "same_as_oracle": same})
                if a == 2:
                    continue
                # the unfused chain: the same work through the existing launches, frame-relative edges
                d_dir = torch.empty(w8 * h8, dtype=torch.uint8, device="cuda")
                d_var = torch.empty(w8 * h8 * 4, dtype=torch.uint8, device="cuda")
                tmp = [ctx.plane_from_host(r, PAD) for r in rec]
                lb = np.zeros(w8 * h8, B.BLOCK_DTYPE)
                lb["x"], lb["y"] = np.tile(np.arange(w8) * 8, h8), np.repeat(np.arange(h8) * 8, w8)
                cb = lb.copy()
                cb["x"] //= 2
                cb["y"] //= 2
                d_lb, d_cb = dev(lb), dev(cb)
                d_scale = dev(np.full((h8 * 2) * (w8 * 2), 16384, np.uint32))
                d_dist = torch.empty(w8 * h8 * 8, dtype=torch.uint8, device="cuda")
                strengths = [dev(np.full(sbw * sbh, v, np.uint8)) for v in ys + us]
                h8p = (H + 7) & ~7

                def unfused():
                    ctx.cdef_find_dir_dev(d_rec[0], bd, d_skip, d_dir, d_var)
                    for i in range(n_idx):
                        for p in range(3):
                            ctx.cdef_filter_plane_dev(d_rec[p], tmp[p], p, int(p > 0), int(p > 0), W, h8p, bd, 5, d_skip,
                                                      d_dir, d_var, strengths[i if p == 0 else 8 + i])
                        ctx.cdef_dist_dev(d_src[0], tmp[0], d_lb, w8 * h8, 8, 8, bd, d_dist)
                        for p in (1, 2):
                            ctx.weighted_sse_dev(d_src[p], tmp[p], d_cb, w8 * h8, 4, 4, d_scale, w8 * 2, d_dist)
                ms2 = timed(unfused, reps=10)
                emit(f"cdef find_dir + (filter x3 + cdef_dist + weighted_sse x2) per index, {bd}-bit cdef_bits "
                     f"{cdef_bits} (lower bound of the unfused composition)", nsb, "superblocks", ms2,
                     nbytes + n_idx * (2 * (64 * 64 + 2 * 32 * 32) * bpp * 2),
                     "frame-relative edges, so its output is NOT the reference's area-relative one; no cost, argmin "
                     "or winner write: a lower bound for today's composition",
                     extra={"bit_depth": bd, "cdef_bits": cdef_bits, "ms_per_frame": ms2,
                            "fused_1x1_speedup": ms2 / ms})
                for p in tmp:
                    ctx.plane_free(p)
        for p in d_rec + d_src + d_out:
            ctx.plane_free(p)


def deblock(ctx):
    """b200_deblock_levels_dev and b200_deblock_filter_dev on a 1080p 4:2:0 frame at 8 and 10 bit (seeded
    partition, half the blocks skip), once as one frame item and once as 2x2-superblock area items, each call
    timed on its own.  Algorithmic bytes: the level search reads rec + src over the items and the 4x4 block
    grid; the filter reads in + the grid and writes out.  Next to it, the oracle with every host thread on the
    same inputs (one thread per item), and a full check of levels, tallies and output against it."""
    from tests.test_deblock_gpu import DevPlanes, frame_setup
    from tests.test_oracle_deblock import orc_levels
    from tests.test_oracle_deblock_spec import PAD, orc_filter, state_array
    W, H = 1920, 1080
    w4, h4 = W // 4, ((H + 7) >> 3) * 2
    frame = [(0, 0, w4, h4, W, H)]
    areas = [(x, y, min(32, w4 - x), min(32, h4 - y), W - 4 * x, H - 4 * y) for y in range(0, h4, 32)
             for x in range(0, w4, 32)]
    st = state_array()
    for bd in (8, 10):
        rng = np.random.default_rng(60 + bd)
        grid, src, rec = frame_setup(rng, "420", bd, W, H, skip_p=0.5)
        bpp = 1 if bd == 8 else 2
        pix = (W * H * 3 // 2) * bpp
        d_rec, d_src = DevPlanes(ctx, rec, "420"), DevPlanes(ctx, src, "420")
        d_out = DevPlanes(ctx, [np.zeros_like(a) for a in rec], "420")
        d_mi = dev(grid)
        for label, items in (("frame item", frame), ("2x2-superblock areas", areas)):
            n = len(items)
            d_lv = torch.empty(n * 4, dtype=torch.uint8, device="cuda")
            d_t = torch.empty(n * 3 * 2 * 64 * 8, dtype=torch.uint8, device="cuda")
            lv_ms = timed(lambda: ctx.deblock_levels_dev(d_rec.views, d_src.views, 1, 1, bd, d_mi, w4, items, d_lv,
                                                          d_t))
            f_ms = timed(lambda: ctx.deblock_filter_dev(d_rec.views, d_out.views, 1, 1, bd, st, d_lv, d_mi, w4, items))
            want_lv, want_t = orc_levels(rec, src, "420", bd, grid, items)
            got_lv = d_lv.cpu().numpy().reshape(n, 4)
            got_t = d_t.cpu().numpy().view(np.int64).reshape(n, 3, 2, 64)
            filt = [a.copy() for a in rec]
            orc_filter(filt, "420", bd, st, want_lv, grid, items)
            got = d_out.download()

            def visible(a, p):
                o, w, h = PAD >> (p > 0), W >> (p > 0), H >> (p > 0)
                return a[o:o + h, o:o + w]
            same = bool((got_lv == want_lv).all() and (got_t == want_t).all() and
                        all((visible(g, p) == visible(f, p)).all() for p, (g, f) in enumerate(zip(got, filt))))
            assert same, f"deblock {label} {bd}-bit disagrees with the oracle"
            cpu_lv = cpu_rate(lambda: orc_levels(rec, src, "420", bd, grid, items), 1)
            cpu_f = cpu_rate(lambda: orc_filter([a.copy() for a in rec], "420", bd, st, want_lv, grid, items), 1)
            extra = {"items": n, "bit_depth": bd, "same_as_oracle": same, "levels_mean": float(want_lv.mean()),
                     "library": os.path.basename(B.LIB_PATH)}
            emit(f"deblock_levels_dev {label} {bd}-bit 4:2:0 (sse_optimize)", 1, "frames", lv_ms,
                 2 * pix + grid.nbytes, "1080p, seeded partition, half skip; bytes: rec + src + 4x4 grid",
                 cpu=cpu_lv, extra=extra)
            emit(f"deblock_filter_dev {label} {bd}-bit 4:2:0 (deblock_filter_frame)", 1, "frames", f_ms,
                 2 * pix + grid.nbytes, "same frame and levels; bytes: in + out + 4x4 grid", cpu=cpu_f, extra=extra)
        for dp in (d_rec, d_src, d_out):
            dp.free()


def lrf(ctx):
    """b200_lrf_filter_dev on a 1080p 4:2:0 frame at 8 and 10 bit (seeded smooth content plus noise), with the
    two unit configurations RestorationState::new gives 1080p (small: luma 64 / chroma 32 at low base_q_idx;
    large: 256 / 256 at base_q_idx above 200) and three unit mixes: all Sgrproj (what rav1e emits), all Wiener,
    and None / Wiener / Sgrproj drawn at random.  Algorithmic bytes: cdeffed read and out written over the
    crop; the deblocked frame's reads (a few rows per stripe) are left out.  Next to it, the oracle on one host
    thread on the same inputs, and a full check of the output against it."""
    from tests.test_lrf_gpu import DevPlanes
    from tests.test_oracle_lrf_spec import PAD, make_frame, orc_lrf, random_units, unit_grid
    W, H = 1920, 1080
    for bd in (8, 10):
        rng = np.random.default_rng(70 + bd)
        cd, db = make_frame(rng, W, H, "420", bd, "smooth")
        bpp = 1 if bd == 8 else 2
        pix = (W * H + 2 * (W // 2) * (H // 2)) * bpp
        d_cd, d_db = DevPlanes(ctx, cd), DevPlanes(ctx, db)
        d_out = DevPlanes(ctx, [np.zeros_like(a) for a in cd])
        for cfg, us in (("small units 64/32", [64, 32, 32]), ("large units 256/256", [256, 256, 256])):
            for mix, kinds in (("all sgrproj", (2,)), ("all wiener", (1,)), ("mixed", (0, 1, 2))):
                units = [random_units(rng, *unit_grid(W, H, p, "420", us[p]), kinds=kinds) for p in range(3)]
                ms = timed(lambda: ctx.lrf_filter_dev(d_cd.views, d_db.views, d_out.views, 1, 1, W, H, bd, 1, us,
                                                      units))
                want = orc_lrf(cd, db, "420", bd, W, H, 1, us, units)
                got = d_out.download()
                same = all((g[PAD:PAD + (H >> (p > 0)), PAD:PAD + (W >> (p > 0))] ==
                            w[PAD:PAD + (H >> (p > 0)), PAD:PAD + (W >> (p > 0))]).all()
                           for p, (g, w) in enumerate(zip(got, want)))
                assert same, f"lrf {cfg} {mix} {bd}-bit disagrees with the oracle"
                cpu = cpu_rate(lambda: orc_lrf(cd, db, "420", bd, W, H, 1, us, units), 1)
                extra = {"bit_depth": bd, "unit_size": us, "units": mix, "same_as_oracle": same,
                         "library": os.path.basename(B.LIB_PATH)}
                emit(f"lrf_filter_dev {cfg} {mix} {bd}-bit 4:2:0 (lrf_filter_frame)", 1, "frames", ms, 2 * pix,
                     "1080p seeded; bytes: cdeffed + out over the crop", cpu=cpu, extra=extra)
        for dp in (d_cd, d_db, d_out):
            dp.free()


def lrf_search(ctx):
    """b200_lrf_search_dev on a 1080p 4:2:0 frame at 8 and 10 bit (seeded smooth content plus noise), every item
    of the frame in one call, for the three unit configurations RestorationState::new picks by base_q_idx (luma
    64 / 128 / 256, chroma half), with the Full and the Reduced set lists.  Algorithmic bytes: lrf_in and src
    read once per item over its unit.  Next to it, orc_lrf_search on one host thread on the same inputs, and a
    full check of every output against it."""
    from tests.test_oracle_lrf_search import areas_and_items, lrf_search as orc_search, make_frame
    W, H = 1920, 1080
    for bd in (8, 10):
        rng = np.random.default_rng(80 + bd)
        lin, src = make_frame(rng, W, H, "420", bd)
        bpp = 1 if bd == 8 else 2
        pix = (W * H + 2 * (W // 2) * (H // 2)) * bpp
        d_in = [ctx.plane_from_host(a, 8) for a in lin]
        d_src = [ctx.plane_from_host(a, 8) for a in src]
        for uy in (64, 128, 256):
            us = [uy, uy >> 1, uy >> 1]
            areas, items = areas_and_items(rng, W, H, "420", us, incoming="mixed")
            n = len(items)
            d_best, d_cost, d_ch = dev(np.zeros(12 * n, np.uint8)), dev(np.zeros(n)), dev(np.zeros(n, np.uint8))
            for reduced in (0, 1):
                ms = timed(lambda: ctx.lrf_search_dev(d_in, d_src, 1, 1, W, H, bd, us, reduced, None, (16384,) * 3,
                                                      500.0, areas, items, d_best, d_cost, d_ch))
                want = orc_search(lin, src, "420", W, H, bd, us, reduced, areas, items, lam=500.0)
                same = bool((d_best.cpu().numpy().view(np.uint8) == want[0].view(np.uint8)).all() and
                            (d_cost.cpu().numpy().view(np.uint64) == want[1].view(np.uint64)).all() and
                            (d_ch.cpu().numpy() == want[2]).all())
                assert same, f"lrf_search {uy} reduced={reduced} {bd}-bit disagrees with the oracle"
                cpu = cpu_rate(lambda: orc_search(lin, src, "420", W, H, bd, us, reduced, areas, items, lam=500.0), 1)
                extra = {"bit_depth": bd, "unit_size": us, "sets": "reduced" if reduced else "full", "items": n,
                         "same_as_oracle": same, "library": os.path.basename(B.LIB_PATH)}
                emit(f"lrf_search_dev units {uy}/{uy >> 1} {'reduced' if reduced else 'full'} sets {bd}-bit 4:2:0",
                     1, "frames", ms, 2 * pix, "1080p seeded, every item in one call; bytes: lrf_in + src once",
                     cpu=cpu, extra=extra)
        for p in d_in + d_src:
            ctx.plane_free(p)


def loop_decision(ctx):
    """b200_loop_decision_dev over a whole 1080p 4:2:0 frame at 8 and 10 bit (seeded smooth content plus noise,
    30% of the 8x8 blocks skipped, 20% of the units lru_skip), every area in one call, for the unit
    configurations of the search leg with the Full and Reduced set lists.  The time includes the per-stage status
    reads.  Next to it, orc_loop_decision on one host thread on the same inputs, and a check of every output."""
    from tests.test_oracle_loop_decision import case, run
    W, H = 1920, 1080
    for bd in (8, 10):
        for uy in (64, 128, 256):
            fx = case(100 + bd + uy, "420", bd, W, H, (uy, uy >> 1, uy >> 1), lam=500.0)
            d_rec = [ctx.plane_from_host(a, 8) for a in fx["rec"]]
            d_src = [ctx.plane_from_host(a, 8) for a in fx["src"]]
            d_work = [ctx.plane_from_host(np.zeros_like(a), 8) for a in fx["rec"]]
            d_skip = dev(fx["skip8"].reshape(-1))
            d_imp = dev(fx["imp"].reshape(-1))
            n, nu = len(fx["areas"]), len(fx["units"])
            # the oracle wrapper's sentinels: areas that run no stage leave their slots and units untouched
            d_best, d_unit = dev(np.full(16 * n, 127, np.int8)), dev(np.full(12 * nu, 0xEE, np.uint8))
            d_ucost, d_wr = dev(np.full(nu, np.nan)), dev(np.full(nu, 7, np.uint8))
            for reduced in (0, 1):
                fx["reduced"] = bool(reduced)
                got = {}

                def call():
                    got["stages"] = ctx.loop_decision_dev(
                        d_rec, d_src, d_work, 1, 1, W, H, bd, 1, fx["damping"], fx["cdef_bits"], fx["ystr"],
                        fx["uvstr"], d_skip, 1, fx["unit_size"], reduced, d_imp, fx["dist_scale"], fx["lam"],
                        fx["areas"], fx["units"], fx["sb_unit"], d_best, d_unit, d_ucost, d_wr)
                ms = timed(call)
                want = run(fx)
                same = bool(got["stages"] == want[0] and (d_best.cpu().numpy().view(np.int8) == want[1][:16 * n]).all() and
                            (d_unit.cpu().numpy().view(np.uint8) == want[2].view(np.uint8)).all() and
                            (d_ucost.cpu().numpy().view(np.uint64) == want[3].view(np.uint64)).all() and
                            (d_wr.cpu().numpy() == want[4]).all())
                assert same, f"loop_decision {uy} reduced={reduced} {bd}-bit disagrees with the oracle"
                cpu = cpu_rate(lambda: run(fx), 1)
                extra = {"bit_depth": bd, "unit_size": list(fx["unit_size"]), "sets": "reduced" if reduced else "full",
                         "areas": n, "units": nu, "stages": got["stages"], "same_as_oracle": same,
                         "library": os.path.basename(B.LIB_PATH)}
                emit(f"loop_decision_dev units {uy}/{uy >> 1} {'reduced' if reduced else 'full'} sets {bd}-bit 4:2:0",
                     1, "frames", ms, 0, "1080p seeded, every area in one call, per-stage status reads included",
                     cpu=cpu, extra=extra, cpu_threads=1)  # orc_loop_decision runs on one thread
            for p in d_rec + d_src + d_work:
                ctx.plane_free(p)


def segmentation(ctx):
    """b200_segmentation_optimize_dev on a 1080p score map (240 x 135 importance blocks, lognormal scores) at 8 and
    10 bit, and b200_select_segment_dev over every block of the 1080p frame at 8x8 and at 64x64 with each level.
    Algorithmic bytes: the score map once (optimize); per block its distortion and activity entries, the item
    and the outputs (select).  Next to each, the oracle on one host thread on the same inputs, and a check of
    every output against it.  A call is tens of microseconds, so each line times 500 back-to-back calls."""
    from tests.test_oracle_segmentation import AC_Q, oracle_optimize, oracle_select, scale_maps, score_maps
    from tests.test_segmentation_gpu import frame_items
    W, H = 1920, 1080
    w, h = (W + 7) // 8, (H + 7) // 8
    name, scores, mw, mh = score_maps()[0]
    assert (mw, mh) == (w, h), name
    d_sc, d_rec = dev(scores), dev(np.zeros(240, np.uint8))
    lib = os.path.basename(B.LIB_PATH)
    for bd in (8, 10):
        ms = timed(lambda: ctx.segmentation_optimize_dev(d_sc, w, h, 120, bd, AC_Q[bd], 1, None, d_rec), reps=500)
        want = oracle_optimize(scores, w, h, 120, bd, 1, None)
        same = d_rec.cpu().numpy().tobytes() == want.tobytes()
        assert same, f"segmentation_optimize {bd}-bit disagrees with the oracle"
        cpu = cpu_rate(lambda: oracle_optimize(scores, w, h, 120, bd, 1, None), 1)
        emit(f"segmentation_optimize_dev 1080p map {bd}-bit", 1, "frames", ms, 4 * w * h,
             "240x135 lognormal scores, base_q_idx 120; launch_ms includes the histogram clear", cpu=cpu,
             extra={"bit_depth": bd, "segments": int(want["max_segment"][0]) + 1, "same_as_oracle": same,
                    "library": lib}, cpu_threads=1)
    d, a = scale_maps(w, h, seed=13)
    d_d, d_a = dev(d), dev(a)
    rec = d_rec.cpu().numpy().view(B.SEGMENTATION_DTYPE)  # the 10-bit record
    for bs, label, imp in ((3, "8x8", 1), (12, "64x64", 64)):  # imp: importance blocks per block
        items = frame_items(W, H, bs)
        n = len(items)
        d_it, d_sidx, d_scale = dev(items), dev(np.zeros(2 * n, np.uint8)), dev(np.zeros(n, np.uint32))
        for level, lname in ((1, "simple"), (2, "complex"), (3, "full")):
            ms = timed(lambda: ctx.select_segment_dev(d_it, n, d_d, d_a, w, h, 0, level, d_rec, d_sidx, d_scale),
                       reps=500)
            want, want_scale = oracle_select(items, d, a, w, h, 0, level, rec)
            same = bool((d_sidx.cpu().numpy().reshape(-1, 2) == want).all() and
                        (d_scale.cpu().numpy().view(np.uint32) == want_scale).all())
            assert same, f"select_segment {label} {lname} disagrees with the oracle"
            cpu = cpu_rate(lambda: oracle_select(items, d, a, w, h, 0, level, rec), n)
            emit(f"select_segment_dev 1080p {label} blocks {lname}", n, "blocks", ms, 8 * imp + 8 + 2 + 4,
                 "every block of the frame, 1/7 skipped; bytes: distortion + activity entries, item, outputs",
                 cpu=cpu, extra={"items": n, "same_as_oracle": same, "library": lib}, cpu_threads=1)


def coeff_rate(ctx):
    """b200_coeff_rate_dev on two batches, each checked against the oracle, next to the oracle's own rate on all
    usable host threads:
    - tx-type decision: every 16x16 block of a seeded 1080p frame quantized by b200_encode_tx_blocks_dev (intra,
      zero-motion prediction, dc/ac quantizer 140/160) for all 16 types; one chain per (block, type of
      TX_SET_INTRA_2), the 5 types rdo_tx_type_decision evaluates there, from the default CDFs;
    - mixed: 4x4 .. 32x32 luma chains of one to four tx blocks plus 4:2:0 chroma chains, seeded coefficients.
    Symbols: every symbol and bypass bit the chains code (the oracle encoder's count).  Algorithmic bytes per chain:
    its items, its coded blocks and its output word - what the kernel must read at least.  Downloading the
    eob-long coefficient runs for the host to count instead moves 2 (i16) bytes per coded position plus the eob:
    given per line as arithmetic; that alternative's time is not measured."""
    from tests import coeff_rate_cases as K
    lib = os.path.basename(B.LIB_PATH)
    T = K.tx_decision_batch(ctx, 1920, 1080, 8, seed=1)
    rng = np.random.default_rng(2)
    b = K.Batch(np.concatenate([K.default_cdfs(), K.random_cdfs(rng, 1)]), 0)
    for _ in range(6000):
        t = int(rng.choice([0, 1, 2, 3, 5, 6, 7, 8, 9, 10, 13, 14, 15, 16]))
        plane = int(rng.choice([0, 0, 1, 2]))
        w4, h4 = 1 << (K.TX_WL[t] - 2), 1 << (K.TX_HL[t] - 2)
        items = []
        for k in range(int(rng.integers(1, 5))):
            tt = int(rng.choice(K.INV_SET[K.tx_set(t, 0, 0)])) if plane == 0 else 0
            eob = int(rng.choice(K.eob_choices(rng, t)[:3]))
            items.append(K.item(b.add_block(K.make_block(rng, t, tt, eob, 0, zero_frac=0.7)), eob, t, tt, plane=plane,
                                bsize=K.bsize_of(64, 64), x4=(k * w4) % (16 - w4 + 1), y4=0))
        b.add_chain(items, snapshot=int(rng.integers(0, 5)))
    batches = [("tx-type decision 1080p 16x16 x 5 intra types", T["cdfs"], T["chains"], T["items"], T["q"]),
               ("mixed 4x4..32x32 luma + 4:2:0 chroma chains", *b.arrays())]
    for label, cdfs, chains, items, q in batches:
        d = [dev(a) for a in (cdfs, chains, items, q)]
        d_rate = dev(np.zeros(len(chains), np.uint32))
        d_cul = dev(np.zeros(len(items), np.uint8))
        call = lambda: ctx.coeff_rate_dev(d[0], len(cdfs), d[1], len(chains), d[2], len(items), d[3], len(q),  # noqa
                                          int(q.dtype == np.int32), d_rate, d_cul)
        ms = timed(call, reps=20)
        want, want_cul = K.oracle_rate(cdfs, chains, items, q)
        same = bool((d_rate.cpu().numpy().view(np.uint32) == want).all() and (d_cul.cpu().numpy() == want_cul).all())
        assert same, f"coeff_rate {label} disagrees with the oracle"
        nsym = sum(K.oracle_encode(cdfs, ch, items, q)[2] for ch in chains[:2000]) * len(chains) / min(2000, len(chains))
        areas = np.array([K.coded(int(t))[0] * K.coded(int(t))[1] for t in items["tx_size"]])
        read = (16 * len(items) + q.itemsize * int(areas.sum()) + 112 * len(chains) + 4 * len(chains)) / len(chains)
        download = (q.itemsize * int(items["eob"].astype(np.int64).sum()) + 2 * len(items)) / len(chains)
        cpu = cpu_rate(lambda: K.oracle_rate(cdfs, chains, items, q), len(chains))
        emit(f"coeff_rate_dev {label}", len(chains), "chains", ms, read,
             "symbols_per_s from the oracle encoder's symbol count (sampled over the first 2000 chains)", cpu=cpu,
             extra={"items": len(items), "symbols_per_s": nsym / (ms * 1e-3), "same_as_oracle": same,
                    "host_count_download_bytes_per_chain": download,
                    "host_count_download_time": "not measured", "library": lib})


def tx_size_type(ctx):
    """b200_intra_tx_size_type_dev on three 1080p 8-bit luma workloads, each checked against the oracle, next to
    the oracle (oracle/tx_size_type.c) on all usable host threads:
    - every 16x16 block x 3 screened modes (DC, V, PAETH), Psychovisual (cdef_dist) distortion;
    - the same items with tx-domain distortion;
    - a mixed-size partition: each 32x32 cell split into one of 32x32, 32x16, 16x32, 16x16, 16x8, 8x16, 8x8,
      one random mode per block.
    Items carry dc/ac quantizers 120/140 and the default CDFs.  Algorithmic bytes per item: the item, its best
    record, its 21 candidate records, and the block's src and rec pixels once - what the kernels must touch at
    least."""
    from tests import coeff_rate_cases as K
    from tests import tx_size_type_cases as T
    lib = os.path.basename(B.LIB_PATH)
    w, h, pad = 1920, 1080, 64
    src, rec = T.make_case(w, h, 8, 11)
    dsrc, drec = ctx.plane_from_host(src, pad), ctx.plane_from_host(rec, pad)
    cdfs = K.default_cdfs()
    lam = 0.0013 * 140 * 140
    rng = np.random.default_rng(12)
    splits = [(32, 32), (32, 16), (16, 32), (16, 16), (16, 8), (8, 16), (8, 8)]
    mixed = []
    for y in range(0, h, 32):
        for x in range(0, w, 32):
            bw, bh = splits[int(rng.integers(0, len(splits)))]
            for yy in range(y, min(y + 32, h), bh):
                for xx in range(x, x + 32, bw):
                    mixed.append(T.grid_items(bw, bh, bw, bh, [int(rng.integers(0, 13))]))
                    mixed[-1]["x"], mixed[-1]["y"] = xx, yy
    mixed = np.concatenate(mixed)
    grid = T.grid_items(w, h, 16, 16, [0, 1, 12])
    loads = [("1080p 16x16 x 3 modes Psychovisual", grid, 2), ("1080p 16x16 x 3 modes tx-domain", grid, 0),
             ("1080p mixed partition 8x8..32x32 Psychovisual", mixed, 2)]
    for label, it, dm in loads:
        n = len(it)
        d_it, d_cdfs = dev(it), dev(cdfs)
        d_best = dev(np.zeros(n, B.TX_BEST_DTYPE))
        d_cands = dev(np.zeros((n, 21), B.TX_CAND_DTYPE))
        call = lambda: ctx.intra_tx_size_type_dev(drec, dsrc, (0, 0, w, h), w, h, 8, dm, 0, lam, 16384, None, 0,  # noqa
                                                  d_cdfs, 1, d_it, n, d_best, d_cands)
        ms = timed(call, reps=10)
        wb, wc = T.oracle(src, rec, pad, (0, 0, w, h), w, h, 8, dm, 0, lam, 16384, None, cdfs, it)
        gb = d_best.cpu().numpy().view(B.TX_BEST_DTYPE)
        gc = d_cands.cpu().numpy().view(B.TX_CAND_DTYPE).reshape(n, 21)
        same = bool((gb.view(np.uint8) == wb.view(np.uint8)).all() and (gc.view(np.uint8) == wc.view(np.uint8)).all())
        assert same, f"tx_size_type {label} disagrees with the oracle"
        px = np.array([T.BS_W[b] * T.BS_H[b] for b in it["bsize"]], np.float64)
        read = 52 + 16 + 21 * 24 + 2 * float(px.mean())
        cpu = cpu_rate(lambda: T.oracle(src, rec, pad, (0, 0, w, h), w, h, 8, dm, 0, lam, 16384, None, cdfs, it), n)
        evaluated = int((gc["state"] == B.TX_EVALUATED).sum())
        emit(f"intra_tx_size_type_dev {label}", n, "items", ms, read, "items = (block, mode); bytes: item, records, "
             "src + rec pixels of the block", cpu=cpu,
             extra={"candidates_evaluated": evaluated, "same_as_oracle": same, "library": lib})


def host_gather(stats, prev, wib, hib, tile, x4, y4, w, h):
    """get_subset_predictors (me.rs:386-534, CORNER, ssdec 0) for a batch of blocks of one size and slot, vectorised:
    -> (CAND_DTYPE list grouped by block, CSR offsets), all_mvs order"""
    x4, y4 = x4.astype(np.int64), y4.astype(np.int64)
    x_min = np.maximum(-x4 * 32 - (128 + 8 * w), -(1 << 14) + 1)
    x_max = np.minimum((wib - x4 - w // 4) * 32 + 128 + 8 * w, (1 << 14) - 1)
    y_min = np.maximum(-y4 * 32 - (128 + 8 * h), -(1 << 14) + 1)
    y_max = np.minimum((hib - y4 - h // 4) * 32 + 128 + 8 * h, (1 << 14) - 1)
    tx, ty = x4 // tile * tile, y4 // tile * tile
    cols, rows = np.minimum(tile, wib - tx), np.minimum(tile, hib - ty)
    bx, by = x4 - tx, y4 - ty
    wb, hb = w // 4, h // 4
    chw, chh = np.minimum(wb >> 1, cols - 1 - bx), np.minimum(hb >> 1, rows - 1 - by)

    def proc(g, x, y):
        s = g[np.clip(y, 0, hib - 1), np.clip(x, 0, wib - 1)]
        q = lambda v: np.fix(v.astype(np.int64) / 8).astype(np.int64) * 8  # noqa: E731  (i16 `/ 8`, toward zero)
        return np.clip(q(s["mv_row"]), y_min, y_max), np.clip(q(s["mv_col"]), x_min, x_max)
    one = np.ones(len(x4), bool)
    cols_ = [(proc(stats, tx + bx + chw, ty + by + chh), one),
             (proc(stats, tx + bx - 1, ty + by + chh), bx > 0),
             (proc(stats, tx + bx + chw, ty + by - 1), by > 0),
             (proc(stats, tx + bx + wb, ty + by + chh), bx + wb < cols),
             (proc(stats, tx + bx + chw, ty + by + hb), by + hb < rows),
             ((0 * x4, 0 * x4), one)]
    if prev is not None:
        hw, hh = np.minimum(wb >> 1, wib - 1 - x4), np.minimum(hb >> 1, hib - 1 - y4)
        cols_ += [(proc(prev, x4 - 1, y4 + hh), x4 > 0), (proc(prev, x4 + hw, y4 - 1), y4 > 0),
                  (proc(prev, x4 + wb, y4 + hh), x4 + wb < wib), (proc(prev, x4 + hw, y4 + hb), y4 + hb < hib),
                  (proc(prev, x4 + hw, y4 + hh), one)]
    rows_m = np.stack([c[0][0] for c in cols_], 1)
    cols_m = np.stack([c[0][1] for c in cols_], 1)
    keep = np.stack([c[1] for c in cols_], 1)
    offs = np.zeros(len(x4) + 1, np.uint32)
    offs[1:] = np.cumsum(keep.sum(1))
    preds = np.zeros(int(offs[-1]), B.CAND_DTYPE)
    preds["mv_row"], preds["mv_col"] = rows_m[keep], cols_m[keep]
    preds["block"] = np.nonzero(keep)[0]
    return preds, offs


def encode_me(ctx):
    """b200_estimate_motion_dev on a 1080p 8-bit frame x 3 reference slots: every 8x8, 16x16 and 32x32 block, and a
    mixed partition (each 32x32 cell split into one of 32x32 .. 8x8), with use_satd_subpel, 1/8 pel and the stats grids
    of b200_lookahead_motion_dev (LAST's grids as subset C).  Next to it, the same results through the composed
    host-orchestrated chain (grids downloaded, predictors gathered on the host, b200_me_search_multi_dev,
    b200_me_candidates_multi_dev with SATD, b200_subpel_search_dev per slot), compared in the same run, and the oracle
    (oracle/encode_me.c) on 8 threads."""
    import time
    from tests.test_lookahead_me_gpu import dev_pyramid
    from tests.test_oracle_encode_me import ITEM_DTYPE, TX_SIZES, Enc, grid_dims
    lib = os.path.basename(B.LIB_PATH)
    W, H, PAD, NS = 1920, 1080, 96, 3
    e = Enc(W, H, bd=8, nslots=NS, tiles=(64, 64), prev=False, seed=31, pad=PAD, use_satd=1, allow_hp=1,
            me_lambda=3.0)
    wib, hib = grid_dims(W, H)
    dcur, dold = dev_pyramid(e.src_img), dev_pyramid(np.ascontiguousarray(np.roll(e.src_img, 3, 1)))
    drefs = [dev_pyramid(r) for r in e.ref_imgs]
    d_stats, d_prev = dev(np.zeros(NS * wib * hib * 8, np.uint8)), dev(np.zeros(NS * wib * hib * 8, np.uint8))
    lp = B.LookaheadMeParams(8, 0, e.me_lambda, 0, 1, 64, 64)
    ctx.lookahead_motion_dev([dold] * NS, drefs, lp, d_prev)
    ctx.lookahead_motion_dev([dcur] * NS, drefs, lp, d_stats)
    torch.cuda.synchronize()
    e.stats = d_stats.cpu().numpy().view(ME_STATS).reshape(NS, hib, wib)
    e.prev = d_prev.cpu().numpy().view(ME_STATS).reshape(NS, hib, wib)
    e.has_prev = [1] * NS
    src = ctx.plane_from_host(e.src_img, PAD)
    refs = [ctx.plane_from_host(r, PAD) for r in e.ref_imgs]
    pairs = B.PlanePairs([src] * NS, refs, [0] * NS, [0] * NS)
    rng = np.random.default_rng(5)

    def grid_of(s):
        bw, bh = TX_SIZES[s]
        xs, ys = np.meshgrid(np.arange(0, W // 4 - bw // 4 + 1, bw // 4), np.arange(0, H // 4 - bh // 4 + 1, bh // 4))
        return xs.ravel(), ys.ravel()
    splits = [3, 10, 9, 2, 8, 7, 1]   # 32x32, 32x16, 16x32, 16x16, 16x8, 8x16, 8x8 (TxSize)
    mixed = {s: ([], []) for s in splits}
    for y in range(0, H - 31, 32):
        for x in range(0, W - 31, 32):
            s = splits[int(rng.integers(0, len(splits)))]
            bw, bh = TX_SIZES[s]
            for yy in range(y, y + 32, bh):
                for xx in range(x, x + 32, bw):
                    mixed[s][0].append(xx // 4)
                    mixed[s][1].append(yy // 4)
    loads = [(f"{TX_SIZES[s][0]}x{TX_SIZES[s][1]}", {s: grid_of(s)}) for s in (1, 2, 3)]
    loads.append(("mixed 32x32 .. 8x8 partition", {s: (np.array(v[0]), np.array(v[1])) for s, v in mixed.items()}))
    p_enc = B.EncMeParams(8, 1, e.me_lambda, 1, 0, 64, 64)
    lam = e.lam()
    for label, groups in loads:
        parts, size_end = [], np.zeros(19, np.uint32)
        for s in range(19):
            if s in groups:
                xs, ys = groups[s]
                it = np.zeros(NS * len(xs), ITEM_DTYPE)
                it["x4"], it["y4"] = np.tile(xs, NS), np.tile(ys, NS)
                it["slot"] = np.repeat(np.arange(NS), len(xs))
                it["pmv"] = rng.integers(-4, 5, (len(it), 2, 2)) * 8
                parts.append(it)
            size_end[s] = sum(len(p) for p in parts)
        items = np.ascontiguousarray(np.concatenate(parts))
        n = len(items)
        d_items, d_out = dev(items), torch.empty(16 * n, dtype=torch.uint8, device="cuda")
        l0 = ctx.launches
        ctx.estimate_motion_dev(src, refs, d_stats, p_enc, size_end, d_items, n, d_out, d_prev, e.has_prev)
        nlaunch = ctx.launches - l0
        ms = timed(lambda: ctx.estimate_motion_dev(src, refs, d_stats, p_enc, size_end, d_items, n, d_out, d_prev,
                                                   e.has_prev), reps=10)
        got = d_out.cpu().numpy().view(B.ME_RESULT_DTYPE).copy()

        def composed():
            st = d_stats.cpu().numpy().view(ME_STATS).reshape(NS, hib, wib)
            pv = d_prev.cpu().numpy().view(ME_STATS).reshape(NS, hib, wib)
            out = np.zeros(n, B.ME_RESULT_DTYPE)
            lo = 0
            for s in range(19):
                hi = int(size_end[s])
                if hi == lo:
                    continue
                w, h = TX_SIZES[s]
                it = items[lo:hi]
                m = hi - lo
                lists, ends = [], []
                for k in range(NS):
                    sel = it["slot"] == k
                    pr, of = host_gather(st[k], pv[k], wib, hib, 16 * 64, it["x4"][sel], it["y4"][sel], w, h)
                    lists.append((pr, of))
                    ends.append(int(sel.sum()))
                base = np.concatenate([[0], np.cumsum(ends)])
                preds = np.concatenate([pr for pr, _ in lists])
                coff = np.concatenate([[0], np.cumsum([len(pr) for pr, _ in lists])])
                offs = np.concatenate([[0]] + [of[1:] + coff[k] for k, (_, of) in enumerate(lists)]).astype(np.uint32)
                blocks = np.zeros(m, B.BLOCK_DTYPE)
                blocks["x"], blocks["y"] = it["x4"] * 4, it["y4"] * 4
                pmv = np.ascontiguousarray(it["pmv"].astype(np.int16))
                d_b, d_pm = dev(blocks), dev(pmv)
                pp = B.PlanePairs([src] * NS, refs, base[1:], base[1:])
                p_sad = B.me_params(w, h, W, H, lam, allow_hp=True)
                p_satd = B.me_params(w, h, W, H, lam, allow_hp=True, use_satd=True)
                d_best = torch.empty(16 * m, dtype=torch.uint8, device="cuda")
                ctx.me_search_multi_dev(pp, d_b, m, dev(preds), dev(offs), 1, p_sad, d_best, d_pm)
                full = d_best.cpu().numpy().view(B.ME_RESULT_DTYPE).copy()
                c = np.zeros(m, B.CAND_DTYPE)
                c["block"] = np.arange(m)
                c["mv_row"], c["mv_col"] = full["mv_row"], full["mv_col"]
                d_sad, d_cost = torch.empty(4 * m, dtype=torch.uint8, device="cuda"), torch.empty(8 * m, dtype=torch.uint8,
                                                                                                device="cuda")
                ctx.me_candidates_multi_dev(pp, d_b, m, dev(c), m, p_satd, None, d_pm, d_sad, d_cost)
                full["sad"] = d_sad.cpu().numpy().view(np.uint32)
                full["cost"] = d_cost.cpu().numpy().view(np.uint64)
                d_full, d_res = dev(full), torch.empty(16 * m, dtype=torch.uint8, device="cuda")
                for k in range(NS):
                    a, b = int(base[k]), int(base[k + 1])
                    ctx.subpel_search_dev(src, refs[k], d_b[4 * a:4 * b], b - a, d_full[16 * a:16 * b], p_satd,
                                          d_res[16 * a:16 * b], 0, d_pmv=d_pm[8 * a:8 * b])
                out[lo:hi] = d_res.cpu().numpy().view(B.ME_RESULT_DTYPE)
                lo = hi
            return out
        want = composed()
        same = bool(got.tobytes() == want.tobytes())
        assert same, f"encode ME {label}: the composed chain and b200_estimate_motion_dev disagree"
        reps, t0 = 0, time.perf_counter()
        while reps < 2 or time.perf_counter() - t0 < 1.0:
            composed()
            reps += 1
        host_ms = (time.perf_counter() - t0) * 1e3 / reps
        oracle = e.oracle(items, size_end, threads=8)
        same_oracle = bool(oracle.tobytes() == got.tobytes())
        assert same_oracle, f"encode ME {label}: the oracle and b200_estimate_motion_dev disagree"
        cpu = cpu_rate(lambda: e.oracle(items, size_end, threads=8), n)
        moved = int((((got["mv_row"] | got["mv_col"]) & 7) != 0).sum())
        emit(f"estimate_motion_dev 1080p 8-bit x {NS} slots, {label}", n, "items", ms, 0,
             "items = (block, slot); one call, one launch per size group; data-dependent work per item (no byte figure)",
             cpu=cpu, cpu_threads=8,
             extra={"launches": nlaunch, "composed_chain_ms": host_ms, "composed_over_call": host_ms / ms,
                    "composed_chain": "grids to host, numpy gather, me_search_multi + me_candidates_multi (SATD) + "
                                      "subpel_search per slot, per size group; host clock",
                    "same_as_composed_chain": same, "same_as_oracle": same_oracle, "subpel_vectors": moved,
                    "library": lib})
    for pyr in [dcur, dold] + drefs:
        for q in pyr:
            ctx.plane_free(q)
    for q in [src] + refs:
        ctx.plane_free(q)


ME_STATS = np.dtype([("mv_row", "<i2"), ("mv_col", "<i2"), ("normalized_sad", "<u4")])


def main():
    torch.cuda.set_device(0)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    ctx = B.Context(0, use_torch_stream=True)
    print(json.dumps(card()))
    if "--subpel-sizes" in sys.argv[1:]:
        subpel_sizes(ctx)
        return
    if "--intra-screen" in sys.argv[1:]:
        intra_screen(ctx)
        return
    if "--inter-screen" in sys.argv[1:]:
        inter_screen(ctx)
        return
    if "--cdef-rdo" in sys.argv[1:]:
        cdef_rdo(ctx)
        return
    if "--cfl-alpha" in sys.argv[1:]:
        cfl_alpha(ctx)
        return
    if "--deblock" in sys.argv[1:]:
        deblock(ctx)
        return
    if "--lrf" in sys.argv[1:]:
        lrf(ctx)
        return
    if "--lrf-search" in sys.argv[1:]:
        lrf_search(ctx)
        return
    if "--loop-decision" in sys.argv[1:]:
        loop_decision(ctx)
        return
    if "--segmentation" in sys.argv[1:]:
        segmentation(ctx)
        return
    if "--coeff-rate" in sys.argv[1:]:
        coeff_rate(ctx)
        return
    if "--tx-size-type" in sys.argv[1:]:
        tx_size_type(ctx)
        return
    if "--encode-me" in sys.argv[1:]:
        encode_me(ctx)
        return
    rng = np.random.default_rng(0)
    W, H, PAD = 1920, 1080, 96

    # ---- config 3: forward-transform sweep over a 1080p residual frame, all 160 pairs, 8 bit
    resid = torch.from_numpy(rng.integers(-255, 256, (H * W,)).astype(np.int16)).cuda()
    out = torch.empty(H * W, dtype=torch.int32, device="cuda")
    sweep_ms = 0.0
    for ts, (w, h) in enumerate(TX_SIZES):
        n = (W // w) * (H // h)
        for tt in range(17):
            if not ctx.L.b200_valid_av1_transform(ts, tt):
                continue
            ms = timed(lambda: ctx.fwd_txfm_dev(resid, w * h, w, out, n, ts, tt, 8, False), reps=10)
            sweep_ms += ms
            if tt == 0:
                cpu = None
                if (w, h) in ((16, 16), (4, 4), (64, 64)):
                    hres = resid.cpu().numpy()[:n * w * h].reshape(n, h, w)
                    cpu = cpu_rate(lambda: O.forward_transform_batch(hres, ts, 0, 8, threads=O.host_threads()), n)
                emit(f"fwd_txfm {w}x{h} DCT_DCT 8-bit", n, "blocks", ms, w * h * 4,
                     "1080p residual frame tiled by this size; i16 in + i16 out", cpu)
    print(json.dumps({"kernel": "fwd_txfm sweep (160 size/type pairs x whole 1080p frame)",
                      "total_ms": sweep_ms, "pixels_per_s": 160 * W * H / (sweep_ms * 1e-3)}))

    # ---- planes
    oplanes = {}

    def mk(key, dtype, bd):
        img = rng.integers(0, 1 << bd, (H, W)).astype(dtype)
        op = O.Plane(W, H, PAD, dtype=dtype)
        op.fill_from(img)
        oplanes[key] = op
        return ctx.plane_from_host(img, PAD)
    cur8, ref8 = mk("cur8", np.uint8, 8), mk("ref8", np.uint8, 8)
    cur10, ref10 = mk("cur10", np.uint16, 10), mk("ref10", np.uint16, 10)
    TH = O.host_threads()
    blocks = grid_blocks(W, H, 16, 16)
    nb = len(blocks)
    d_blocks = dev(blocks)

    # ---- mc: put_8tap HV, 16x16, REGULAR, 8 sub-pel vectors per block (config 4 shape)
    pattern = np.array([(r * s, c * s) for s in (4, 2) for r, c in ((1, 0), (0, 1), (-1, 0), (0, -1))])
    centre = rng.integers(-16, 17, (nb, 2)) * 8 + 3
    mvs = (centre[:, None, :] + pattern[None]).reshape(-1, 2).astype(np.int16)
    mblocks = np.repeat(blocks, len(pattern))
    n = len(mblocks)
    d_mb, d_mv = dev(mblocks), dev(mvs)
    for name, ref, oref, bd, bpp in (("8-bit", ref8, "ref8", 8, 1), ("10-bit", ref10, "ref10", 10, 2)):
        d_pred = torch.empty(n * 256 * bpp, dtype=torch.uint8, device="cuda")
        ms = timed(lambda: ctx.mc_blocks_dev(ref, d_mb, d_mv, n, 16, 16, 0, 0, bd, 0, 0, 0, d_pred), reps=10)
        cpu = cpu_rate(lambda: O.mc_blocks(oplanes[oref], mblocks, mvs, 16, 16, 0, 0, bd, threads=TH), n)
        emit(f"put_8tap HV 16x16 {name}", n, "blocks", ms, (23 * 23 + 256) * bpp, cpu=cpu)

    # ---- config 4: sub-pel candidates (MC + SATD + cost + argmin), 10-bit, 8 per block
    cands = np.zeros(n, B.CAND_DTYPE)
    cands["block"] = np.repeat(np.arange(nb, dtype=np.uint32), len(pattern))
    cands["mv_row"], cands["mv_col"] = mvs[:, 0], mvs[:, 1]
    offs = (np.arange(nb + 1) * len(pattern)).astype(np.uint32)
    d_c, d_o = dev(cands), dev(offs)
    d_best = torch.empty(nb * 16, dtype=torch.uint8, device="cuda")
    for name, cur, ref, ocur, oref, bd, bpp in (("8-bit", cur8, ref8, "cur8", "ref8", 8, 1),
                                                ("10-bit", cur10, ref10, "cur10", "ref10", 10, 2)):
        p = B.me_params(16, 16, W, H, 6400, allow_hp=True, use_satd=True, bit_depth=bd)
        ms = timed(lambda: ctx.me_subpel_candidates_dev(cur, ref, d_blocks, nb, d_c, n, p, 0, d_o, None,
                                                        None, None, d_best), reps=10)
        cpu = cpu_rate(lambda: O.subpel_candidates(oplanes[ocur], oplanes[oref], blocks, cands, 16, 16, True,
                                                   6400, None, True, 0, bd, threads=TH), n)
        emit(f"subpel candidates (put_8tap + SATD + cost + argmin) 16x16 {name}", n, "candidates", ms,
             23 * 23 * bpp + 256 * bpp + 4, "two launches + argmin; prediction round-trips through HBM", cpu)
    # chain tail: winners' prediction -> residual -> 16x16 DCT (10-bit)
    d_pred = torch.empty(nb * 256 * 2, dtype=torch.uint8, device="cuda")
    d_coef = torch.empty(nb * 256, dtype=torch.int32, device="cuda")
    d_wmv = dev(mvs[::len(pattern)].copy())

    def chain():
        ctx.mc_blocks_dev(ref10, d_blocks, d_wmv, nb, 16, 16, 0, 0, 10, 0, 0, 0, d_pred)
        ctx.fwd_txfm_pred_dev(cur10, d_pred, d_blocks, nb, d_coef, 2, 0, 10)
    ms = timed(chain, reps=10)
    emit("winner put_8tap + residual + fwd_txfm 16x16 10-bit", nb, "blocks", ms, 2598,
         "SURVEY §8d fused MC->SATD->txfm figure (2598 B/block)")

    # ---- config 4, fused: sub-pel refinement + winner's residual + 16x16 DCT in ONE kernel
    # (b200_subpel_rdo_dev): no prediction touches HBM
    for name, cur, ref, bd, bpp in (("8-bit", cur8, ref8, 8, 1), ("10-bit", cur10, ref10, 10, 2)):
        p = B.me_params(16, 16, W, H, 6400, allow_hp=True, use_satd=True, bit_depth=bd)
        d_fc = torch.empty(nb * 256, dtype=torch.int16 if bd == 8 else torch.int32, device="cuda")
        ms = timed(lambda: ctx.subpel_rdo_dev(cur, ref, d_blocks, nb, d_c, n, d_o, p, 0, 2, 0, None, None, None,
                                              d_best, d_fc), reps=10)
        emit(f"FUSED subpel RDO (8 x [put_8tap + SATD + cost] + argmin + residual + DCT 16x16) {name}", nb, "blocks",
             ms, 8 * 23 * 23 * bpp + 256 * bpp + 256 * (2 if bd == 8 else 4) + 16,
             "BASELINE configs[3]; bytes: 8 source footprints + org block + coefficients + winner "
             "(SURVEY 8d quotes 2598 B per single-candidate block at 10 bit)")

    # ---- lookahead (api/lookahead.rs): pyramid, intra / inter cost maps, importance-block difference
    hres = ctx.plane_alloc(W // 2, H // 2, PAD // 2, 1)
    qres = ctx.plane_alloc(W // 4, H // 4, PAD // 4, 1)

    def pyramid():
        ctx.plane_downsample_dev(cur8, hres, W // 2, H // 2)
        ctx.plane_downsample_dev(hres, qres, W // 4, H // 4)
    ms = timed(pyramid, reps=10)
    emit("Plane::downsampled x2 (half + quarter resolution ME pyramid) 1080p 8-bit", W * H, "source pixels", ms,
         1 + 0.25 + 0.25 + 0.0625, "reads the level above, writes the padded level below")
    nimp = (W // 8) * (H // 8)
    d_ic = torch.empty(nimp, dtype=torch.int32, device="cuda")
    ms = timed(lambda: ctx.estimate_intra_costs_dev(cur8, 8, d_ic), reps=10)
    hic = np.zeros(nimp, np.uint32)
    OLk = O.lib()
    OLk.orc_estimate_intra_costs.restype = None
    OLk.orc_estimate_intra_costs.argtypes = [C.c_void_p, C.c_ssize_t] + [C.c_int] * 4 + [C.c_void_p]
    oc = oplanes["cur8"]
    cpu = cpu_rate(lambda: OLk.orc_estimate_intra_costs(oc.at(0, 0), oc.stride, W, H, 1, 8, hic.ctypes.data), nimp)
    emit("estimate_intra_costs (edges + DC + SATD 8x8, fused) 1080p 8-bit", nimp, "8x8 blocks", ms, 64 + 16 + 4, cpu=cpu)
    d_imv = dev((rng.integers(-32, 33, (nimp, 2)) * 4).astype(np.int16))
    d_scr, d_mean = torch.zeros(1, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.float64, device="cuda")
    ms = timed(lambda: ctx.estimate_inter_costs_dev(cur8, ref8, d_imv, d_ic, d_scr, d_mean), reps=10)
    emit("estimate_inter_costs cost part (SATD 8x8 vs displaced reference + f64 mean) 1080p 8-bit", nimp, "8x8 blocks",
         ms, 128 + 4 + 4)
    ms = timed(lambda: ctx.importance_block_difference_dev(cur8, ref8, d_scr, d_mean), reps=10)
    emit("estimate_importance_block_difference 1080p 8-bit", nimp, "8x8 blocks", ms, 128)

    # ---- temporal RDO (api/internal.rs:912-1230): speed 6's window (20 lookahead frames + the coded one)
    from tests.test_oracle_temporal_rdo import oracle_importances, oracle_intra_costs, window_1080p
    win = window_1080p()
    oracle_intra_costs(win)
    tplanes = [ctx.plane_from_host(im, win.pad) for im in win.imgs]
    d_ti, d_tm = dev(win.intra), dev(win.mvs)
    d_timp = torch.empty(len(win.imgs) * win.n_imp, dtype=torch.float32, device="cuda")

    def window():
        ctx.block_importances_dev(tplanes, 8, d_ti, d_tm, win.steps, d_timp)
    l0 = ctx.launches
    window()
    nlaunch = ctx.launches - l0
    ms = timed(window, reps=5)
    units = len(win.steps) * win.n_imp
    # per propagated source block: source + reference 8x8 blocks, its vector, intra cost and importance,
    # and one read-modify-write of a destination importance (n_imp destinations per step)
    bpu = 2 * 64 * 1 + 4 + 4 + 4 + 2 * 4
    cpu = cpu_rate(lambda: oracle_importances(win), units)
    emit("temporal RDO window 1080p 8-bit (block importances, 21 frames / 57 steps)", units, "propagated source blocks",
         ms, bpu, "launch_ms = one whole window; the oracle's CPU rate is ONE thread (the propagation is serial)", cpu,
         extra={"window_ms": ms, "launches_per_window": nlaunch,
                "launch_count_note": "ctx launch counter: pass A, the CUB radix sort (counted once), bucket bounds, "
                                     "one pass B per step"})
    for p in tplanes:
        ctx.plane_free(p)

    # ---- lookahead motion vectors (me.rs:153-337): one 1080p pair, one reference slot, three levels, one tile
    import time
    from tests.test_oracle_lookahead_me import Params, downsample, images, oracle_motion
    from tests.test_oracle_lookahead_me import pyramid as la_pyramid
    la_cur, la_ref = images(W, H, 8, True, 5)

    def la_dev(img):
        lv = [img, downsample(img)]
        lv.append(downsample(lv[1]))
        return [ctx.plane_from_host(im, 64) for im in lv]
    la_dc, la_dr = la_dev(la_cur), la_dev(la_ref)
    la_oc, la_or = la_pyramid(la_cur), la_pyramid(la_ref)
    d_st = torch.empty(8 * (W // 4) * (H // 4 + 2), dtype=torch.uint8, device="cuda")
    for label, fs in (("speed-6 settings: no full search", 0), ("with full search", 1)):
        lp = Params(bit_depth=8, me_lambda=16.0, full_search=fs)
        bp = B.LookaheadMeParams(8, 0, lp.me_lambda, fs, 1, 64, 64)
        l0 = ctx.launches
        ctx.lookahead_motion_dev([la_dc], [la_dr], bp, d_st)
        nlaunch = ctx.launches - l0
        ms = timed(lambda: ctx.lookahead_motion_dev([la_dc], [la_dr], bp, d_st), reps=5)
        t0 = time.perf_counter()
        oracle_motion(la_oc, la_or, W, H, lp)
        cpu_s = time.perf_counter() - t0
        emit(f"lookahead ME 1080p 8-bit, one ref, 3 levels ({label})", 1, "frames", ms, 2 * W * H * (1 + 0.25 + 0.0625),
             "launch_ms = one frame (refinement + one launch per anti-diagonal); smooth pattern shifted by (5, -3) px, "
             "me_lambda 16; the oracle's CPU rate is ONE thread (the serial reference order)", 1.0 / cpu_s,
             extra={"frame_ms": ms, "launches_per_frame": nlaunch, "oracle_ms_per_frame": cpu_s * 1e3})
    for p in la_dc + la_dr:
        ctx.plane_free(p)

    # ---- get_intra_edges for every 16x16 block of a frame x 13 modes, then the predictions from them
    eitems = np.zeros(nb * 13, B.EDGE_ITEM_DTYPE)
    eitems["po_x"], eitems["po_y"] = np.repeat(blocks["x"], 13), np.repeat(blocks["y"], 13)
    eitems["part_x"], eitems["part_y"] = eitems["po_x"] // 4, eitems["po_y"] // 4
    eitems["bsize"], eitems["tx_size"] = 6, 2                                  # BLOCK_16X16, TX_16X16
    eitems["mode"] = np.tile([0, 2, 1, 9, 11, 10, 12, 3, 4, 5, 6, 7, 8], nb)   # RAV1E_INTRA_MODES
    eitems["enable_ief"] = 1
    d_ei = dev(eitems)
    d_eb = torch.empty(len(eitems) * 257, dtype=torch.uint8, device="cuda")
    d_el = torch.empty(len(eitems) * 2, dtype=torch.uint8, device="cuda")
    ms = timed(lambda: ctx.get_intra_edges_dev(cur8, (0, 0, W, H), 0, 0, 8, d_ei, len(eitems), d_eb, d_el), reps=10)
    emit("get_intra_edges 16x16 x 13 modes 1080p 8-bit", len(eitems), "edge buffers", ms, 257 + 16 + 2,
         "item + up to 65 plane pixels in, 257-pixel buffer + lengths out")

    # ---- compute_rd_cost: 16 candidates per block, cost + first minimum
    nrd = nb * 16
    d_rate = dev(rng.integers(0, 1 << 16, nrd).astype(np.uint32))
    d_dist = dev(rng.integers(0, 1 << 30, nrd).astype(np.uint64))
    d_roffs = dev((np.arange(nb + 1) * 16).astype(np.uint32))
    d_rc = torch.empty(nrd, dtype=torch.float64, device="cuda")
    d_rb = torch.empty(nb, dtype=torch.int32, device="cuda")
    ms = timed(lambda: ctx.compute_rd_cost_dev(117.25, d_rate, d_dist, nrd, d_rc, d_roffs, nb, d_rb), reps=10)
    emit("compute_rd_cost (f64 fma) + first minimum per block, 16 candidates per block", nrd, "candidates", ms, 4 + 8 + 8)

    # ---- device-side search stages of full_pixel_me (me.rs:692-856), 1080p, 16x16 blocks.
    # Structured content (low-passed noise displaced by (+6, -3) px + noise) so the walks are real;
    # predictors scatter within +-8 px of the true motion like neighbouring blocks' vectors do.
    from scipy.ndimage import uniform_filter
    base = uniform_filter(rng.integers(0, 256, (H + 64, W + 64)).astype(np.float32), 9)
    base = (base - base.min()) / (base.max() - base.min()) * 255
    s_ref = np.rint(base[32:32 + H, 32:32 + W]).astype(np.uint8)
    s_cur = np.clip(np.rint(base[32 - 3:32 - 3 + H, 32 + 6:32 + 6 + W] + rng.normal(0, 1.5, (H, W))), 0, 255).astype(np.uint8)
    os_cur, os_ref = O.Plane(W, H, PAD), O.Plane(W, H, PAD)
    os_cur.fill_from(s_cur)
    os_ref.fill_from(s_ref)
    ds_cur, ds_ref = ctx.plane_from_host(s_cur, PAD), ctx.plane_from_host(s_ref, PAD)
    p_srch = B.me_params(16, 16, W, H, 1600)
    d_sbest = torch.empty(nb * 16, dtype=torch.uint8, device="cuda")
    for label, nsub, per, umh_range in (("predictors + diamond (non-extensive)", 1, (10,), 0),
                                        ("extensive ladder through UMH-24 + hexagon", 3, (1, 5, 4), 24)):
        counts = np.tile(np.array(per), nb)
        soffs = np.zeros(nb * nsub + 1, np.uint32)
        soffs[1:] = np.cumsum(counts)
        spreds = np.zeros(int(soffs[-1]), B.CAND_DTYPE)
        smv = (np.array([-3, 6]) + rng.integers(-8, 9, (len(spreds), 2))) * 8
        spreds["mv_row"], spreds["mv_col"] = smv[:, 0], smv[:, 1]
        sthresh = np.zeros(nb, np.uint32)                     # never exit early: every stage runs
        d_sp, d_so, d_st = dev(spreds), dev(soffs), dev(sthresh)
        ms = timed(lambda: ctx.me_search_dev(ds_cur, ds_ref, d_blocks, nb, d_sp, d_so, nsub, p_srch, d_sbest,
                                             None, d_st if nsub == 3 else None, umh_range), reps=10)
        cpu = cpu_rate(lambda: O.full_pixel_me_blocks(os_cur, os_ref, blocks, spreds, soffs, nsub, 16, 16, 1600,
                                                      None, sthresh if nsub == 3 else None, umh_range, threads=TH), nb)
        emit(f"me_search 16x16 8-bit: {label}", nb, "blocks", ms, 0,
             "data-dependent number of SAD evaluations per block (no SURVEY byte figure); one warp per block", cpu)

    # ---- intra: 13 modes per 16x16 block
    edges = rng.integers(0, 256, (nb, 257)).astype(np.uint8)
    modes = [(0, 3, 0), (2, 3, 180), (1, 3, 90), (9, 3, 0), (11, 3, 0), (10, 3, 0), (12, 3, 0), (3, 3, 45),
             (4, 3, 135), (5, 3, 113), (6, 3, 157), (7, 3, 203), (8, 3, 67)]        # RAV1E_INTRA_MODES
    items = np.zeros(nb * len(modes), B.INTRA_ITEM_DTYPE)
    items["edge"] = np.repeat(np.arange(nb, dtype=np.uint32), len(modes))
    items["mode"] = np.tile([m[0] for m in modes], nb)
    items["variant"] = 3
    items["angle"] = np.tile([m[2] for m in modes], nb)
    items["ief"] = 0
    items["left_len"] = items["above_len"] = 32
    items["x"] = np.repeat(blocks["x"], len(modes))
    items["y"] = np.repeat(blocks["y"], len(modes))
    d_e, d_i = dev(edges), dev(items)
    d_p = torch.empty(len(items) * 256, dtype=torch.uint8, device="cuda")
    ms = timed(lambda: ctx.predict_intra_dev(d_e, d_i, len(items), None, 16, 16, 8, W, H, d_p), reps=10)
    hout = np.zeros((len(items), 256), np.uint8)
    OL = O.lib()
    OL.orc_predict_intra_batch.restype = None
    OL.orc_predict_intra_batch.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p] + [C.c_int] * 5 + [C.c_void_p]
    cpu = cpu_rate(lambda: OL.orc_predict_intra_batch(edges.ctypes.data, 1, items.ctypes.data, len(items), None,
                                                      16, 16, 8, W, H, hout.ctypes.data), len(items))
    emit("predict_intra 16x16 x 13 modes 8-bit", len(items), "predictions", ms, 257 + 256, cpu=cpu)

    # ---- quantize -> dequantize -> tx-domain distortion on the 16x16 DCT coefficients of a frame
    d_coef16 = torch.empty(nb * 256, dtype=torch.int16, device="cuda")
    ctx.fwd_txfm_residual_dev(cur8, ref8, d_blocks, nb, None, d_coef16, 2, 0, 8)
    d_q16 = torch.empty(nb * 256, dtype=torch.int16, device="cuda")
    d_r16 = torch.empty(nb * 256, dtype=torch.int16, device="cuda")
    d_eob = torch.empty(nb, dtype=torch.int16, device="cuda")
    d_txd = torch.empty(nb, dtype=torch.int64, device="cuda")
    ms = timed(lambda: ctx.quantize_dev(d_coef16, nb, 2, 0, 120, 96, False, False, d_q16, d_r16, d_eob, d_txd), reps=10)
    hcoef = d_coef16.cpu().numpy().reshape(nb, 256)
    hq, hr = np.zeros_like(hcoef), np.zeros_like(hcoef)
    he, hd = np.zeros(nb, np.uint16), np.zeros(nb, np.uint64)
    OLq = O.lib()
    OLq.orc_quantize_chain_batch.restype = None
    OLq.orc_quantize_chain_batch.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_uint32, C.c_uint32,
                                             C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    cpu = cpu_rate(lambda: OLq.orc_quantize_chain_batch(hcoef.ctypes.data, nb, 2, 0, 120, 96, 0, 0, hq.ctypes.data,
                                                        hr.ctypes.data, he.ctypes.data, hd.ctypes.data, TH), nb)
    emit("quantize + dequantize + tx-dist 16x16 8-bit (noise residual: long scans)", nb, "blocks", ms,
         3 * 512 + 10, "coefficients in, qcoeffs + rcoeffs + eob + distortion out", cpu)

    # ---- inverse transform + reconstruct, and encode_tx_block's numeric core in one call
    rec = ctx.plane_from_host(np.zeros((H, W), np.uint8) + 128, 0)
    ms = timed(lambda: ctx.inverse_transform_add_dev(d_r16, rec, d_blocks, nb, 2, 0, 8), reps=10)
    emit("inverse_transform_add 16x16 DCT_DCT 8-bit", nb, "blocks", ms, 512 + 2 * 256, "rcoeffs in, plane read-modify-write")
    d_co2 = torch.empty(nb * 256, dtype=torch.int16, device="cuda")
    ms = timed(lambda: ctx.encode_tx_blocks_dev(cur8, ref8, rec, d_blocks, nb, None, 2, 0, 8, 120, 96, False, True,
                                                d_co2, d_q16, d_r16, d_eob, d_txd), reps=10)
    emit("encode_tx_blocks (diff + fwd txfm + quantize + dequantize + tx-dist + inverse add) 16x16 8-bit", nb, "blocks",
         ms, 2 * 256 + 3 * 512 + 10 + 2 * 256, "")

    # ---- RDO distortion kernels on the 1080p 8-bit planes: every 16x16 block / every 8x8 block
    d_scale = dev(rng.integers(1 << 12, 1 << 16, ((H + 3) // 4, W // 4)).astype(np.uint32))
    d_wsse = torch.empty(nb * 8, dtype=torch.uint8, device="cuda")
    ms = timed(lambda: ctx.weighted_sse_dev(cur8, ref8, d_blocks, nb, 16, 16, d_scale, W // 4, d_wsse), reps=10)
    emit("get_weighted_sse 16x16 8-bit", nb, "blocks", ms, 2 * 256 + 16 * 4 + 8,
         "two 16x16 blocks + 16 chunk scales in, one u64 out")
    b8 = grid_blocks(W, H, 8, 8)
    d_b8 = dev(b8)
    d_cd = torch.empty(len(b8) * 4, dtype=torch.uint8, device="cuda")
    ms = timed(lambda: ctx.cdef_dist_dev(cur8, ref8, d_b8, len(b8), 8, 8, 8, d_cd, None), reps=10)
    emit("cdef_dist_kernel 8x8 8-bit (+ ssim boost)", len(b8), "8x8 blocks", ms, 2 * 64 + 4)

    # ---- config 5: CDEF on a 4K frame (luma + one 4:2:0 chroma plane)
    W4, H4 = 3840, 2160
    luma = rng.integers(0, 256, (H4, W4)).astype(np.uint8)
    chroma = rng.integers(0, 256, (H4 // 2, W4 // 2)).astype(np.uint8)
    pl, plo = ctx.plane_from_host(luma, 0), ctx.plane_from_host(np.zeros_like(luma), 0)
    pc, pco = ctx.plane_from_host(chroma, 0), ctx.plane_from_host(np.zeros_like(chroma), 0)
    n8 = (W4 // 8) * (H4 // 8)
    d_dir = torch.empty(n8, dtype=torch.uint8, device="cuda")
    d_var = torch.empty(n8, dtype=torch.int32, device="cuda")
    d_str = dev(np.full(((H4 + 63) // 64) * ((W4 + 63) // 64), 4 * 7 + 2, np.uint8))
    ms = timed(lambda: ctx.cdef_find_dir_dev(pl, 8, None, d_dir, d_var), reps=10)
    cpu = cpu_rate(lambda: O.cdef_analyze_frame(luma, 8), n8)
    emit("cdef_find_dir 4K luma", n8, "8x8 blocks", ms, 64 + 8, cpu=cpu)
    hdirs, hvar = O.cdef_analyze_frame(luma, 8)
    hstr = np.full(((H4 + 63) // 64, (W4 + 63) // 64), 4 * 7 + 2, np.uint8)
    ms = timed(lambda: ctx.cdef_filter_plane_dev(pl, plo, 0, 0, 0, W4, H4, 8, 5, None, d_dir, d_var, d_str), reps=10)
    cpu = cpu_rate(lambda: O.cdef_filter_plane(luma, 0, 0, 0, W4, H4, 8, 5, None, hdirs, hvar, hstr), n8)
    emit("cdef_filter 4K luma", n8, "8x8 blocks", ms, 208, cpu=cpu)
    ms = timed(lambda: ctx.cdef_filter_plane_dev(pc, pco, 1, 1, 1, W4, H4, 8, 5, None, d_dir, d_var, d_str), reps=10)
    emit("cdef_filter 4K chroma 4:2:0", n8, "4x4 blocks", ms, 8 * 8 + 16)

    # ---- sub-pel diamond search at the sizes the fused kernel gained (also alone: --subpel-sizes)
    subpel_sizes(ctx)


if __name__ == "__main__":
    main()
