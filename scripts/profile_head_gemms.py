"""Per-kernel device time of the bench step (bench.py's flagship training step, run eagerly in situ under torch.profiler),
with the tensor-core work of the head's three GEMM kernels counted from the shapes they run at.

For k1a_shuffle_convt_kernel (layer 1), convt_rows_kernel (layer 2 + two-pass softmax) and wgrad_kernel (both layers) it
prints two counts of mma.sync m16n8k16 FLOPs and the rate each implies over the measured kernel time:
  all tiles  -- every tile of the kernels' 4-shift tiling (4 shifts x 10 n8 tiles for k1a, 4 x 6 per warp for the banded
                kernel, 4 x 5 m16 tiles for the weight gradient), zero-weight tiles included;
  non-zero   -- only the tiles whose weights hold one of the 9 real (class, shift) taps of 16 (head_prep.cuh NZ_N8 /
                NZ_M16; for the banded kernel, of the columns its epilogue reads).
Kernels that skip the zero tiles issue the non-zero count; kernels that do not, the all-tiles count.  The card's name, power limit and SM clocks are read in the same run.
For b3a_dgrad_kernel (layer-1 data gradient) it prints the FLOPs it issues and the useful ones (2 x 9 taps x c1 per d
feature), with the rate each implies.
It also prints the head backward's fixed-order gradient sums (every reduce_partials* launch) as one row: µs and launches per step.

    python scripts/profile_head_gemms.py [--clips 16] [--steps 10] [--warmup 3] [--json OUT]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

MMA_FLOP = 2 * 16 * 8 * 16  # one mma.sync m16n8k16
NCLS, CLS = 4, 20           # 4 output classes x 20 columns (class-major, head_bf16.cu)


def tap(cls: int, sh: int) -> bool:
    """(output class, input shift) pairs that carry a real 3x3 tap (head_prep.cuh)."""
    return not ((cls >> 1) == 0 and (sh >> 1) == 1) and not ((cls & 1) == 0 and (sh & 1) == 1)


def nz_tiles(sh: int, width: int, lo: int = 0, hi: int = NCLS * CLS) -> int:
    """tiles of `width` columns (rows) within [lo, hi) of the class-major 80 that hold a non-zero weight for shift sh"""
    return sum(any(tap(k // CLS, sh) for k in range(c, c + width)) for c in range(lo, hi, width))


def k1a_flops(frames: int, cin: int, h: int, w: int) -> tuple[float, float]:
    """k1a: per (frame, band) item, the band's m16 tiles x 10 n8 x 4 shifts x 2 k16 per 32-channel stage; the bands are as
    head_bf16.cu's make_k1a_geom cuts them (the fewest whose largest band fits 8 warps x 3 m16 tiles = 384 raster rows)"""
    p = 2 * w + 1
    g = next(g for g in range(1, h + 1) if 2 * -(-h // g) * p <= 384)
    m16 = sum(-(-2 * (h // g + (i < h % g)) * p // 16) for i in range(g))  # m16 tiles per frame
    per_stage = m16 * 2  # x k16
    nst = cin // 32
    all_t = frames * nst * per_stage * 4 * 10
    nonzero = frames * nst * per_stage * sum(nz_tiles(sh, 8) for sh in range(4))
    return all_t * MMA_FLOP, nonzero * MMA_FLOP


def rows_flops(frames: int, hi: int, wi: int, npass: int) -> tuple[float, float]:
    """banded kernel, K = 32 (one stage): per 128-row tile, warps (q, e) accumulate columns [32e, 32e + 48) and use
    [40e, 40e + 40)"""
    pp = wi + 1
    r = min(256 // pp, hi)
    tiles = sum((min(r, hi - y0) * pp + 127) // 128 for y0 in range(0, hi, r))
    per = frames * tiles * npass * 4 * 2 * 2  # q warps x m16 x k16
    all_t = per * 2 * 4 * 6
    nonzero = per * sum(nz_tiles(sh, 8, 40 * e, 40 * e + 40) for e in range(2) for sh in range(4))
    return all_t * MMA_FLOP, nonzero * MMA_FLOP


def wgrad_flops(frames: int, hi: int, wi: int, nkc: int) -> tuple[float, float]:
    """weight gradient: M = 80 (class, o) rows = 5 m16 tiles per shift, N = 8 channels per K-chunk, K = the raster in
    units of R image rows (R * (Wi + 1) rounded up to 16); the launch picks R as launch_wgrad does"""
    kcx = 8 if nkc % 8 == 0 else 4
    r = next(r for r in range(min(hi, 8), 0, -1)
             if hi % r == 0 and 2 * 10 * ((r * (wi + 1) + 15) & ~15) * 16 + 2 * kcx * ((((r * (wi + 1) + 15) & ~15) + wi + 2 + 7) & ~7) * 16 + 64 <= 225 * 1024)
    kr = (r * (wi + 1) + 15) & ~15
    per = frames * (hi // r) * (kr // 16) * (nkc // kcx) * 2 * (kcx // 2)  # units x k16 x groups x halves x n8 tiles
    all_t = per * 4 * 5
    nonzero = per * sum(nz_tiles(sh, 16) for sh in range(4))
    return all_t * MMA_FLOP, nonzero * MMA_FLOP


def b3a_flops(frames: int, c: int, h: int, w: int, c1: int) -> tuple[float, float]:
    """b3a: per (frame, 128-channel tile, (di, feature-row pair) item), 4 warps x W / 2 n8 tiles x 2 m16 tiles x the 14
    non-zero (shift, k16) steps; useful: 9 taps x c1 multiply-adds per d feature"""
    tiles = -(-c // 4 // 128)
    issued = frames * tiles * h * 4 * (w // 2) * 2 * 14
    return issued * MMA_FLOP, frames * c * h * w * 2 * 9 * c1


def gpu_info() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), [c.strip() for c in out.strip().split(",")]))
    except Exception as exc:  # noqa: BLE001
        return {"error": repr(exc)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=16)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the table as JSON to this path")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profile_head_gemms.py measures on the GPU"
    from torch.profiler import ProfilerActivity, profile

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    import lightning_pose_b200  # noqa: F401

    prob = bench.make_problem(args.clips, seed=1234, device=dev)
    hp = bench.HotPath(prob, dev, fwd_only=False)
    feats = prob["feats"].to(torch.bfloat16).to(dev)
    for _ in range(args.warmup):
        hp.step(feats)
    torch.cuda.synchronize()
    info = gpu_info()
    with bench.ClockSampler(0) as clk:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                hp.step(feats)
            torch.cuda.synchronize()
    clocks = clk.summary()
    per, calls = {}, {}
    for e in prof.key_averages():
        if e.device_time_total > 0:
            per[e.key] = per.get(e.key, 0.0) + e.device_time_total / args.steps
            calls[e.key] = calls.get(e.key, 0) + e.count / args.steps
    total = sum(per.values())
    # the head backward's fixed-order gradient sums (dW2, db2, db1, dW1 of each chain), all launches of reduce_partials*
    sums = [k for k in per if "reduce_partials" in k]
    fixed_sums = {"us_per_step": round(sum(per[k] for k in sums), 1), "launches_per_step": round(sum(calls[k] for k in sums), 2)}

    nf = args.clips * (bench.B_LABELED + bench.T_UNLABELED)
    c4, h = bench.FEAT_C // 4, bench.FEAT_HW
    gemms = {
        "k1a_shuffle_convt_kernel": k1a_flops(nf, c4, h, h),
        "convt_rows_kernel": rows_flops(nf, 4 * h, 4 * h, 2),
        "wgrad_kernel": tuple(a + b for a, b in zip(wgrad_flops(nf, 2 * h, 2 * h, c4 // 8), wgrad_flops(nf, 4 * h, 4 * h, 4))),
    }
    b3a_us = sum(v for k, v in per.items() if "b3a_dgrad_kernel" in k)
    issued, useful = b3a_flops(nf, bench.FEAT_C, h, h, bench.K_PTS)
    b3a = {"kernel": "b3a_dgrad_kernel", "us_per_step": round(b3a_us, 1), "issued_tflop": round(issued / 1e12, 4), "useful_tflop": round(useful / 1e12, 4),
           "issued_tflops": round(issued / b3a_us / 1e6, 1) if b3a_us else None, "useful_tflops": round(useful / b3a_us / 1e6, 1) if b3a_us else None}
    rows = []
    for name, (all_t, nz) in gemms.items():
        us = sum(v for k, v in per.items() if name in k)
        rows.append({"kernel": name, "us_per_step": round(us, 1), "all_tiles_tflop": round(all_t / 1e12, 4), "nonzero_tflop": round(nz / 1e12, 4),
                     "all_tiles_tflops": round(all_t / us / 1e6, 1) if us else None, "nonzero_tflops": round(nz / us / 1e6, 1) if us else None})
    top = sorted(per.items(), key=lambda kv: -kv[1])[:15]
    res = {"gpu": info, "clocks_during_profile": clocks, "frames_per_step": nf, "steps": args.steps,
           "kernel_us_per_step_total": round(total, 1), "head_gemms": rows, "b3a": b3a, "fixed_order_sums": fixed_sums,
           "top_kernels": [{"kernel": k[:90], "us_per_step": round(v, 1)} for k, v in top]}
    print(f"{info.get('name')}  power limit {info.get('power.limit')}  SM clock {clocks.get('sm_mhz')} MHz (max {clocks.get('sm_max_mhz')})  "
          f"{nf} frames/step, {args.steps} steps")
    print(f"{'kernel':28s} {'us/step':>9s} {'all-tiles TFLOP':>16s} {'non-zero TFLOP':>15s} {'all-tiles TFLOP/s':>18s} {'non-zero TFLOP/s':>17s}")
    for r in rows:
        print(f"{r['kernel']:28s} {r['us_per_step']:9.1f} {r['all_tiles_tflop']:16.4f} {r['nonzero_tflop']:15.4f} {r['all_tiles_tflops'] or 0:18.1f} {r['nonzero_tflops'] or 0:17.1f}")
    print(f"{'b3a_dgrad_kernel':28s} {b3a['us_per_step']:9.1f}  issued {b3a['issued_tflop']:.4f} TFLOP ({b3a['issued_tflops'] or 0:.1f} TFLOP/s), "
          f"useful {b3a['useful_tflop']:.4f} TFLOP ({b3a['useful_tflops'] or 0:.1f} TFLOP/s)")
    print(f"{'fixed-order sums':28s} {fixed_sums['us_per_step']:9.1f} us/step in {fixed_sums['launches_per_step']:g} launches/step (reduce_partials*)")
    print(f"all kernels: {total:.1f} us/step (summed over both streams)")
    for t in res["top_kernels"]:
        print(f"  {t['us_per_step']:9.1f}  {t['kernel']}")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
