#!/usr/bin/env python
"""Measured HBM ceilings of this GPU for three read:write mixes, written to MEASURED_PEAKS.json.

bench.py quotes every stage's bandwidth as a share of `hbm_gbs`.  The data sheet's 3.35 TB/s (H100 SXM) is never reached
in practice, and what is reached depends on the mix of reads and writes, so the ceiling is measured with plain torch
kernels on buffers far larger than L2:
  read    a reduction (torch.sum):                 N bytes read
  copy    dst.copy_(src), 1:1 read:write:         N read + N written
  add21   torch.add(a, b, out=c), 2:1 read:write: 2N read + N written (the closest mix to k_skin's 44 B read : 24 B written)
Each pattern is timed with CUDA events around one launch, median of `--reps` launches after `--warmup`.  `hbm_gbs` is the
HIGHEST of the three rates, so a fraction of it is never inflated by choosing a slow pattern.  The card's name, power limit
and SM clock are recorded beside the numbers: they are part of them.

    python tools/hbm_peaks.py [--gib 4] [--reps 30] [--warmup 5] [--out MEASURED_PEAKS.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card_info() -> dict:
    """Name, power limit and clocks as nvidia-smi reports them (read-only queries)."""
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={q}", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        vals = [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]
        info.update(dict(zip(["smi_name", "power_limit", "sm_clock", "sm_clock_max", "mem_clock"], vals)))
    except Exception as e:  # nvidia-smi missing: the numbers still stand, the card description is thinner
        info["nvidia_smi_error"] = str(e)
    return info


def time_op(fn, reps: int, warmup: int) -> float:
    """Median milliseconds of one call of fn, CUDA events around each call."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def measure(gib: float, reps: int, warmup: int) -> dict:
    n = int(gib * (1 << 30)) // 4  # f32 elements per buffer
    nbytes = 4 * n
    out = {}
    a = torch.ones(n, dtype=torch.float32, device="cuda")
    b = torch.ones(n, dtype=torch.float32, device="cuda")
    c = torch.empty(n, dtype=torch.float32, device="cuda")
    acc = torch.empty((), dtype=torch.float32, device="cuda")
    patterns = {
        "read": (lambda: torch.sum(a, dim=0, out=acc), nbytes, 0),
        "copy": (lambda: c.copy_(a), nbytes, nbytes),
        "add21": (lambda: torch.add(a, b, out=c), 2 * nbytes, nbytes),
    }
    for name, (fn, rd, wr) in patterns.items():
        ms = time_op(fn, reps, warmup)
        out[name] = {"ms": round(ms, 4), "bytes_read": rd, "bytes_written": wr, "gbs": round((rd + wr) / ms / 1e6, 1)}
    del a, b, c
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--gib", type=float, default=4.0, help="size of each buffer in GiB (>= 4: far beyond the 50 MB L2)")
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(REPO, "MEASURED_PEAKS.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("hbm_peaks: no CUDA device; the ceilings can only be measured on the GPU")
    rates = measure(args.gib, args.reps, args.warmup)
    res = {
        "hbm_gbs": max(r["gbs"] for r in rates.values()),
        "patterns": rates,
        "card": card_info(),
        "method": f"CUDA events around one launch, median of {args.reps} after {args.warmup} warm-up, {args.gib:g} GiB per buffer",
        "datasheet_gbs": 3350.0,
    }
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
