"""Kernel-level timing of the dense prefill attention (one layer) at the benchmark's shapes.

    python tools/attn_bench.py [--lib PATH] [--seconds S] [--heads HQ/HKV] [--out FILE]

Times sb200_attn_prefill_dense on seeded bf16 operands, qwen-3-4b heads (32 query, 8 kv heads,
G = 4) unless --heads says otherwise (40/8 is qwen-3-14b, G = 5), with CUDA events over
>= --seconds of work per shape after a warm-up, and prints one JSON line.  Shapes, one
32k-token prefill step each:
  headline   306 rows of 107 own tokens after a 46-token shared prefix (the sentiment job)
  documents  64 rows of 512 tokens, no prefix (the 512-token documents job)
For each: ms per launch, the HBM floor (Q and K/V read once, O written once, over 3.35 TB/s),
the bytes/s that implies, and the useful causal FLOP/s (QK^T and PV over visible keys only).
  --lib       load another build of libsutro_b200.so (sets SB200_LIB), so two builds can be
              timed alternately on the same card
The card's name, power limit and SM clock are read with nvidia-smi while the last shape runs.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

HQ, HKV, HD = 32, 8, 128
HBM_BYTES_PER_S = 3.35e12       # H100 SXM data sheet
SHAPES = {"headline": (306, 107, 46), "documents": (64, 512, 0)}   # rows, own tokens, prefix


def gpu_info(fields: str) -> str:
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else ""
    except (OSError, subprocess.SubprocessError):
        return ""


def shape_costs(rows: int, own: int, past: int):
    """(bytes, flops) the shape needs: Q and O once per token, own K/V once per token, the
    prefix K/V once; 4 * 128 flops per (query head, visible key)."""
    T = rows * own
    tok = 2 * HD                                        # bytes of one head's row
    nbytes = T * HQ * tok * 2 + T * 2 * HKV * tok + past * 2 * HKV * tok
    visible = rows * sum(past + j + 1 for j in range(own))
    return nbytes, 4.0 * HD * HQ * visible


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None)
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--heads", default="32/8",
                    help="query/kv heads, e.g. 40/8 for qwen-3-14b (default: qwen-3-4b's 32/8)")
    ap.add_argument("--out", default=None, help="append the JSON line to this file as well")
    args = ap.parse_args()
    global HQ, HKV
    HQ, HKV = (int(x) for x in args.heads.split("/"))
    if args.lib:
        os.environ["SB200_LIB"] = os.path.abspath(args.lib)
    sys.path.insert(0, ROOT)
    import torch
    from sutro_b200 import _lib as L

    if not torch.cuda.is_available():
        sys.exit("attn_bench: needs a CUDA device")
    lib = L.lib()
    qt = lib.sb200_attn_prefill_q_tile(HQ, HKV)
    ldq = (HQ + 2 * HKV) * HD
    n_layers, layer = 2, 1
    result = {"lib": os.environ.get("SB200_LIB", "default"), "shapes": {}}
    for name, (rows, own, past) in SHAPES.items():
        T = rows * own
        g = torch.Generator(device="cpu").manual_seed(rows * 1000 + own)
        qkv = torch.randn(T + 32, ldq, generator=g).to("cuda", torch.bfloat16)
        pre = torch.randn(n_layers, max(past, 1), 2 * HKV * HD, generator=g).to("cuda",
                                                                             torch.bfloat16)
        out = torch.empty(T, HQ * HD, dtype=torch.bfloat16, device="cuda")
        i32 = lambda x: torch.tensor(x, dtype=torch.int32, device="cuda")
        items = i32([x for i in range(rows) for t0 in range(0, own, qt) for x in (i, t0)])
        qs, ql, pa = i32([i * own for i in range(rows)]), i32([own] * rows), i32([past] * rows)
        stream = torch.cuda.current_stream().cuda_stream

        def launch():
            L.check(lib.sb200_attn_prefill_dense(
                L.ptr(qkv), qkv.shape[0], L.ptr(out), L.ptr(pre) if past else None,
                past if past else 0, n_layers, layer, L.ptr(items), items.numel() // 2, L.ptr(qs),
                L.ptr(ql), L.ptr(pa), HQ, HKV, 1.0 / math.sqrt(HD), stream))

        for _ in range(5):
            launch()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            launch()
        e1.record()
        torch.cuda.synchronize()
        n = max(10, int(args.seconds * 1e3 / (e0.elapsed_time(e1) / 5)))
        e0.record()
        for _ in range(n):
            launch()
        e1.record()
        if name == list(SHAPES)[-1]:
            card = gpu_info("name,power.limit,clocks.sm")
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / n
        nbytes, flops = shape_costs(rows, own, past)
        floor_ms = nbytes / HBM_BYTES_PER_S * 1e3
        result["shapes"][name] = {
            "rows": rows, "own_tokens": own, "prefix": past, "tokens": T, "launches": n,
            "ms": round(ms, 4), "hbm_floor_ms": round(floor_ms, 4),
            "gb_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1),
            "share_of_hbm_floor": round(floor_ms / ms, 3),
            "useful_tflop_per_s": round(flops / (ms * 1e-3) / 1e12, 1)}
    result["card"] = card
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
