"""Cost of presence / frequency / repetition penalties and min_p on the configs[2]-shaped job.

    python tools/sampling_bench.py [--rows N] [--rounds R] [--out FILE]

BASELINE.json configs[2] shape: synthetic documents (~512-token prompts), qwen-3-4b bf16 with
seeded weights, 64 generated tokens with ignore_eos, no schema, one GPU, through the one-call
entry point (sb200_infer_text).  Two settings run alternately, R rounds each, on one engine:
  off  temperature 0.7
  on   temperature 0.7, presence_penalty 1.5, frequency_penalty 0.5, repetition_penalty 1.1,
       min_p 0.05
Each timed job ends in a device synchronise.  Then one profile=True job per setting gives the
device time per kernel class (CUDA events around every launch).  The card's name and power
limit are read with nvidia-smi in the same run.  Prints one JSON line (and writes it to --out).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SETTINGS = {
    "off": dict(temperature=0.7, seed=1),
    "on": dict(temperature=0.7, seed=1, presence_penalty=1.5, frequency_penalty=0.5,
               repetition_penalty=1.1, min_p=0.05),
}


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, power, clock = (s.strip() for s in (q.stdout.strip().split(",") + ["?", "?", "?"])[:3])
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    from sutro_b200 import synth
    from sutro_b200.engine import KERNEL_CLASSES, LocalEngine
    assert torch.cuda.is_available(), "sampling_bench measures on the GPU; none is visible"

    eng = LocalEngine.from_seed("qwen-3-4b", seed=0, device=0, max_slots=1024,
                                max_prefill_tokens=32768)
    rows = synth.documents(args.rows, seed=11, words=475)
    kw = dict(system_prompt=None, json_schema=None, max_new_tokens=64, ignore_eos=True)

    def job(setting, n=None, **extra):
        torch.cuda.synchronize()
        t = time.perf_counter()
        r = eng.infer_one_call(rows[:n] if n else rows, return_tokens=False, **kw,
                               **SETTINGS[setting], **extra)
        torch.cuda.synchronize()
        return r, time.perf_counter() - t

    for s in SETTINGS:                        # warm-up: every shape of the timed jobs
        job(s, n=256)
    times = {s: [] for s in SETTINGS}
    info = card()
    for _ in range(args.rounds):
        for s in SETTINGS:
            r, dt = job(s)
            times[s].append(dt)
    out = {"config": "BASELINE.json configs[2] shape: synthetic documents, ~512-token prompts, "
                     "64 generated tokens (ignore_eos), no schema, qwen-3-4b bf16, 1 GPU, "
                     "sb200_infer_text",
           "rows": len(rows), "rounds": args.rounds, **info}
    for s in SETTINGS:
        med = statistics.median(times[s])
        prof, _ = job(s, profile=True)
        st = prof.stats
        out[s] = {"params": SETTINGS[s], "rows_per_sec_median": len(rows) / med,
                  "rows_per_sec_each": [len(rows) / t for t in times[s]],
                  "kernel_ms": {k: round(v, 3) for k, v in st["kernel_ms"].items()},
                  "kernel_launches": st["kernel_launches"]}
    out["sample_ms_added"] = out["on"]["kernel_ms"]["sample"] - out["off"]["kernel_ms"]["sample"]
    out["rows_per_sec_ratio_on_off"] = (out["on"]["rows_per_sec_median"]
                                        / out["off"]["rows_per_sec_median"])
    assert set(out["on"]["kernel_ms"]) == set(KERNEL_CLASSES)
    eng.close()
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
