"""Kernel-level timing of the bf16 GEMM at the qwen-3-4b prefill shapes (M = 32,768 tokens).

    python tools/gemm_bench.py [--lib PATH] [--m ROWS] [--plain] [--sweep] [--cublas] [--out FILE]

Times sb200_gemm_bf16_tn / sb200_gemm_qkv_rope with their real epilogues on seeded operands,
with CUDA events over >= --seconds of work per shape after a warm-up, and prints one JSON line.
  --lib       load another build of libsutro_b200.so (sets SB200_LIB), so two builds can be
              timed alternately on the same card
  --m         rows (tokens) per GEMM; the default is a full 32k-token prefill step, 128 or the
              decode batch (3584) time the decode-sized calls
  --plain     also time each shape with a plain bf16 store (EPI_STORE_BF16 at the same N and K),
              so the cost of each fused epilogue over a plain store can be read off directly
  --sweep     also time the down shape at block_n = 64 / 128 / 256 and report the implied
              operand feed, rate x (128 + BN) / (128 BN) bytes per flop into shared memory
  --cublas    also time torch.matmul (cuBLAS) at the same shapes and name its kernels
The card's name, power limit and SM clock are read with nvidia-smi while the largest shape runs.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

M = 32768
HQ, HKV, HD, PAGE = 32, 8, 128, 16
# name, N, K, epilogue (0 store, 1 +residual, 2 SwiGLU, 4 QKV_ROPE)
SHAPES = [("gate_up", 19456, 2560, 2), ("down", 2560, 9728, 1), ("qkv", 6144, 2560, 4),
          ("o", 2560, 4096, 1)]


def gpu_info(fields: str) -> str:
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else ""
    except (OSError, subprocess.SubprocessError):
        return ""


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None)
    ap.add_argument("--m", type=int, default=32768)
    ap.add_argument("--plain", action="store_true")
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--cublas", action="store_true")
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--out", default=None, help="append the JSON line to this file as well")
    args = ap.parse_args()
    global M
    M = args.m
    if args.lib:
        os.environ["SB200_LIB"] = os.path.abspath(args.lib)
    sys.path.insert(0, ROOT)
    import torch
    from sutro_b200 import _lib as L

    assert torch.cuda.is_available(), "gemm_bench needs a GPU"
    lib = L.lib()
    dev = "cuda"
    stream = torch.cuda.current_stream()
    g = torch.Generator(device=dev).manual_seed(0)

    def rand(*shape, scale=1.0):
        return (torch.randn(*shape, device=dev, generator=g) * scale).to(torch.bfloat16)

    # operands shared by every shape (sized for the largest K and N)
    a_big = rand(M, 9728)
    # QKV epilogue operands: the tokens of 32 sequences back to back (1024 each at M = 32768),
    # pages laid out per slot
    slots = 32
    seq = (M + slots - 1) // slots
    max_pages = (seq + PAGE - 1) // PAGE
    tok_slot = (torch.arange(M, device=dev, dtype=torch.int32) // seq).contiguous()
    tok_pos = (torch.arange(M, device=dev, dtype=torch.int32) % seq).contiguous()
    page_table = torch.arange(slots * max_pages, device=dev, dtype=torch.int32)
    kv = torch.zeros(slots * max_pages, HKV, 2, PAGE, HD, dtype=torch.bfloat16, device=dev)
    inv = 1.0 / (1e6 ** (torch.arange(0, HD, 2, dtype=torch.float32, device=dev) / HD))
    fr = torch.arange(seq, dtype=torch.float32, device=dev)[:, None] * inv[None, :]
    cos, sin = fr.cos().to(torch.bfloat16), fr.sin().to(torch.bfloat16)
    qn = (torch.rand(HD, device=dev, generator=g) + 0.5).to(torch.bfloat16)
    kn = (torch.rand(HD, device=dev, generator=g) + 0.5).to(torch.bfloat16)

    def make_call(N, K, epi, block_n):
        a = a_big[:, :K].contiguous()
        w = rand(N, K, scale=1.0 / math.sqrt(K))
        if epi == 2:
            out = torch.empty(M, N // 2, dtype=torch.bfloat16, device=dev)
        else:
            out = rand(M, N)
        s = stream.cuda_stream
        if epi == 4:
            return lambda: L.check(lib.sb200_gemm_qkv_rope(
                a.data_ptr(), M, w.data_ptr(), out.data_ptr(), M, K, block_n, qn.data_ptr(),
                kn.data_ptr(), cos.data_ptr(), sin.data_ptr(), tok_slot.data_ptr(),
                tok_pos.data_ptr(), page_table.data_ptr(), max_pages, kv.data_ptr(), HQ, HKV,
                1e-6, s))
        resid = out.data_ptr() if epi == 1 else 0     # in place, as the engine runs it
        return lambda: L.check(lib.sb200_gemm_bf16_tn(
            a.data_ptr(), M, w.data_ptr(), out.data_ptr(), resid, M, N, K, out.shape[1], epi,
            block_n, s))

    def time_fn(fn, flops, read_clock=False):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(3):
            fn()
        e1.record()
        torch.cuda.synchronize()
        per = e0.elapsed_time(e1) / 3 * 1e-3
        n = max(5, math.ceil(args.seconds / per))
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        clock = gpu_info("clocks.sm") if read_clock else None   # read while the queue runs
        torch.cuda.synchronize()
        sec = e0.elapsed_time(e1) * 1e-3 / n
        return {"ms": sec * 1e3, "tflops": flops / sec / 1e12, "iters": n, "clock_sm": clock}

    res = {"lib": L.LIB_PATH, "gpu": gpu_info("name,power.limit,clocks.max.sm"),
           "M": M, "shapes": {}}
    for i, (name, N, K, epi) in enumerate(SHAPES):
        t = time_fn(make_call(N, K, epi, 0), 2.0 * M * N * K, read_clock=(i == 0))
        if t["clock_sm"]:
            res["clock_sm_under_load"] = t["clock_sm"]
        del t["clock_sm"]
        res["shapes"][name] = {"N": N, "K": K, "epi": epi, **t}
        torch.cuda.empty_cache()

    if args.plain:
        res["plain"] = {}
        for name, N, K, _ in SHAPES:
            t = time_fn(make_call(N, K, 0, 0), 2.0 * M * N * K)
            del t["clock_sm"]
            res["plain"][name] = t
            torch.cuda.empty_cache()

    if args.sweep:
        _, N, K, epi = SHAPES[1]
        res["down_block_n_sweep"] = {}
        for bn in (64, 128, 256):
            t = time_fn(make_call(N, K, epi, bn), 2.0 * M * N * K)
            del t["clock_sm"]
            # A (128 x 64) and W (BN x 64) bf16 per 2 * 128 * BN * 64 flop
            t["feed_TBps"] = t["tflops"] * (128 + bn) / (128 * bn)
            res["down_block_n_sweep"][bn] = t

    if args.cublas:
        res["cublas"] = {}
        for name, N, K, _ in SHAPES:
            a = a_big[:, :K].contiguous()
            w = rand(N, K, scale=1.0 / math.sqrt(K))
            t = time_fn(lambda: torch.matmul(a, w.t()), 2.0 * M * N * K)
            del t["clock_sm"]
            res["cublas"][name] = t
            del a, w
            torch.cuda.empty_cache()
        from torch.profiler import ProfilerActivity, profile
        _, N, K, _ = SHAPES[0]
        a = a_big[:, :K].contiguous()
        w = rand(N, K, scale=1.0 / math.sqrt(K))
        torch.matmul(a, w.t())
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            torch.matmul(a, w.t())
            torch.cuda.synchronize()
        res["cublas_kernels"] = sorted({e.key for e in prof.key_averages()
                                        if e.device_type == torch.autograd.DeviceType.CUDA})

    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
