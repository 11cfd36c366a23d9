"""Long-context timing: split-KV decode attention per layer, and one end-to-end long-document job.

    python tools/long_context_bench.py [--seconds S] [--docs N] [--doc-tokens T] [--heads HQ/HKV]
                                       [--max-position W] [--skip-e2e] [--out FILE]

1. Decode attention, one layer, qwen-3-4b heads (32 query, 8 kv heads; --heads 40/8 gives
   qwen-3-14b's), through sb200_attn_decode on seeded bf16 operands, CUDA events over
   >= --seconds of launches per shape after a warm-up:
     12 x 32k, 24 x 16k, 48 x 8k    rows x tokens of context (about 12 GB of KV each)
     mixed       1 x 32k + 3,583 x 128, against the 3,583 short rows alone
   For each: ms per launch, the HBM floor (every row's K/V read once, over the 3.35 TB/s data
   sheet figure) and the bytes/s reached.  The C-ABI bounds contexts by the page table's width, so
   the mixed launch (width 2,049 pages) lets every row split and carries the empty units of the
   short rows; the engine lists only its long rows.
2. End-to-end: --docs synthetic documents of about --doc-tokens tokens, 64 output tokens each,
   qwen-3-4b (seeded weights), no schema, default engine options: rows/s and input tokens/s of a
   timed run, then a profiled run's per-class device times, with the prefill attention's useful
   causal TFLOP/s.
3. With --max-position W (e.g. 131072): the end-to-end job serves a W-token window (qwen-3-4b
   switches to YaRN past 32,768; pass --doc-tokens near W, e.g. 120000), decode attention adds
   4 rows x W tokens, and the prefill attention of one W-token row is timed per layer both ways:
   one sb200_attn_prefill_dense call over the row, and the 32,768-token chunks the engine runs
   (sb200_attn_prefill_chunked, each chunk's earlier tokens read from the paged pool), with the
   useful causal TFLOP/s of each and their ratio.
The card's name, power limit and SM clock are read with nvidia-smi during the measurements.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

HQ, HKV, HD, PAGE = 32, 8, 128, 16
HBM_BYTES_PER_S = 3.35e12       # H100 SXM data sheet
SHAPES = {"12x32k": [32768] * 12, "24x16k": [16384] * 24, "48x8k": [8192] * 48,
          "mixed_1x32k_3583x128": [32768] + [128] * 3583, "short_3583x128": [128] * 3583}


def gpu_info(fields: str) -> str:
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else ""
    except (OSError, subprocess.SubprocessError):
        return ""


def kv_bytes(lens) -> int:
    """K and V of every context token of every kv head, read once."""
    return sum(lens) * HKV * 2 * HD * 2


def time_launches(launch, seconds: float, torch) -> tuple:
    for _ in range(3):
        launch()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(3):
        launch()
    e1.record()
    torch.cuda.synchronize()
    n = max(10, int(seconds * 1e3 / (e0.elapsed_time(e1) / 3)))
    e0.record()
    for _ in range(n):
        launch()
    e1.record()
    card = gpu_info("name,power.limit,clocks.sm")
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n, n, card


def decode_shapes(args, torch, L) -> dict:
    lib = L.lib()
    out = {}
    shapes = dict(SHAPES)
    window = max(32768, args.max_position or 0)
    if window > 32768:
        shapes[f"4x{window // 1024}k"] = [window] * 4
    for name, lens in shapes.items():
        B = len(lens)
        n_pages = [(n + PAGE - 1) // PAGE for n in lens]
        # the short-only launch keeps today's page-table width (no split); the rest the engine's
        width = (4096 // PAGE) if max(lens) <= 4096 else window // PAGE + 1
        total = sum(n_pages)
        g = torch.Generator(device="cuda").manual_seed(B)
        pool = torch.randn(total, HKV, 2, PAGE, HD, device="cuda", generator=g).to(torch.bfloat16)
        pt = torch.zeros(B, width, dtype=torch.int32)
        at = 0
        perm = torch.randperm(total, generator=torch.Generator().manual_seed(B)).to(torch.int32)
        for i, n in enumerate(n_pages):
            pt[i, :n] = perm[at:at + n]
            at += n
        pt = pt.cuda()
        qkv = torch.randn(B, (HQ + 2 * HKV) * HD, device="cuda", generator=g).to(torch.bfloat16)
        o = torch.empty(B, HQ * HD, dtype=torch.bfloat16, device="cuda")
        rs = torch.arange(B, dtype=torch.int32, device="cuda")
        ctx = torch.tensor(lens, dtype=torch.int32, device="cuda")
        stream = torch.cuda.current_stream().cuda_stream

        def launch():
            L.check(lib.sb200_attn_decode(L.ptr(qkv), L.ptr(o), L.ptr(pool), L.ptr(pt), width,
                                          L.ptr(rs), L.ptr(ctx), B, HQ, HKV, 1.0 / math.sqrt(HD),
                                          stream))

        ms, n, card = time_launches(launch, args.seconds, torch)
        nbytes = kv_bytes(lens)
        out[name] = {"rows": B, "context_tokens": sum(lens), "launches": n, "ms": round(ms, 4),
                     "hbm_floor_ms": round(nbytes / HBM_BYTES_PER_S * 1e3, 4),
                     "tb_per_s": round(nbytes / (ms * 1e-3) / 1e12, 3),
                     "share_of_3_35_tb_per_s": round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3),
                     "card": card}
        print(name, out[name], flush=True)
        del pool, pt, qkv, o
        torch.cuda.empty_cache()
    return out


def causal_flops(n_tok: int, hq: int) -> float:
    """Useful causal attention FLOPs of one layer over an n_tok-token row: 4 * 128 per (query
    head, visible key)."""
    return 4.0 * HD * hq * n_tok * (n_tok + 1) / 2


def chunked_vs_dense(args, torch, L, chunk: int = 32768) -> dict:
    """Per-layer prefill attention of one max_position-token row (no shared prefix): one dense
    call, against the engine's chunks of `chunk` tokens reading their history from the pool."""
    lib = L.lib()
    n = args.max_position
    g = torch.Generator(device="cuda").manual_seed(11)
    w = (HQ + 2 * HKV) * HD
    qkv = torch.randn(n + 32, w, device="cuda", generator=g).to(torch.bfloat16)
    out = torch.empty(n + 32, HQ * HD, dtype=torch.bfloat16, device="cuda")
    # the pool holds the row's K/V at positions [0, n) (values need only be finite for timing)
    pages = n // PAGE
    pool = torch.randn(pages, HKV, 2, PAGE, HD, device="cuda", generator=g).to(torch.bfloat16)
    pt = torch.randperm(pages, generator=torch.Generator().manual_seed(3)).to(torch.int32)
    pt = torch.cat([pt, torch.zeros(1, dtype=torch.int32)]).cuda()
    qt = lib.sb200_attn_prefill_q_tile(HQ, HKV)
    align = lib.sb200_attn_prefill_hist_align(HQ, HKV)
    chunk = chunk // align * align
    i32 = lambda x: torch.tensor(x, dtype=torch.int32, device="cuda")   # noqa: E731
    stream = torch.cuda.current_stream().cuda_stream
    scale = 1.0 / math.sqrt(HD)
    dense_args = (i32([x for t0 in range(0, n, qt) for x in (0, t0)]), i32([0]), i32([n]),
                  i32([0]))

    def dense():
        it, qs, ql, past = dense_args
        L.check(lib.sb200_attn_prefill_dense(L.ptr(qkv), n + 32, L.ptr(out), None, 0, 1, 0,
                                             L.ptr(it), len(range(0, n, qt)), L.ptr(qs),
                                             L.ptr(ql), L.ptr(past), HQ, HKV, scale, stream))
    chunks = []
    for h in range(0, n, chunk):
        m = min(chunk, n - h)
        chunks.append((m, i32([x for t0 in range(0, m, qt) for x in (0, t0)]), i32([0]),
                       i32([m]), i32([0]), i32([0]), i32([h])))

    def chunked():
        for m, it, qs, ql, past, slot, hist in chunks:
            L.check(lib.sb200_attn_prefill_chunked(
                L.ptr(qkv), n + 32, L.ptr(out), None, 0, 1, 0, L.ptr(it), len(range(0, m, qt)),
                L.ptr(qs), L.ptr(ql), L.ptr(past), HQ, HKV, scale, L.ptr(pool), L.ptr(pt),
                pages + 1, L.ptr(slot), L.ptr(hist), stream))
    res = {"row_tokens": n, "chunk_tokens": chunk, "chunks": len(chunks)}
    flops = causal_flops(n, HQ)
    for name, fn in (("dense", dense), ("chunked", chunked)):
        ms, k, card = time_launches(fn, args.seconds, torch)
        res[name] = {"ms": round(ms, 3), "launches": k,
                     "tflop_per_s": round(flops / (ms * 1e-3) / 1e12, 1), "card": card}
        print(name, res[name], flush=True)
    res["chunked_over_dense"] = round(res["chunked"]["ms"] / res["dense"]["ms"], 3)
    del qkv, out, pool
    torch.cuda.empty_cache()
    return res


def end_to_end(args, torch) -> dict:
    from sutro_b200 import modelspec as MS, synth, vocab as VB
    from sutro_b200.engine import LocalEngine
    spec = MS.with_window(MS.get_spec("qwen-3-4b"), args.max_position)
    w = MS.make_engine_weights_on_device(spec, seed=0, device="cuda")
    v = VB.build_vocab(spec.family, spec.vocab_size, seed=0)
    eng = LocalEngine(spec, w, v, device=0)
    # calibrate words per token on one document, then draw the job's documents at that length
    probe = synth.documents(1, seed=7, words=2000)[0]
    ratio = len(probe.split()) / len(eng.tokenizer.encode([probe])[0])
    docs = synth.documents(args.docs, seed=7, words=int(args.doc_tokens * ratio))
    kw = dict(max_new_tokens=64, ignore_eos=True)
    eng.generate(docs[:1 if args.max_position else 2], **kw)     # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = eng.generate(docs, **kw)
    dt = time.perf_counter() - t0
    card = gpu_info("name,power.limit,clocks.sm")
    prof = eng.generate(docs, profile=True, **kw).stats
    kms = prof["kernel_ms"]
    # useful causal prefill attention FLOPs: 4 * 128 per (query head, visible key), every layer
    rows_tok = prof["input_tokens"] / args.docs
    attn_flops = (args.docs * 4.0 * HD * spec.n_q_heads * spec.n_layers * rows_tok *
                  (rows_tok + 1) / 2)
    res = {"docs": args.docs, "input_tokens": r.stats["input_tokens"],
           "rows_truncated": r.stats["rows_truncated"], "seconds": round(dt, 2),
           "rows_per_sec": round(args.docs / dt, 3),
           "input_tok_per_sec": round(r.stats["input_tokens"] / dt, 1),
           "kernel_ms": {k: round(kms[k], 1) for k in ("attn_prefill", "gemm", "attn_decode")
                         if k in kms},
           "gemm_tflop_per_s": round(prof["gemm_flops"] / (kms["gemm"] * 1e-3) / 1e12, 1),
           "prefill_attn_tflop_per_s": round(attn_flops / (kms["attn_prefill"] * 1e-3) / 1e12, 1),
           "kv_pages": eng.kv_pages, "max_position": spec.max_position,
           "prefill_steps": r.stats["prefill_steps"], "card": card}
    eng.close()
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--docs", type=int, default=64)
    ap.add_argument("--doc-tokens", type=int, default=30000)
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--heads", default="32/8",
                    help="query/kv heads, e.g. 40/8 for qwen-3-14b (default: qwen-3-4b's 32/8)")
    ap.add_argument("--max-position", type=int, default=None,
                    help="serve this window (e.g. 131072) and time the chunked prefill attention")
    ap.add_argument("--skip-decode", action="store_true")
    ap.add_argument("--out", default=None, help="append the JSON line to this file as well")
    args = ap.parse_args()
    global HQ, HKV
    HQ, HKV = (int(x) for x in args.heads.split("/"))
    sys.path.insert(0, ROOT)
    import torch
    from sutro_b200 import _lib as L

    if not torch.cuda.is_available():
        sys.exit("long_context_bench: needs a CUDA device")
    result = {}
    if not args.skip_decode:
        result["decode_attention_per_layer"] = decode_shapes(args, torch, L)
    if args.max_position:
        result["prefill_attention_per_layer"] = chunked_vs_dense(args, torch, L)
    if not args.skip_e2e:
        result["end_to_end"] = end_to_end(args, torch)
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
