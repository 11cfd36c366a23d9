"""Save the outputs of the fused GEMMs at the qwen-3-4b prefill shapes, to compare two builds.

    python tools/gemm_dump.py --lib PATH --out DIR [--no-dense]

Runs, on seeded operands, the four prefill GEMMs of one layer at M = 32,768 tokens in engine
order: QKV (+q/k-norm, RoPE, paged K/V, dense K/V copy), O (+residual, in place), gate/up
(+SwiGLU) and down (+residual, in place), then QKV at M = 3,584.  Writes each output buffer as
raw bytes to DIR: qkv.bin, kv.bin (the paged pool), x.bin (the residual stream after O and
down), act.bin (the SwiGLU output), qkv_3584.bin and kv_3584.bin.  With --no-dense only the
M = 3,584 QKV runs, without the dense K/V copy (SB200_QKV_DENSE=0, as a decode step), into
qkv_3584_nodense.bin and kv_3584_nodense.bin.  Each build runs in its own process; the files of
two builds are then compared byte for byte (cmp).
"""
from __future__ import annotations

import argparse
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HQ, HKV, HD, PAGE = 32, 8, 128, 16
D, FF = 2560, 9728


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", required=True)
    ap.add_argument("--out", required=True)
    ap.add_argument("--no-dense", action="store_true")
    args = ap.parse_args()
    os.environ["SB200_LIB"] = os.path.abspath(args.lib)
    if args.no_dense:
        os.environ["SB200_QKV_DENSE"] = "0"
    sys.path.insert(0, ROOT)
    import torch
    from sutro_b200 import _lib as L

    assert torch.cuda.is_available(), "gemm_dump needs a GPU"
    lib = L.lib()
    dev = "cuda"
    s = torch.cuda.current_stream().cuda_stream
    g = torch.Generator(device=dev).manual_seed(0)
    os.makedirs(args.out, exist_ok=True)

    def rand(*shape, scale=1.0):
        return (torch.randn(*shape, device=dev, generator=g) * scale).to(torch.bfloat16)

    def save(name, t):
        torch.cuda.synchronize()
        t.contiguous().view(torch.uint8).cpu().numpy().tofile(os.path.join(args.out, name))

    n_qkv = (HQ + 2 * HKV) * HD
    w_qkv = rand(n_qkv, D, scale=1.0 / math.sqrt(D))
    w_o = rand(D, HQ * HD, scale=1.0 / math.sqrt(HQ * HD))
    w_gu = rand(2 * FF, D, scale=1.0 / math.sqrt(D))
    w_down = rand(D, FF, scale=1.0 / math.sqrt(FF))
    qn = (torch.rand(HD, device=dev, generator=g) + 0.5).to(torch.bfloat16)
    kn = (torch.rand(HD, device=dev, generator=g) + 0.5).to(torch.bfloat16)
    inv = 1.0 / (1e6 ** (torch.arange(0, HD, 2, dtype=torch.float32, device=dev) / HD))

    def qkv(m, slots, tag):
        """QKV of m tokens, `slots` sequences back to back, into a fresh pool."""
        seq = (m + slots - 1) // slots
        max_pages = (seq + PAGE - 1) // PAGE
        tok_slot = (torch.arange(m, device=dev, dtype=torch.int32) // seq).contiguous()
        tok_pos = (torch.arange(m, device=dev, dtype=torch.int32) % seq).contiguous()
        perm = torch.randperm(slots * max_pages + 8, device=dev, generator=g)
        page_table = perm[:slots * max_pages].to(torch.int32).contiguous()
        kv = torch.zeros(slots * max_pages + 8, HKV, 2, PAGE, HD, dtype=torch.bfloat16, device=dev)
        fr = torch.arange(seq, dtype=torch.float32, device=dev)[:, None] * inv[None, :]
        cos, sin = fr.cos().to(torch.bfloat16), fr.sin().to(torch.bfloat16)
        a = rand(m, D)
        out = torch.zeros(m, n_qkv, dtype=torch.bfloat16, device=dev)
        L.check(lib.sb200_gemm_qkv_rope(
            a.data_ptr(), m, w_qkv.data_ptr(), out.data_ptr(), m, D, 0, qn.data_ptr(),
            kn.data_ptr(), cos.data_ptr(), sin.data_ptr(), tok_slot.data_ptr(), tok_pos.data_ptr(),
            page_table.data_ptr(), max_pages, kv.data_ptr(), HQ, HKV, 1e-6, s))
        save(f"qkv{tag}.bin", out)
        save(f"kv{tag}.bin", kv)
        return out

    def gemm(a, w, out, resid, n, k, epi):
        L.check(lib.sb200_gemm_bf16_tn(a.data_ptr(), a.shape[0], w.data_ptr(), out.data_ptr(),
                                       L.ptr(resid), a.shape[0], n, k, out.shape[1], epi, 0, s))

    if args.no_dense:
        qkv(3584, 16, "_3584_nodense")
        return
    m = 32768
    q = qkv(m, 32, "")
    x = rand(m, D)
    gemm(q[:, :HQ * HD].contiguous(), w_o, x, x, D, HQ * HD, 1)       # O + residual, in place
    act = torch.empty(m, FF, dtype=torch.bfloat16, device=dev)
    gemm(x, w_gu, act, None, 2 * FF, D, 2)                            # gate/up + SwiGLU
    save("act.bin", act)
    gemm(act, w_down, x, x, D, FF, 1)                                 # down + residual, in place
    save("x.bin", x)
    qkv(3584, 16, "_3584")


if __name__ == "__main__":
    main()
