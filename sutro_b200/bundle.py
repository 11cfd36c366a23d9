"""Model bundles: a LocalEngine's model written to disk in the form `sb200_model_open` reads
(csrc/model_bundle.cu), so that a host without Python can serve it through the C-ABI.

    python -m sutro_b200.bundle --model qwen-3-4b --out /models/qwen-3-4b.sb200 [--seed 0]
    python -m sutro_b200.bundle --hf-dir /ckpt/Qwen3-4B --out /models/qwen3-4b.sb200
    python -m sutro_b200.bundle --model qwen-3-4b --max-position 131072 --out /models/q4b-128k

Layout: `manifest.json` (format 1: spec, tokenizer parameters, special-token ids, and for every
tensor its byte offset / size in `data.bin`) + `data.bin` (bf16 weights in the engine's layout
— wqkv rows q|k|v, gate/up rows interleaved —, bf16 RoPE tables, tokenizer tables)."""
from __future__ import annotations

import json
import os
from typing import Dict

import numpy as np
import torch


def _bytes(t) -> bytes:
    if isinstance(t, np.ndarray):
        return np.ascontiguousarray(t).tobytes()
    t = t.detach().contiguous().cpu()
    return t.view(torch.uint8).numpy().tobytes() if t.dtype != torch.uint8 else t.numpy().tobytes()


def export_bundle(engine, out_dir: str) -> str:
    """Write `engine`'s model (weights, RoPE tables, tokenizer) as a bundle directory."""
    from .unicode_tables import class_table
    os.makedirs(out_dir, exist_ok=True)
    spec, w, v = engine.spec, engine.weights, engine.vocab
    tensors: Dict[str, Dict[str, int]] = {}
    with open(os.path.join(out_dir, "data.bin"), "wb") as f:
        def put(name, t):
            b = _bytes(t)
            pad = (-f.tell()) % 256
            f.write(b"\0" * pad)
            tensors[name] = {"offset": f.tell(), "bytes": len(b)}
            f.write(b)
        put("embed", w.embed)
        if not spec.tied_embeddings:
            put("lm_head", w.lm_head)
        put("final_norm", w.final_norm)
        put("rope_cos", engine.cos)
        put("rope_sin", engine.sin)
        for l in range(spec.n_layers):
            p = f"layers.{l}."
            for name in ("ln1", "ln2", "wqkv", "wo", "wgu", "wd"):
                put(p + name, getattr(w, name)[l])
            if spec.qk_norm:
                put(p + "q_norm", w.q_norm[l])
                put(p + "k_norm", w.k_norm[l])
        blob, off = v.byte_blob()
        put("tok.merges", np.ascontiguousarray(v.merge_array(), dtype=np.int32))
        if v.merged_ids is not None:
            put("tok.merged_ids", np.ascontiguousarray(v.merged_ids, dtype=np.int32))
        put("tok.cls_table", np.ascontiguousarray(class_table(), dtype=np.uint8))
        put("tok.bytes", np.ascontiguousarray(blob, dtype=np.uint8))
        put("tok.offsets", np.ascontiguousarray(off, dtype=np.int32))
        if v.word_overrides:      # ignore_merges (vocab.Vocab.word_overrides)
            from .engine import word_override_arrays
            o_toks, o_off, o_ids = word_override_arrays(v)
            put("tok.override_tokens", o_toks)
            put("tok.override_offsets", o_off)
            put("tok.override_ids", o_ids)
    manifest = {
        "format": 1,
        "spec": {"name": spec.name, "family": spec.family, "n_layers": spec.n_layers,
                 "d_model": spec.d_model, "n_q_heads": spec.n_q_heads,
                 "n_kv_heads": spec.n_kv_heads, "d_ff": spec.d_ff, "vocab_size": spec.vocab_size,
                 "max_position": spec.max_position, "rms_eps": spec.rms_eps,
                 "qk_norm": int(spec.qk_norm), "embedding_model": int(spec.embedding_model),
                 "eos_id": int(v.eos_id), "tied_embeddings": int(spec.tied_embeddings)},
        "tokenizer": {"digits": int(v.digits), "n_merges": len(v.merges)},
        "specials": {k: int(i) for k, i in v.specials.items()},
        "tensors": tensors,
    }
    with open(os.path.join(out_dir, "manifest.json"), "w") as f:
        json.dump(manifest, f, ensure_ascii=True)
    return out_dir


def main():
    import argparse
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument("--model", default=None, help="named architecture, seeded random weights")
    ap.add_argument("--hf-dir", default=None, help="Hugging Face model directory (safetensors)")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--max-position", type=int, default=None,
                    help="context window to serve (default: the model's registered window); "
                         "the bundle holds RoPE tables for it")
    ap.add_argument("--out", required=True)
    a = ap.parse_args()
    from .engine import LocalEngine
    if a.hf_dir:
        from .pretrained import load_pretrained
        kw = {} if a.max_position is None else {"max_position": a.max_position}
        eng = load_pretrained(a.hf_dir, 0, kv_pages=64, max_slots=8, max_prefill_tokens=256, **kw)
    elif a.model:
        eng = LocalEngine.from_seed(a.model, seed=a.seed, device=0, kv_pages=64, max_slots=8,
                                    max_prefill_tokens=256, max_position=a.max_position)
    else:
        ap.error("--model or --hf-dir")
    print(export_bundle(eng, a.out))


if __name__ == "__main__":
    main()
