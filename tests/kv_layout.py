"""Test helper: pack / unpack the swizzled paged KV layout (csrc/kernels.h).

pool[page][kv_head][K|V][16 tokens][128 dims] bf16; inside a [16][128] tile the
16-byte chunk c (8 dims) of token row r sits at chunk position c ^ (r & 7).
"""
import torch

PAGE = 16
HD = 128


def _perm(device):
    r = torch.arange(PAGE, device=device).view(PAGE, 1)
    c = torch.arange(16, device=device).view(1, 16)
    return (c ^ (r & 7))  # [16,16]: physical chunk of logical chunk c in row r


def pack_tile(x):
    """x: [..., 16, 128] logical -> physical (swizzled) tile."""
    shp = x.shape
    xc = x.reshape(*shp[:-1], 16, 8)
    out = torch.empty_like(xc)
    p = _perm(x.device)
    idx = p.view(*([1] * (xc.dim() - 3)), PAGE, 16, 1).expand_as(xc)
    out.scatter_(-2, idx, xc)
    return out.reshape(shp)


def unpack_tile(x):
    shp = x.shape
    xc = x.reshape(*shp[:-1], 16, 8)
    p = _perm(x.device)
    idx = p.view(*([1] * (xc.dim() - 3)), PAGE, 16, 1).expand_as(xc)
    return torch.gather(xc, -2, idx).reshape(shp)


def build_cache(k_seqs, v_seqs, hkv, num_pages, device, seed=0):
    """k_seqs[i], v_seqs[i]: [L_i, hkv, 128] bf16.  Returns (pool, page_table, max_pages).
    Pages are assigned in a shuffled order so page ids are non-trivial."""
    g = torch.Generator().manual_seed(seed)
    order = torch.randperm(num_pages, generator=g).tolist()
    n_seq = len(k_seqs)
    max_pages = max((k.shape[0] + PAGE - 1) // PAGE for k in k_seqs) + 1
    pool = torch.zeros(num_pages, hkv, 2, PAGE, HD, dtype=torch.bfloat16, device=device)
    pt = torch.zeros(n_seq, max_pages, dtype=torch.int32)
    nxt = 0
    for i, (k, v) in enumerate(zip(k_seqs, v_seqs)):
        L = k.shape[0]
        for p in range((L + PAGE - 1) // PAGE):
            page = order[nxt]
            nxt += 1
            pt[i, p] = page
            n = min(PAGE, L - p * PAGE)
            kt = torch.zeros(hkv, PAGE, HD, dtype=torch.bfloat16, device=device)
            vt = torch.zeros_like(kt)
            kt[:, :n] = k[p * PAGE:p * PAGE + n].transpose(0, 1)
            vt[:, :n] = v[p * PAGE:p * PAGE + n].transpose(0, 1)
            pool[page, :, 0] = pack_tile(kt)
            pool[page, :, 1] = pack_tile(vt)
    return pool, pt.to(device), max_pages


# ---- long positions -------------------------------------------------------------------------
MAX_POS = 32768                   # the longest window the engine serves
MAX_PAGES = MAX_POS // PAGE + 1   # the engine's page-table width: 2,049 entries
# positions every long-position test includes: each end of the first splits, 16k and the last
EDGE_POSITIONS = (0, 4095, 4096, 8191, 8192, 16384, 32767)


def long_positions(M, n_slots, seed):
    """M tokens over n_slots slots (token i in slot i % n_slots) at positions distinct per slot,
    drawn from [0, 32,768); every slot with at least 7 tokens holds all of EDGE_POSITIONS, at
    shuffled token indices.  -> (tok_slot, tok_pos) int64 on the CPU."""
    g = torch.Generator().manual_seed(seed)
    edges = torch.tensor(EDGE_POSITIONS)
    tok_slot = torch.arange(M) % n_slots
    tok_pos = torch.empty(M, dtype=torch.long)
    for s in range(n_slots):
        idx = (tok_slot == s).nonzero().flatten()
        rest = torch.randperm(MAX_POS, generator=g)
        pos = torch.cat([edges, rest[~torch.isin(rest, edges)]])[:len(idx)]
        tok_pos[idx] = pos[torch.randperm(len(idx), generator=g)]
    return tok_slot, tok_pos


def sparse_page_table(tok_slot, tok_pos, n_slots, seed, spare=16):
    """The engine's [n_slots, 2,049] page table over a pool holding only the pages the tokens
    touch (shuffled ids) and `spare` pages nothing maps; every other entry points at one
    sentinel page, which no write may reach.  -> (page table int32 cpu, num_pages, sentinel)."""
    g = torch.Generator().manual_seed(seed)
    used = torch.unique(tok_slot * MAX_PAGES + tok_pos // PAGE)
    num_pages = len(used) + 1 + spare
    ids = torch.randperm(num_pages, generator=g).to(torch.int32)
    sentinel = int(ids[-1])
    pt = torch.full((n_slots, MAX_PAGES), sentinel, dtype=torch.int32)
    pt.view(-1)[used] = ids[:len(used)]
    return pt, num_pages, sentinel
