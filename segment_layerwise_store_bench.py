#!/usr/bin/env python
"""segment_layerwise_store_bench.py -- a RAG prompt's documents stored from inside it, layer by layer, on one GPU.

  python segment_layerwise_store_bench.py [--steps K] [--warmup W] [--tiers cpu,cuda,host-cachegen,host-lossless]
                                          [--ffn F]

Workload (segment_bench.py's): L = 32 layers, 8 KV heads x 128 dims, bf16, chunk 256, a paged KV cache (block 16,
scrambled slot mapping) holding eight 2048-token documents back to back and a 512-token question (16896 tokens); the
first document is at token 0 and is stored under its prefix keys, the other seven are turned back by -start.  The
forward pass is layerwise_store_bench.py's stand-in: per layer one [T, 4096] x [4096, F] bf16 GEMM (F = --ffn, default
14336), then the layer's K and V rows written into the cache.  Two legs alternate in one process, each on a fresh
sequence every step (every chunk is stored):
  whole       the forward, then LMCacheEngine.store_paged_segments on the forward stream
  layerwise   store_paged_segments_layerwise before the forward, save_layer(l) after each layer's write, finish()
Per leg, from CUDA events on the forward stream, as layerwise_store_bench.py defines them: step_ms (start -> the end of
the store's call or finish()), fwd_ms (start -> the last layer's write), store_tail_ms (the last layer's write -> the
step's end), and call_ms (host time of the store_paged_segments / store_paged_segments_layerwise call).  Medians.
gather: one b200kv_pack_chunks_layers_rope launch of one layer of the seven documents (CUDA events over 200
launches), with its bytes (each staged element read once and written once) over 3.35 TB/s, the H100 SXM's HBM3 data
sheet figure.  After the timed steps both legs store one more sequence into fresh engines and their stored bytes are
compared by digest (containers on the CacheGen and lossless tiers, raw blobs on the raw tiers).  A layer-wise store
into a compressed tier keeps the chunks that fit LMCACHE_B200_LAYERWISE_STORE_MB (default 1024; this workload's 64
chunks of 32 MB of raw KV need more for all of them to fit), so chunks_stored gives each leg's count and
equal_where_both_hold compares the chunks both hold.  Prints one JSON line with the card's name and power limit.
Writes nothing into the tree.
"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

L, H, D, CS, BS = 32, 8, 128, 256, 16
DOC, N_DOCS, QUESTION = 2048, 8, 512
T = N_DOCS * DOC + QUESTION
SEGMENTS = [(i * DOC, (i + 1) * DOC) for i in range(N_DOCS)]


def _gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def _config(tier):
    from lmcache_b200.config import LMCacheEngineConfig
    if tier in ("cpu", "cuda"):
        return LMCacheEngineConfig(CS, tier, None, None, False, False, None)
    return LMCacheEngineConfig.from_legacy(chunk_size=CS, backend="cpu", local_serde=tier.split("-")[1],
                                           local_capacity_bytes=8 << 30)


def _keys(eng, tokens):
    """every key a store of SEGMENTS of `tokens` writes: prefix keys of the first document, derived keys of the rest"""
    out = [eng._make_key(h, "vllm") for h in eng._prefix_hash(tokens[:DOC])]
    for a, b in SEGMENTS[1:]:
        out += [eng._derived_key(h, "vllm") for h in eng._prefix_hash(tokens[a:b])]
    return out


def _digests(eng, keys):
    """sha256 of what the tier holds under each key (a container, or a raw blob), None for a chunk it does not hold"""
    import torch
    torch.cuda.synchronize()
    out = []
    for k in keys:
        e = eng.engine_.dict.get(k)
        if e is None:
            out.append(None)
        elif hasattr(e, "ready"):
            e.ready.wait()
            out.append(None if e.rec is None else hashlib.sha256(bytes(e.rec.blk.view())[:e.rec.nbytes]).hexdigest())
        else:
            if hasattr(e, "wait"):
                e.wait()
                e = e.host
            out.append(hashlib.sha256(e.contiguous().view(-1).view(torch.uint8).cpu().numpy()).hexdigest())
    return out


def gather_kernel(caches, slots, reps=200):
    """one layer's b200kv_pack_chunks_layers_rope over the seven documents inside the prompt"""
    import torch
    from lmcache_b200.codec import KvView
    from lmcache_b200.rope import RopeSpec, StagedGather, plan_segment_store, plan_segments, pack_rope_layers
    plans = plan_segments(T, SEGMENTS[1:], CS)
    runs, rows, _, shifts = plan_segment_store(plans, [(0, 0)] * len(plans), CS)
    view = KvView.from_paged(caches, slots)
    side = torch.cuda.current_stream()
    g = StagedGather(view, runs, shifts, "vllm", False, RopeSpec.from_base(D, 10000.0), side, KvView.blob_shape)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def launch(l):
        pack_rope_layers(view, g.ptrs.data_ptr() + 8 * g.R * l, g.arrays, g.chunk_tokens, l, l + 1, g.table, g.rope,
                         side)
    for l in range(L):
        launch(l)
    ev[0].record(side)
    for i in range(reps):
        launch(i % L)
    ev[1].record(side)
    torch.cuda.synchronize()
    us = ev[0].elapsed_time(ev[1]) * 1e3 / reps
    nbytes = 2 * len(rows) * 2 * H * D * 2                  # every staged element of one layer read once, written once
    return {"tokens_staged": len(rows), "layer_us": round(us, 2), "bytes_per_layer": nbytes,
            "share_of_3350_GBps": round(nbytes / (us * 1e-6) / 3.35e12, 3)}


def run_tier(tier, steps, warmup, ffn, caches, slots, base, x, w):
    import torch
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineMetadata
    from lmcache_b200.rope import RopeSpec
    dev = slots.device
    spec = RopeSpec.from_base(D, 10000.0)
    meta = LMCacheEngineMetadata("lmsys/longchat-7b-16k", 1, 0, "vllm", "bfloat16")
    fwd = torch.cuda.current_stream()
    reps = -(-T // base.shape[2])

    def layer(l):
        torch.mm(x, w)
        for kv in (0, 1):
            src = base[l, kv].repeat(reps, 1, 1)[:T] if reps > 1 else base[l, kv][:T]
            caches[l][kv].view(-1, H, D)[slots] = src

    def step(eng, mode, tokens):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        torch.cuda.synchronize()
        ev[0].record(fwd)
        call, h = 0.0, None
        if mode == "layerwise":
            c0 = time.perf_counter()
            h = eng.store_paged_segments_layerwise(tokens, caches, slots, SEGMENTS, spec)
            call = time.perf_counter() - c0
        for l in range(L):
            layer(l)
            if h is not None:
                h.save_layer(l)
        ev[1].record(fwd)
        if mode == "whole":
            c0 = time.perf_counter()
            eng.store_paged_segments(tokens, caches, slots, SEGMENTS, spec)
            call = time.perf_counter() - c0
        else:
            h.finish()
        ev[2].record(fwd)
        torch.cuda.synchronize()
        return {"step_ms": ev[0].elapsed_time(ev[2]), "fwd_ms": ev[0].elapsed_time(ev[1]),
                "store_tail_ms": ev[1].elapsed_time(ev[2]), "call_ms": call * 1e3}

    eng = LMCacheEngine(_config(tier), meta)
    res = {"whole": [], "layerwise": []}
    seq = 1
    for i in range(warmup + steps):
        for m in ("whole", "layerwise") if i % 2 == 0 else ("layerwise", "whole"):
            r = step(eng, m, torch.arange(T, device=dev) + seq * T)
            seq += 1
            if tier in ("cpu", "cuda"):
                eng.engine_.dict.clear()             # unbounded raw tier: the next step's sequence is a fresh one
            if i >= warmup:
                res[m].append(r)
    eng.close()
    digests = []
    for m in ("whole", "layerwise"):
        e = LMCacheEngine(_config(tier), meta)
        tokens = torch.arange(T, device=dev) + 10 ** 7
        step(e, m, tokens)
        digests.append(_digests(e, _keys(e, tokens)))
        e.close()

    def summ(rows):
        return {k: round(statistics.median(r[k] for r in rows), 3) for k in rows[0]}
    both = [(a, b) for a, b in zip(*digests) if a is not None and b is not None]
    return {"tier": tier, "runs_per_leg": steps, "whole": summ(res["whole"]), "layerwise": summ(res["layerwise"]),
            "chunks": len(digests[0]), "chunks_stored": [sum(d is not None for d in ds) for ds in digests],
            "stored_bytes_equal": digests[0] == digests[1], "equal_where_both_hold": all(a == b for a, b in both)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ffn", type=int, default=14336)
    ap.add_argument("--tiers", default="cpu,cuda,host-cachegen,host-lossless")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("segment_layerwise_store_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    import bench
    dev = torch.device("cuda", 0)
    base = bench.synth_kv_torch(8192, dev, seed=0)[:, :, :, :H].to(torch.bfloat16)
    nblk = T // BS + 8
    caches = [(torch.zeros((nblk, BS, H, D), dtype=torch.bfloat16, device=dev),
               torch.zeros((nblk, BS, H, D), dtype=torch.bfloat16, device=dev)) for _ in range(L)]
    slots = torch.randperm(nblk * BS, device=dev, generator=torch.Generator(device=dev).manual_seed(1))[:T]
    x = torch.randn((T, 4096), dtype=torch.bfloat16, device=dev)
    w = torch.randn((4096, a.ffn), dtype=torch.bfloat16, device=dev) * 0.01
    out = {"bench": "segment_layerwise_store", "gpu": _gpu_info(), "ffn": a.ffn, "tokens": T,
           "segments": len(SEGMENTS), "arena_budget_mb": int(os.environ.get("LMCACHE_B200_LAYERWISE_STORE_MB", "1024")),
           "gather": gather_kernel(caches, slots),
           "results": [run_tier(t, a.steps, a.warmup, a.ffn, caches, slots, base, x, w) for t in a.tiers.split(",")]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
