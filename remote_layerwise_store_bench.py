#!/usr/bin/env python
"""remote_layerwise_store_bench.py -- the layer-by-layer store on the lm:// remote and hybrid tiers during a prefill step.

  python remote_layerwise_store_bench.py [--steps K] [--warmup W] [--tokens 8192,65536] [--ffn F]
                                         [--serde cachegen|lossless] [--tier remote|hybrid]

The model step is layerwise_store_bench.py's: L = 32 layers, bf16, chunk 256, a paged KV cache (block 16, scrambled slot
mapping), and per layer one [T, 4096] x [4096, F] bf16 GEMM on the forward stream followed by the layer's K and V
writes.  Here the KV has 8 of the 32 heads (a GQA shape), so that 65536 tokens of containers fit the server's memory.
The server is this project's lm:// server on loopback, started and stopped by the bench (b200kv_lm_server_start); with
--tier hybrid the engine also has a page-locked local tier of the same serde (local_device "cpu", 8 GiB), so both parts
keep the same containers and every store is encoded once.  Every leg rewrites one token sequence (skip_existing=False),
so the server holds one sequence.  Legs alternate in one process, the order reversed every other step:
  bare          the forward alone
  store_paged   the forward, then store_paged(blocking=True) -- what finish() ran before the remote and hybrid tiers went
                layer-wise: it returns once the server holds every chunk
  layerwise     store_paged_layerwise before the forward, save_layer(l) after each layer's write, finish() at the end
  store_paged_2enc (--tier hybrid) store_paged with the one-encode rule switched off: each part encodes the store
                itself, the hybrid's path before it encoded once
Per leg, medians over the timed steps:
  step_ms   host clock, from the start (after a device synchronise) to the store's return: the server holds every chunk
  fwd_ms    CUDA events on the forward stream, start -> the last layer's write
  tail_ms   step_ms - fwd_ms: what the store adds behind the forward, sends included
  store_ms  host clock of the store_paged call alone (store_paged legs)
The forward's slowdown by a leg is its fwd_ms - bare fwd_ms.  After the timed steps the containers a store_paged and a
layer-wise store put on the server for the same KV under two token sequences are compared by digest
(containers_equal, over the chunks both hold: a layer-wise store keeps the prefix of chunks that fit its device arena,
LMCACHE_B200_LAYERWISE_STORE_MB, and chunks_on_server says how many each holds).  Prints one JSON line; writes nothing
into the tree.
"""
import argparse
import ctypes
import hashlib
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from layerwise_store_bench import _gpu_info  # noqa: E402


class _Server:
    """this project's lm:// server, in this process, on a loopback port the system picks"""

    def __init__(self):
        from lmcache_b200 import _native as N
        self.lib = N.lib()
        self.h = ctypes.c_void_p()
        N.check(self.lib.b200kv_lm_server_start(b"127.0.0.1", 0, ctypes.byref(self.h)))
        self.url = f"lmn://127.0.0.1:{self.lib.b200kv_lm_server_port(self.h)}"

    def stop(self):
        if self.h is not None:
            self.lib.b200kv_lm_server_stop(self.h)
            self.h = None


def _server_digests(url, eng, tokens):
    from lmcache_b200.storage_backend.connector import CreateConnector
    c = CreateConnector(url)
    try:
        out = []
        for d in eng._prefix_hash(tokens):
            b = c.get(eng._make_key(d, "vllm").to_string())
            out.append(hashlib.sha256(bytes(b)).hexdigest() if b else None)
        return out
    finally:
        c.close()


def run(T, steps, warmup, ffn, serde, tier, url):
    import torch

    import bench
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    from lmcache_b200.storage_backend.hybrid_backend import LMCHybridBackend
    L, H, D, cs, bs = 32, 8, 128, 256, 16
    dev = torch.device("cuda", 0)
    base = bench.synth_kv_torch(min(T, 8192), dev, seed=0)[:, :, :, :H].to(torch.bfloat16)
    reps = -(-T // base.shape[2])
    nblk = T // bs + 8
    caches = [(torch.zeros((nblk, bs, H, D), dtype=torch.bfloat16, device=dev),
               torch.zeros((nblk, bs, H, D), dtype=torch.bfloat16, device=dev)) for _ in range(L)]
    x = torch.randn((T, 4096), dtype=torch.bfloat16, device=dev)
    w = torch.randn((4096, ffn), dtype=torch.bfloat16, device=dev) * 0.01
    slots = torch.randperm(nblk * bs, device=dev)[:T]
    meta = LMCacheEngineMetadata("lmsys/longchat-7b-16k", 1, 0, "vllm", "bfloat16")

    def new_engine():
        if tier == "hybrid":
            cfg = LMCacheEngineConfig(cs, "cpu", url, serde, False, False, serde, 8 << 30)
        else:
            cfg = LMCacheEngineConfig(cs, None, url, serde, False, False)
        return LMCacheEngine(cfg, meta)
    eng = new_engine()
    fwd = torch.cuda.current_stream()
    shares = LMCHybridBackend._shares_containers

    def layer(l):
        torch.mm(x, w)
        for kv in (0, 1):
            src = base[l, kv].repeat(reps, 1, 1)[:T] if reps > 1 else base[l, kv][:T]
            caches[l][kv].view(-1, H, D)[slots] = src

    tokens = torch.arange(T, device=dev)

    def step(mode):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ev[0].record(fwd)
        h = eng.store_paged_layerwise(tokens, caches, slots, skip_existing=False) if mode == "layerwise" else None
        for l in range(L):
            layer(l)
            if h is not None:
                h.save_layer(l)
        ev[1].record(fwd)
        store = 0.0
        if h is not None:
            h.finish()
        elif mode != "bare":
            if mode == "store_paged_2enc":
                LMCHybridBackend._shares_containers = lambda self, chunk_size, view: False
            try:
                c0 = time.perf_counter()
                eng.store_paged(tokens, caches, slots, skip_existing=False, blocking=True)
                store = time.perf_counter() - c0
            finally:
                LMCHybridBackend._shares_containers = shares
        else:
            torch.cuda.synchronize()
        wall = (time.perf_counter() - t0) * 1e3
        torch.cuda.synchronize()
        f = ev[0].elapsed_time(ev[1])
        return {"step_ms": wall, "fwd_ms": f, "tail_ms": wall - f, "store_ms": store * 1e3}

    legs = ["bare", "store_paged", "layerwise"] + (["store_paged_2enc"] if tier == "hybrid" else [])
    res = {m: [] for m in legs}
    for i in range(warmup + steps):
        for m in legs if i % 2 == 0 else legs[::-1]:
            r = step(m)
            if i >= warmup:
                res[m].append(r)
    # equality: the same KV stored by store_paged and by the layer-wise store, under two token sequences
    ta, tb = tokens + 10 ** 7, tokens + 2 * 10 ** 7
    for l in range(L):
        layer(l)
    eng.store_paged(ta, caches, slots)
    h = eng.store_paged_layerwise(tb, caches, slots)
    layered = h._enc is not None
    for l in range(L):
        h.save_layer(l)
    h.finish()
    a, b = _server_digests(url, eng, ta), _server_digests(url, eng, tb)
    eng.close()

    def summ(rows):
        return {k: round(statistics.median(r[k] for r in rows), 3) for k in rows[0]}
    out = {"tokens": T, "runs_per_leg": steps, "layer_wise": layered}
    out.update({m: summ(res[m]) for m in legs})
    out.update(chunks=-(-T // cs), chunks_on_server=[sum(d is not None for d in ds) for ds in (a, b)],
               containers_equal=all(x == y for x, y in zip(a, b) if x is not None and y is not None))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--tokens", default="8192,65536")
    ap.add_argument("--ffn", type=int, default=14336)
    ap.add_argument("--serde", choices=("cachegen", "lossless"), default="cachegen")
    ap.add_argument("--tier", choices=("remote", "hybrid"), default="remote")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("remote_layerwise_store_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    srv = _Server()
    try:
        results = [run(int(t), a.steps, a.warmup, a.ffn, a.serde, a.tier, srv.url) for t in a.tokens.split(",")]
    finally:
        srv.stop()
    print(json.dumps({"bench": "remote_layerwise_store", "gpu": _gpu_info(), "ffn": a.ffn, "serde": a.serde,
                      "tier": a.tier, "kv_heads": 8,
                      "arena_budget_mb": int(os.environ.get("LMCACHE_B200_LAYERWISE_STORE_MB", "1024")),
                      "results": results}))


if __name__ == "__main__":
    main()
