#!/usr/bin/env python
"""layerwise_store_bench.py -- what a layer-by-layer store costs and hides during a prefill step, on one GPU.

  python layerwise_store_bench.py [--steps K] [--warmup W] [--tokens 8192,65536] [--ffn F]
                                  [--local-serde cachegen|lossless] [--dtype bf16|fp16|e4m3] [--raw cpu|cuda]

Model of a prefill step: L = 32 layers, 32 KV heads x 128 dims, bf16, chunk 256, a paged KV cache (block 16, scrambled
slot mapping).  Per layer the forward stream runs a stand-in for the layer's compute -- one [T, 4096] x [4096, F] bf16
GEMM (F = --ffn, default 14336: about one MLP up-projection of a 7-8B model) -- and then writes the layer's K and V rows
into the cache (a scatter of bench.py's synthetic 8192-token KV, repeated for longer sequences).  Two legs alternate in
one process, each on a fresh sequence every step (every chunk is stored):
  store_paged   the whole forward, then LMCacheEngine.store_paged(blocking=False) on the forward stream
  layerwise     store_paged_layerwise before the forward, save_layer(l) after each layer's write, finish() at the end
Per leg, from CUDA events on the forward stream (start = before layer 0's GEMM):
  step_ms       start -> the forward stream's end (after the store's enqueue / finish())
  fwd_ms        start -> the last layer's write (the forward itself: the layer-wise encode shares SMs with it)
  store_tail_ms the last layer's write -> the step's end: what the store adds behind the forward
  landed_ms     start -> every container in host memory (host clock until a retrieve of the keys returns)
  call_ms       host time of the store_paged / store_paged_layerwise call (the hash chain and the skip_existing scan)
A forward without any store is timed too (bare_fwd_ms), so the store's slowdown of the forward is fwd_ms - bare_fwd_ms.
Containers of both legs are compared through digests of their bytes after the timed steps (same tokens, same KV), over
the chunks both legs hold; chunks_landed says how many each leg holds (a layer-wise store keeps the prefix of chunks that
fit its device arena, LMCACHE_B200_LAYERWISE_STORE_MB).  --local-serde lossless stores lossless containers (versions 5
and 6) instead of CacheGen ones, --dtype fp16 keeps an fp16 KV cache; the JSON line names them when they are not the
defaults.  --raw cpu / --raw cuda store into a raw tier instead (local_device "cpu" / "cuda" without a serde: chunk
blobs packed one layer at a time), with 8 of the 32 KV heads (a GQA shape: 65536 tokens of raw blobs fit the card) and
--dtype e4m3 for an FP8 E4M3 cache; a raw tier is unbounded, so each step's blobs are dropped after it, and
peak_hbm_mb is the step's peak of allocated device memory above what was allocated at its start.  Prints one JSON line.
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


def _gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def _container_digests(engine, keys):
    """sha256 of every chunk's container, None for a chunk the tier does not hold"""
    out = []
    for k in keys:
        e = engine.engine_.dict[k]
        e.ready.wait()
        out.append(None if e.rec is None else hashlib.sha256(bytes(e.rec.blk.view())[:e.rec.nbytes]).hexdigest())
    return out


def _raw_digests(engine, keys):
    """sha256 of every chunk's raw blob, None for a chunk the tier does not hold"""
    import torch

    from lmcache_b200.storage_backend.local_backend import _HostEntry
    out = []
    for k in keys:
        v = engine.engine_.dict.get(k)
        if isinstance(v, _HostEntry):
            v.wait()
            v = v.host
        out.append(None if v is None else hashlib.sha256(v.contiguous().view(-1).view(torch.uint8).cpu().numpy()).hexdigest())
    return out


def run(T, steps, warmup, ffn, serde="cachegen", dt="bf16", raw=None):
    import torch

    import bench
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    L, H, D, cs, bs = 32, 32 if raw is None else 8, 128, 256, 16
    dev = torch.device("cuda", 0)
    dtype = {"fp16": torch.float16, "bf16": torch.bfloat16, "e4m3": torch.float8_e4m3fn}[dt]
    base = bench.synth_kv_torch(min(T, 8192), dev, seed=0)[:, :, :, :H].to(dtype)  # SURVEY 8d data, as bench.py's headline
    reps = -(-T // base.shape[2])
    nblk = T // bs + 8
    try:
        caches = [(torch.zeros((nblk, bs, H, D), dtype=dtype, device=dev),
                   torch.zeros((nblk, bs, H, D), dtype=dtype, device=dev)) for _ in range(L)]
        x = torch.randn((T, 4096), dtype=torch.bfloat16, device=dev)
        w = torch.randn((4096, ffn), dtype=torch.bfloat16, device=dev) * 0.01
    except torch.cuda.OutOfMemoryError:
        return {"tokens": T, "skipped": "does not fit on the card"}
    slots = torch.randperm(nblk * bs, device=dev)[:T]
    meta = LMCacheEngineMetadata("lmsys/longchat-7b-16k", 1, 0, "vllm", "float16" if dt == "fp16" else "bfloat16")
    # a fresh sequence per step: the tier is bounded (8 GiB), so older sequences are evicted
    def new_engine(capacity=None):
        if raw is not None:
            return LMCacheEngine(LMCacheEngineConfig(cs, raw, None, None, False, False, None), meta)
        return LMCacheEngine(LMCacheEngineConfig.from_legacy(chunk_size=cs, backend="cpu", local_serde=serde,
                                                             local_capacity_bytes=capacity), meta)
    eng = new_engine(8 << 30)
    fwd = torch.cuda.current_stream()

    def layer(l):
        torch.mm(x, w)
        for kv in (0, 1):
            src = base[l, kv].repeat(reps, 1, 1)[:T] if reps > 1 else base[l, kv][:T]
            caches[l][kv].view(-1, H, D)[slots] = src

    def step(mode, seq):
        tokens = torch.arange(T, device=dev) + seq * T
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        mem0 = torch.cuda.memory_allocated()
        t0 = time.perf_counter()
        ev[0].record(fwd)
        call = 0.0
        h = None
        if mode == "layerwise":
            c0 = time.perf_counter()
            h = eng.store_paged_layerwise(tokens, caches, slots)
            call = time.perf_counter() - c0
        for l in range(L):
            layer(l)
            if h is not None:
                h.save_layer(l)
        ev[1].record(fwd)
        if mode == "store_paged":
            c0 = time.perf_counter()
            eng.store_paged(tokens, caches, slots, blocking=False)
            call = time.perf_counter() - c0
        elif h is not None:
            h.finish()
        ev[2].record(fwd)
        held = 0
        if mode != "bare" and raw is not None:
            for k in [eng._make_key(d, "vllm") for d in eng._prefix_hash(tokens)]:
                e = eng.engine_.dict.get(k)
                if e is not None and hasattr(e, "wait"):
                    e.wait()                         # the entry's last device->host copy
                held += e is not None
            torch.cuda.current_stream().synchronize()
        elif mode != "bare":
            eng.retrieve(tokens[:1])                 # waits for the landing of chunk 0 ...
            for k in [eng._make_key(d, "vllm") for d in eng._prefix_hash(tokens)]:
                e = eng.engine_.dict[k]
                e.ready.wait()                       # ... and of every other chunk
                held += e.error is None and e.rec is not None
        landed = time.perf_counter() - t0
        torch.cuda.synchronize()
        peak = (torch.cuda.max_memory_allocated() - mem0) / 2 ** 20
        if raw is not None:
            eng.engine_.dict.clear()                 # unbounded tier: the next step's sequence is a fresh one
        return {"step_ms": ev[0].elapsed_time(ev[2]), "fwd_ms": ev[0].elapsed_time(ev[1]),
                "store_tail_ms": ev[1].elapsed_time(ev[2]), "landed_ms": landed * 1e3, "call_ms": call * 1e3,
                "chunks_held": held, "peak_hbm_mb": round(peak, 1)}, tokens

    res = {m: [] for m in ("bare", "store_paged", "layerwise")}
    seq = 1
    for i in range(warmup + steps):
        for m in ("bare", "store_paged", "layerwise") if i % 2 == 0 else ("layerwise", "store_paged", "bare"):
            r, _ = step(m, seq)
            seq += 1
            if i >= warmup:
                res[m].append(r)
    # equality of the legs: the same tokens and KV stored by both, compared by container digests
    digests = []
    for m in ("store_paged", "layerwise"):
        e2 = new_engine()
        eng, keep = e2, eng
        tokens = torch.arange(T, device=dev) + 10 ** 7
        if m == "store_paged":
            for l in range(L):
                layer(l)
            eng.store_paged(tokens, caches, slots)
        else:
            h = eng.store_paged_layerwise(tokens, caches, slots)
            for l in range(L):
                layer(l)
                h.save_layer(l)
            h.finish()
        keys = [eng._make_key(d, "vllm") for d in eng._prefix_hash(tokens)]
        digests.append(_container_digests(eng, keys) if raw is None else _raw_digests(eng, keys))
        e2.close()
        eng = keep
    eng.close()

    def summ(rows):
        return {k: round(statistics.median(r[k] for r in rows), 3) for k in rows[0]} if rows else {}
    out = {"tokens": T, "runs_per_leg": steps, "bare_fwd_ms": summ(res["bare"]).get("fwd_ms"),
           "store_paged": summ(res["store_paged"]), "layerwise": summ(res["layerwise"]),
           "chunks": -(-T // cs), "chunks_landed": [sum(d is not None for d in ds) for ds in digests],
           "containers_equal": all(a == b for a, b in zip(*digests) if a is not None and b is not None)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--tokens", default="8192,65536")
    ap.add_argument("--ffn", type=int, default=14336)
    ap.add_argument("--local-serde", choices=("cachegen", "lossless"), default="cachegen")
    ap.add_argument("--dtype", choices=("bf16", "fp16", "e4m3"), default="bf16")
    ap.add_argument("--raw", choices=("cpu", "cuda"), default=None)
    a = ap.parse_args()
    if a.dtype == "e4m3" and a.raw is None and a.local_serde == "cachegen":
        raise SystemExit("--dtype e4m3 needs --raw or --local-serde lossless: CacheGen codes 16-bit KV only")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("layerwise_store_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    results = [run(int(t), a.steps, a.warmup, a.ffn, a.local_serde, a.dtype, a.raw) for t in a.tokens.split(",")]
    out = {"bench": "layerwise_store", "gpu": _gpu_info(), "ffn": a.ffn}
    if a.raw is not None:
        out.update(raw=a.raw, dtype=a.dtype, kv_heads=8)
    elif a.local_serde != "cachegen" or a.dtype != "bf16":
        out.update(local_serde=a.local_serde, dtype=a.dtype)
    out.update(arena_budget_mb=int(os.environ.get("LMCACHE_B200_LAYERWISE_STORE_MB", "1024")), results=results)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
