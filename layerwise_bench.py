#!/usr/bin/env python
"""layerwise_bench.py -- what a layer-by-layer retrieve buys on the compressed host tier, on one GPU.

  python layerwise_bench.py [--steps K] [--warmup W] [--tokens 8192,65536] [--chunk C] [--cold N]
                            [--raw cpu|cuda] [--dtype bf16|e4m3]

Workload: bench.py's e2e shape (32 layers / 32 heads / 128 dims, bf16 KV, chunk 256, synthetic SURVEY 8d data), stored
once through LMCacheEngine.store into the compressed host tier, then retrieved again and again, alternating
  retrieve            LMCacheEngine.retrieve(tokens): chunk-major waves, the whole blob is there at the end
  retrieve_layerwise  LMCacheEngine.retrieve_layerwise(tokens): layer-major upload + decode, one ready event per layer
Per leg, from CUDA events (the start event is recorded on the caller's stream right before the call):
  total_ms            start -> the end of the retrieve (retrieve: an event after the call; layer-wise: ready[L-1])
  ready*_ms           layer-wise only: start -> ready[0], ready[L/2], ready[L-1] (the handle's per-layer events)
  layer_ms            layer-wise only: ready[l+1] - ready[l], mean and max over the layers
  call_ms             host wall clock of the call itself (layer-wise: until the hit count is known)
  enqueue_ms          layer-wise only: host time the worker spent enqueueing the fixed sections + plan, and per layer
                      (mean and max): when it is not below layer_ms, the host paces the layers
The layer-wise leg runs warm (the same sequence again and again) and cold (`--cold` sequences stored before the timed
loop and retrieved once each).  The last warm step's KV of the two legs is compared through per-layer digests of the bit
patterns.  Sequences longer than 8192 tokens repeat bench.py's 8192-token KV.  A token count that does not fit on the card
is reported as skipped.  --raw cpu / --raw cuda measure the raw tiers instead (local_device "cpu" / "cuda" without a
serde: chunk blobs copied and unpacked one layer at a time); they keep 8 of the 32 KV heads (a GQA shape, so that 65536
tokens of raw blobs and the retrieved KV fit the card), and --dtype e4m3 stores an FP8 E4M3 KV.  Prints one JSON line.
Writes nothing into the tree.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def _power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def _digest(kv, w_cache={}):
    """per-layer position-weighted sums of the K and V bit patterns: equal KV gives equal digests; both legs' blobs never
    need to be alive at once"""
    import torch
    out = []
    for k, v in kv:
        for x in (k, v):
            b = x.contiguous().view(-1).view(torch.int16).to(torch.int32)
            w = w_cache.get(b.numel())
            if w is None:
                w = w_cache[b.numel()] = torch.arange(b.numel(), device=b.device, dtype=torch.int32) % 65521 + 1
            out.append(torch.stack((b.sum(dtype=torch.int64), (b * w).sum(dtype=torch.int64))))
    return torch.stack(out).cpu()


def run(T, cs, steps, warmup, cold_steps, raw=None, dt="bf16"):
    import torch

    import bench
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata

    dev = torch.device("cuda", 0)
    meta = LMCacheEngineMetadata(bench.MODEL, 1, 0, "vllm", "bfloat16")
    if raw is None:
        cfg = LMCacheEngineConfig.from_legacy(chunk_size=cs, backend="cpu", local_serde="cachegen")
    else:
        cfg = LMCacheEngineConfig(cs, raw, None, None, False, False, None)
    engine = LMCacheEngine(cfg, meta)
    g = torch.Generator(device=dev).manual_seed(3)
    try:
        tokens = torch.randint(0, 32000, (T,), device=dev, generator=g)
        # bench.py's 8192-token KV, repeated along the tokens for longer sequences (generating 65536 tokens at once needs
        # more memory than the card has): same statistics, same bytes per chunk
        base_T = min(T, 8192)
        kv = bench.synth_kv_torch(base_T, dev, 1236, "kv8d")                # [L,2,t,H,D]
        if raw is not None:
            kv = kv[:, :, :, :8].contiguous()
            if dt == "e4m3":
                kv = kv.to(torch.float8_e4m3fn)
        if T > base_T:
            kv = torch.cat([kv] * (T // base_T), dim=2)
        L = kv.shape[0]
        kv_tuple = tuple((kv[l, 0], kv[l, 1]) for l in range(L))
        engine.store(tokens, kv_tuple, blocking=True)
        cold_tokens = []
        for _ in range(cold_steps):                    # sequences stored now, retrieved once each, later
            t = torch.randint(0, 32000, (T,), device=dev, generator=g)
            engine.store(t, kv_tuple, blocking=True)
            cold_tokens.append(t)
        del kv, kv_tuple
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        cur = torch.cuda.current_stream()
        host_bytes = engine.engine_.host_bytes() // (1 + cold_steps) if raw is None else None

        def plain():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record(cur)
            t0 = time.perf_counter()
            ret, mask = engine.retrieve(tokens)
            t1 = time.perf_counter()
            e.record(cur)
            e.synchronize()
            assert int(mask.sum()) == T
            return {"total_ms": s.elapsed_time(e), "call_ms": 1e3 * (t1 - t0)}, ret

        def layerwise(tok):
            s = torch.cuda.Event(enable_timing=True)
            s.record(cur)
            t0 = time.perf_counter()
            r = engine.retrieve_layerwise(tok)
            t1 = time.perf_counter()
            r.synchronize()
            assert int(r.ret_mask.sum()) == T
            ready = [r._upload.ready(l) for l in range(L)]          # timing events, recorded after each layer's decode
            at = [s.elapsed_time(e) for e in ready]
            step = [b - a for a, b in zip(at, at[1:])]
            enq = r._upload.enqueue_s
            return {"total_ms": at[-1], "call_ms": 1e3 * (t1 - t0), "ready0_ms": at[0], "ready_mid_ms": at[L // 2],
                    "ready_last_ms": at[-1], "layer_ms_mean": sum(step) / len(step), "layer_ms_max": max(step),
                    "enqueue_plan_ms": 1e3 * enq[0], "enqueue_layer_ms_mean": 1e3 * sum(enq[1:]) / L,
                    "enqueue_layer_ms_max": 1e3 * max(enq[1:])}, r

        for _ in range(warmup):
            plain()
            layerwise(tokens)
        legs = {"retrieve": [], "retrieve_layerwise": [], "retrieve_layerwise_cold": []}
        equal = True
        for i in range(steps):
            m, out = plain()
            legs["retrieve"].append(m)
            want = _digest(out) if i == steps - 1 else None
            del out
            m, out = layerwise(tokens)
            legs["retrieve_layerwise"].append(m)
            if want is not None:
                equal = torch.equal(want, _digest(out.kv))
            del out
        for t in cold_tokens:
            m, out = layerwise(t)
            legs["retrieve_layerwise_cold"].append(m)
            del out

        def summary(p):
            return {k: round(sum(x[k] for x in p) / len(p), 3) for k in p[0]} | \
                {"total_ms_each": [round(x["total_ms"], 3) for x in p]}

        res = {"tokens": T, "container_bytes": host_bytes, "bit_equal": bool(equal)}
        for k, p in legs.items():
            if p:
                res[k] = summary(p)
        a, b = res["retrieve"]["total_ms"], res["retrieve_layerwise"]["total_ms"]
        res["layerwise_total_vs_retrieve"] = round(b / a - 1.0, 4)
        return res
    finally:
        engine.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--tokens", type=str, default="8192,65536")
    ap.add_argument("--chunk", type=int, default=256)
    ap.add_argument("--cold", type=int, default=3)
    ap.add_argument("--raw", choices=("cpu", "cuda"), default=None)
    ap.add_argument("--dtype", choices=("bf16", "e4m3"), default="bf16")
    args = ap.parse_args()
    if args.dtype != "bf16" and args.raw is None:
        raise SystemExit("--dtype e4m3 needs --raw: CacheGen codes 16-bit KV only")
    import torch

    import __graft_entry__ as ge
    ge.build_cuda()
    torch.cuda.set_device(0)
    results = []
    for T in (int(x) for x in args.tokens.split(",")):
        try:
            results.append(run(T, args.chunk, args.steps, args.warmup, args.cold, args.raw, args.dtype))
        except torch.cuda.OutOfMemoryError:
            results.append({"tokens": T, "skipped": "does not fit on the card"})
        torch.cuda.empty_cache()
    out = {"metric": "layerwise_retrieve_ms", "chunk": args.chunk, "steps": args.steps, "warmup": args.warmup,
           "gpu": torch.cuda.get_device_name(0), "power_limit": _power_limit()}
    if args.raw is not None:
        out.update(raw=args.raw, dtype=args.dtype, kv_heads=8)
    out["results"] = results
    print(json.dumps(out))


if __name__ == "__main__":
    main()
