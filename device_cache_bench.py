#!/usr/bin/env python
"""device_cache_bench.py -- what the device level of the compressed host tier (device_cache_bytes) gains, on one GPU.

  python device_cache_bench.py [--steps K] [--warmup W] [--tokens 8192,65536] [--chunk C]

Workload: bench.py's e2e shape (32 layers / 32 heads / 128 dims, bf16 KV, chunk 256, synthetic SURVEY 8d data) through
LMCacheEngine.  Two engines live in one process and alternate step by step after their warm-ups:
  host    local_device="cpu", local_serde="cachegen": every retrieve uploads its containers over PCIe
  level   the same plus device_cache_bytes = 2 sequences' containers: every retrieve of the stored sequence is all hits
Per leg and size: retrieve() wall clock of the stored sequence; retrieve_layerwise's ready[0] and ready[L-1] (CUDA event
time from the call's start); store() of a fresh sequence (the level adds a device-to-device copy per container); and,
for the level, one retrieve right after a restart-like drop of every device copy (a promotion).  The retrieved KV's
digest must be equal across legs.  Prints one JSON line with the GPU's name and power limit.  Writes nothing into the
tree.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def _power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--tokens", default="8192,65536")
    ap.add_argument("--chunk", type=int, default=256)
    args = ap.parse_args()
    import torch

    import __graft_entry__ as ge
    ge.build_cuda()
    import bench
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    from lmcache_b200.slab import block_bytes

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cs = args.chunk
    meta = LMCacheEngineMetadata(bench.MODEL, 1, 0, "vllm", "bfloat16")
    cur = torch.cuda.current_stream()
    result = {"metric": "device_cache_retrieve_ms", "chunk": cs, "steps": args.steps, "warmup": args.warmup,
              "gpu": torch.cuda.get_device_name(dev), "power_limit": _power_limit(), "sizes": {}}

    def digest(ret):
        return int(sum(int(t.view(torch.int16).sum(dtype=torch.int64)) for kv in ret for t in kv))

    for T in [int(t) for t in args.tokens.split(",")]:
        kv = bench.synth_kv_torch(T, dev, 1236, "kv8d")
        kv_tuple = tuple((kv[l, 0], kv[l, 1]) for l in range(kv.shape[0]))
        g = torch.Generator(device=dev).manual_seed(12)

        def fresh():
            return torch.randint(0, 32000, (T,), device=dev, generator=g)

        def engine_for(level_bytes):
            cfg = LMCacheEngineConfig.from_legacy(chunk_size=cs, backend="cpu", local_serde="cachegen",
                                                  device_cache_bytes=level_bytes)
            return LMCacheEngine(cfg, meta)

        host = engine_for(None)
        tokens = fresh()
        host.store(tokens, kv_tuple)
        seq = sum(block_bytes(e.nbytes) for e in host.engine_.dict.values())
        level = engine_for(2 * seq)
        level.engine_.reserve_device()
        level.store(tokens, kv_tuple)
        steps = args.warmup + args.steps
        host.engine_.reserve_host((steps + 3) * seq)
        level.engine_.reserve_host((steps + 3) * seq)
        legs = {"host": host, "level": level}
        runs = {name: {"retrieve_ms": [], "ready0_ms": [], "readyL_ms": [], "store_ms": []} for name in legs}
        digests = {}

        def one(name, eng):
            r = runs[name]
            cur.synchronize()
            t0 = time.perf_counter()
            ret, mask = eng.retrieve(tokens)
            cur.synchronize()
            r["retrieve_ms"].append(1e3 * (time.perf_counter() - t0))
            assert int(mask.sum()) == T
            digests.setdefault(name, set()).add(digest(ret))
            del ret
            start = torch.cuda.Event(enable_timing=True)
            start.record(cur)
            lw = eng.retrieve_layerwise(tokens)
            lw.synchronize()
            n = lw.num_layers
            r["ready0_ms"].append(start.elapsed_time(lw._upload.ready(0)))
            r["readyL_ms"].append(start.elapsed_time(lw._upload.ready(n - 1)))
            digests[name].add(digest(lw.kv))
            del lw
            tok = fresh()
            cur.synchronize()
            t0 = time.perf_counter()
            eng.store(tok, kv_tuple, skip_existing=False, blocking=True)
            r["store_ms"].append(1e3 * (time.perf_counter() - t0))

        for i in range(steps):
            for name, eng in legs.items():
                one(name, eng)
            if i == args.warmup - 1:
                for r in runs.values():
                    for v in r.values():
                        v.clear()
                level.engine_._dcache.hits = 0
        # one promoted retrieve: drop every device copy, then retrieve (uploads and promotes), then all hits again
        be = level.engine_
        cur.synchronize()
        with be.update_lock:
            for e in be.dict.values():
                if e.rec is not None and e.rec.dev is not None:
                    be._dcache.drop(e)
        p0 = be._dcache.promotions
        t0 = time.perf_counter()
        ret, _ = level.retrieve(tokens)
        cur.synchronize()
        promoted_ms = 1e3 * (time.perf_counter() - t0)
        digests["level"].add(digest(ret))
        del ret
        out = {name: {k: round(statistics.median(v), 3) for k, v in r.items()} for name, r in runs.items()}
        out["level"]["promoted_retrieve_ms"] = round(promoted_ms, 3)
        out["level"]["promoted_chunks"] = be._dcache.promotions - p0
        out["level"]["device_cache"] = be.device_cache_stats()
        out["container_bytes_per_sequence"] = seq
        out["digest_equal"] = len(digests["host"] | digests["level"]) == 1
        result["sizes"][str(T)] = out
        host.close()
        level.close()
        del kv, kv_tuple
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
