#!/usr/bin/env python
"""evict_bench.py -- what eviction costs the compressed host tier (local_capacity_bytes), on one GPU.

  python evict_bench.py [--steps K] [--warmup W] [--tokens T] [--chunk C]

Workload: bench.py's e2e shape (32 layers / 32 heads / 128 dims, 8192-token bf16 KV, chunk 256, synthetic SURVEY 8d data)
through LMCacheEngine.store(tokens, kv, blocking=True) then LMCacheEngine.retrieve(tokens).  Every step stores a FRESH
sequence (new token ids, the same KV), so the two legs below differ in one thing only:
  unbounded  local_capacity_bytes=None: nothing is evicted (the slab grows by one sequence's containers per step)
  evicting   local_capacity_bytes = 2.5 sequences' containers: from the third store on, every store evicts about one
             sequence (the tails of the coldest chains) on the store worker before it lands its waves
The legs alternate step by step after their warm-ups.  Wall clock of the newest sequence's store and retrieve; for the
evicting leg also the time the store worker spent making room -- choosing and retiring victims, waiting for their
uploads, allocating the blocks (`make_room_ms`), the chunks evicted per
step, the slab bytes reserved, and a bit-exact parity spot check of the last retrieve against the reference decode.

Prints one JSON line.  Writes nothing into the tree.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--tokens", type=int, default=8192)
    ap.add_argument("--chunk", type=int, default=256)
    args = ap.parse_args()
    import torch

    import __graft_entry__ as ge
    ge.build_cuda()
    import bench
    from lmcache_b200 import _native as N
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.codec import PinnedBuffer
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    T, cs = args.tokens, args.chunk
    kv = bench.synth_kv_torch(T, dev, 1236, "kv8d")                 # [L,2,T,H,D], bench.py's e2e data
    kv_tuple = tuple((kv[l, 0], kv[l, 1]) for l in range(kv.shape[0]))
    meta = LMCacheEngineMetadata(bench.MODEL, 1, 0, "vllm", "bfloat16")
    lib = N.lib()
    cur = torch.cuda.current_stream()
    digest = PinnedBuffer(4096)
    g = torch.Generator(device=dev).manual_seed(11)

    def engine_for(capacity):
        cfg = LMCacheEngineConfig.from_legacy(chunk_size=cs, backend="cpu", local_serde="cachegen",
                                              local_capacity_bytes=capacity)
        return LMCacheEngine(cfg, meta)

    def one_step(engine, keep=False):
        tokens = torch.randint(0, 32000, (T,), device=dev, generator=g)
        cur.synchronize()
        be = engine.engine_
        ev0, ms0 = be.evicted, evict_s[0]
        t0 = time.perf_counter()
        engine.store(tokens, kv_tuple, skip_existing=False, blocking=True)
        t1 = time.perf_counter()
        ret, mask = engine.retrieve(tokens)
        N.check(lib.b200kv_copy_async(digest.host_ptr, ret[0][0].data_ptr(), 4096, cur.cuda_stream))
        cur.synchronize()
        t2 = time.perf_counter()
        assert int(mask.sum()) == T
        return t1 - t0, t2 - t1, be.evicted - ev0, evict_s[0] - ms0, ret if keep else None

    # the time the store worker spends making room for each wave (LMCLocalCompressedBackend._make_room)
    evict_s = [0.0]

    def timed(orig):
        def f(*a):
            t = time.perf_counter()
            try:
                return orig(*a)
            finally:
                evict_s[0] += time.perf_counter() - t
        return f

    free = engine_for(None)
    one_step(free)
    seq_bytes = sum(e.blk.cap for e in free.engine_.dict.values() if e.blk is not None)
    cap = int(2.5 * seq_bytes)
    free.engine_.reserve_host((args.warmup + args.steps + 2) * seq_bytes)
    bounded = engine_for(cap)
    bounded.engine_.reserve_host(cap)
    bounded.engine_._make_room = timed(bounded.engine_._make_room)
    for _ in range(args.warmup):
        one_step(free)
        one_step(bounded)                                 # from the third store on, every store evicts
    parts = {"unbounded": [], "evicting": []}
    for i in range(args.steps):
        parts["unbounded"].append(one_step(free))
        parts["evicting"].append(one_step(bounded, keep=(i == args.steps - 1)))
    ret = parts["evicting"][-1][4]
    out = torch.stack([torch.stack((k, v)) for k, v in ret])
    parity = bench.parity_spot_check(kv, out, cs)
    del out, ret

    def summary(p):
        n = len(p)
        return {"store_ms": round(1e3 * sum(x[0] for x in p) / n, 2),
                "store_ms_each": [round(1e3 * x[0], 2) for x in p],
                "retrieve_ms": round(1e3 * sum(x[1] for x in p) / n, 2),
                "retrieve_ms_each": [round(1e3 * x[1], 2) for x in p]}

    ev = summary(parts["evicting"])
    ev.update({"capacity_bytes": cap, "evicted_chunks_per_step": round(sum(x[2] for x in parts["evicting"]) / args.steps, 2),
               "make_room_ms": round(1e3 * sum(x[3] for x in parts["evicting"]) / args.steps, 3),
               "slab_reserved_bytes": bounded.engine_.slab.stats()[1], "host_tier_bytes": bounded.engine_.host_bytes(),
               "parity_spot_check": parity})
    print(json.dumps({"metric": "evicting_store_retrieve_ms", "tokens": T, "chunk": cs, "steps": args.steps,
                      "warmup": args.warmup, "gpu": torch.cuda.get_device_name(dev),
                      "unbounded": summary(parts["unbounded"]), "evicting": ev}))
    bounded.close()
    free.close()
    digest.close()


if __name__ == "__main__":
    main()
