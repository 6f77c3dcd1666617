"""Measure the local tiers end to end: raw `cpu` blobs, the lossless host tier, the CacheGen host tier and the lossless
disk tier (local_serde="lossless" in a temporary directory).

32 layers x 8 KV heads x 128 dims, chunks of 256 tokens, bf16 and fp16, at 8192 and 65536 tokens, on bench.py's kv8d
data and on its high-entropy uniform_signed data.  Per tier: LMCacheEngine.store() and retrieve() wall times around a
device synchronise (medians of --steps after --warmup, a fresh engine per step, its page-locked slab reserved before the
clock starts), the bytes the tier holds, and for the two compressed host tiers the times from the call of
retrieve_layerwise() to the completion of layer 0's and of the last layer's decode (CUDA events).  Every timed lossless
and raw retrieve is compared bit for bit with its input.

Prints the card and its power limit, then one JSON line per measurement.  Writes nothing in the tree."""
import argparse
import json
import shutil
import statistics
import tempfile
import time

import torch

import bench
from lmcache_b200 import _native as N
from lossless_bench import card

MODEL = "lmsys/longchat-7b-16k"
CHUNK = 256
bench.H, bench.C = 8, 8 * bench.D          # 32 layers x 8 KV heads x 128 dims (bench.synth_kv_torch reads these)
TIERS = ("raw_cpu", "lossless_host", "cachegen_host", "lossless_disk")


def _engine(tier: str, dtype: torch.dtype, tmp: str):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    local, serde = {"raw_cpu": ("cpu", None), "lossless_host": ("cpu", "lossless"), "cachegen_host": ("cpu", "cachegen"),
                    "lossless_disk": (tmp + "/", "lossless")}[tier]
    cfg = LMCacheEngineConfig(CHUNK, local, None, None, False, False, serde)
    return LMCacheEngine(cfg, LMCacheEngineMetadata(MODEL, 1, 0, "vllm", str(dtype).replace("torch.", "")))


def _held(eng, tier: str, tmp: str) -> int:
    if tier == "raw_cpu":
        return sum(v.host.numel() * v.host.element_size() for v in eng.engine_.dict.values())
    if tier == "lossless_disk":
        import os
        return sum(os.path.getsize(os.path.join(tmp, f)) for f in os.listdir(tmp))
    return eng.engine_.host_bytes()


def tier_leg(tier: str, tokens: int, dtype: torch.dtype, kind: str, steps: int, warmup: int) -> dict:
    kv = bench.synth_kv_torch(tokens, "cuda", 1, kind).to(dtype)
    pairs = tuple((kv[l, 0], kv[l, 1]) for l in range(kv.shape[0]))
    raw = kv.numel() * 2
    st_ms, rt_ms, l0_ms, ll_ms, exact, held = [], [], [], [], True, 0
    check = tier != "cachegen_host"
    for it in range(warmup + steps):
        tmp = tempfile.mkdtemp(prefix="b200kv-tier-bench-")
        eng = _engine(tier, dtype, tmp)
        try:
            if tier in ("lossless_host", "cachegen_host"):
                eng.engine_.reserve_host(raw + (1 << 20))
            toks = torch.randint(0, 32000, (tokens,), generator=torch.Generator().manual_seed(100 + it))
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            eng.store(toks, pairs)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            got, mask = eng.retrieve(toks)
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            assert int(mask.sum()) == tokens
            if check:
                back = torch.stack([torch.stack([k, v]) for k, v in got])
                exact = exact and torch.equal(back.view(torch.int16), kv.view(torch.int16))
                del back
            del got
            held = _held(eng, tier, tmp)
            if tier in ("lossless_host", "cachegen_host"):
                start = torch.cuda.Event(enable_timing=True)
                start.record()
                r = eng.retrieve_layerwise(toks)
                ev0, evl = r._upload.ready(0), r._upload.ready(r.num_layers - 1)
                r.synchronize()
                if it >= warmup:
                    l0_ms.append(start.elapsed_time(ev0))
                    ll_ms.append(start.elapsed_time(evl))
                if check:
                    back = torch.stack([torch.stack([k, v]) for k, v in r.kv])
                    exact = exact and torch.equal(back.view(torch.int16), kv.view(torch.int16))
                    del back
                del r
            if it >= warmup:
                st_ms.append(1e3 * (t1 - t0))
                rt_ms.append(1e3 * (t2 - t1))
        finally:
            eng.close()
            shutil.rmtree(tmp, ignore_errors=True)
            torch.cuda.empty_cache()
    out = {"leg": "tier", "tier": tier, "tokens": tokens, "dtype": str(dtype).replace("torch.", ""), "data": kind,
           "raw_bytes": raw, "held_bytes": held, "ratio": round(raw / held, 3),
           "store_ms": round(statistics.median(st_ms), 2), "retrieve_ms": round(statistics.median(rt_ms), 2)}
    if l0_ms:
        out["layerwise_layer0_ms"] = round(statistics.median(l0_ms), 2)
        out["layerwise_last_ms"] = round(statistics.median(ll_ms), 2)
    out["bit_exact"] = bool(exact) if check else None
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--tokens", type=int, nargs="+", default=[8192, 65536])
    ap.add_argument("--data", nargs="+", default=["kv8d", "uniform_signed"])
    ap.add_argument("--tiers", nargs="+", default=list(TIERS), choices=TIERS)
    args = ap.parse_args()
    N.require_cuda()
    torch.cuda.set_device(0)
    print(json.dumps({"card": card()}), flush=True)
    for tokens in args.tokens:
        for dtype in (torch.bfloat16, torch.float16):
            for kind in args.data:
                for tier in args.tiers:
                    print(json.dumps(tier_leg(tier, tokens, dtype, kind, args.steps, args.warmup)), flush=True)


if __name__ == "__main__":
    main()
