"""Paged store / retrieve in vLLM's three paged cache layouts: FlashAttention rows, FlashInfer's block-strided rows and
PagedAttention's (xFormers') split pair, at 32 layers x 8 KV heads x 128 channels, chunks of 256 tokens.

Legs (medians over --reps runs, the layouts alternating inside every run, seeded inputs):
  mover    b200kv_pack_chunks of the whole call, device -> device and into mapped page-locked memory: GB/s of KV moved
  tiers    store_paged / retrieve_paged ms on the raw cpu and cuda tiers and the lossless host tier
  layers   retrieve_paged_layerwise on the cpu tier: ms until layer 0 and until the last layer are ready
  staging  peak HBM above the caches during a store_paged on the lossless host tier (the split layout's staging blob)
Prints one JSON line per leg and the card's name and power limit."""
import argparse
import json
import statistics
import subprocess
import time

import torch

from lmcache_b200.cache_engine import LMCacheEngine
from lmcache_b200.codec import KvView, PinnedBuffer
from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata

L, H, D, BS, CS = 32, 8, 128, 16, 256
LAYOUTS = ("flash", "strided", "split")
MODEL = "lmsys/longchat-7b-16k"


def make_caches(kind, T, dtype, seed):
    """the caches of T tokens in layout `kind`, vLLM's slot map of a shuffled block table, seeded"""
    nb = (T + BS - 1) // BS + 4
    g = torch.Generator(device="cuda").manual_seed(seed)
    es = torch.empty((), dtype=dtype).element_size()
    caches = []
    for _ in range(L):
        if kind == "flash":
            pair = tuple(torch.randint(0, 256, (nb * BS * H * D * es,), dtype=torch.uint8, device="cuda", generator=g)
                         .view(dtype).view(nb, BS, H, D) for _ in range(2))
        elif kind == "strided":
            kv = torch.randint(0, 256, (nb * 2 * BS * H * D * es,), dtype=torch.uint8, device="cuda", generator=g) \
                .view(dtype).view(nb, 2, BS, H, D)
            pair = (kv[:, 0], kv[:, 1])
        else:
            x = 16 // es
            c = torch.randint(0, 256, (2 * nb * BS * H * D * es,), dtype=torch.uint8, device="cuda", generator=g) \
                .view(dtype).view(2, nb, BS * H * D)
            pair = (c[0].view(nb, H, D // x, BS, x), c[1].view(nb, H, D, BS))
        caches.append(pair)
    gen = torch.Generator().manual_seed(seed)
    blocks = torch.randperm(nb, generator=gen)
    slots = (blocks.view(-1, 1) * BS + torch.arange(BS).view(1, -1)).flatten()[:T].cuda()
    return caches, slots


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def mover_leg(T, dtype, reps):
    out = {}
    kv_bytes = 2 * L * T * H * D * torch.empty((), dtype=dtype).element_size()
    pinned = PinnedBuffer(kv_bytes)
    ms = {(k, m): [] for k in LAYOUTS for m in ("d2d", "pinned")}
    views = {}
    for k in LAYOUTS:
        caches, slots = make_caches(k, T, dtype, 1)
        views[k] = (KvView.from_paged(caches, slots), caches)
    dev = torch.empty(kv_bytes, dtype=torch.uint8, device="cuda")
    from lmcache_b200 import _native as N
    import ctypes

    def pack(view, ptr):
        N.check(N.lib().b200kv_pack_chunks(ctypes.byref(view.desc), 0, (T + CS - 1) // CS, CS, T - (T - 1) // CS * CS, 0,
                                           ctypes.c_void_p(ptr), L * 2 * H * D * CS * view.dtype.itemsize,
                                           torch.cuda.current_stream().cuda_stream), "pack")
    for k in LAYOUTS:                                      # warm-up
        pack(views[k][0], dev.data_ptr())
        pack(views[k][0], pinned.dev_ptr)
    for _ in range(reps):
        for k in LAYOUTS:
            ms[(k, "d2d")].append(timed(lambda: [pack(views[k][0], dev.data_ptr()) for _ in range(5)]) / 5)
            ms[(k, "pinned")].append(timed(lambda: pack(views[k][0], pinned.dev_ptr)))
    for (k, m), v in ms.items():
        med = statistics.median(v)
        out[f"{k}_{m}_ms"] = round(med, 3)
        out[f"{k}_{m}_GBps"] = round(kv_bytes / med / 1e6, 1)
    pinned.close()
    return out


def tier_config(tier):
    if tier == "lossless":
        return LMCacheEngineConfig(CS, "cpu", None, None, False, False, "lossless")
    return LMCacheEngineConfig(CS, tier, None, None, False, False, None)


def tiers_leg(T, dtype, reps, tier):
    ms = {(k, op): [] for k in LAYOUTS for op in ("store", "retrieve")}
    tokens = torch.randint(0, 32000, (T,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    for r in range(reps + 1):                              # run 0 warms every shape up
        for k in LAYOUTS:
            caches, slots = make_caches(k, T, dtype, 2)
            eng = LMCacheEngine(tier_config(tier), LMCacheEngineMetadata(MODEL, 1, 0, "vllm", "bfloat16"))
            st = timed(lambda: eng.store_paged(tokens, caches, slots))
            rt = timed(lambda: eng.retrieve_paged(tokens, caches, slots))
            eng.close()
            del eng, caches
            torch.cuda.empty_cache()
            if r:
                ms[(k, "store")].append(st)
                ms[(k, "retrieve")].append(rt)
    return {f"{k}_{op}_ms": round(statistics.median(v), 2) for (k, op), v in ms.items()}


def layers_leg(T, dtype, reps):
    res = {(k, w): [] for k in LAYOUTS for w in ("first", "last")}
    tokens = torch.randint(0, 32000, (T,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(6))
    for r in range(reps + 1):
        for k in LAYOUTS:
            caches, slots = make_caches(k, T, dtype, 3)
            eng = LMCacheEngine(tier_config("cpu"), LMCacheEngineMetadata(MODEL, 1, 0, "vllm", "bfloat16"))
            eng.store_paged(tokens, caches, slots)
            torch.cuda.synchronize()
            start = torch.cuda.Event(enable_timing=True)
            start.record()
            h = eng.retrieve_paged_layerwise(tokens, caches, slots)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            h.wait_layer(0)
            e0.record()
            h.wait_layer(L - 1)
            e1.record()
            torch.cuda.synchronize()
            if r:
                res[(k, "first")].append(start.elapsed_time(e0))
                res[(k, "last")].append(start.elapsed_time(e1))
            eng.close()
            del eng, caches
            torch.cuda.empty_cache()
    return {f"{k}_layer_{w}_ready_ms": round(statistics.median(v), 2) for (k, w), v in res.items()}


def staging_leg(T, dtype):
    out = {}
    tokens = torch.randint(0, 32000, (T,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(7))
    for k in LAYOUTS:
        caches, slots = make_caches(k, T, dtype, 4)
        eng = LMCacheEngine(tier_config("lossless"), LMCacheEngineMetadata(MODEL, 1, 0, "vllm", "bfloat16"))
        eng.store_paged(tokens[:CS], caches, slots[:CS])   # the codec's own buffers exist before the measurement
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        eng.store_paged(tokens, caches, slots)
        torch.cuda.synchronize()
        out[f"{k}_peak_extra_MB"] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
        eng.close()
        del eng, caches
        torch.cuda.empty_cache()
    out["raw_bytes_MB"] = round(2 * L * (T - CS) * H * D * torch.empty((), dtype=dtype).element_size() / 2 ** 20, 1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, nargs="+", default=[8192, 65536])
    ap.add_argument("--dtypes", nargs="+", default=["bfloat16", "float8_e4m3fn"])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--legs", nargs="+", default=["mover", "tiers", "layers", "staging"])
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": card}), flush=True)
    for name in a.dtypes:
        dtype = getattr(torch, name)
        for T in a.tokens:
            common = {"dtype": name, "tokens": T, "L": L, "H": H, "D": D, "block_size": BS, "chunk": CS}
            if "mover" in a.legs:
                print(json.dumps({"leg": "mover", **common, **mover_leg(T, dtype, a.reps)}), flush=True)
            if "tiers" in a.legs:
                for tier in ("cpu", "cuda", "lossless"):
                    print(json.dumps({"leg": "tiers", "tier": tier, **common, **tiers_leg(T, dtype, a.reps, tier)}),
                          flush=True)
            if "layers" in a.legs:
                print(json.dumps({"leg": "layers", "tier": "cpu", **common, **layers_leg(T, dtype, a.reps)}), flush=True)
            if "staging" in a.legs:
                print(json.dumps({"leg": "staging", "tier": "lossless", **common, **staging_leg(T, dtype)}), flush=True)


if __name__ == "__main__":
    main()
