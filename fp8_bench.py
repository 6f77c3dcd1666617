"""Measure one-byte (FP8) KV caches against bf16 on the native paths.

Shape: 32 layers x 8 KV heads x 128 dims, chunks of 256 tokens, 8192 and 65536 tokens.  Data: randn, and randn with
per-channel scales (exp of a normal per channel), cast to float8_e4m3fn, float8_e5m2 or bfloat16.
  codec leg   lossless container ratio and encode / decode GB/s of raw KV (CUDA events around each call), E4M3, E5M2 and
              bf16 side by side; every decode compared bit for bit with its input
  engine leg  store_paged / retrieve_paged ms (host clock around work that ends in a device synchronise) of vLLM-shaped
              paged caches, on the raw cpu tier and on the lossless host tier (local_serde: lossless), FP8 and bf16
  mover leg   b200kv_pack_chunks / b200kv_unpack_chunks GB/s between paged caches and mapped pinned host memory, one-byte
              against 16-bit elements
Legs of one measurement alternate their variants step by step; numbers are medians of --steps (at least 3) after
--warmup.  Prints the card and its power limit, then one JSON line per measurement.  Writes nothing in the tree."""
import argparse
import ctypes
import json
import statistics
import time

import torch

from lmcache_b200 import _native as N
from lmcache_b200.codec import KvView, LosslessCodec, PinnedBuffer
from lossless_bench import card

MODEL = "lmsys/longchat-7b-16k"
L, H, D, CHUNK = 32, 8, 128, 256
DTYPES = {"e4m3": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2, "bf16": torch.bfloat16}


def synth(tokens: int, dtype: torch.dtype, kind: str, seed: int) -> torch.Tensor:
    """[L, 2, T, H, D] of `dtype`, made one layer at a time (no float32 copy of the whole KV)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = torch.empty((L, 2, tokens, H, D), dtype=dtype, device="cuda")
    for l in range(L):
        x = torch.randn((2, tokens, H, D), device="cuda", generator=g)
        if kind == "scaled":
            x *= torch.exp(torch.randn((2, 1, H, D), device="cuda", generator=g))
        out[l] = x.to(dtype)
    return out


def _bits(x: torch.Tensor) -> torch.Tensor:
    return x.view(torch.uint8)


def codec_leg(tokens: int, kind: str, steps: int, warmup: int) -> list:
    codec = LosslessCodec()                      # one staging for every dtype: grown once, to the 16-bit bound
    n = (tokens + CHUNK - 1) // CHUNK
    kvs = {name: synth(tokens, dt, kind, 1) for name, dt in DTYPES.items()}
    res = {name: {"enc": [], "dec": [], "bytes": 0, "exact": True} for name in DTYPES}
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for it in range(warmup + steps):
        for name, kv in kvs.items():
            out = torch.empty_like(kv)
            view, dst = KvView.from_blob(kv, "vllm"), KvView.from_blob(out, "vllm")
            s.record()
            batch = codec.encode(view, 0, tokens, CHUNK)
            e.record()
            torch.cuda.synchronize()
            enc = s.elapsed_time(e)
            s.record()
            codec.decode_raw(batch.buf.data_ptr(), batch.buf.numel(), [j * batch.stride for j in range(n)], batch.sizes,
                             [min(CHUNK, tokens - j * CHUNK) for j in range(n)], dst, [j * CHUNK for j in range(n)],
                             batch.max_dtype, batch.coder)
            e.record()
            torch.cuda.synchronize()
            r = res[name]
            if it >= warmup:
                r["enc"].append(enc)
                r["dec"].append(s.elapsed_time(e))
                r["exact"] = r["exact"] and torch.equal(_bits(out), _bits(kv)) and not any(codec.decode_status())
            r["bytes"] = sum(batch.sizes)
            del out, batch
    rows = []
    for name, kv in kvs.items():
        r, raw = res[name], kv.numel() * kv.element_size()
        enc, dec = statistics.median(r["enc"]), statistics.median(r["dec"])
        rows.append({"leg": "codec", "tokens": tokens, "data": kind, "dtype": name, "raw_bytes": raw,
                     "container_bytes": r["bytes"], "ratio": round(raw / r["bytes"], 4), "encode_ms": round(enc, 3),
                     "decode_ms": round(dec, 3), "encode_GBps": round(raw / enc / 1e6, 1),
                     "decode_GBps": round(raw / dec / 1e6, 1), "bit_exact": r["exact"]})
    return rows


def _paged(kv: torch.Tensor, seed: int):
    """vLLM-shaped caches [num_blocks, 16, H, D] per layer holding kv's tokens at shuffled slots"""
    T = kv.shape[2]
    nslots = (T + 15) // 16 * 16
    slots = torch.randperm(nslots, generator=torch.Generator().manual_seed(seed))[:T].cuda()
    caches = []
    for l in range(L):
        pair = []
        for kvi in range(2):
            c = torch.zeros((nslots // 16, 16, H, D), dtype=kv.dtype, device="cuda")
            _bits(c).view(nslots, -1)[slots] = _bits(kv[l, kvi].contiguous()).view(T, -1)
            pair.append(c)
        caches.append(tuple(pair))
    return caches, slots


def engine_leg(tokens: int, steps: int, warmup: int) -> list:
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    variants = [(tier, name) for tier in ("cpu", "lossless") for name in ("e4m3", "bf16")]
    src = {name: _paged(synth(tokens, DTYPES[name], "randn", 2), 3) for name in ("e4m3", "bf16")}
    times = {v: ([], []) for v in variants}
    exact = {v: True for v in variants}
    for it in range(warmup + steps):
        for tier, name in variants:
            caches, slots = src[name]
            cfg = LMCacheEngineConfig(CHUNK, "cpu", None, None, False, False, "lossless" if tier == "lossless" else None)
            eng = LMCacheEngine(cfg, LMCacheEngineMetadata(MODEL, 1, 0, "vllm", name))
            toks = torch.randint(0, 32000, (tokens,), generator=torch.Generator().manual_seed(100 + it))
            dst = [(torch.zeros_like(k), torch.zeros_like(v)) for k, v in caches]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            eng.store_paged(toks, caches, slots)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            mask = eng.retrieve_paged(toks, dst, slots)
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            if it >= warmup:
                times[(tier, name)][0].append(1e3 * (t1 - t0))
                times[(tier, name)][1].append(1e3 * (t2 - t1))
                exact[(tier, name)] = exact[(tier, name)] and int(mask.sum()) == tokens and all(
                    torch.equal(_bits(x), _bits(y)) for p, q in zip(dst, caches) for x, y in zip(p, q))
            eng.close()
            del dst
    return [{"leg": "engine", "tier": "cpu (raw)" if tier == "cpu" else "cpu, local_serde: lossless", "dtype": name,
             "tokens": tokens, "store_paged_ms": round(statistics.median(times[(tier, name)][0]), 2),
             "retrieve_paged_ms": round(statistics.median(times[(tier, name)][1]), 2), "bit_exact": exact[(tier, name)]}
            for tier, name in variants]


def mover_leg(tokens: int, steps: int, warmup: int) -> list:
    lib, sp = N.lib(), torch.cuda.current_stream().cuda_stream
    n = (tokens + CHUNK - 1) // CHUNK
    last = tokens - (n - 1) * CHUNK
    legs = {}
    for name in ("e4m3", "bf16"):
        caches, slots = _paged(synth(tokens, DTYPES[name], "randn", 4), 5)
        view = KvView.from_paged(caches, slots)
        es = 1 if name == "e4m3" else 2
        stride = 2 * L * CHUNK * H * D * es
        legs[name] = (view, PinnedBuffer(n * stride), stride, caches)
    times = {name: ([], []) for name in legs}
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for it in range(warmup + steps):
        for name, (view, pin, stride, caches) in legs.items():
            s.record()
            N.check(lib.b200kv_pack_chunks(ctypes.byref(view.desc), 0, n, CHUNK, last, 0, ctypes.c_void_p(pin.dev_ptr),
                                           stride, sp), "pack_chunks")
            e.record()
            torch.cuda.synchronize()
            pk = s.elapsed_time(e)
            s.record()
            N.check(lib.b200kv_unpack_chunks(ctypes.c_void_p(pin.dev_ptr), stride, n, CHUNK, last, 0,
                                             ctypes.byref(view.desc), 0, sp), "unpack_chunks")
            e.record()
            torch.cuda.synchronize()
            if it >= warmup:
                times[name][0].append(pk)
                times[name][1].append(s.elapsed_time(e))
    rows = []
    for name, (view, pin, stride, caches) in legs.items():
        raw = 2 * L * tokens * H * D * (1 if name == "e4m3" else 2)
        pk, up = statistics.median(times[name][0]), statistics.median(times[name][1])
        rows.append({"leg": "mover", "tokens": tokens, "element_bytes": 1 if name == "e4m3" else 2,
                     "chunks": "mapped pinned host", "pack_ms": round(pk, 3), "unpack_ms": round(up, 3),
                     "pack_GBps": round(raw / pk / 1e6, 1), "unpack_GBps": round(raw / up / 1e6, 1)})
        pin.close()
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--tokens", type=int, nargs="+", default=[8192, 65536])
    args = ap.parse_args()
    if args.steps < 3:
        ap.error("--steps must be at least 3: the numbers are medians")
    N.require_cuda()
    torch.cuda.set_device(0)
    print(json.dumps({"card": card()}), flush=True)
    for tokens in args.tokens:
        for kind in ("randn", "scaled"):
            for row in codec_leg(tokens, kind, args.steps, args.warmup):
                print(json.dumps(row), flush=True)
            torch.cuda.empty_cache()
        for row in mover_leg(tokens, args.steps, args.warmup):
            print(json.dumps(row), flush=True)
        torch.cuda.empty_cache()
        for row in engine_leg(tokens, args.steps, args.warmup):
            print(json.dumps(row), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
