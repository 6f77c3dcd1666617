#!/usr/bin/env python
"""deep_model_bench.py -- the KV of an 80-layer model (Llama-3.1-70B's geometry) through the codec and the engine, on one GPU.

  python deep_model_bench.py [--steps K] [--warmup W] [--tokens 8192] [--heads 8,2,1]

Workload: 80 layers, D = 128, bf16 KV, synthetic SURVEY 8d data (bench.py's kv8d distribution), chunk 256, the bins of
a cachegen_config that applies the reference table's rule to 80 layers (keys 32 bins for layers 0-9, values 32 for
layers 0-1, 16 after).  Run per tensor-parallel rank: H = 8 / 2 / 1 KV heads per rank is TP 1 / 4 / 8 of the model's
8 KV heads.  Per H:
  encode_GBps / decode_GBps   KV bytes over the device time of CacheGenCodec.encode / decode_device_batch of every
                              chunk in one call (CUDA events on the call's stream, median over the steps)
  store_ms / retrieve_ms      LMCacheEngine.store / retrieve of the whole sequence, host clock around the call and a
                              device synchronise (median), on the compressed host tier (local_serde = "cachegen") and on
                              the raw "cpu" tier
  container_bytes             the compressed tier's containers for the sequence, and their ratio to the KV bytes
  oracle                      the first and last chunk the compressed tier returns, against the CPU oracle's decode
At H = 1 a chunk has 160 tiles of 128 streams, one per plane: the GPU is under-filled there, and the number says so.
Prints one JSON line with the card's name and power limit.  Writes nothing into the tree.
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

MODEL = "meta-llama/Llama-3.1-70B-Instruct"
L, D = 80, 128
CACHEGEN_CONFIG = dict(key_first_layers=10, key_second_layers=20, key_third_layers=L, key_first_bins=32,
                       key_second_bins=16, key_third_bins=16, value_first_layers=2, value_first_bins=32,
                       value_second_bins=16)


def _power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def synth_kv(T, H, device, seed):
    """[L,2,T,H,D] bf16: bench.py's kv8d distribution at this geometry"""
    import torch
    C = H * D
    g = torch.Generator(device=device).manual_seed(seed)
    sigma = torch.exp(0.5 * torch.randn((L, 2, 1, C), device=device, generator=g)).clamp_(0.1, 8.0)
    outl = torch.rand((L, 2, 1, C), device=device, generator=g) < 0.01
    sigma = torch.where(outl, sigma * 10.0, sigma)
    kv = torch.empty((L, 2, T, C), dtype=torch.bfloat16, device=device)
    for t0 in range(0, T, 512):
        n = min(512, T - t0)
        kv[:, :, t0:t0 + n] = (torch.randn((L, 2, n, C), device=device, generator=g) * sigma).to(torch.bfloat16)
    return kv.reshape(L, 2, T, H, D)


def _bits(x):
    """bf16 tensor -> numpy uint16 bit pattern"""
    import torch
    return x.contiguous().cpu().view(torch.int16).numpy().view("uint16")


def run(T, H, cs, steps, warmup):
    import numpy as np
    import torch

    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.codec import CacheGenCodec, KvView
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    from oracle import oracle as O

    dev = torch.device("cuda", 0)
    cur = torch.cuda.current_stream()
    kv = synth_kv(T, H, dev, 1236 + H)
    kv_bytes = kv.numel() * 2
    res = {"heads": H, "tp": 8 // H, "tokens": T, "kv_bytes": kv_bytes}

    # ---- kernels: encode every chunk in one call, decode them all in one call, device time from events
    codec = CacheGenCodec(MODEL, cachegen_config=CACHEGEN_CONFIG)
    src = KvView.from_blob(kv, "vllm")
    out = torch.empty_like(kv)
    dst = KvView.from_blob(out, "vllm")
    n = (T + cs - 1) // cs
    ntok = [min(cs, T - j * cs) for j in range(n)]
    enc_ms, dec_ms = [], []
    for i in range(warmup + steps):
        s, m, e = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        s.record(cur)
        batch = codec.encode(src, 0, T, cs)
        m.record(cur)
        codec.decode_device_batch(batch, ntok, dst, [j * cs for j in range(n)])
        e.record(cur)
        e.synchronize()
        if i >= warmup:
            enc_ms.append(s.elapsed_time(m))
            dec_ms.append(m.elapsed_time(e))
    # the encode call's time includes waiting for its sizes on the host (encode() = encode_async + wait): the events
    # bracket the device work of the call in stream order either way
    res["encode_ms"] = round(statistics.median(enc_ms), 3)
    res["decode_ms"] = round(statistics.median(dec_ms), 3)
    res["encode_GBps"] = round(kv_bytes / res["encode_ms"] / 1e6, 1)
    res["decode_GBps"] = round(kv_bytes / res["decode_ms"] / 1e6, 1)
    res["container_bytes"] = int(sum(batch.sizes))
    res["ratio"] = round(kv_bytes / res["container_bytes"], 2)
    res["codec_status"] = codec.decode_status() == [0] * n
    del batch, out, dst, src

    # ---- engine: store() / retrieve() of the whole sequence on the compressed host tier and on the raw cpu tier
    meta = LMCacheEngineMetadata(MODEL, 1, 0, "vllm", "bfloat16")
    tokens = torch.randint(0, 32000, (T,), device=dev, generator=torch.Generator(device=dev).manual_seed(7))
    kv_tuple = tuple((kv[l, 0], kv[l, 1]) for l in range(L))
    tiers = {"compressed": dict(local_serde="cachegen", cachegen_config=CACHEGEN_CONFIG), "raw_cpu": {}}
    spot = None
    for name, kw in tiers.items():
        eng = LMCacheEngine(LMCacheEngineConfig.from_legacy(chunk_size=cs, backend="cpu", **kw), meta)
        try:
            st, rt = [], []
            for i in range(warmup + steps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                eng.store(tokens, kv_tuple, skip_existing=False)
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                ret, mask = eng.retrieve(tokens)
                torch.cuda.synchronize()
                t2 = time.perf_counter()
                assert int(mask.sum()) == T, name
                if i >= warmup:
                    st.append(1e3 * (t1 - t0))
                    rt.append(1e3 * (t2 - t1))
                if name == "compressed" and i == warmup + steps - 1:
                    spot = [(a, torch.stack([torch.stack([k[a:a + cs], v[a:a + cs]]) for k, v in ret]))
                            for a in sorted({0, (n - 1) * cs})]
                del ret, mask
            res[name] = {"store_ms": round(statistics.median(st), 3), "retrieve_ms": round(statistics.median(rt), 3)}
            if name == "compressed":
                res[name]["host_bytes"] = int(eng.engine_.host_bytes())
        finally:
            eng.close()
    del kv_tuple

    # ---- the compressed tier's first and last chunk against the CPU oracle (not timed)
    from lmcache_b200.storage_backend.serde.cachegen_basics import CacheGenConfig
    cfg = CacheGenConfig(**CACHEGEN_CONFIG)
    kb = np.array(cfg.key_bins_list(), np.float32)
    vb = np.array(cfg.value_bins_list(), np.float32)
    ok = True
    for a, got in spot:
        t = got.shape[2]
        bits = _bits(kv[:, :, a:a + t]).reshape(L, 2, t, H * D)
        want = O.decode_chunk(O.encode_chunk(bits, O.DT_BF16, kb, vb, O.CODER_RANS), O.DT_BF16, kb, vb, O.DT_BF16)
        ok = ok and np.array_equal(_bits(got).reshape(L, 2, t, H * D), want)
    res["oracle"] = "bit-exact" if ok else "MISMATCH"
    del kv, spot
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--tokens", type=int, default=8192)
    ap.add_argument("--chunk", type=int, default=256)
    ap.add_argument("--heads", type=str, default="8,2,1", help="KV heads per rank (8 = TP 1, 2 = TP 4, 1 = TP 8)")
    args = ap.parse_args()
    import torch

    from lmcache_b200 import _native as N
    N.require_cuda()
    torch.cuda.set_device(0)
    results = [run(args.tokens, int(h), args.chunk, args.steps, args.warmup) for h in args.heads.split(",")]
    print(json.dumps({"metric": "deep_model_80L", "model_geometry": f"{L}L x D{D}", "chunk": args.chunk,
                      "steps": args.steps, "warmup": args.warmup, "gpu": torch.cuda.get_device_name(0),
                      "power_limit": _power_limit(), "results": results}))


if __name__ == "__main__":
    main()
