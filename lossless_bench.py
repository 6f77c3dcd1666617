"""Measure the lossless codec (B2KV versions 5 and 6) and the `lossless` remote serde.

Kernel leg: 32 layers x 8 heads x 128 dims at 8192 and 65536 tokens, bf16 and fp16, each of bench.py's DATA_KINDS, chunks
of 256 tokens: encode and decode GB/s of raw KV (CUDA events, after warm-up, median of --steps), container bytes and
ratio, and every timed decode compared bit for bit with its input.
Engine leg: LMCacheEngine.store() / retrieve() of 8192 tokens through an in-process native lm:// server (port 0), for the
lossless, torch and cachegen serdes: medians of --steps.

Prints the card and its power limit, then one JSON line per measurement.  Writes nothing in the tree."""
import argparse
import ctypes
import json
import statistics
import subprocess
import time

import torch

import bench
from lmcache_b200 import _native as N
from lmcache_b200.codec import KvView, LosslessCodec

MODEL = "lmsys/longchat-7b-16k"
CHUNK = 256
bench.H, bench.C = 8, 8 * bench.D          # 32 layers x 8 KV heads x 128 dims (bench.synth_kv_torch reads these)


def card() -> dict:
    d = {"gpu": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        d["power_limit_w"] = float(out.splitlines()[0])
    except Exception:       # noqa: BLE001
        d["power_limit_w"] = None
    return d


def kernel_leg(tokens: int, dtype: torch.dtype, kind: str, steps: int, warmup: int) -> dict:
    kv = bench.synth_kv_torch(tokens, "cuda", 1, kind).to(dtype)
    view = KvView.from_blob(kv, "vllm")
    codec = LosslessCodec()
    raw = kv.numel() * 2
    n = (tokens + CHUNK - 1) // CHUNK
    out = torch.empty_like(kv)
    dst = KvView.from_blob(out, "vllm")
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    enc_ms, dec_ms, exact = [], [], True
    batch = None
    for it in range(warmup + steps):
        s.record()
        batch = codec.encode(view, 0, tokens, CHUNK)         # waits for the sizes: the event pair brackets the kernels
        e.record()
        torch.cuda.synchronize()
        if it >= warmup:
            enc_ms.append(s.elapsed_time(e))
        out.view(torch.int16).fill_(0)
        s.record()
        codec.decode_raw(batch.buf.data_ptr(), batch.buf.numel(), [j * batch.stride for j in range(n)], batch.sizes,
                         [min(CHUNK, tokens - j * CHUNK) for j in range(n)], dst, [j * CHUNK for j in range(n)],
                         batch.max_dtype, batch.coder)
        e.record()
        torch.cuda.synchronize()
        if it >= warmup:
            dec_ms.append(s.elapsed_time(e))
            exact = exact and torch.equal(out.view(torch.int16), kv.view(torch.int16)) and \
                not any(codec.decode_status())
    total = sum(batch.sizes)
    enc, dec = statistics.median(enc_ms), statistics.median(dec_ms)
    del kv, out, batch
    return {"leg": "kernel", "tokens": tokens, "dtype": str(dtype).replace("torch.", ""), "data": kind,
            "raw_bytes": raw, "container_bytes": total, "ratio": round(raw / total, 4),
            "encode_ms": round(enc, 3), "decode_ms": round(dec, 3),
            "encode_GBps": round(raw / enc / 1e6, 1), "decode_GBps": round(raw / dec / 1e6, 1), "bit_exact": exact}


def engine_leg(serde: str, tokens: int, steps: int, warmup: int) -> dict:
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    lib = N.lib()
    h = ctypes.c_void_p()
    N.check(lib.b200kv_lm_server_start(b"127.0.0.1", 0, ctypes.byref(h)), "lm_server_start")
    try:
        url = f"lm://127.0.0.1:{lib.b200kv_lm_server_port(h)}"
        kv = bench.synth_kv_torch(tokens, "cuda", 2, "kv8d")
        pairs = tuple((kv[l, 0], kv[l, 1]) for l in range(kv.shape[0]))
        meta = LMCacheEngineMetadata(MODEL, 1, 0, "vllm", "bfloat16")
        st_ms, rt_ms, exact = [], [], None
        for it in range(warmup + steps):
            cfg = LMCacheEngineConfig(CHUNK, None, url, serde, False, False)
            w, r = LMCacheEngine(cfg, meta), LMCacheEngine(cfg, meta)
            toks = torch.randint(0, 32000, (tokens,), generator=torch.Generator().manual_seed(100 + it))
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            w.store(toks, pairs)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            got, mask = r.retrieve(toks)
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            assert int(mask.sum()) == tokens
            if it >= warmup:
                st_ms.append(1e3 * (t1 - t0))
                rt_ms.append(1e3 * (t2 - t1))
            if exact is None:
                back = torch.stack([torch.stack([k, v]) for k, v in got])
                exact = torch.equal(back.view(torch.int16), kv.view(torch.int16))
            w.close()
            r.close()
        return {"leg": "engine", "serde": serde, "tokens": tokens, "store_ms": round(statistics.median(st_ms), 2),
                "retrieve_ms": round(statistics.median(rt_ms), 2), "bit_exact": bool(exact)}
    finally:
        lib.b200kv_lm_server_stop(h)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--tokens", type=int, nargs="+", default=[8192, 65536])
    ap.add_argument("--engine-steps", type=int, default=5)
    ap.add_argument("--no-engine", action="store_true")
    args = ap.parse_args()
    N.require_cuda()
    torch.cuda.set_device(0)
    print(json.dumps({"card": card()}), flush=True)
    for tokens in args.tokens:
        for dtype in (torch.bfloat16, torch.float16):
            for kind in bench.DATA_KINDS:
                print(json.dumps(kernel_leg(tokens, dtype, kind, args.steps, args.warmup)), flush=True)
                torch.cuda.empty_cache()
    if not args.no_engine:
        for serde in ("lossless", "torch", "cachegen"):
            print(json.dumps(engine_leg(serde, 8192, args.engine_steps, 1)), flush=True)


if __name__ == "__main__":
    main()
