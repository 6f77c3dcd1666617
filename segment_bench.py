"""Non-prefix KV reuse on the H100: LMCacheEngine.retrieve_paged_segments against retrieve_paged, and the rope shift
kernel on its own.

Workload: a RAG request of eight 2048-token documents and a 512-token question (16896 tokens), 32 layers x 8 KV heads x
128 channels, bf16, chunk 256, a FlashAttention paged cache of 16-token blocks.  Each document is stored as a prompt of
its own; the same request is also stored whole, so that retrieve_paged of its 16896-token prefix moves the same kind of
bytes (the segments hit 16384 tokens: the question was never stored as a document).  Tiers: the raw cpu tier, and the
CacheGen and lossless page-locked host tiers.

The kernel leg times b200kv_rope_table + b200kv_rope_shift with CUDA events over many launches, for the seven documents
that do not start at token 0 (14336 tokens), in the FlashAttention and the split (PagedAttention) layouts, and reports
bytes read plus written -- rotary channels of every key row, from the shapes -- per second against the H100 SXM's
3.35 TB/s.  Prints the card's name and power limit with the numbers.

    python segment_bench.py [--steps 5] [--warmup 2] [--tiers cpu,host-cachegen,host-lossless] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

L, H, D, CS, BS = 32, 8, 128, 256, 16
N_DOCS, DOC, QUESTION = 8, 2048, 512
HBM_BYTES_PER_S = 3.35e12
MODEL = "meta-llama/Llama-3.1-8B-Instruct"         # 32 layers, 8 KV heads of 128 channels: its CacheGen bins


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return name, out


def config(tier):
    from lmcache_b200.config import LMCacheEngineConfig
    if tier == "cpu":
        return LMCacheEngineConfig(CS, "cpu", None, None, False, False, None)
    return LMCacheEngineConfig(CS, "cpu", None, None, False, False, tier.split("-")[1])


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts), min(ts), out


def engine_leg(tier, steps, warmup, src, slots, tokens, segs):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineMetadata
    from lmcache_b200.rope import RopeSpec
    eng = LMCacheEngine(config(tier), LMCacheEngineMetadata(MODEL, 1, 0, "vllm", "bfloat16"))
    try:
        for a, b in segs:
            eng.store_paged(tokens[a:b], src, slots[a:b])
        prefix = tokens + 1_000_000                          # the same bytes under the request's own prefix keys
        eng.store_paged(prefix, src, slots)
        if hasattr(eng.engine_, "drain"):
            eng.engine_.drain()
        dst = [(torch.empty_like(k), torch.empty_like(v)) for k, v in src]
        rope = RopeSpec.from_base(D, 10000.0)
        seg_ms, seg_min, ret_s = timed(lambda: eng.retrieve_paged_segments(tokens, dst, slots, segs, rope), steps,
                                       warmup)
        pre_ms, pre_min, ret_p = timed(lambda: eng.retrieve_paged(prefix, dst, slots), steps, warmup)
        return {"tier": tier, "segments_ms_p50": round(seg_ms, 3), "segments_ms_min": round(seg_min, 3),
                "segments_tokens": int(ret_s.sum()), "prefix_ms_p50": round(pre_ms, 3), "prefix_ms_min": round(pre_min, 3),
                "prefix_tokens": int(ret_p.sum())}
    finally:
        eng.close()


def kernel_leg(layout, iters, src_rows, slots, segs):
    from lmcache_b200.codec import KvView
    from lmcache_b200.rope import RopeSpec, plan_segments, rope_shift, seg_of_tok
    nb = src_rows[0][0].shape[0] // BS
    if layout == "flash":
        caches = [tuple(r.view(nb, BS, H, D).clone() for r in p) for p in src_rows]
    else:                                                   # vLLM's PagedAttention.split_kv_cache, x = 8 at bf16
        caches = [(k.view(nb, BS, H, D // 8, 8).permute(0, 2, 3, 1, 4).contiguous(),
                   v.view(nb, BS, H, D).permute(0, 2, 3, 1).contiguous()) for k, v in src_rows]
    view = KvView.from_paged(caches, slots)
    rope = RopeSpec.from_base(D, 10000.0)
    plans = plan_segments(len(slots), segs, CS)
    sot, lo, hi, shifts = seg_of_tok(len(slots), [(p, p.end - p.start) for p in plans])
    seg = torch.tensor(sot, dtype=torch.int32, device="cuda")
    sh = torch.tensor(shifts, dtype=torch.int64, device="cuda")
    n_rot = sum(1 for s in sot if s >= 0)
    nbytes = 2 * n_rot * L * H * rope.rotary_dim * 2          # read + write, bf16
    for _ in range(5):
        rope_shift(view, lo, seg, sh, rope)
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        rope_shift(view, lo, seg, sh, rope)
    stop.record()
    stop.synchronize()
    us = start.elapsed_time(stop) * 1e3 / iters
    rate = nbytes / (us * 1e-6)
    return {"layout": layout, "rotated_tokens": n_rot, "bytes": nbytes, "us_per_launch_pair": round(us, 2),
            "GBps": round(rate / 1e9, 1), "share_of_3.35TBps": round(rate / HBM_BYTES_PER_S, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--tiers", default="cpu,host-cachegen,host-lossless")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "segment_bench measures on a CUDA device; there is no CPU fallback"
    name, power = card()
    T = N_DOCS * DOC + QUESTION
    gen = torch.Generator(device="cuda").manual_seed(0)
    nb = (T + BS - 1) // BS + 8
    src_rows = [tuple(torch.randn(nb * BS, H, D, device="cuda", generator=gen).to(torch.bfloat16) for _ in range(2))
                for _ in range(L)]
    src = [tuple(r.view(nb, BS, H, D) for r in p) for p in src_rows]
    slots = (torch.randperm(nb, device="cuda", generator=gen)[:, None] * BS +
             torch.arange(BS, device="cuda")[None, :]).flatten()[:T].contiguous()
    tokens = torch.randint(0, 32000, (T,), generator=torch.Generator().manual_seed(1))
    segs = [(i * DOC, (i + 1) * DOC) for i in range(N_DOCS)]
    results = {"card": name, "power_limit": power, "workload": {"L": L, "H": H, "D": D, "dtype": "bfloat16",
               "chunk": CS, "tokens": T, "documents": N_DOCS, "doc_tokens": DOC, "question_tokens": QUESTION},
               "kernel": [], "engine": []}
    for layout in ("flash", "split"):
        r = kernel_leg(layout, args.iters, src_rows, slots, segs)
        results["kernel"].append(r)
        print(json.dumps(r), flush=True)
    for tier in args.tiers.split(","):
        r = engine_leg(tier, args.steps, args.warmup, src, slots, tokens, segs)
        results["engine"].append(r)
        print(json.dumps(r), flush=True)
    print(json.dumps({"card": name, "power_limit": power}))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "segment_bench.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
