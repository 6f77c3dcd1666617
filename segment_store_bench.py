"""Storing a prompt's documents from inside it, on the H100: b200kv_pack_chunks_rope against the two launches it fuses,
LMCacheEngine.store_paged_segments against store_paged, and what the derived-key continuation costs a segment retrieve.

Workload (segment_bench.py's): a RAG request of eight 2048-token documents and a 512-token question (16896 tokens),
32 layers x 8 KV heads x 128 channels, bf16, chunk 256, a paged cache of 16-token blocks.  Request 1 holds the
documents in order from token 0; request 2 holds them in reverse order after a 512-token question, so every document
moves.

  (a) kernel: one rope table + one b200kv_pack_chunks_rope launch against b200kv_pack_chunks + rope table +
      b200kv_rope_shift of the packed rows, for the seven documents that do not start at token 0 (14336 tokens), in the
      FlashAttention and split (PagedAttention) layouts: microseconds over many launches (CUDA events), bytes read plus
      written from the shapes, and their rate against the H100 SXM's 3.35 TB/s.
  (b) engine: store_paged_segments of the eight documents against store_paged of the whole 16896-token request 1
      (skip_existing=False, so every call stores everything), on the raw cpu, CacheGen host and lossless host tiers:
      median and minimum of --steps calls.
  (c) engine: request 2's retrieve_paged_segments after (b)'s segment store (chunks 0.. of seven documents come from
      their derived keys), and the same call on an engine where the first seven of each document's eight chunks were
      stored alone and no derived key exists: every segment misses its last prefix key, so each pays the one extra
      (missing) derived-key lookup the continuation adds.  With --baseline-root DIR
      the second call is also timed with the package of another checkout (e.g. the parent commit), alternating.

Prints the card's name and power limit with the numbers.

    python segment_store_bench.py [--steps 5] [--warmup 2] [--iters 200] [--tiers cpu,host-cachegen,host-lossless]
                                  [--baseline-root DIR] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if "--leg-root" in sys.argv:                       # a (c) leg run with another checkout's package
    sys.path.insert(0, sys.argv[sys.argv.index("--leg-root") + 1])
else:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

L, H, D, CS, BS = 32, 8, 128, 256, 16
N_DOCS, DOC, QUESTION = 8, 2048, 512
HBM_BYTES_PER_S = 3.35e12
MODEL = "meta-llama/Llama-3.1-8B-Instruct"


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
    import statistics
    import time
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


def workload():
    T = N_DOCS * DOC + QUESTION
    gen = torch.Generator(device="cuda").manual_seed(0)
    nb = (T + BS - 1) // BS + 8
    src_rows = [tuple(torch.randn(nb * BS, H, D, device="cuda", generator=gen).to(torch.bfloat16) for _ in range(2))
                for _ in range(L)]
    slots = (torch.randperm(nb, device="cuda", generator=gen)[:, None] * BS +
             torch.arange(BS, device="cuda")[None, :]).flatten()[:T].contiguous()
    docs = torch.randint(0, 32000, (N_DOCS, DOC), generator=torch.Generator().manual_seed(1))
    question = torch.randint(0, 32000, (QUESTION,), generator=torch.Generator().manual_seed(2))
    tok1 = torch.cat([docs.flatten(), question])                                  # documents from token 0
    tok2 = torch.cat([question] + [docs[i] for i in reversed(range(N_DOCS))])     # reversed, after the question
    seg1 = [(i * DOC, (i + 1) * DOC) for i in range(N_DOCS)]
    seg2 = [(QUESTION + (N_DOCS - 1 - i) * DOC, QUESTION + (N_DOCS - i) * DOC) for i in range(N_DOCS)]
    return nb, src_rows, slots, tok1, tok2, seg1, seg2


def caches(layout, src_rows, nb):
    if layout == "flash":
        return [tuple(r.view(nb, BS, H, D) for r in p) for p in src_rows]
    return [(k.view(nb, BS, H, D // 8, 8).permute(0, 2, 3, 1, 4).contiguous(),   # vLLM's split_kv_cache, x = 8 at bf16
             v.view(nb, BS, H, D).permute(0, 2, 3, 1).contiguous()) for k, v in src_rows]


def kernel_leg(layout, iters, src_rows, nb, slots, seg1):
    import ctypes
    from lmcache_b200 import _native as N
    from lmcache_b200.codec import KvView
    from lmcache_b200.rope import RopeSpec, pack_rope, plan_segment_store, plan_segments, rope_shift, rope_table
    view = KvView.from_paged(caches(layout, src_rows, nb), slots)
    rope = RopeSpec.from_base(D, 10000.0)
    inner = [p for p in plan_segments(len(slots), seg1, CS) if p.start > 0]
    _, rows, sot, shifts = plan_segment_store(inner, [(0, 0)] * len(inner), CS)
    src = view.rows(torch.tensor(rows, dtype=torch.int64, device="cuda"))
    n = len(rows)
    seg = torch.tensor(sot, dtype=torch.int32, device="cuda")
    sh = torch.tensor(shifts, dtype=torch.int64, device="cuda")
    blob = torch.empty(L, 2, n, H, D, dtype=torch.bfloat16, device="cuda")
    blob2 = torch.empty_like(blob)

    def fused():
        pack_rope(src, blob, seg, rope_table(sh, rope), rope)

    def composed():
        N.check(N.lib().b200kv_pack_chunks(ctypes.byref(src.desc), 0, 1, n, n, 0, ctypes.c_void_p(blob2.data_ptr()),
                                           blob2.numel() * 2, None), "pack_chunks")
        rope_shift(KvView.from_blob(blob2, "vllm"), 0, seg, sh, rope)
    fused()
    composed()
    torch.cuda.synchronize()
    same = bool(torch.equal(blob.view(torch.int16), blob2.view(torch.int16)))
    kv_bytes = n * L * 2 * H * D * 2
    rot_bytes = n * L * H * rope.rotary_dim * 2
    out = {"layout": layout, "tokens": n, "bit_identical": same}
    for name, fn, nbytes in (("fused", fused, 2 * kv_bytes), ("pack_then_shift", composed, 2 * kv_bytes + 2 * rot_bytes)):
        for _ in range(5):
            fn()
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record()
        for _ in range(iters):
            fn()
        stop.record()
        stop.synchronize()
        us = start.elapsed_time(stop) * 1e3 / iters
        rate = nbytes / (us * 1e-6)
        out[name] = {"us": round(us, 1), "bytes": nbytes, "TBps": round(rate / 1e12, 3),
                     "share_of_3.35TBps": round(rate / HBM_BYTES_PER_S, 3)}
    return out


def drain(eng):
    if hasattr(eng.engine_, "drain"):
        eng.engine_.drain()


def engine_leg(tier, steps, warmup, w):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineMetadata
    from lmcache_b200.rope import RopeSpec
    nb, src_rows, slots, tok1, tok2, seg1, seg2 = w
    src = caches("flash", src_rows, nb)
    rope = RopeSpec.from_base(D, 10000.0)
    eng = LMCacheEngine(config(tier), LMCacheEngineMetadata(MODEL, 1, 0, "vllm", "bfloat16"))
    try:
        def seg_store():
            eng.store_paged_segments(tok1, src, slots, seg1, rope, skip_existing=False)
            drain(eng)

        def whole_store():
            eng.store_paged(tok1 + 1_000_000, src, slots, skip_existing=False)
            drain(eng)
        s_ms, s_min, _ = timed(seg_store, steps, warmup)
        w_ms, w_min, _ = timed(whole_store, steps, warmup)
        dst = [(torch.empty_like(k), torch.empty_like(v)) for k, v in src]
        slots2 = slots.flip(0).contiguous()
        r_ms, r_min, ret = timed(lambda: eng.retrieve_paged_segments(tok2, dst, slots2, seg2 + [(0, QUESTION)], rope),
                                 steps, warmup)
        return {"tier": tier, "store_segments_ms_p50": round(s_ms, 3), "store_segments_ms_min": round(s_min, 3),
                "store_paged_whole_ms_p50": round(w_ms, 3), "store_paged_whole_ms_min": round(w_min, 3),
                "retrieve_derived_ms_p50": round(r_ms, 3), "retrieve_derived_ms_min": round(r_min, 3),
                "retrieve_derived_tokens": int(ret.sum())}
    finally:
        eng.close()


def alone_leg(tier, steps, warmup):
    """(c) without derived keys: the first DOC - CS tokens of each document stored alone, request 2's segments
    retrieved; the only API used is one the parent commit had"""
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineMetadata
    from lmcache_b200.rope import RopeSpec
    nb, src_rows, slots, tok1, tok2, seg1, seg2 = workload()
    src = caches("flash", src_rows, nb)
    rope = RopeSpec.from_base(D, 10000.0)
    eng = LMCacheEngine(config(tier), LMCacheEngineMetadata(MODEL, 1, 0, "vllm", "bfloat16"))
    try:
        for a, b in seg1:
            eng.store_paged(tok1[a:b - CS], src, slots[a:b - CS])
        drain(eng)
        dst = [(torch.empty_like(k), torch.empty_like(v)) for k, v in src]
        slots2 = slots.flip(0).contiguous()
        ms, mn, ret = timed(lambda: eng.retrieve_paged_segments(tok2, dst, slots2, seg2 + [(0, QUESTION)], rope),
                            steps, warmup)
        return {"tier": tier, "retrieve_alone_ms_p50": round(ms, 3), "retrieve_alone_ms_min": round(mn, 3),
                "retrieve_alone_tokens": int(ret.sum())}
    finally:
        eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--tiers", default="cpu,host-cachegen,host-lossless")
    ap.add_argument("--baseline-root", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--leg-alone", default=None, help=argparse.SUPPRESS)    # internal: one (c) leg, as JSON
    ap.add_argument("--leg-root", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "segment_store_bench measures on a CUDA device; there is no CPU fallback"
    if args.leg_alone:
        print(json.dumps(alone_leg(args.leg_alone, args.steps, args.warmup)))
        return
    name, power = card()
    w = workload()
    results = {"card": name, "power_limit": power,
               "workload": {"L": L, "H": H, "D": D, "dtype": "bfloat16", "chunk": CS, "tokens": len(w[3]),
                            "documents": N_DOCS, "doc_tokens": DOC, "question_tokens": QUESTION},
               "kernel": [], "engine": [], "alone": []}
    for layout in ("flash", "split"):
        r = kernel_leg(layout, args.iters, w[1], w[0], w[2], w[5])
        results["kernel"].append(r)
        print(json.dumps(r), flush=True)
    for tier in args.tiers.split(","):
        r = engine_leg(tier, args.steps, args.warmup, w)
        results["engine"].append(r)
        print(json.dumps(r), flush=True)
    roots = [("this", ROOT)] + ([("baseline", args.baseline_root)] if args.baseline_root else [])
    for rnd in range(args.rounds if args.baseline_root else 1):
        for tag, root in roots:
            for tier in args.tiers.split(","):
                out = subprocess.run([sys.executable, os.path.abspath(__file__), "--leg-alone", tier, "--leg-root", root,
                                      "--steps", str(args.steps), "--warmup", str(args.warmup)],
                                     capture_output=True, text=True, check=True).stdout
                r = dict(json.loads(out.strip().splitlines()[-1]), tree=tag, round=rnd)
                results["alone"].append(r)
                print(json.dumps(r), flush=True)
    print(json.dumps({"card": name, "power_limit": power}))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "segment_store_bench.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
