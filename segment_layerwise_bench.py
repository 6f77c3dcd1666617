"""The layer-wise segment retrieve on the H100: when layer 0 and the last layer of a RAG request's documents are ready
with LMCacheEngine.retrieve_paged_segments_layerwise, against retrieve_paged_segments on the same data.

Workload (segment_bench.py's): a request of eight 2048-token documents and a 512-token question (16896 tokens), 32
layers x 8 KV heads x 128 channels, bf16, chunk 256, a FlashAttention paged cache of 16-token blocks.  Each document is
stored as a prompt of its own; the segments hit 16384 tokens, seven of the eight documents turned by their start.

Per tier, each step runs the layer-wise form then the whole form (alternating, so both see the same machine state), and
the medians over the steps are reported: host milliseconds from the call to layer 0's ready event having completed, to
the last layer's, and the whole retrieve_paged_segments.  From the layer-wise run's own timing events it also reports
the mean device time between consecutive layers' ready events: on the cuda tier, where nothing waits for a copy, that
is one layer's b200kv_unpack_chunks_layers_rope launch, reported with the bytes it moves (one layer of every hit chunk
read and written) against the H100 SXM's 3.35 TB/s.  A kernel leg times one layer of every hit chunk with the fused
b200kv_unpack_chunks_layers_rope against b200kv_unpack_chunks_layers per document plus b200kv_rope_shift_layers (CUDA
events over --iters launches), with the bytes each moves.  Prints the card's name and power limit with the numbers.

    python segment_layerwise_bench.py [--steps 5] [--warmup 2] [--tiers cpu,cuda,host-cachegen,host-lossless] [--out DIR]
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from segment_bench import BS, CS, D, DOC, H, HBM_BYTES_PER_S, L, MODEL, N_DOCS, QUESTION, card  # noqa: E402


def config(tier):
    from lmcache_b200.config import LMCacheEngineConfig
    if tier in ("cpu", "cuda"):
        return LMCacheEngineConfig(CS, tier, None, None, False, False, None)
    return LMCacheEngineConfig(CS, "cpu", None, None, False, False, tier.split("-")[1])


def engine_leg(tier, steps, warmup, src, slots, tokens, segs):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineMetadata
    from lmcache_b200.rope import RopeSpec
    eng = LMCacheEngine(config(tier), LMCacheEngineMetadata(MODEL, 1, 0, "vllm", "bfloat16"))
    try:
        for a, b in segs:
            eng.store_paged(tokens[a:b], src, slots[a:b])
        if hasattr(eng.engine_, "drain"):
            eng.engine_.drain()
        dst = [(torch.empty_like(k), torch.empty_like(v)) for k, v in src]
        rope = RopeSpec.from_base(D, 10000.0)

        def layerwise():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = eng.retrieve_paged_segments_layerwise(tokens, dst, slots, segs, rope)
            r._upload.ready(0).synchronize()
            t1 = time.perf_counter()
            r.synchronize()
            t2 = time.perf_counter()
            evs = [r._upload.ready(l) for l in range(r.num_layers)]
            distinct = len({id(e) for e in evs}) == r.num_layers
            gap = statistics.mean(evs[l - 1].elapsed_time(evs[l]) for l in range(1, len(evs))) if distinct else None
            return (t1 - t0) * 1e3, (t2 - t0) * 1e3, gap, int(r.ret_mask.sum()), distinct

        def whole():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ret = eng.retrieve_paged_segments(tokens, dst, slots, segs, rope)
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1e3, int(ret.sum())
        for _ in range(warmup):
            layerwise()
            whole()
        lw, wh = [], []
        for _ in range(steps):
            lw.append(layerwise())
            wh.append(whole())
        gaps = [x[2] for x in lw if x[2] is not None]
        out = {"tier": tier, "layer0_ms_p50": round(statistics.median(x[0] for x in lw), 3),
               "last_layer_ms_p50": round(statistics.median(x[1] for x in lw), 3),
               "whole_ms_p50": round(statistics.median(x[0] for x in wh), 3),
               "layer_major": lw[0][4], "tokens": lw[0][3], "whole_tokens": wh[0][1]}
        if gaps:
            us = statistics.median(gaps) * 1e3
            n_tok = lw[0][3]
            nbytes = 2 * n_tok * 2 * H * D * 2           # the fused unpack reads each chunk row and writes it once
            out.update({"per_layer_us": round(us, 1), "per_layer_bytes": nbytes,
                        "per_layer_GBps": round(nbytes / (us * 1e-6) / 1e9, 1),
                        "share_of_3.35TBps": round(nbytes / (us * 1e-6) / HBM_BYTES_PER_S, 3)})
        return out
    finally:
        eng.close()


def kernel_leg(iters, src, slots, segs):
    """One layer of every hit chunk (64 chunks of 256 tokens, the document at 0 copied) into the FlashAttention cache:
    one b200kv_unpack_chunks_layers_rope launch, against one b200kv_unpack_chunks_layers per document plus one
    b200kv_rope_shift_layers -- what the raw tiers launch per layer with and without the fused kernel."""
    import ctypes

    import numpy as np

    from lmcache_b200 import _native as N
    from lmcache_b200.codec import KvView
    from lmcache_b200.rope import RopeSpec, Rotation, chunk_arrays, rope_shift_layers, rope_table, unpack_rope_layers
    view = KvView.from_paged([tuple(t.clone() for t in p) for p in src], slots)
    rope = RopeSpec.from_base(D, 10000.0)
    table = rope_table(torch.tensor([a for a, _ in segs[1:]], dtype=torch.int64, device="cuda"), rope)
    rot = Rotation(rope, table, [-1] + list(range(len(segs) - 1)), [b for _, b in segs])
    placed = [(r, a + k * CS, CS) for r, (a, b) in enumerate(segs) for k in range((b - a) // CS)]
    row = 2 * H * D * 2
    chunks = torch.randn(len(placed) * CS * row // 2, device="cuda").to(torch.bfloat16)
    ptrs = torch.tensor(chunks.data_ptr() + np.arange(len(placed)) * CS * row, dtype=torch.int64, device="cuda")
    arrays = tuple(torch.from_numpy(a).cuda() for a in chunk_arrays(placed, rot.run_rows))
    lo, sot = 0, np.full(segs[-1][1], -1, np.int32)
    for r, (a, b) in enumerate(segs[1:]):
        sot[a:b] = r
    seg = torch.from_numpy(sot).cuda()
    per_doc = (segs[0][1] - segs[0][0]) // CS
    st = torch.cuda.current_stream()

    def fused():
        unpack_rope_layers(view, ptrs.data_ptr(), arrays, CS, 5, 6, rot, st)

    def composed():
        for r, (a, b) in enumerate(segs):
            N.check(N.lib().b200kv_unpack_chunks_layers(ctypes.c_void_p(ptrs.data_ptr() + 8 * r * per_doc), per_doc, CS,
                                                        CS, 0, 5, 6, ctypes.byref(view.desc), a, st.cuda_stream))
        rope_shift_layers(view, 5, 6, lo, seg, table, rope, st)
    n_tok = len(placed) * CS
    n_rot = n_tok - (segs[0][1] - segs[0][0])
    out = []
    for name, fn, nbytes in (("fused", fused, 2 * n_tok * row),
                             ("unpack+shift", composed, 2 * n_tok * row + 2 * n_rot * H * D * 2)):
        for _ in range(5):
            fn()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(iters):
            fn()
        t1.record()
        t1.synchronize()
        us = t0.elapsed_time(t1) * 1e3 / iters
        out.append({"kernel": name, "per_layer_us": round(us, 1), "bytes": nbytes,
                    "GBps": round(nbytes / (us * 1e-6) / 1e9, 1),
                    "share_of_3.35TBps": round(nbytes / (us * 1e-6) / HBM_BYTES_PER_S, 3)})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--tiers", default="cpu,cuda,host-cachegen,host-lossless")
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "segment_layerwise_bench measures on a CUDA device; there is no CPU fallback"
    name, power = card()
    T = N_DOCS * DOC + QUESTION
    gen = torch.Generator(device="cuda").manual_seed(0)
    nb = (T + BS - 1) // BS + 8
    src = [tuple(torch.randn(nb * BS, H, D, device="cuda", generator=gen).to(torch.bfloat16).view(nb, BS, H, D)
                 for _ in range(2)) for _ in range(L)]
    slots = (torch.randperm(nb, device="cuda", generator=gen)[:, None] * BS +
             torch.arange(BS, device="cuda")[None, :]).flatten()[:T].contiguous()
    tokens = torch.randint(0, 32000, (T,), generator=torch.Generator().manual_seed(1))
    segs = [(i * DOC, (i + 1) * DOC) for i in range(N_DOCS)]
    results = {"card": name, "power_limit": power, "workload": {"L": L, "H": H, "D": D, "dtype": "bfloat16",
               "chunk": CS, "tokens": T, "documents": N_DOCS, "doc_tokens": DOC, "question_tokens": QUESTION},
               "engine": []}
    results["kernel"] = kernel_leg(args.iters, src, slots, segs)
    for r in results["kernel"]:
        print(json.dumps(r), flush=True)
    for tier in args.tiers.split(","):
        r = engine_leg(tier, args.steps, args.warmup, src, slots, tokens, segs)
        results["engine"].append(r)
        print(json.dumps(r), flush=True)
    print(json.dumps({"card": name, "power_limit": power}))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "segment_layerwise_bench.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
