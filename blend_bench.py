"""CacheBlend's selective recomputation on the H100: the deviation and select kernels, BlendPlan.check, and a synthetic
quality table.

Workload (segment_bench.py's): a RAG request of eight 2048-token documents and a 512-token question (T = 16896 tokens),
32 layers x 8 KV heads x 128 channels, bf16, 16-token blocks.  Legs:

  * deviation: b200kv_blend_deviation over all T tokens of one layer, in the FlashAttention, FlashInfer block-strided,
    PagedAttention split and dense (retrieve_segments' views) layouts, timed with CUDA events over many launches; bytes
    = 2 * n * H * D * 2 + 4 n (fresh and cached key rows read, dev written) against the H100 SXM's 3.35 TB/s.
  * select: b200kv_blend_select at n = 16896 and n = 2^20 (85 % candidates, k = 15 % of them), against torch.topk of the
    masked deviations followed by torch.sort of the indices.
  * check: BlendPlan.check at the first check layer with a device sync, keeping 100 % and 15 % of the retrieved tokens.
  * quality: the toy decoder of tests/blend_model.py (random weights, not a real model) with two documents stored alone
    on the raw cuda tier and served inside [system][A][B][question]; the relative error of the question's last-layer
    output against a full prefill, at ratios 0, 0.05, 0.15, 0.3 and 1, for the deviation's choice and for a random
    choice of the same size.

Prints the card's name and power limit with the numbers, one JSON document; --out DIR also writes it there.

    python blend_bench.py [--iters 200] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

L, H, D, BS = 32, 8, 128, 16
N_DOCS, DOC, QUESTION = 8, 2048, 512
T = N_DOCS * DOC + QUESTION
HBM_BYTES_PER_S = 3.35e12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return name, out


def event_us(fn, iters):
    for _ in range(5):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / iters


def views():
    """the same key rows of layers 0..1 in the four layouts, over T tokens in shuffled blocks"""
    from lmcache_b200.codec import KvView
    nb = (T + BS - 1) // BS + 8
    g = torch.Generator(device="cuda").manual_seed(0)
    blocks = torch.randperm(nb, device="cuda", generator=g)
    slots = (blocks[:, None] * BS + torch.arange(BS, device="cuda")[None, :]).flatten()[:T].contiguous()
    out = {}
    flash = [tuple(torch.randn(nb, BS, H, D, generator=g, device="cuda").to(torch.bfloat16) for _ in range(2))
             for _ in range(L)]
    out["flash"] = KvView.from_paged(flash, slots)
    strided = []
    for k, v in flash:
        kv = torch.stack((k, v), dim=1)                      # FlashInfer: [nb, 2, bs, H, D]
        strided.append((kv[:, 0], kv[:, 1]))
    out["strided"] = KvView.from_paged(strided, slots)
    split = []
    for k, v in flash:
        c = torch.empty(2, nb, BS * H * D, dtype=torch.bfloat16, device="cuda")
        kc, vc = c[0].view(nb, H, D // 8, BS, 8), c[1].view(nb, H, D, BS)
        kc.copy_(k.view(nb, BS, H, D // 8, 8).permute(0, 2, 3, 1, 4))
        vc.copy_(v.view(nb, BS, H, D).permute(0, 2, 3, 1))
        split.append((kc, vc))
    out["split"] = KvView.from_paged(split, slots)
    blob = torch.empty(L, 2, T, H, D, dtype=torch.bfloat16, device="cuda")
    for l, (k, v) in enumerate(flash):
        blob[l, 0], blob[l, 1] = k.view(-1, H, D)[slots], v.view(-1, H, D)[slots]
    out["dense"] = KvView.from_tuple(tuple((blob[l, 0], blob[l, 1]) for l in range(L)), "vllm")
    return out, flash, slots


def deviation_leg(vs, iters):
    from lmcache_b200.blend import deviation
    st = torch.cuda.current_stream()
    tok = torch.arange(T, device="cuda")
    fresh = torch.randn(T, H * D, device="cuda").to(torch.bfloat16)
    dev = torch.empty(T, dtype=torch.float32, device="cuda")
    nbytes = 2 * T * H * D * 2 + 4 * T
    res, ref = {}, None
    for name, v in vs.items():
        us = event_us(lambda: deviation(v, 1, tok, fresh, H * D, dev, st), iters)
        torch.cuda.synchronize()
        if ref is None:
            ref = dev.clone()
        res[name] = {"us": round(us, 2), "bytes": nbytes, "frac_of_3.35TBps": round(nbytes / (us * 1e-6) / HBM_BYTES_PER_S, 3),
                     "bit_identical_to_flash": bool(torch.equal(dev, ref))}
    return res


def select_leg(iters):
    from lmcache_b200.blend import select
    st = torch.cuda.current_stream()
    res = {}
    for n in (T, 1 << 20):
        g = torch.Generator(device="cuda").manual_seed(n)
        dev = torch.rand(n, generator=g, device="cuda") * 100
        cand = (torch.rand(n, generator=g, device="cuda") < 0.85).to(torch.uint8)
        n_cand = int(cand.sum())
        k = -(-15 * n_cand // 100)
        n_out = n - n_cand + k
        us = event_us(lambda: select(dev, cand, k, n_out, st), iters)
        masked = dev.masked_fill(cand == 0, float("-inf"))

        def torch_way():
            return torch.sort(torch.topk(masked, k).indices).values
        us_t = event_us(torch_way, iters)
        got = select(dev, cand, k, n_out, st)[n - n_cand:]
        same = bool(torch.equal(got, torch_way()))
        res[str(n)] = {"k": k, "select_us": round(us, 2), "topk_sort_us": round(us_t, 2),
                       "same_candidates_as_topk": same}
    return res


def check_leg(vs, reps):
    from lmcache_b200.blend import BlendPlan, BlendSpec
    mask = torch.ones(T, dtype=torch.bool)
    mask[:DOC] = False                                      # the first document sits at token 0: recomputed
    mask[-QUESTION:] = False
    fresh = torch.randn(T, H, D, device="cuda").to(torch.bfloat16)
    res = {}
    for r in (1.0, 0.15):
        ts = []
        for i in range(reps + 3):
            plan = BlendPlan(vs["flash"], mask, BlendSpec([1], [r]), vs["flash"].slots)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            plan.check(1, fresh)
            torch.cuda.synchronize()
            if i >= 3:
                ts.append((time.perf_counter() - t0) * 1e6)
        ts.sort()
        res[f"{int(r * 100)}%"] = {"median_us": round(ts[len(ts) // 2], 1), "min_us": round(ts[0], 1),
                                    "rows_kept": plan.sizes[0][2]}
    return res


def quality_leg():
    import blend_model as M
    from lmcache_b200.blend import BlendSpec, BlendStep
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    from lmcache_b200.rope import RopeSpec
    model = M.ToyDecoder(seed=0)
    g = torch.Generator().manual_seed(1)
    sysp, A, B, q = (torch.randint(0, M.VOCAB, (n,), generator=g) for n in (12, 48, 40, 10))
    eng = LMCacheEngine(LMCacheEngineConfig(16, "cuda", None, None, False, False, None),
                        LMCacheEngineMetadata("lmsys/longchat-7b-16k", 1, 0, "vllm", "bfloat16"))
    try:
        for doc in (A, B):
            c = M.PagedKV("flash")
            s = torch.arange(len(doc), device="cuda")
            model.prefill(doc.cuda(), c, s)
            eng.store_paged(doc, c.caches, s)
        tokens = torch.cat([sysp, A, B, q])
        n = len(tokens)
        segs = [(12, 60), (60, 100)]
        slots = torch.arange(n, device="cuda")
        full = model.prefill(tokens.cuda(), M.PagedKV("flash"), slots)[-10:]
        rope = RopeSpec(M.D, model.inv_freq, "neox")
        rows = []
        for r in (0.0, 0.05, 0.15, 0.3, 1.0):
            errs = {}
            for how in ("deviation", "random"):
                cache = M.PagedKV("flash")
                ret = eng.retrieve_paged_segments(tokens, cache.caches, slots, segs, rope)
                plan = eng.blend_paged(cache.caches, slots, ret, BlendSpec([1], [r]))
                choose = None
                if how == "random":
                    def choose(layer, step, ret=ret):
                        forced = torch.nonzero(~ret).flatten()
                        retr = torch.nonzero(ret).flatten()
                        k = step.tokens.numel() - forced.numel()
                        pick = retr[torch.randperm(retr.numel(), generator=torch.Generator().manual_seed(5))[:k]]
                        t = torch.cat([forced, pick.sort().values]).cuda()
                        return BlendStep(t, t, slots[t])
                x, _, _ = model.blended_prefill(tokens.cuda(), cache, slots, plan, choose=choose)
                errs[how] = round(M.rel_err(x[-10:], full), 4)
            rows.append({"ratio": r, "rel_err_deviation": errs["deviation"], "rel_err_random": errs["random"]})
        return {"model": "toy decoder, random weights (not a real model): 4 layers, GQA 4q/2kv heads, D 64",
                "rows": rows}
    finally:
        eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    vs, _, _ = views()
    res = {"card": name, "power_limit": power, "workload": f"T={T} L={L} H={H} D={D} bf16 bs={BS}",
           "deviation": deviation_leg(vs, a.iters), "select": select_leg(a.iters), "check": check_leg(vs, 20),
           "quality": quality_leg()}
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "blend_bench.json"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
