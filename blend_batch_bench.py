"""A batched blend on the H100: b200kv_blend_select_batch against B one-request selects, and BatchBlendPlan.check
against a loop of BlendPlan.check over the same requests.

Workloads, 8 KV heads x 128 channels bf16, 16-token blocks (only the check layer's key plane is read, so the cache holds
the two layers the check uses):
  * 8 x 16896: blend_bench.py's request (eight 2048-token documents and a 512-token question), eight times;
  * 64 x 2048: 64 prompts of 2048 tokens;
  * 256 mixed: 32 RAG prompts of 4096 tokens and 224 one-token decode rows.
Each RAG request retrieved every token but its first 512 and its last 256 (none for a decode row); the budget is 15 %.
Legs, each pair run alternately and repeated, medians reported:
  * select: one b200kv_blend_select_batch over the batch's deviations against B b200kv_blend_select calls over the same
    rows, timed with CUDA events; and at B = 1 (n = 16896 and n = 2^20, 85 % candidates, k = 15 %) the segmented kernels
    against b200kv_blend_select;
  * check: BatchBlendPlan.check against the loop of BlendPlan.check, wall time with a device sync.

Prints the card's name and power limit with the numbers, one JSON document; --out DIR also writes it there.

    python blend_batch_bench.py [--iters 50] [--reps 5] [--out DIR]
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from blend_bench import card, event_us  # noqa: E402

H, D, BS = 8, 128, 16


def workloads():
    rag = lambda n: (n, 512, n - 256)                      # noqa: E731  (tokens, retrieved range)
    return {"8x16896": [rag(16896)] * 8, "64x2048": [rag(2048)] * 64,
            "256-mixed": [rag(4096) if i % 8 == 0 else (1, 0, 0) for i in range(256)]}


def masks_of(reqs):
    out = []
    for n, a, b in reqs:
        m = torch.zeros(n, dtype=torch.bool)
        m[a:b] = True
        out.append(m)
    return out


def med(xs):
    xs = sorted(xs)
    return round(xs[len(xs) // 2], 2)


def select_leg(iters, reps):
    from lmcache_b200.blend import select, select_batch
    st = torch.cuda.current_stream()
    res = {}
    for name, reqs in workloads().items():
        masks = masks_of(reqs)
        n = sum(m.numel() for m in masks)
        g = torch.Generator(device="cuda").manual_seed(n)
        dev = torch.rand(n, generator=g, device="cuda") * 100
        cand = torch.cat(masks).to(torch.uint8).cuda()
        starts = [0]
        for m in masks:
            starts.append(starts[-1] + m.numel())
        ks = [-(-15 * int(m.sum()) // 100) for m in masks]
        outs = [m.numel() - int(m.sum()) + k for m, k in zip(masks, ks)]
        seg_t, k_t = torch.tensor(starts, device="cuda"), torch.tensor(ks, device="cuda")
        slices = [(dev[a:b], cand[a:b], k, o) for a, b, k, o in zip(starts, starts[1:], ks, outs)]

        def batched():
            return select_batch(dev, cand, seg_t, k_t, sum(outs), st)

        def loop():
            return [select(d, c, k, o, st) for d, c, k, o in slices]
        same = torch.equal(batched(), torch.cat([r + a for r, a in zip(loop(), starts)]))
        tb, tl = [], []
        for _ in range(reps):
            tb.append(event_us(batched, iters))
            tl.append(event_us(loop, iters))
        res[name] = {"B": len(reqs), "n": n, "batched_us": med(tb), "loop_of_selects_us": med(tl),
                     "identical_rows": bool(same)}
    for n in (16896, 1 << 20):
        g = torch.Generator(device="cuda").manual_seed(n)
        dev = torch.rand(n, generator=g, device="cuda") * 100
        cand = (torch.rand(n, generator=g, device="cuda") < 0.85).to(torch.uint8)
        n_cand = int(cand.sum())
        k = -(-15 * n_cand // 100)
        n_out = n - n_cand + k
        seg_t, k_t = torch.tensor([0, n], device="cuda"), torch.tensor([k], device="cuda")
        same = torch.equal(select_batch(dev, cand, seg_t, k_t, n_out, st), select(dev, cand, k, n_out, st))
        tb, t1 = [], []
        for _ in range(reps):
            tb.append(event_us(lambda: select_batch(dev, cand, seg_t, k_t, n_out, st), iters))
            t1.append(event_us(lambda: select(dev, cand, k, n_out, st), iters))
        res[f"B=1 n={n}"] = {"segmented_us": med(tb), "b200kv_blend_select_us": med(t1), "identical_rows": bool(same)}
    return res


def cache_for(n):
    from lmcache_b200.codec import KvView
    nb = -(-n // BS) + 4
    g = torch.Generator(device="cuda").manual_seed(0)
    caches = [tuple(torch.randn(nb, BS, H, D, generator=g, device="cuda").to(torch.bfloat16) for _ in range(2))
              for _ in range(2)]
    blocks = torch.randperm(nb, device="cuda", generator=g)
    slots = (blocks[:, None] * BS + torch.arange(BS, device="cuda")[None, :]).flatten()[:n].contiguous()
    return caches, slots, KvView


def check_leg(reps):
    from lmcache_b200.blend import BatchBlendPlan, BlendPlan, BlendSpec
    spec = BlendSpec([1], [0.15])
    res = {}
    for name, reqs in workloads().items():
        masks = masks_of(reqs)
        n = sum(m.numel() for m in masks)
        caches, slots, KvView = cache_for(n)
        starts = [0]
        for m in masks:
            starts.append(starts[-1] + m.numel())
        fresh = torch.randn(n, H, D, device="cuda").to(torch.bfloat16)
        views = [KvView.from_paged(caches, slots[a:b]) for a, b in zip(starts, starts[1:])]
        bview = KvView.from_paged(caches, slots)

        def batched():
            plan = BatchBlendPlan(bview, masks, spec, slots)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            plan.check(1, fresh)
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1e6

        def loop():
            plans = [BlendPlan(v, m, spec, slots[a:b]) for v, m, a, b in zip(views, masks, starts, starts[1:])]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for p, a, b in zip(plans, starts, starts[1:]):
                p.check(1, fresh[a:b])
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1e6
        for _ in range(3):
            batched(), loop()
        tb, tl = [], []
        for _ in range(reps):
            tb.append(batched())
            tl.append(loop())
        res[name] = {"B": len(reqs), "n": n, "batched_check_us": med(tb), "loop_of_checks_us": med(tl)}
    # B = 1: blend_bench.py's request, BlendPlan.check
    reqs = workloads()["8x16896"][:1]
    masks = masks_of(reqs)
    caches, slots, KvView = cache_for(16896)
    view = KvView.from_paged(caches, slots)
    fresh = torch.randn(16896, H, D, device="cuda").to(torch.bfloat16)
    ts = []
    for i in range(reps + 3):
        plan = BlendPlan(view, masks[0], spec, slots)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        plan.check(1, fresh)
        torch.cuda.synchronize()
        if i >= 3:
            ts.append((time.perf_counter() - t0) * 1e6)
    res["B=1 BlendPlan.check n=16896"] = {"median_us": med(ts)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    res = {"card": name, "power_limit": power, "shape": f"H={H} D={D} bf16 bs={BS}, budget 15 %",
           "select": select_leg(a.iters, a.reps), "check": check_leg(max(a.reps, 20))}
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "blend_batch_bench.json"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
