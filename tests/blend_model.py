"""A seeded toy decoder for the blend tests and blend_bench.py: random weights, not a trained model.

4 layers, 4 query heads over 2 KV heads (GQA) of D = 64, neox RoPE, RMS norms, fp32 compute, and its KV in a bf16 paged
cache (FlashAttention rows or PagedAttention's split blocks).  prefill() is a full prefill; blended_prefill() is
CacheBlend's: it computes every token up to the first check layer, asks BlendPlan.check which tokens to keep computing,
and from there on computes those only, attending to the cache, whose other rows hold the retrieved KV."""
import math

import torch

L, HQ, HKV, D, HIDDEN, FFN, VOCAB = 4, 4, 2, 64, 256, 512, 1000


class PagedKV:
    """L layers of a paged bf16 (K, V) cache of nb blocks of bs slots, in the FlashAttention ("flash") or split
    PagedAttention ("split") layout; caches is what the engine's paged calls take"""

    def __init__(self, kind, nb=16, bs=16, device="cuda"):
        self.kind, self.nb, self.bs = kind, nb, bs
        x = 8                                                    # 16 bytes of bf16
        if kind == "flash":
            self.caches = [tuple(torch.zeros(nb, bs, HKV, D, dtype=torch.bfloat16, device=device) for _ in range(2))
                           for _ in range(L)]
        else:
            self.caches = []
            for _ in range(L):
                c = torch.zeros(2, nb, bs * HKV * D, dtype=torch.bfloat16, device=device)
                self.caches.append((c[0].view(nb, HKV, D // x, bs, x), c[1].view(nb, HKV, D, bs)))

    def write(self, l, slots, k, v):
        kc, vc = self.caches[l]
        k, v = k.to(torch.bfloat16), v.to(torch.bfloat16)
        if self.kind == "flash":
            kc.view(-1, HKV, D)[slots] = k
            vc.view(-1, HKV, D)[slots] = v
        else:
            b, o = torch.div(slots, self.bs, rounding_mode="floor"), torch.remainder(slots, self.bs)
            kc[b, :, :, o, :] = k.view(-1, HKV, D // 8, 8)
            vc[b, :, :, o] = v

    def read(self, l, slots):
        """(K, V) of the slots as fp32 [n, HKV, D]"""
        kc, vc = self.caches[l]
        if self.kind == "flash":
            return kc.view(-1, HKV, D)[slots].float(), vc.view(-1, HKV, D)[slots].float()
        b, o = torch.div(slots, self.bs, rounding_mode="floor"), torch.remainder(slots, self.bs)
        return kc[b, :, :, o, :].reshape(-1, HKV, D).float(), vc[b, :, :, o].float()


class ToyDecoder:
    def __init__(self, seed=0, device="cuda", qk_gain=1.0):
        g = torch.Generator().manual_seed(seed)

        def w(*shape, scale=1.0):
            return (torch.randn(*shape, generator=g) * scale).to(device)
        self.emb = w(VOCAB, HIDDEN)
        self.layers = [dict(wq=w(HIDDEN, HQ * D, scale=qk_gain / math.sqrt(HIDDEN)),
                            wk=w(HIDDEN, HKV * D, scale=qk_gain / math.sqrt(HIDDEN)),
                            wv=w(HIDDEN, HKV * D, scale=1 / math.sqrt(HIDDEN)),
                            wo=w(HQ * D, HIDDEN, scale=1 / math.sqrt(HQ * D)),
                            w1=w(HIDDEN, FFN, scale=1 / math.sqrt(HIDDEN)),
                            w2=w(FFN, HIDDEN, scale=1 / math.sqrt(FFN))) for _ in range(L)]
        self.inv_freq = 1.0 / (10000.0 ** (torch.arange(0, D, 2, dtype=torch.float) / D))   # float32, CPU: RopeSpec's
        self._inv = self.inv_freq.to(device)

    @staticmethod
    def _norm(x):
        return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-6)

    def _rope(self, x, pos):
        ang = pos.float()[:, None] * self._inv[None, :]
        c, s = torch.cos(ang)[:, None, :], torch.sin(ang)[:, None, :]
        a, b = x[..., :D // 2], x[..., D // 2:]
        return torch.cat((a * c - b * s, b * c + a * s), dim=-1)

    def qkv(self, l, x, pos):
        p, h = self.layers[l], self._norm(x)
        q = (h @ p["wq"]).view(-1, HQ, D)
        k = (h @ p["wk"]).view(-1, HKV, D)
        v = (h @ p["wv"]).view(-1, HKV, D)
        return self._rope(q, pos), self._rope(k, pos), v

    def finish(self, l, x, q, pos, K, V):
        """attention of the rows at positions pos over the request's keys K, V (token order), then the MLP"""
        p, T = self.layers[l], K.shape[0]
        rep = HQ // HKV
        Kx, Vx = K.repeat_interleave(rep, dim=1), V.repeat_interleave(rep, dim=1)
        logits = torch.einsum("nhd,thd->hnt", q, Kx) / math.sqrt(D)
        future = torch.arange(T, device=x.device)[None, :] > pos[:, None]
        logits = logits.masked_fill(future[None], float("-inf"))
        o = torch.einsum("hnt,thd->nhd", torch.softmax(logits, dim=-1), Vx).reshape(-1, HQ * D)
        x = x + o @ p["wo"]
        return x + torch.nn.functional.gelu(self._norm(x) @ p["w1"]) @ p["w2"]

    def prefill(self, tokens, cache, slots):
        """full prefill of tokens at positions 0..T-1, its KV written to cache at slots; the last layer's output of every
        token"""
        T = tokens.numel()
        x, pos = self.emb[tokens], torch.arange(T, device=slots.device)
        for l in range(L):
            q, k, v = self.qkv(l, x, pos)
            cache.write(l, slots, k, v)
            K, V = cache.read(l, slots)
            x = self.finish(l, x, q, pos, K, V)
        return x

    def blended_prefill(self, tokens, cache, slots, plan, wait=None, choose=None):
        """CacheBlend's prefill over a cache whose retrieved rows are in place: (the last layer's output of the tokens
        computed to the end, those tokens, the BlendSteps).  Rows are kept in token order; the fresh keys go to
        plan.check in the plan's row order.  wait(l) runs before layer l (a layer-wise retrieve's wait_layer);
        choose(layer, step) may replace a step's choice (the random baseline of blend_bench.py)."""
        T = tokens.numel()
        x = self.emb[tokens]
        toks = torch.arange(T, device=slots.device)
        perm = toks                                          # the plan's row i is our row perm[i]
        steps = []
        for l in range(L):
            if wait is not None:
                wait(l)
            q, k, v = self.qkv(l, x, toks)
            step = None
            if l in plan.spec.check_layers:
                step = plan.check(l, k[perm].to(torch.bfloat16))
                if choose is not None:
                    step = choose(l, step)
                steps.append(step)
            cache.write(l, slots[toks], k, v)                # the model writes the KV it computed
            K, V = cache.read(l, slots)
            x = self.finish(l, x, q, toks, K, V)
            if step is not None:
                order = torch.argsort(step.tokens)
                x = x[perm][step.rows][order]
                toks = step.tokens[order]
                perm = torch.argsort(order)
        return x, toks, steps


def rel_err(got, want):
    return float((got - want).norm() / want.norm())
