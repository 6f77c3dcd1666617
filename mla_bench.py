"""Latent (MLA) KV through the codec at DeepSeek-V3's geometry: the one-plane path (container version 4) against the
workaround of coding the latent tensor as both K and V (version 3 of the pair `(latent, latent)`).

    python mla_bench.py [--tokens 8192] [--steps 20] [--warmup 3]
    python mla_bench.py --engine [--engine-tokens 8192,65536] [--steps 5] [--warmup 1]

61 layers, D = 576 (kv_lora_rank 512 + rope 64), bf16, 256-token chunks, bench.py's kv8d distribution.  The two legs
alternate in one process; per leg: encode and decode GB/s of LATENT bytes (L * T * 576 * 2, the same for both legs;
CUDA events, medians), container bytes, and (one-plane leg) the reconstruction error against the input, max abs and
relative RMS per layer.  Prints one JSON line with the card's name and power limit; writes nothing.

With --engine the same latent goes through LMCacheEngine instead (engine_legs): an MLA engine (use_mla) against the
pair workaround through a (K, V) engine, on the CacheGen host tier, the raw cpu tier and the layer-wise retrieve."""
import argparse
import json
import statistics
import subprocess
import time

import torch

L, D, CHUNK = 61, 576, 256


def _synth_latent(T, seed):
    """bench.py's kv8d (synth_kv_torch) at this geometry, generated the same way: N(0,1) * sigma[l, c], sigma ~
    LogNormal(0, 0.5) clipped to [0.1, 8], 1% outlier channels x10, drawn in 512-token blocks and cast to bf16 block by
    block (no fp32 tensor of the whole KV).  [L, T, D]"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    sigma = torch.exp(0.5 * torch.randn((L, 1, D), device="cuda", generator=g)).clamp_(0.1, 8.0)
    outl = torch.rand((L, 1, D), device="cuda", generator=g) < 0.01
    sigma = torch.where(outl, sigma * 10.0, sigma)
    x = torch.empty((L, T, D), dtype=torch.bfloat16, device="cuda")
    step = 512
    for t0 in range(0, T, step):
        n = min(step, T - t0)
        x[:, t0:t0 + n] = (torch.randn((L, n, D), device="cuda", generator=g) * sigma).to(torch.bfloat16)
    return x


def _power_limit_w():
    try:
        import pynvml as n
        n.nvmlInit()
        h = n.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        return n.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
    except Exception:       # noqa: BLE001 -- no NVML: ask nvidia-smi (a query, nothing is set)
        try:
            out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                                  "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=10)
            return float(out.stdout.strip().splitlines()[0])
        except Exception:   # noqa: BLE001
            return None


def _timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


_CFG = dict(key_first_layers=10, key_second_layers=20, key_third_layers=L, key_first_bins=32, key_second_bins=16,
            key_third_bins=16, value_first_layers=2, value_first_bins=32, value_second_bins=16)


def _engine(tier, mla):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    cfg = LMCacheEngineConfig(CHUNK, "cpu", None, None, False, False, "cachegen" if tier == "host_cachegen" else None,
                              cachegen_config=_CFG)
    return LMCacheEngine(cfg, LMCacheEngineMetadata("deepseek-ai/DeepSeek-V3", 1, 0, "vllm", "bfloat16", mla))


def _held_bytes(eng):
    """bytes the local tier keeps: CacheGen containers, or the raw tier's page-locked chunk blobs"""
    f = getattr(eng.engine_, "host_bytes", None)
    if f is not None:
        return int(f())
    return sum(v.host.numel() * v.host.element_size() for v in eng.engine_.dict.values())


def _wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def engine_legs(T, steps, warmup):
    """LMCacheEngine.store / retrieve of one T-token latent: the MLA engine (one plane per layer) against the pair
    workaround (the latent as K and V through a (K, V) engine), on the CacheGen host tier and the raw cpu tier, plus the
    layer-wise retrieve on the CacheGen host tier (host ms until layer 0 and until the last layer are ready).  Host wall
    ms around a device synchronise, medians; both kinds alternate step by step."""
    x = _synth_latent(T, seed=2)
    tokens = torch.arange(T, dtype=torch.int64)
    kvs = {"mla": tuple(x[l] for l in range(L)),
           "pair_workaround": tuple((x[l].unsqueeze(1), x[l].unsqueeze(1)) for l in range(L))}
    res = {}
    for tier in ("host_cachegen", "raw_cpu"):
        engines = {k: _engine(tier, k == "mla") for k in kvs}
        ms = {k: {"store": [], "retrieve": [], "layer0": [], "last_layer": []} for k in kvs}
        for step in range(warmup + steps):
            for k, eng in engines.items():
                s, _ = _wall(lambda: eng.store(tokens, kvs[k], skip_existing=False))
                r, (kv, mask) = _wall(lambda: eng.retrieve(tokens))
                assert int(mask.sum()) == T
                del kv
                if step >= warmup:
                    ms[k]["store"].append(s)
                    ms[k]["retrieve"].append(r)
                if tier != "host_cachegen":
                    continue
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                lw = eng.retrieve_layerwise(tokens)
                lw._upload.ready(0).synchronize()
                t1 = time.perf_counter()
                lw.synchronize()
                t2 = time.perf_counter()
                del lw
                if step >= warmup:
                    ms[k]["layer0"].append((t1 - t0) * 1e3)
                    ms[k]["last_layer"].append((t2 - t0) * 1e3)
        for k, eng in engines.items():
            leg = {f"{op}_ms": statistics.median(v) for op, v in ms[k].items() if v}
            leg["bytes_held"] = _held_bytes(eng)
            res.setdefault(tier, {})[k] = leg
            eng.close()
        del engines
        torch.cuda.empty_cache()
    for tier, legs in res.items():
        legs["ratios_mla_over_pair"] = {k: legs["mla"][k] / legs["pair_workaround"][k] for k in legs["mla"]}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--engine", action="store_true",
                    help="run the LMCacheEngine legs instead of the codec legs, at --engine-tokens")
    ap.add_argument("--engine-tokens", default="8192,65536")
    args = ap.parse_args()
    from lmcache_b200.codec import CacheGenCodec, KvView
    if args.engine:
        torch.cuda.set_device(0)
        props = torch.cuda.get_device_properties(0)
        legs = {int(t): engine_legs(int(t), args.steps, args.warmup) for t in args.engine_tokens.split(",")}
        print(json.dumps(dict(metric="mla_latent_engine", card=props.name, power_limit_w=_power_limit_w(), layers=L,
                              D=D, chunk=CHUNK, dtype="bf16", data="kv8d", steps=args.steps, tokens=legs)))
        return
    T = args.tokens
    torch.cuda.set_device(0)
    x = _synth_latent(T, seed=1)
    cfg = dict(key_first_layers=10, key_second_layers=20, key_third_layers=L, key_first_bins=32, key_second_bins=16,
               key_third_bins=16, value_first_layers=2, value_first_bins=32, value_second_bins=16)
    codec = CacheGenCodec("deepseek-ai/DeepSeek-V3", cachegen_config=cfg)
    nchunk = (T + CHUNK - 1) // CHUNK
    ntok = [min(CHUNK, T - j * CHUNK) for j in range(nchunk)]
    starts = [j * CHUNK for j in range(nchunk)]
    latent_bytes = L * T * D * 2
    legs = {
        "one_plane": (KvView.from_blob(x, "vllm"), lambda: torch.empty_like(x),
                      lambda o: KvView.from_blob(o, "vllm"), lambda o: o),
        "pair_workaround": (KvView.from_tuple([(x[l].unsqueeze(1), x[l].unsqueeze(1)) for l in range(L)], "vllm"),
                            lambda: torch.empty((L, 2, T, 1, D), dtype=x.dtype, device="cuda"),
                            lambda o: KvView.from_tuple([(o[l, 0], o[l, 1]) for l in range(L)], "vllm"),
                            lambda o: o[:, 0, :, 0]),
    }
    outs = {k: mk() for k, (_, mk, _, _) in legs.items()}
    dsts = {k: mkv(outs[k]) for k, (_, _, mkv, _) in legs.items()}
    stride = {k: codec.out_stride(L, 1, D, CHUNK, v.latent) for k, (v, _, _, _) in legs.items()}
    bufs = {k: torch.empty(stride[k] * nchunk + 1024, dtype=torch.uint8, device="cuda") for k in legs}
    enc_ms = {k: [] for k in legs}
    dec_ms = {k: [] for k in legs}
    batches = {}
    for step in range(args.warmup + args.steps):
        for k, (view, _, _, _) in legs.items():          # the legs alternate: same clocks, same thermal state
            holder = {}
            e = _timed(lambda: holder.__setitem__("t", codec.encode_async(view, 0, T, CHUNK, out=bufs[k])))
            batches[k] = holder["t"].wait()
            d = _timed(lambda: codec.decode_device_batch(batches[k], ntok, dsts[k], starts))
            if step >= args.warmup:
                enc_ms[k].append(e)
                dec_ms[k].append(d)
    torch.cuda.synchronize()
    res = {}
    for k, (_, _, _, first) in legs.items():
        res[k] = dict(encode_GBps=latent_bytes / statistics.median(enc_ms[k]) / 1e6,
                      decode_GBps=latent_bytes / statistics.median(dec_ms[k]) / 1e6,
                      encode_ms=statistics.median(enc_ms[k]), decode_ms=statistics.median(dec_ms[k]),
                      container_bytes=int(sum(batches[k].sizes)))
    # both legs decode the latent plane to the same bits; the one-plane leg's error against the input
    same = torch.equal(outs["one_plane"].view(torch.int16),
                       outs["pair_workaround"][:, 0, :, 0].contiguous().view(torch.int16))
    max_abs, rel_rms = torch.empty(L), torch.empty(L)
    for l in range(L):                                      # one layer at a time: no fp32 copy of the whole KV
        xf, err = x[l].float(), outs["one_plane"][l].float() - x[l].float()
        max_abs[l] = err.abs().amax()
        rel_rms[l] = err.pow(2).mean().sqrt() / xf.pow(2).mean().sqrt()
    res["one_plane"]["max_abs_err_per_layer"] = [round(v, 5) for v in max_abs.tolist()]
    res["one_plane"]["rel_rms_err_per_layer"] = [round(v, 5) for v in rel_rms.tolist()]
    props = torch.cuda.get_device_properties(0)
    line = dict(metric="mla_latent_codec", card=props.name, power_limit_w=_power_limit_w(), layers=L, D=D,
                tokens=T, chunk=CHUNK, dtype="bf16", data="kv8d", latent_bytes=latent_bytes, steps=args.steps,
                legs_decode_identical=bool(same),
                bytes_ratio=res["one_plane"]["container_bytes"] / res["pair_workaround"]["container_bytes"],
                encode_time_ratio=res["one_plane"]["encode_ms"] / res["pair_workaround"]["encode_ms"],
                decode_time_ratio=res["one_plane"]["decode_ms"] / res["pair_workaround"]["decode_ms"],
                max_rel_rms_err=max(rel_rms.tolist()), **res)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
