#!/usr/bin/env python
"""remote_layerwise_bench.py -- what a layer-by-layer retrieve from the lm:// remote tier gives a decode replica, on one GPU.

  python remote_layerwise_bench.py [--steps K] [--warmup W] [--tokens 8192,65536] [--serde cachegen,lossless]
                                   [--ffn F]

Model: L = 32 layers, 8 KV heads x 128 dims, bf16 (bench.py's synthetic SURVEY 8d data, its first 8 heads), chunk 256,
stored once per size and serde into a native lm:// server in this process (loopback, LMCACHE_B200_REMOTE_CONNS
connections).  Two legs alternate in one process, each reading the whole sequence back:
  retrieve    LMCacheEngine.retrieve(), then the stand-in forward pass
  layerwise   retrieve_layerwise(), then the forward pass, which waits on wait_layer(l) before layer l's GEMM
The forward pass is one [T, 4096] x [4096, F] bf16 GEMM per layer (F = --ffn, default 14336), as layerwise_store_bench.py.
Per leg (medians over the timed steps):
  retrieve_ms   host time of retrieve() until its KV is on the device (retrieve leg)
  call_ms       host time of the retrieve_layerwise() call: the OPENs and the match (layerwise leg)
  ready_ms      [layer 0, layer L/2, layer L-1]: device time from the call's start to the layer's ready event
  enqueue_ms    the uploader's host time per layer, not counting its waits for the layer's bytes (mean over the layers)
  wait_ms       the uploader's wait per layer for the layer's bytes to arrive (mean over the layers)
  match_ms      host time of the call's match (OPENs in flight, header checks)
  open_ms       host time of one OPEN exchange on a pool thread (mean; the slab allocation and the prefix included)
  read_ms       host time of one READ exchange on a network thread (mean)
  thread_ms     one network thread's whole life (mean; read_ms x its READs + its own Python work)
  step_ms       the call's start -> the forward pass's end (device events; both legs)
  fetched_MB, reads  bytes fetched by OPEN / READ and READ round trips per step (layerwise leg)
Every step's KV is digested per layer; every step of both legs must agree (digests_equal).  The layer-major remote get
is opt-in: this bench sets LMCACHE_B200_REMOTE_LAYERWISE=1 for its engines.  Loopback only: a real NIC is not measured.
Prints one JSON line.  Writes nothing into the tree.
"""
import argparse
import ctypes
import hashlib
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def _gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def _digests(kv):
    import torch
    out = []
    for k, v in kv:
        h = hashlib.sha256()
        for t in (k, v):
            h.update(t.contiguous().view(torch.int16).cpu().numpy().tobytes())
        out.append(h.hexdigest())
    return out


def run(T, serde, steps, warmup, ffn, port):
    import torch

    import bench
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    os.environ["LMCACHE_B200_REMOTE_LAYERWISE"] = "1"
    L, H, D, cs = 32, 8, 128, 256
    dev = torch.device("cuda", 0)
    base = bench.synth_kv_torch(min(T, 8192), dev, seed=0)[:, :, :, :H]          # [L, 2, t, H, D]: the first 8 heads
    reps = -(-T // base.shape[2])
    blob = (base.repeat(1, 1, reps, 1, 1)[:, :, :T] if reps > 1 else base).contiguous()
    kv = tuple((blob[l, 0], blob[l, 1]) for l in range(L))
    meta = LMCacheEngineMetadata("lmsys/longchat-7b-16k", 1, 0, "vllm", "bfloat16")
    cfg = LMCacheEngineConfig(cs, None, f"lmn://127.0.0.1:{port}", serde, False, False, None)
    eng = LMCacheEngine(cfg, meta)
    tokens = torch.arange(T, device=dev) + (7 << 20) * (1 + ["cachegen", "lossless"].index(serde))
    eng.store(tokens, kv)
    del kv, blob, base
    x = torch.randn((T, 4096), dtype=torch.bfloat16, device=dev)
    w = torch.randn((4096, ffn), dtype=torch.bfloat16, device=dev) * 0.01
    fwd = torch.cuda.current_stream()
    be = eng.engine_
    res = {"retrieve": [], "layerwise": []}
    digests = []

    def step(mode):
        torch.cuda.synchronize()
        s0 = dict(be.ranged_stats)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(fwd)
        t0 = time.perf_counter()
        out = {}
        if mode == "retrieve":
            got, mask = eng.retrieve(tokens)
            torch.cuda.synchronize()
            out["retrieve_ms"] = 1e3 * (time.perf_counter() - t0)
            for _ in range(L):
                torch.mm(x, w)
        else:
            r = eng.retrieve_layerwise(tokens)
            out["call_ms"] = 1e3 * (time.perf_counter() - t0)
            got, mask = r.kv, r.ret_mask
            for layer in range(L):
                r.wait_layer(layer, fwd)
                torch.mm(x, w)
        e1.record(fwd)
        torch.cuda.synchronize()
        assert int(mask.sum()) == T, "the whole sequence must hit"
        out["step_ms"] = e0.elapsed_time(e1)
        if mode == "layerwise":
            up = r._upload
            out["ready_ms"] = [e0.elapsed_time(up.ready(i)) for i in (0, L // 2, L - 1)]
            enq, wait = getattr(up, "enqueue_s", [])[1:], getattr(up, "wait_s", [])[1:]
            out["enqueue_ms"] = 1e3 * statistics.mean(enq) if enq else None
            out["wait_ms"] = 1e3 * statistics.mean(wait) if wait else None
            st = be.ranged_stats
            d = {k: st[k] - s0[k] for k in st}
            out["fetched_MB"] = d["bytes"] / 1e6
            out["reads"] = d["reads"]
            out["match_ms"] = 1e3 * d["match_s"]
            out["open_ms"] = 1e3 * d["open_s"] / max(1, d["opens"])
            out["read_ms"] = 1e3 * d["read_s"] / max(1, d["reads"])
            out["thread_ms"] = 1e3 * d["thread_s"] / int(os.environ.get("LMCACHE_B200_REMOTE_CONNS", "4"))
        digests.append(_digests(got))
        return out

    for i in range(warmup + steps):
        for mode in (("retrieve", "layerwise") if i % 2 == 0 else ("layerwise", "retrieve")):
            out = step(mode)
            if i >= warmup:
                res[mode].append(out)
    eng.close()

    def med(rows, key):
        vals = [r[key] for r in rows if r.get(key) is not None]
        if not vals:
            return None
        if isinstance(vals[0], list):
            return [round(statistics.median(v), 2) for v in zip(*vals)]
        return round(statistics.median(vals), 2)
    summary = {"tokens": T, "serde": serde,
               "retrieve": {k: med(res["retrieve"], k) for k in ("retrieve_ms", "step_ms")},
               "layerwise": {k: med(res["layerwise"], k) for k in ("call_ms", "ready_ms", "enqueue_ms", "wait_ms",
                                                                   "step_ms", "fetched_MB", "reads", "match_ms",
                                                                   "open_ms", "read_ms", "thread_ms")},
               "digests_equal": all(d == digests[0] for d in digests)}
    return summary


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--tokens", default="8192,65536")
    ap.add_argument("--serde", default="cachegen,lossless")
    ap.add_argument("--ffn", type=int, default=14336)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "remote_layerwise_bench.py needs a CUDA device"
    torch.cuda.set_device(0)
    from lmcache_b200 import _native as N
    lib = N.lib()
    h = ctypes.c_void_p()
    N.check(lib.b200kv_lm_server_start(b"127.0.0.1", 0, ctypes.byref(h)), "lm_server_start")
    try:
        port = lib.b200kv_lm_server_port(h)
        rows = [run(int(t), s, a.steps, a.warmup, a.ffn, port) for t in a.tokens.split(",") for s in a.serde.split(",")]
    finally:
        lib.b200kv_lm_server_stop(h)
    print(json.dumps({"bench": "remote_layerwise", "gpu": _gpu_info(), "conns": int(os.environ.get(
        "LMCACHE_B200_REMOTE_CONNS", "4")), "ffn": a.ffn, "rows": rows}))


if __name__ == "__main__":
    main()
