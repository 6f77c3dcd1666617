#!/usr/bin/env python
"""fused_absmax_bench.py -- where the encode half of bench.py's step goes: the per-token maxima against the coder.

  python fused_absmax_bench.py [--tokens 8192] [--wave 8] [--steps 10] [--data kv8d] [--heads 32]

Workload: bench.py's headline block (32 layers, 32 heads x 128, bf16, 256-token chunks, waves of 8 chunks), encode only
(container version 3).  Prints one JSON line:
  encode_call_ms   device time of one step's b200kv_encode_chunks calls (every wave), events on the stream, profiling off
  slots_ms         the library's per-kernel event slots, summed over a step's waves (absmax, encode, compact); a slot
                   that a path does not launch is absent
  absmax_plus_encode_ms / encode_only_ms
                   what the maxima pass costs beside the coder: the separate absmax_kernel runs alone on the HBM before
                   encode_kernel, so absmax + encode minus encode alone is the most folding the maxima into the coder
                   can recover
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

MODEL = "lmsys/longchat-7b-16k"
L, D = 32, 128


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=8192)
    ap.add_argument("--chunk", type=int, default=256)
    ap.add_argument("--heads", type=int, default=32)
    ap.add_argument("--wave", type=int, default=8)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--data", default="kv8d")
    args = ap.parse_args()

    import torch

    import __graft_entry__ as ge
    ge.build_cuda()
    import bench
    bench.H, bench.C = args.heads, args.heads * D
    from lmcache_b200 import _native as N
    from lmcache_b200.codec import CacheGenCodec, KvView

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    H = args.heads
    T, cs = args.tokens, args.chunk
    n_chunks = (T + cs - 1) // cs
    W = max(1, min(args.wave, n_chunks))
    lib = N.lib()
    codec = CacheGenCodec(MODEL)
    kv = bench.synth_kv_torch(T, dev, 1236, args.data)
    view = KvView.from_blob(kv, "vllm")
    stride = codec.out_stride(L, H, D, cs)
    staging = torch.empty(stride * W + N.READ_SLACK, dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream()
    waves = [(c0, min(W * cs, T - c0 * cs)) for c0 in range(0, n_chunks, W)]

    def step():
        for c0, nt in waves:
            codec.encode_async(view, c0 * cs, nt, cs, out=staging)

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()

    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    call_ms = []
    for _ in range(args.steps):
        ev0.record(stream)
        step()
        ev1.record(stream)
        torch.cuda.synchronize()
        call_ms.append(ev0.elapsed_time(ev1))

    lib.b200kv_profile_enable(1)
    slots = {k: [] for k in N.PROFILE_SLOTS}
    for _ in range(args.steps):
        tot = {}
        for c0, nt in waves:
            codec.encode_async(view, c0 * cs, nt, cs, out=staging)
            buf = (ctypes.c_float * 8)()
            N.check(lib.b200kv_profile_last(buf, 8))
            for i, name in enumerate(N.PROFILE_SLOTS):
                if buf[i] >= 0:
                    tot[name] = tot.get(name, 0.0) + buf[i]
        for k, v in tot.items():
            slots[k].append(v)
    lib.b200kv_profile_enable(0)
    torch.cuda.synchronize()

    def med(v):
        v = sorted(v)
        return v[len(v) // 2]

    s = {k: round(med(v), 4) for k, v in slots.items() if v}
    raw = L * 2 * T * H * D * 2
    line = {"card": card(), "shape": f"{L}L/{H}H/{D}D {T} tokens, chunk {cs}, waves of {W}", "data": args.data,
            "steps": args.steps, "encode_call_ms": round(med(call_ms), 4),
            "encode_call_ms_min_max": [round(min(call_ms), 4), round(max(call_ms), 4)],
            "encode_call_GBps": round(raw / (med(call_ms) * 1e-3) / 1e9, 1), "slots_ms": s,
            "absmax_plus_encode_ms": round(s.get("absmax", 0.0) + s.get("encode", 0.0), 4),
            "encode_only_ms": s.get("encode")}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
