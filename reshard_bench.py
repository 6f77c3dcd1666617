#!/usr/bin/env python
"""reshard_bench.py -- what a retrieve across tensor-parallel layouts costs against the ordinary one, on one GPU.

  python reshard_bench.py [--steps K] [--warmup W] [--tokens 8192] [--serde cachegen|lossless]

Workload: a 32-layer / 8-KV-head / 128-dim model in bf16 (Llama-3-8B-shaped, Mistral-7B's bin table), chunks of 256
tokens, synthetic KV (SURVEY 8d: log-normal channel scales, 1 % outlier channels).  1, 2, 4 and 8 all divide the 8 KV
heads, so every pair of layouts below is served.  One process starts the native lm:// server in-process (stopped at
exit); engines of layouts W = 1, 2 and 4 store their head shards of the same KV under three token sequences (one per
layout, so that a retrieving engine's own layout holds nothing of the sequences it reshards).  Legs, alternated step by
step after the warm-ups:
  own1      retrieve() at W' = 1 of the W = 1 sequence
  2to1      retrieve() at W' = 1 of the W = 2 sequence (two containers per chunk, each decoded whole)
  4to1      retrieve() at W' = 1 of the W = 4 sequence (four containers per chunk)
  own2      retrieve() at W' = 2, rank 0, of the W = 2 sequence
  1to2      retrieve() at W' = 2, rank 0, of the W = 1 sequence (the whole container fetched, half of it decoded)
Per leg: the median wall clock of retrieve() (host clock around the call and a device synchronize), the container bytes
fetched, and the decode kernel time (CUDA events, median of repeated calls on device-resident containers) of the leg's
decode against a whole decode of the same containers.  Every resharded result is checked bit for bit against the
source layout's own retrieve.  Prints one JSON line with the GPU's name and power limit.  Writes nothing into the tree.

--serde lossless runs the same legs with remote_serde "lossless" and reshard_lossless (container version 5): the
containers are then the KV's own bits, and every resharded result is also checked bit for bit against the original
KV's heads of the retrieving rank.  The JSON line then carries "serde": "lossless"; the default (cachegen) prints
what it always printed.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

MODEL = "mistralai/Mistral-7B-Instruct-v0.2"
L, HG, D, CS = 32, 8, 128, 256


def _power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--tokens", type=int, default=8192)
    ap.add_argument("--serde", choices=("cachegen", "lossless"), default="cachegen")
    args = ap.parse_args()
    import torch

    import __graft_entry__ as ge
    ge.build_cuda()
    from lmcache_b200 import _native as N
    from lmcache_b200.cache_engine import LMCacheEngine, sha256_prefix_chain
    from lmcache_b200.codec import KvView
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    from lmcache_b200.reshard import source_shards
    from lmcache_b200.utils import CacheEngineKey

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cur = torch.cuda.current_stream()
    T = args.tokens
    lib = N.lib()
    srv = ctypes.c_void_p()
    N.check(lib.b200kv_lm_server_start(b"127.0.0.1", 0, ctypes.byref(srv)), "server_start")
    url = f"lm://127.0.0.1:{lib.b200kv_lm_server_port(srv)}"
    engines = []
    try:
        g = torch.Generator(device=dev).manual_seed(8)
        sigma = torch.exp(0.5 * torch.randn((L, 2, 1, HG, D), device=dev, generator=g)).clamp(0.1, 8.0)
        sigma = torch.where(torch.rand(sigma.shape, device=dev, generator=g) < 0.01, sigma * 10, sigma)
        kv = (torch.randn((L, 2, T, HG, D), device=dev, generator=g) * sigma).to(torch.bfloat16)
        seqs = {W: torch.randint(0, 32000, (T,), device=dev, generator=g) for W in (1, 2, 4)}

        def engine(W, r, reshard=None):
            cfg = LMCacheEngineConfig(CS, None, url, args.serde, False, False, reshard_world_sizes=reshard,
                                      reshard_lossless=reshard is not None and args.serde == "lossless")
            e = LMCacheEngine(cfg, LMCacheEngineMetadata(MODEL, W, r, "vllm", "bfloat16"))
            engines.append(e)
            return e

        for W, tok in seqs.items():
            for r in range(W):
                a, b = r * HG // W, (r + 1) * HG // W
                engine(W, r).store(tok, tuple((kv[l, 0, :, a:b], kv[l, 1, :, a:b]) for l in range(L)))

        conn = ctypes.c_void_p()
        N.check(lib.b200kv_lm_connect(b"127.0.0.1", lib.b200kv_lm_server_port(srv), ctypes.byref(conn)), "connect")

        def fetch(W, r, tok):
            """the containers layout W's rank r stored for `tok`, as host bytes"""
            out = []
            for h in sha256_prefix_chain(tok, CS):
                key = CacheEngineKey("vllm", MODEL, W, r, h).to_string().encode()
                n = lib.b200kv_lm_get_begin(conn, key)
                assert n > 0, "a stored chunk is missing"
                buf = ctypes.create_string_buffer(n)
                N.check(lib.b200kv_lm_read(conn, buf, n), "read")
                out.append(buf.raw)
            return out

        legs = {"own1": (1, 0, 1, None), "2to1": (1, 0, 2, [2, 4]), "4to1": (1, 0, 4, [2, 4]),
                "own2": (2, 0, 2, None), "1to2": (2, 0, 1, [1])}
        retr = {name: engine(Wd, rd, rs) for name, (Wd, rd, _, rs) in legs.items()}
        runs = {name: [] for name in legs}
        for i in range(args.warmup + args.steps):
            for name, (Wd, rd, W, _) in legs.items():
                cur.synchronize()
                t0 = time.perf_counter()
                ret, mask = retr[name].retrieve(seqs[W])
                cur.synchronize()
                ms = 1e3 * (time.perf_counter() - t0)
                assert int(mask.sum()) == T, f"{name}: {int(mask.sum())} of {T} tokens"
                if i >= args.warmup:
                    runs[name].append(ms)
                del ret

        # bit identity against the source layout's own retrieves
        own = {(W, r): engine(W, r) for W in (1, 2, 4) for r in range(W)}
        for name, (Wd, rd, W, rs) in legs.items():
            if rs is None:
                continue
            got, _ = retr[name].retrieve(seqs[W])
            parts = []
            for s in source_shards(HG, W, Wd, rd):
                src, _ = own[(W, s.rank)].retrieve(seqs[W])
                parts.append([(k[:, s.src_head0:s.src_head0 + s.n_heads], v[:, s.src_head0:s.src_head0 + s.n_heads])
                              for k, v in src])
            for l in range(L):
                for x in range(2):
                    want = torch.cat([p[l][x] for p in parts], dim=1)
                    assert torch.equal(got[l][x].view(torch.int16), want.view(torch.int16)), f"{name} differs"
                    if args.serde == "lossless":        # and the bits this rank's heads had before any store
                        a, b = rd * HG // Wd, (rd + 1) * HG // Wd
                        assert torch.equal(got[l][x].view(torch.int16), kv[l, x, :, a:b].view(torch.int16)), \
                            f"{name} differs from the original KV"

        # decode kernel time of each leg's decode against a whole decode of the same containers
        codec = retr["own1"].engine_.deserializer.codec

        def kernel_ms(W, Wd, rd):
            shards = source_shards(HG, W, Wd, rd)
            hs = HG // W
            blobs, offs, tot, ntok, toks, src0, dst0, nh = [], [], [], [], [], [], [], []
            o = 0
            for s in shards:
                for j, c in enumerate(fetch(W, s.rank, seqs[W])):
                    blobs.append(c + b"\0" * ((-len(c)) % 16))
                    offs.append(o)
                    o += len(blobs[-1])
                    tot.append(len(c))
                    ntok.append(min(CS, T - j * CS))
                    toks.append(j * CS)
                    src0.append(s.src_head0)
                    dst0.append(s.dst_head0)
                    nh.append(s.n_heads)
            raw = b"".join(blobs) + b"\0" * N.READ_SLACK
            buf = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(dev)
            hd = N.Header.from_buffer_copy(raw[:N.HEADER_BYTES])
            md = int(hd.max_dtype)
            cd = int(hd.version) - 1 if args.serde == "cachegen" else codec.coder_for(CS)
            win = torch.empty((L, 2, T, HG // Wd, D), dtype=torch.bfloat16, device=dev)
            whole = torch.empty((L, 2, T, hs, D), dtype=torch.bfloat16, device=dev)
            vw, vf = KvView.from_blob(win, "vllm"), KvView.from_blob(whole, "vllm")
            per_shard = len(offs) // len(shards)

            def time_it(fn, reps=20):
                fn()
                out = []
                for _ in range(reps):
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record(cur)
                    fn()
                    b.record(cur)
                    b.synchronize()
                    out.append(a.elapsed_time(b))
                return statistics.median(out)

            def windowed():
                codec.decode_raw_heads(buf.data_ptr(), buf.numel(), offs, tot, ntok, vw, toks, md, cd, hs, src0, dst0, nh)

            def full():       # each shard's containers decoded whole, one call per shard
                for k in range(len(shards)):
                    sl = slice(k * per_shard, (k + 1) * per_shard)
                    codec.decode_raw(buf.data_ptr(), buf.numel(), offs[sl], tot[sl], ntok[sl], vf, toks[sl], md, cd)
            return round(time_it(windowed), 3), round(time_it(full), 3), sum(tot)

        result = {"metric": "reshard_retrieve_ms", "tokens": T, "layers": L, "kv_heads": HG, "head_dim": D,
                  "chunk": CS, "steps": args.steps, "warmup": args.warmup, "gpu": torch.cuda.get_device_name(dev),
                  "power_limit": _power_limit(), "legs": {}}
        if args.serde != "cachegen":
            result["serde"] = args.serde
        for name, (Wd, rd, W, rs) in legs.items():
            k_win, k_full, fetched = kernel_ms(W, Wd, rd)         # the leg fetches every container it decodes
            leg = {"retrieve_ms_median": round(statistics.median(runs[name]), 3),
                   "retrieve_ms_runs": [round(x, 3) for x in runs[name]], "bytes_fetched": fetched,
                   "decode_kernel_ms": k_win, "whole_decode_kernel_ms": k_full}
            if rs:
                st = retr[name].reshard_stats()[W]
                n_ret = args.warmup + args.steps + 1
                assert st["chunks"] == n_ret * len(sha256_prefix_chain(seqs[W], CS)) and st["bytes"] == n_ret * fetched
            result["legs"][name] = leg
        lib.b200kv_lm_close(conn)
        print(json.dumps(result))
    finally:
        for e in engines:
            e.close()
        lib.b200kv_lm_server_stop(srv)


if __name__ == "__main__":
    main()
