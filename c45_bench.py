"""bench.py --config c4 | c5 : BASELINE.json configs[3] and configs[4] -- cache engines sharing KV through ONE lm:// server.

  c4  "2 vLLM instances sharing KV via lmcache.server, longchat-7b-16k-shaped synthetic prompts" (reference recipe
      README.md:55-58, test tests/test_backends.py:181-203): rank 0 stores prompts of 16 384 tokens (8 GiB of bf16 KV each)
      through LMCacheEngine.store() -> lm:// + CacheGen, rank 1 retrieves them with LMCacheEngine.retrieve() -- a replica
      that never stored anything.  With one process (python bench.py --config c4) both roles run back to back on one GPU
      with two engine objects and separate connections.
  c5  "8 independent cache engines, RAG-style 16 x 4096-token chunk mix, non-prefix retrieve": every rank stores 16
      independent 4096-token sequences (own hash chains), then retrieves a random 8 of them, one retrieve() per sequence
      (the reference has no blend API, README.md:71; SURVEY.md 8d).  All ranks talk to the one server on rank 0.

Run under torchrun for N > 1 exactly like bench.py (one rank per GPU; NCCL only lines ranks up and gathers timings; the data
path is host sockets, SURVEY.md 8e).  Rank 0 hosts the native lm:// server of libb200kv in-process (csrc/lmnet.cu: threads
outside the GIL), which speaks the reference's wire protocol (lmcache/protocol.py).

One JSON line on rank 0: aggregate store / retrieve GB/s of raw bf16 KV, per-sequence retrieve latency percentiles, the wire
bytes, and ttft_saved_ms_p50 = t_prefill - t_retrieve(p50), with t_prefill a STATED model constant (no LLM is run,
SURVEY.md 8d): 2 * 6.74e9 FLOPs per token for the 7B weights plus causal attention, at 60 % of the sustained bf16 peak in
MEASURED_PEAKS.json, or of the H100 SXM data sheet's dense bf16 rate (989 TFLOP/s) where that file is absent."""
import ctypes
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
MODEL = "lmsys/longchat-7b-16k"
L, H, D = 32, 32, 128
C = H * D


def prefill_ms(tokens: int) -> float:
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except OSError:
        pass
    tflops = 0.6 * float(peaks.get("bf16_tflops_sustained", 989.0))
    flops = 2.0 * 6.74e9 * tokens + 2.0 * L * tokens * tokens * C        # weights + causal QK^T/PV (4 L T^2 C / 2)
    return flops / (tflops * 1e12) * 1e3


def main(args):
    import torch

    import __graft_entry__ as ge
    ge.build_cuda()
    import bench
    from lmcache_b200 import _native as N
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist = None
    if world > 1:
        import torch.distributed as dist
        sys.stdout.flush()
        saved = os.dup(1)
        os.dup2(2, 1)
        try:
            dist.init_process_group("nccl", device_id=dev)
            dist.barrier(device_ids=[local])
            torch.cuda.synchronize()
        finally:
            sys.stdout.flush()
            os.dup2(saved, 1)
            os.close(saved)

    def barrier():
        torch.cuda.synchronize()
        if dist is not None:
            dist.barrier()

    def gather(obj):
        if dist is None:
            return [obj]
        out = [None] * world
        dist.all_gather_object(out, obj)
        return out

    lib = N.lib()
    os.environ["LMCACHE_B200_CODER"] = args.coder
    # ---- one shared server, on rank 0
    server = ctypes.c_void_p()
    port = [0]
    if rank == 0:
        N.check(lib.b200kv_lm_server_start(b"127.0.0.1", 0, ctypes.byref(server)), "lm_server_start")
        port[0] = int(lib.b200kv_lm_server_port(server))
    if dist is not None:
        dist.broadcast_object_list(port, src=0)
    url = f"lm://127.0.0.1:{port[0]}"
    cs = args.chunk
    cfg = LMCacheEngineConfig.from_legacy(chunk_size=cs, backend=url, remote_serde="cachegen")

    def engine(worker_id):
        # every engine keys its chunks by (world_size, worker_id): c5 ranks stay disjoint, c4's reader uses the writer's id
        return LMCacheEngine(cfg, LMCacheEngineMetadata(MODEL, max(world, 1), worker_id, "vllm", "bfloat16"))

    c4 = args.config == "c4"
    T = 16384 if c4 else 4096
    n_seq = (8 if c4 else 16)                   # c4: enough prompts for a stable median (the wire's share of a retrieve varies)
    if args.tokens not in (8192, T):
        T = args.tokens                         # smaller shapes for smoke runs
    raw_seq = L * 2 * T * C * 2
    # a few distinct KV blocks, cycled over the sequences (keys differ through the token ids)
    n_kv = 1 if c4 else 2
    kvs = [bench.synth_kv_torch(T, dev, 555 + 17 * rank + i, args.data) for i in range(n_kv)]
    tuples = [tuple((kv[l, 0], kv[l, 1]) for l in range(L)) for kv in kvs]
    g = torch.Generator(device=dev).manual_seed(1000 + rank)
    if c4:
        # both roles need the same prompts: derive them from a seed every rank knows
        gs = torch.Generator(device=dev).manual_seed(4242)
        toks = [torch.randint(0, 32000, (T,), device=dev, generator=gs) for _ in range(n_seq)]
    else:
        toks = [torch.randint(0, 32000, (T,), device=dev, generator=g) for _ in range(n_seq)]

    writer = (rank == 0) if c4 else True
    reader = (rank == (1 if world > 1 else 0)) if c4 else True
    store_s = retr_lat = None
    eng_w = engine(0 if c4 else rank) if writer else None
    # warm the pipelines (page-locked slab segments, rings, upload slots) outside the timed regions: one full-length
    # sequence that is stored and read back before anything is timed
    gw = torch.Generator(device=dev).manual_seed(31337 + (0 if c4 else rank))
    warm = torch.randint(0, 32000, (T,), device=dev, generator=gw)
    if writer:
        eng_w.store(warm, tuples[0])
    barrier()
    if writer:
        t0 = time.perf_counter()
        for i in range(n_seq):
            eng_w.store(toks[i], tuples[i % n_kv], blocking=True)
        torch.cuda.synchronize()
        store_s = time.perf_counter() - t0
    barrier()            # a blocking store ends with one EXIST round trip per connection, so the server holds every chunk
    eng_r = None
    if reader:
        # c4: a replica that never stored anything (its geometry comes from a container header); c5: the storing engine
        eng_r = engine(0) if c4 else eng_w
        wr, wm = eng_r.retrieve(warm)
        torch.cuda.synchronize()
        assert int(wm.sum()) == T
        del wr
        import random
        order = list(range(n_seq)) if c4 else random.Random(7 + rank).sample(range(n_seq), n_seq // 2)
        retr_lat = []
        ok = True
        for i in order:
            t0 = time.perf_counter()
            ret, mask = eng_r.retrieve(toks[i])
            torch.cuda.synchronize()
            retr_lat.append(time.perf_counter() - t0)
            ok = ok and int(mask.sum()) == T and len(ret) == L
            del ret
        assert ok, "a stored sequence did not come back in full"
        # parity spot check on the last retrieved sequence: first chunk vs the reference decode (tests/ref_torch.py)
        ret, _ = eng_r.retrieve(toks[order[-1]])
        blob = torch.stack((torch.stack([k for k, _ in ret]), torch.stack([v for _, v in ret]))).permute(1, 0, 2, 3, 4)
        src = kvs[order[-1] % n_kv] if (not c4 or world == 1) else bench.synth_kv_torch(T, dev, 555 + 0, args.data)
        parity = bench.parity_spot_check(src, blob.contiguous(), cs)
    else:
        parity = None
    barrier()
    keys = int(lib.b200kv_lm_server_num_keys(server)) if rank == 0 else None
    res = gather({"rank": rank, "store_s": store_s, "retr_lat": retr_lat, "parity": parity,
                  "n_stored": n_seq if writer else 0, "n_read": len(retr_lat) if retr_lat else 0})
    for e in (eng_w, eng_r):
        if e is not None:
            e.close()
    barrier()
    if rank == 0:
        stored = sum(r["n_stored"] for r in res)
        read = sum(r["n_read"] for r in res)
        t_store = max(r["store_s"] for r in res if r["store_s"])
        lats = sorted(x for r in res if r["retr_lat"] for x in r["retr_lat"])
        t_retr = max(sum(r["retr_lat"]) for r in res if r["retr_lat"])
        p50 = lats[len(lats) // 2]
        tp = prefill_ms(T)
        line = {
            "metric": "kv_share_raw_GBps", "config_id": args.config, "n_gpus": world, "unit": "GB/s",
            "store_GBps": round(stored * raw_seq / t_store / 1e9, 2), "retrieve_GBps": round(read * raw_seq / t_retr / 1e9, 2),
            "value": round(read * raw_seq / t_retr / 1e9, 2), "higher_is_better": True, "data": "synthetic",
            "config": {"workload": ("BASELINE configs[3]: writer engine -> one lm:// server -> reader engine, " if c4 else
                                    "BASELINE configs[4]: N engines x 16 sequences, retrieve a random 8 of 16 each, one shared lm:// server, ") +
                                   f"{T}-token sequences ({raw_seq / 2**30:.1f} GiB raw bf16 each), {L}L/{H}H/{D}D, chunk_size {cs}, "
                                   f"CacheGen ({args.coder}) over lm://, {os.environ.get('LMCACHE_B200_REMOTE_CONNS', '4')} connections per engine",
                       "data_kind": args.data, "sequences_stored": stored, "sequences_retrieved": read,
                       "server": "native lm:// server of libb200kv on rank 0 (reference wire protocol)", "server_keys": keys},
            "retrieve_latency_ms": {"p50": round(p50 * 1e3, 1), "min": round(lats[0] * 1e3, 1), "max": round(lats[-1] * 1e3, 1)},
            "ttft": {"t_prefill_ms_model": round(tp, 1), "t_retrieve_ms_p50": round(p50 * 1e3, 1),
                     "ttft_saved_ms_p50": round(tp - p50 * 1e3, 1),
                     "model": "t_prefill = (2 * 6.74e9 * T + 2 * L * T^2 * C) FLOPs / (0.6 * bf16_tflops_sustained of "
                              "MEASURED_PEAKS.json); a stated constant, no LLM is run (SURVEY.md 8d)"},
            "parity_spot_check": [r["parity"] for r in res if r["parity"]],
        }
        print(json.dumps(line))
        N.check(lib.b200kv_lm_server_stop(server))
    if dist is not None:
        dist.destroy_process_group()
