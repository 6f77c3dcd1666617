"""Generate golden vectors by importing the *reference's own* functions (CPU, this container).

Run once on a CPU machine with a checkout of the reference (GPU test runs only read the outputs):

    python tests/golden/make_golden.py <path of an LMCache v0.1.2 tree>

Outputs (committed): tests/golden/golden_codec.npz, tests/golden/golden_hash.json,
tests/golden/golden_engine.json.

What is pinned, and by which reference code (paths relative to the reference tree):
  * quantise           lmcache/storage_backend/serde/cachegen_encoder.py:40-61  torch_quant_vectorized
                       + _split_kv :76-91 and the K/V concat :284-285
  * dequantise + cast  lmcache/storage_backend/serde/cachegen_decoder.py:24-35 do_dequantize
                       + assembly :182-200
  * CDF                in-tree spec CacheGenEncoderImpl.compute_cdf :174-222 (process_batch :185-196)
                       + _convert_to_int_and_normalize :95-126   (torch CPU semantics)
  * bins               CacheGenSerializer.make_key_bins / make_value_bins :339-350 (with .cuda() -> identity)
  * hash chain         lmcache/cache_engine.py:58-96  LMCacheEngine._prefix_hash/_chunk_tokens
  * engine semantics   lmcache/cache_engine.py store/retrieve on LMCLocalBackend("cpu")
The arithmetic-coder bitstream cannot be pinned this way (torchac_cuda wheel absent).
"""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.join(HERE, "..", "_refstubs"), sys.argv[1]]

import numpy as np  # noqa: E402
import torch  # noqa: E402

torch.Tensor.cuda = lambda self, *a, **k: self  # reference ctors call .cuda(); CPU-only here

from lmcache.cache_engine import LMCacheEngine  # noqa: E402
from lmcache.config import LMCacheEngineConfig, LMCacheEngineMetadata  # noqa: E402
from lmcache.storage_backend.serde.cachegen_basics import CacheGenConfig  # noqa: E402
from lmcache.storage_backend.serde.cachegen_decoder import do_dequantize  # noqa: E402
from lmcache.storage_backend.serde.cachegen_encoder import (  # noqa: E402
    CacheGenEncoderImpl, CacheGenSerializer, _convert_to_int_and_normalize, _split_kv, torch_quant_vectorized)
from lmcache.utils import CacheEngineKey  # noqa: E402

MODEL = "lmsys/longchat-7b-16k"


def bits(t: torch.Tensor) -> np.ndarray:
    return t.contiguous().view(torch.int16).numpy().view(np.uint16).copy()


def make_bins():
    cfg = CacheGenConfig.from_model_name(MODEL)
    ser = CacheGenSerializer.__new__(CacheGenSerializer)
    kb = CacheGenSerializer.make_key_bins(ser, cfg)
    vb = CacheGenSerializer.make_value_bins(ser, cfg)
    return cfg, kb, vb


def synth(rng, L, t, H, D, dtype, kind):
    C = H * D
    if kind == "normal":
        sigma = np.clip(rng.lognormal(0.0, 0.5, size=(L, 2, 1, C)), 0.1, 8.0)
        outl = rng.random(size=(L, 2, 1, C)) < 0.01
        sigma = np.where(outl, sigma * 10.0, sigma)
        x = rng.standard_normal(size=(L, 2, t, C)) * sigma
    elif kind == "uniform":  # like the reference tests' torch.rand
        x = rng.random(size=(L, 2, t, C))
    else:
        raise ValueError(kind)
    x = torch.from_numpy(x.astype(np.float32)).to(dtype).reshape(L, 2, t, H, D)
    # edge rows: all-zero token row (-> NaN -> symbol 0), a +/- max row, a tiny-magnitude row
    if t >= 3:
        x[0, 0, 1] = 0
        x[1, 1, 2] = 0
        x[2, 0, 0, :, :] = -x[2, 0, 0, :, :].abs()
        x[3, 1, 0, 0, 0] = 3.0
        x[3, 1, 0, 0, 1] = -3.0
    return x


def codec_case(rng, name, L, t, H, D, dtype, kind, out):
    cfg, kb, vb = make_bins()
    kb, vb = kb[:L], vb[:L]
    x = synth(rng, L, t, H, D, dtype, kind)
    fp_k, fp_v = _split_kv(x)
    new_key, max_k = torch_quant_vectorized(kb, fp_k)
    new_val, max_v = torch_quant_vectorized(vb, fp_v)
    sym = torch.cat((new_key, new_val), dim=0).reshape(2 * L, t, H * D)
    # reference decode side: out.float() of uint8 symbols, do_dequantize, stack/reshape/permute/cast
    key_f = new_key.to(torch.uint8).float()
    val_f = new_val.to(torch.uint8).float()
    key = do_dequantize(key_f, kb, max_k)
    value = do_dequantize(val_f, vb, max_v)
    blob = torch.stack([key, value]).reshape(2, L, t, H, D)
    out_bf16 = blob.permute(1, 0, 2, 3, 4).to(torch.bfloat16)          # vllm
    out_fp16 = blob.permute(1, 0, 3, 2, 4).to(torch.float16)           # huggingface [L,2,H,t,D]
    # in-tree CDF spec
    impl = CacheGenEncoderImpl(fp_k=fp_k, fp_v=fp_v, config=cfg)
    impl.quantized_key = {i: new_key[i] for i in range(L)}
    impl.quantized_value = {i: new_val[i] for i in range(L)}
    cdf_k = _convert_to_int_and_normalize(impl.compute_cdf(is_key=True), True)
    cdf_v = _convert_to_int_and_normalize(impl.compute_cdf(is_key=False), True)
    cdf = torch.cat([cdf_k, cdf_v])
    out[f"{name}/x"] = bits(x)
    out[f"{name}/dtype"] = np.array([0 if dtype == torch.bfloat16 else 1])
    out[f"{name}/sym"] = sym.numpy().copy()
    out[f"{name}/max_k"] = bits(max_k)
    out[f"{name}/max_v"] = bits(max_v)
    out[f"{name}/cdf"] = cdf.numpy().copy()
    out[f"{name}/deq_vllm_bf16"] = bits(out_bf16)
    out[f"{name}/deq_hf_fp16"] = bits(out_fp16)
    print(name, tuple(x.shape), "sym range", int(sym.min()), int(sym.max()))


def hash_cases():
    cfg = LMCacheEngineConfig.from_legacy(chunk_size=256, backend="cpu")
    meta = LMCacheEngineMetadata("m", 1, 0, "vllm", "half")
    cases = []
    rng = np.random.default_rng(1234)

    def run(tokens_np, chunk_size, label):
        eng = LMCacheEngine.__new__(LMCacheEngine)
        eng.chunk_size = chunk_size
        toks = torch.from_numpy(tokens_np)
        hashes = eng._prefix_hash(eng._chunk_tokens(toks))
        cases.append(dict(label=label, dtype=str(tokens_np.dtype), chunk_size=chunk_size,
                          tokens_sha256=hashlib.sha256(tokens_np.tobytes()).hexdigest(),
                          gen=label, n=int(tokens_np.shape[0]), hashes=hashes))

    run(np.arange(600, dtype=np.int64), 256, "arange600_i64")
    run(np.arange(600, dtype=np.int32), 256, "arange600_i32")
    run(np.arange(0, dtype=np.int64), 256, "arange0_i64")
    run(np.arange(1, dtype=np.int64), 256, "arange1_i64")
    for n, cs in [(16, 16), (17, 16), (255, 256), (256, 256), (257, 256), (2000, 128), (8192, 256), (1000, 7)]:
        run(rng.integers(0, 32000, n, dtype=np.int64), cs, f"rng1234_{n}_{cs}")
    key = CacheEngineKey("vllm", "m", 1, 0, cases[0]["hashes"][0]).to_string()
    LMCacheEngine  # noqa
    del cfg, meta
    return dict(cases=cases, key_string_example=key,
                note="rng cases are generated sequentially from numpy default_rng(1234).integers(0,32000,n,int64) "
                     "in the listed order")


def engine_cases():
    """Prefix / mask semantics of store+retrieve on the reference engine (local cpu backend)."""
    res = {}
    cfg = LMCacheEngineConfig.from_legacy(chunk_size=256, backend="cpu")
    meta = LMCacheEngineMetadata("test_model", 3, 123, "vllm", "half")
    eng = LMCacheEngine(cfg, meta)
    eng.engine_.dst_device = "cpu"  # hard-coded "cuda" at local_backend.py:53
    g = torch.Generator().manual_seed(0)
    T = 600
    tokens = torch.arange(T, dtype=torch.int64)
    kv = tuple((torch.rand(T, 2, 8, generator=g).bfloat16(), torch.rand(T, 2, 8, generator=g).bfloat16())
               for _ in range(3))
    r0, m0 = eng.retrieve(tokens)
    res["empty_retrieve"] = dict(n_layers=len(r0), mask_sum=int(m0.sum()))
    eng.store(tokens, kv)
    r1, m1 = eng.retrieve(tokens)
    res["full_retrieve"] = dict(mask_sum=int(m1.sum()), ntok=int(r1[0][0].shape[0]),
                                equal=bool(all(torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
                                               for a, b in zip(r1, kv))))
    longer = torch.cat([tokens, torch.arange(1000, 1400, dtype=torch.int64)])
    r2, m2 = eng.retrieve(longer)
    res["prefix_of_longer"] = dict(mask_sum=int(m2.sum()), ntok=int(r2[0][0].shape[0]),
                                   mask_true_idx=[int(m2.nonzero()[0]), int(m2.nonzero()[-1])])
    mask = torch.ones(T, dtype=torch.bool)
    mask[:300] = False
    r3, m3 = eng.retrieve(tokens, mask)
    res["suffix_mask_300"] = dict(mask_sum=int(m3.sum()), ntok=int(r3[0][0].shape[0]),
                                  first_true=int(m3.nonzero()[0]),
                                  equal=bool(torch.equal(r3[0][0], kv[0][0][300:])))
    other = torch.arange(5000, 5300, dtype=torch.int64)
    r4, m4 = eng.retrieve(other)
    res["miss"] = dict(n_layers=len(r4), mask_sum=int(m4.sum()))
    eng.close()
    return res


def main():
    out = {}
    rng = np.random.default_rng(20240921)
    codec_case(rng, "bf16_t1", 12, 1, 2, 32, torch.bfloat16, "normal", out)
    codec_case(rng, "bf16_t7_L32", 32, 7, 2, 32, torch.bfloat16, "normal", out)
    codec_case(rng, "bf16_t40", 12, 40, 2, 32, torch.bfloat16, "normal", out)
    codec_case(rng, "bf16_t236", 12, 236, 1, 16, torch.bfloat16, "normal", out)
    codec_case(rng, "bf16_t256", 12, 256, 1, 16, torch.bfloat16, "normal", out)
    codec_case(rng, "bf16_t300", 12, 300, 1, 8, torch.bfloat16, "normal", out)
    codec_case(rng, "bf16_uniform_t16", 12, 16, 1, 32, torch.bfloat16, "uniform", out)
    codec_case(rng, "fp16_t40", 12, 40, 1, 32, torch.float16, "normal", out)
    codec_case(rng, "fp16_uniform_t128", 12, 128, 1, 16, torch.float16, "uniform", out)
    cfg, kb, vb = make_bins()
    out["key_bins"] = kb.numpy().copy()
    out["value_bins"] = vb.numpy().copy()
    np.savez_compressed(os.path.join(HERE, "golden_codec.npz"), **out)
    with open(os.path.join(HERE, "golden_hash.json"), "w") as f:
        json.dump(hash_cases(), f, indent=1)
    with open(os.path.join(HERE, "golden_engine.json"), "w") as f:
        json.dump(engine_cases(), f, indent=1)
    print("wrote goldens; torch", torch.__version__, "numpy", np.__version__)


if __name__ == "__main__":
    main()
