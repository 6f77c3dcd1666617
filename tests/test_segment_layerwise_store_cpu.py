"""CPU: the host-side parts of the layer-by-layer segment store -- the kernel's per-run arrays and the staging layout
from plan_segment_store's runs, the arena split across runs (pipeline.begin_runs), the handle's forwarding to the
segment-at-0 handle and the run handles (pipeline.SegmentsEncode under a LayerwiseStore), and the fallback choice."""
import numpy as np
import pytest
import torch

from lmcache_b200.cache_engine import LayerwiseStore, LMCacheEngine
from lmcache_b200.codec import KvView
from lmcache_b200.pipeline import FanOutEncode, NoEncode, SegmentsEncode, arena_of, begin_runs
from lmcache_b200.rope import RopeSpec, plan_segment_store, plan_segments, staging_layout, store_run_arrays

CS = 256


def _runs():
    plans = plan_segments(6000, [(300, 1000), (1000, 1001), (2000, 4100), (5000, 5600)], CS)
    return plan_segment_store(plans, [(0, 0), (0, 0), (2, 3), (1, 0)], CS)


def test_run_arrays_one_chunk_per_run():
    runs, rows, sot, shifts = _runs()
    ntok, src, seg = store_run_arrays(runs)
    assert ntok.dtype == np.int32 and src.dtype == np.int64 and seg.dtype == np.int32
    assert ntok.tolist() == [700, 1, 2100 - 5 * CS, 600 - CS]
    assert src.tolist() == [300, 1000, 2000 + 5 * CS, 5000 + CS]
    assert seg.tolist() == [0, 1, 2, 3] and shifts == [-300, -1000, -2000, -5000]
    # the tokens the kernel reads are the rows the whole form stages, in the same order
    assert [t for n, a in zip(ntok, src) for t in range(a, a + n)] == rows
    assert [int(s) for n, s in zip(ntok, seg) for _ in range(n)] == sot


@pytest.mark.parametrize("fmt,latent", [("vllm", False), ("huggingface", False), ("vllm", True)])
def test_staging_layout_is_each_runs_blob_back_to_back(fmt, latent):
    runs, rows, _, _ = _runs()
    L, H, D = 5, (1 if latent else 8), (576 if latent else 128)
    per_tok = (1 if latent else 2) * H * D
    shapes, offs, layer_offs = staging_layout(runs, lambda t: KvView.blob_shape(fmt, L, H, D, t, latent),
                                              lambda t: per_tok * t, L)
    assert shapes == [KvView.blob_shape(fmt, L, H, D, r.n_tok, latent) for r in runs]
    sizes = [int(np.prod(s)) for s in shapes]
    assert offs == [sum(sizes[:i]) for i in range(len(runs))]
    # as much staging as the whole form's one blob of every staged token
    assert sum(sizes) == int(np.prod(KvView.blob_shape(fmt, L, H, D, len(rows), latent)))
    assert layer_offs.shape == (L, len(runs))
    for l in range(L):
        for r, run in enumerate(runs):
            assert layer_offs[l, r] == offs[r] + l * per_tok * run.n_tok
    assert staging_layout([], lambda t: (t,), lambda t: t, 3)[1] == []


class _Handle:
    def __init__(self, log, name, arena=0):
        self.log, self.name, self.arena_bytes = log, name, arena

    def encode_layer(self, layer, stream, ready=None):
        self.log.append(("encode", self.name, layer, stream, ready))

    def finish(self):
        self.log.append(("finish", self.name))
        return f"fin-{self.name}"

    def abandon(self):
        self.log.append(("abandon", self.name))


def test_begin_runs_splits_one_budget_in_plan_order():
    log, budgets = [], []
    bound = 300

    def begin(view, tok_begin, cs, budget):
        assert tok_begin == 0 and cs == CS
        budgets.append(budget)
        return _Handle(log, view, min(view * bound, budget))
    hs = begin_runs(begin, [2, 1, 4, 3], CS, 1000)
    assert budgets == [1000, 400, 100, 1]                     # each run gets what the ones before it left
    assert [h.arena_bytes for h in hs] == [600, 300, 100, 1]
    assert sum(arena_of(h) for h in hs[:3]) == 1000 and not log
    # a raw tier's handles take no arena: every run sees the whole budget
    budgets.clear()
    begin_runs(lambda v, t, c, budget: budgets.append(budget) or NoEncode(), [1, 2, 3], CS, 1000)
    assert budgets == [1000, 1000, 1000]


def test_fan_out_takes_the_larger_part():
    assert FanOutEncode([_Handle([], "a", 7), _Handle([], "b", 9), NoEncode()], None).arena_bytes == 9


def test_begin_runs_abandons_on_refusal_and_error():
    log = []

    def begin(view, tok_begin, cs, budget):
        if view == "none":
            return None
        if view == "boom":
            raise RuntimeError("boom")
        return _Handle(log, view)
    assert begin_runs(begin, ["a", "b", "none", "c"], CS, 10) is None
    assert log == [("abandon", "a"), ("abandon", "b")]
    log.clear()
    with pytest.raises(RuntimeError):
        begin_runs(begin, ["a", "boom"], CS, 10)
    assert log == [("abandon", "a")]


class _Stream:
    def __init__(self, name="s"):
        self.name, self.waited = name, []

    def wait_event(self, ev):
        self.waited.append(ev)


class _Gather:
    def __init__(self, log):
        self.log, self.side = log, _Stream("side")

    def layer(self, layer, stream):
        self.log.append(("gather", layer, stream))
        return f"g{layer}"

    def join(self, events):
        self.log.append(("join", list(events)))
        return "joined"


def _segments_handle(L=3, head=True, runs=2):
    log = []
    head_log = []
    h0 = LayerwiseStore(L, _Handle(head_log, "head"), lambda s, e: head_log.append(("publish", s))) if head else None
    handles = [_Handle(log, f"r{i}") for i in range(runs)]
    published = []

    def publish(stream, enc):
        if enc is None:
            return
        if enc.head is not None:
            enc.head.finish(stream)
        published.extend(h.name for h in enc.handles)
    enc = SegmentsEncode(h0, handles, _Gather(log) if runs else None)
    return LayerwiseStore(L, enc, publish), log, head_log, published


def test_forwarding_to_the_head_and_every_run_in_save_order():
    h, log, head_log, published = _segments_handle()
    s = _Stream()
    for layer in (2, 0, 1):
        h.save_layer(layer, s)
    assert [e[2] for e in head_log if e[0] == "encode"] == [2, 0, 1]
    # one gather per save on the caller's stream, then every run's encode on the side stream behind its event
    want = []
    for layer in (2, 0, 1):
        want += [("gather", layer, s)] + [("encode", f"r{i}", layer, "side", f"g{layer}") for i in range(2)]
    got = [(e[0], e[1], e[2], e[3].name, e[4]) if e[0] == "encode" else e for e in log]
    assert got == want
    with pytest.raises(ValueError, match="saved before"):
        h.save_layer(1, s)
    h.finish(s)
    assert log[-3:] == [("finish", "r0"), ("finish", "r1"), ("join", ["fin-r0", "fin-r1"])]
    assert s.waited == ["joined", "fin-head"]                   # the runs and gathers, then the head's encode
    assert ("publish", s) in head_log and published == ["r0", "r1"]
    with pytest.raises(ValueError, match="before"):
        h.finish(s)
    assert not any(e[0] == "abandon" for e in log + head_log)


def test_missing_layer_and_close_abandon_every_part():
    h, log, head_log, published = _segments_handle()
    s = _Stream()
    h.save_layer(0, s)
    h.save_layer(2, s)
    with pytest.raises(ValueError, match=r"\[1\]"):
        h.finish(s)
    assert ("abandon", "head") in head_log and ("abandon", "r0") in log and ("abandon", "r1") in log
    assert not published and not any(e[0] == "finish" for e in log)
    h, log, head_log, published = _segments_handle()
    h.close()
    assert ("abandon", "head") in head_log and [e for e in log if e[0] == "abandon"] == [("abandon", "r0"),
                                                                                       ("abandon", "r1")]
    h, log, head_log, _ = _segments_handle()
    h.save_layer(0, _Stream())
    del h
    assert ("abandon", "head") in head_log and ("abandon", "r1") in log


def test_head_only_and_runs_only():
    h, log, head_log, published = _segments_handle(L=2, runs=0)
    s = _Stream()
    h.save_layer(0, s)
    h.save_layer(1, s)
    h.finish(s)
    assert not log and published == [] and ("publish", s) in head_log
    h, log, head_log, published = _segments_handle(L=2, head=False)
    h.save_layer(1, s)
    h.save_layer(0, s)
    h.finish(s)
    assert published == ["r0", "r1"] and not head_log


# ---------------------------------------------------------------------------------------------- fallback choice
class _Tier:
    def __init__(self, view=True, max_tokens=4096):
        self._view, self.layerwise_max_tokens = view, max_tokens

    def supports_kv_view(self):
        return self._view

    def begin_layerwise_store(self, view, tok_begin, chunk_size, budget=None):
        raise AssertionError("the fallback begins no layer-wise store")


class _Meta:
    fmt, dtype, model_name, world_size, worker_id = "vllm", "bfloat16", "m", 1, 0


def _engine(tier, chunk_size=CS, fmt="vllm"):
    eng = object.__new__(LMCacheEngine)
    eng.engine_, eng.chunk_size, eng._mla, eng._seg_stream = tier, chunk_size, False, None
    eng.metadata = _Meta()
    eng.metadata.fmt = fmt
    calls = []
    eng.store_paged_segments = lambda *a, **kw: calls.append(("paged", a, kw))
    eng.store_segments = lambda *a, **kw: calls.append(("dense", a, kw))
    return eng, calls


@pytest.mark.parametrize("tier,cs", [(_Tier(max_tokens=0), CS), (_Tier(max_tokens=256), 512), (_Tier(view=False), CS)])
def test_paged_fallback_runs_the_whole_form_at_finish(tier, cs):
    """a torch-serde remote tier (layerwise_max_tokens 0), a chunk over the tier's limit, a tier without KV views"""
    eng, calls = _engine(tier, cs)
    T, L = 600, 2
    caches = [(torch.zeros(40, 16, 2, 64, dtype=torch.bfloat16), torch.zeros(40, 16, 2, 64, dtype=torch.bfloat16))
              for _ in range(L)]
    spec = RopeSpec.from_base(64, 1e4)
    tokens, slots = torch.arange(T), torch.arange(T)
    h = eng.store_paged_segments_layerwise(tokens, caches, slots, [(100, 400)], spec, skip_existing=False)
    s = _Stream()
    for layer in range(L):
        h.save_layer(layer, s)
    assert not calls
    h.finish(s)
    assert len(calls) == 1 and calls[0][0] == "paged"
    assert calls[0][1][3] == [(100, 400)] and calls[0][1][4] is spec and calls[0][1][5] is False


@pytest.mark.parametrize("fmt", ["vllm", "huggingface"])
def test_dense_fallback_for_kv_not_on_the_gpu(fmt):
    eng, calls = _engine(_Tier(), CS, fmt)
    T, L = 300, 2
    shape = (T, 2, 64) if fmt == "vllm" else (2, T, 64)
    kv = tuple((torch.zeros(shape, dtype=torch.bfloat16), torch.zeros(shape, dtype=torch.bfloat16)) for _ in range(L))
    h = eng.store_segments_layerwise(torch.arange(T), kv, [(0, 100), (120, 300)], RopeSpec.from_base(64, 1e4))
    s = _Stream()
    for layer in range(L):
        h.save_layer(layer, s)
    h.finish(s)
    assert [c[0] for c in calls] == ["dense"]


def test_refusals_come_first_even_on_a_fallback_tier():
    eng, calls = _engine(_Tier(max_tokens=0))
    caches = [(torch.zeros(40, 16, 2, 64, dtype=torch.bfloat16), torch.zeros(40, 16, 2, 64, dtype=torch.bfloat16))]
    tokens, slots = torch.arange(600), torch.arange(600)
    with pytest.raises(ValueError, match="overlap"):
        eng.store_paged_segments_layerwise(tokens, caches, slots, [(10, 100), (50, 200)], RopeSpec.from_base(64, 1e4))
    with pytest.raises(ValueError, match="do not fit"):
        eng.store_paged_segments_layerwise(tokens, caches, slots, [(10, 100)], RopeSpec.from_base(64, 1e4, "neox", 8))
    with pytest.raises(TypeError):
        eng.store_paged_segments_layerwise(tokens, caches, slots, [(10, 100)], "not a spec")
    fp8 = [(torch.zeros(40, 16, 2, 64, dtype=torch.float8_e4m3fn),) * 2]
    with pytest.raises(TypeError):
        eng.store_paged_segments_layerwise(tokens, fp8, slots, [(10, 100)], RopeSpec.from_base(64, 1e4))
    assert not calls
