"""GPU: the prefix-hash chain and the KV mover against plain references, bit for bit.

* b200kv_sha256_chain[_ready] and sha256_prefix_chain[_lazy] against hashlib (hash_mover_ref.ref_chain, the reference
  engine's own hash call): element sizes 1, 2, 4 and 8 at every SHA-256 padding class on chained chunks, every ragged
  last chunk, token bases that are not 4-byte aligned, up to 200 sequences (several CTAs of the chain kernel) with empty
  and long chains, ready words and guard bands, two streams sharing the library's scratch buffer, and every refusal.
* b200kv_pack_chunks / b200kv_unpack_chunks against torch indexing: blob, tuple, padded-blob, paged and latent KVs, both
  chunk layouts, the vector and the scalar path, chunks in device and in mapped page-locked host memory, gaps between
  chunks, grids too small for the work; every byte outside what a call covers keeps its sentinel.
* b200kv_copy_batch_async: ~1000 odd-sized copies at odd offsets in every direction, zero-size entries, stream order
  on both sides of the batch, refusals.
KV data are random int16 bit patterns (NaN payloads and +-0 among them) viewed as bf16 / fp16 and compared as int16."""
import ctypes
import threading

import numpy as np
import pytest
import torch

from hash_mover_ref import NP_DTYPE, PAD_CHUNK_SIZES, n_chunks, random_tokens, ref_chain, ref_chain_seqs

pytestmark = pytest.mark.gpu

GUARD = 96          # sentinel bytes checked past the end of every output
SENT8 = 0xAA        # byte sentinel of digest and chunk buffers
SENT16 = -0x5A5B    # int16 sentinel of KV destinations (0xA5A5)


def _N():
    from lmcache_b200 import _native as N
    return N


def _s(stream=None):
    return (stream or torch.cuda.current_stream()).cuda_stream


@pytest.fixture(scope="module")
def pinned():
    from lmcache_b200.codec import PinnedBuffer
    buf = PinnedBuffer(8 << 20)
    yield buf
    buf.close()


def _host(pin, nbytes, dtype=np.uint8, offset=0):
    return np.frombuffer(pin.view(offset, nbytes * np.dtype(dtype).itemsize), dtype)


# ==================================================================================================== hash chain
def _dev_tokens(toks: np.ndarray, k: int = 0) -> torch.Tensor:
    """toks on the device, k elements into a larger allocation: a base that is not 4-byte aligned when k * es % 4 != 0."""
    full = np.concatenate([random_tokens(np.random.default_rng(k), k, toks.dtype.itemsize), toks,
                           random_tokens(np.random.default_rng(k + 1), 8, toks.dtype.itemsize)])
    return torch.from_numpy(full).cuda()[k:k + toks.shape[0]]


def _chain(tokens_ptr: int, es: int, offs, cs: int, stream=None):
    """b200kv_sha256_chain into a sentinel-filled device buffer; returns the hex digests and checks the guard band."""
    N = _N()
    n = n_chunks(offs, cs)
    out = torch.full((32 * n + GUARD,), SENT8, dtype=torch.uint8, device="cuda")
    N.check(N.lib().b200kv_sha256_chain(ctypes.c_void_p(tokens_ptr), es, N.i64_array(offs), len(offs) - 1, cs,
                                        ctypes.c_void_p(out.data_ptr()), _s(stream)), "sha256_chain")
    host = out.cpu().numpy()
    assert (host[32 * n:] == SENT8).all(), "digest written past the last chunk"
    return [bytes(host[32 * i:32 * i + 32]).hex() for i in range(n)]


SWEEP_CS = {1: 57, 2: 27, 4: 14, 8: 7}


@pytest.mark.parametrize("es", [1, 2, 4, 8])
def test_chain_padding_classes(es):
    """Every padding class of the element size on chained chunks (three or more per sequence, full and ragged last
    chunks), then, for one small chunk size, every length of the ragged last chunk after two chained ones (one sequence
    each, so the call spans two CTAs of the chain kernel)."""
    rng = np.random.default_rng(10 + es)
    for cs in PAD_CHUNK_SIZES[es]:
        lens = [3 * cs, 3 * cs + 1, 4 * cs - 1, 5 * cs + cs // 2]
        offs = np.concatenate([[0], np.cumsum(lens)]).tolist()
        toks = random_tokens(rng, offs[-1], es)
        assert _chain(_dev_tokens(toks).data_ptr(), es, offs, cs) == ref_chain_seqs(toks, offs, cs), (es, cs)
    cs = SWEEP_CS[es]
    lens = [2 * cs + r for r in range(1, cs + 1)]
    offs = np.concatenate([[0], np.cumsum(lens)]).tolist()
    toks = random_tokens(rng, offs[-1], es)
    assert _chain(_dev_tokens(toks).data_ptr(), es, offs, cs) == ref_chain_seqs(toks, offs, cs)


@pytest.mark.parametrize("es,k", [(1, 1), (1, 2), (1, 3), (2, 1)])
def test_chain_misaligned_tokens(es, k):
    """Token bases 1, 2 or 3 bytes past a word boundary: the expand kernel reads every word of such a chunk byte by byte.
    Odd chunk sizes make chunk starts alternate in alignment; odd sequence offsets do the same for sequence starts.
    The device tensor is hashed where it is; a host tensor is uploaded to an aligned buffer first."""
    from lmcache_b200.cache_engine import sha256_prefix_chain
    rng = np.random.default_rng(20 + 4 * es + k)
    for cs in ([55, 57, 63, 119] if es == 1 else [27, 59]):
        n = 5 * cs + 3
        toks = random_tokens(rng, n, es)
        want = ref_chain(toks, cs)
        dev = _dev_tokens(toks, k)
        assert dev.data_ptr() % 4 != 0
        assert _chain(dev.data_ptr(), es, [0, n], cs) == want, cs
        assert sha256_prefix_chain(dev, cs) == want, cs
        host = torch.from_numpy(np.concatenate([toks[:k], toks]))[k:]
        assert host.storage_offset() == k
        assert sha256_prefix_chain(host, cs) == want, cs
        offs = [0, 3, 3 + 2 * cs + 1, n]
        assert _chain(dev.data_ptr(), es, offs, cs) == ref_chain_seqs(toks, offs, cs), cs
        assert sha256_prefix_chain(dev, cs, offs) == ref_chain_seqs(toks, offs, cs), cs


@pytest.mark.parametrize("n_seq,es", [(31, 1), (32, 2), (33, 4), (64, 8), (65, 2), (200, 8)])
def test_chain_many_sequences(n_seq, es):
    """Chains of very different lengths in one call: empty sequences first, last and several in a row, 1, cs - 1, cs
    and cs + 1 tokens, and three chains of 64 or more chunks; the digests come back to back in sequence order."""
    rng = np.random.default_rng(n_seq)
    cs = 16
    lens = rng.choice([0, 1, cs - 1, cs, cs + 1, 2 * cs + 3, 5 * cs], n_seq).tolist()
    lens[0] = lens[-1] = 0
    lens[5:9] = [0, 0, 0, 0]
    for i in (2, n_seq // 2, n_seq - 3):
        lens[i] = 64 * cs + int(rng.integers(0, cs))
    offs = np.concatenate([[0], np.cumsum(lens)]).tolist()
    toks = random_tokens(rng, offs[-1], es)
    want = ref_chain_seqs(toks, offs, cs)
    assert len(want) == n_chunks(offs, cs)
    assert _chain(_dev_tokens(toks).data_ptr(), es, offs, cs) == want


def test_chain_ready_words_and_guard_bands(pinned):
    """b200kv_sha256_chain_ready into mapped page-locked memory larger than needed: every ready word of a digest slot
    holds the epoch afterwards, every digest byte and ready word past the last slot keeps its sentinel (a stale epoch).
    The same into device buffers, and with ready = NULL."""
    N = _N()
    lib = N.lib()
    rng = np.random.default_rng(30)
    cs, es = 32, 4
    lens = [0, 5 * cs + 7, 1, 0, cs] + [int(x) for x in rng.integers(0, 4 * cs, 40)] + [0]
    offs = np.concatenate([[0], np.cumsum(lens)]).tolist()
    toks = random_tokens(rng, offs[-1], es)
    dev = _dev_tokens(toks)
    want = ref_chain_seqs(toks, offs, cs)
    n = len(want)
    cap = n + 37
    epoch, stale = 0x5EED0002, 0x5EED0001
    dig = _host(pinned, 32 * cap)
    ready = _host(pinned, cap, np.uint32, offset=32 * cap)
    dig[:] = SENT8
    ready[:] = stale
    N.check(lib.b200kv_sha256_chain_ready(dev.data_ptr(), es, N.i64_array(offs), len(lens), cs, pinned.dev_ptr,
                                          pinned.dev_ptr + 32 * cap, epoch, _s()), "sha256_chain_ready")
    torch.cuda.synchronize()
    assert [bytes(dig[32 * i:32 * i + 32]).hex() for i in range(n)] == want
    assert (dig[32 * n:] == SENT8).all()
    assert (ready[:n] == epoch).all() and (ready[n:] == stale).all()
    # device digests and ready words
    ddig = torch.full((32 * cap,), SENT8, dtype=torch.uint8, device="cuda")
    dready = torch.full((cap,), stale, dtype=torch.int32, device="cuda")
    N.check(lib.b200kv_sha256_chain_ready(dev.data_ptr(), es, N.i64_array(offs), len(lens), cs, ddig.data_ptr(),
                                          dready.data_ptr(), epoch, _s()), "sha256_chain_ready")
    hd, hr = ddig.cpu().numpy(), dready.cpu().numpy().view(np.uint32)
    assert [bytes(hd[32 * i:32 * i + 32]).hex() for i in range(n)] == want
    assert (hd[32 * n:] == SENT8).all()
    assert (hr[:n] == epoch).all() and (hr[n:] == stale).all()
    # ready = NULL: the same digests
    ddig.fill_(SENT8)
    N.check(lib.b200kv_sha256_chain_ready(dev.data_ptr(), es, N.i64_array(offs), len(lens), cs, ddig.data_ptr(), None,
                                          epoch, _s()), "sha256_chain_ready")
    hd = ddig.cpu().numpy()
    assert [bytes(hd[32 * i:32 * i + 32]).hex() for i in range(n)] == want and (hd[32 * n:] == SENT8).all()


def test_chain_shared_scratch_two_streams():
    """The library's grow-only scratch buffer: one call larger than any other in the suite (it must grow the buffer;
    ~34 MB of scratch), then two threads on two streams, each with 20 calls that alternate small and large inputs and
    no host synchronisation between them.  Calls on different streams reuse the same scratch, ordered by the library's
    event; every digest must equal hashlib's."""
    rng = np.random.default_rng(40)
    big = random_tokens(rng, 1 << 20, 8)
    assert _chain(_dev_tokens(big).data_ptr(), 8, [0, big.shape[0]], 256) == ref_chain(big, 256)

    # per thread: (element size, chunk size, sequences x tokens) of the large and the small inputs
    plans = [((8, 256, 32, 8192), (4, 16, 1, 300)), ((4, 128, 48, 4096), (2, 32, 3, 200))]
    jobs = []
    for (large, small) in plans:
        calls = []
        for i in range(20):
            es, cs, nseq, per = large if i % 2 == 0 else small
            offs = [per * s for s in range(nseq + 1)]
            toks = random_tokens(rng, offs[-1], es)
            calls.append((es, cs, offs, toks, _dev_tokens(toks)))
        jobs.append(calls)
    torch.cuda.synchronize()
    N = _N()
    results = [[] for _ in jobs]
    errors = []

    def worker(t):
        try:
            stream = torch.cuda.Stream()
            with torch.cuda.stream(stream):
                for es, cs, offs, _, dev in jobs[t]:
                    out = torch.empty(32 * n_chunks(offs, cs), dtype=torch.uint8, device="cuda")
                    rc = N.lib().b200kv_sha256_chain(dev.data_ptr(), es, N.i64_array(offs), len(offs) - 1, cs,
                                                     out.data_ptr(), stream.cuda_stream)
                    results[t].append((rc, out))
            stream.synchronize()
        except Exception as e:       # noqa: BLE001 -- re-raised in the test's thread
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(len(jobs))]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for t, calls in enumerate(jobs):
        for i, ((es, cs, offs, toks, _), (rc, out)) in enumerate(zip(calls, results[t])):
            assert rc == 0, N.last_error()
            host = out.cpu().numpy()
            got = [bytes(host[32 * k:32 * k + 32]).hex() for k in range(host.shape[0] // 32)]
            assert got == ref_chain_seqs(toks, offs, cs), (t, i)


def test_chain_refusals_write_nothing():
    """Refused calls return < 0 and write no digest and no ready word; a call whose sequences are all empty returns 0
    and writes nothing."""
    N = _N()
    lib = N.lib()
    toks = torch.arange(64, dtype=torch.int64, device="cuda")
    dig = torch.full((32 * 8 + GUARD,), SENT8, dtype=torch.uint8, device="cuda")
    ready = torch.full((16,), 7, dtype=torch.int32, device="cuda")
    tp, dp, rp = toks.data_ptr(), dig.data_ptr(), ready.data_ptr()

    def call(tokens, es, offs, n_seq, cs, digests=dp):
        return lib.b200kv_sha256_chain_ready(tokens, es, None if offs is None else N.i64_array(offs), n_seq, cs,
                                             digests, rp, 9, _s())

    refused = {
        "elem_size 3": call(tp, 3, [0, 8], 1, 4),
        "elem_size 0": call(tp, 0, [0, 8], 1, 4),
        "chunk_size 0": call(tp, 8, [0, 8], 1, 0),
        "chunk_size < 0": call(tp, 8, [0, 8], 1, -4),
        "decreasing offsets": call(tp, 8, [0, 8, 4], 2, 4),
        "n_seq 0": call(tp, 8, [0], 0, 4),
        "NULL offsets": call(tp, 8, None, 1, 4),
        "NULL tokens": call(None, 8, [0, 8], 1, 4),
        "NULL digests": call(tp, 8, [0, 8], 1, 4, digests=None),
    }
    for what, rc in refused.items():
        assert rc < 0, what
    assert call(tp, 8, [0, 0, 0, 0], 3, 4) == 0
    assert call(None, 8, [5, 5], 1, 4) == 0
    assert lib.b200kv_sha256_chain(tp, 8, N.i64_array([0, 0]), 1, 4, dp, _s()) == 0
    torch.cuda.synchronize()
    assert (dig.cpu().numpy() == SENT8).all() and (ready.cpu().numpy() == 7).all()


@pytest.mark.parametrize("dtype", [torch.int16, torch.uint8])
def test_prefix_chain_wrappers(dtype):
    """sha256_prefix_chain and its lazy form hash a tensor's native bytes: int16 and uint8 tensors, a non-contiguous
    view and a slice at an odd storage offset, one or several sequences; lazy digests read in any order."""
    from lmcache_b200.cache_engine import sha256_prefix_chain, sha256_prefix_chain_lazy
    es = torch.empty((), dtype=dtype).element_size()
    rng = np.random.default_rng(50 + es)
    base = torch.from_numpy(random_tokens(rng, 4001, es).view(NP_DTYPE[es])).cuda()
    for t in (base, base[::2], base[3:], base[1:3000]):
        want_src = t.cpu().numpy()
        for cs in (57, 256):
            want = ref_chain(want_src, cs)
            assert sha256_prefix_chain(t, cs) == want, (t.storage_offset(), cs)
            lz = sha256_prefix_chain_lazy(t, cs)
            assert [lz[i] for i in reversed(range(len(lz)))] == want[::-1]
        offs = [0, 7, 7, 1000, t.shape[0]]
        assert list(sha256_prefix_chain_lazy(t, 61, offs)) == ref_chain_seqs(want_src, offs, 61)


# ==================================================================================================== pack / unpack
KINDS = ["blob_vllm", "blob_hf", "tuple_vllm", "tuple_hf", "blob_pad_d", "blob_pad_tok", "paged", "latent_blob",
         "latent_tuple", "latent_paged"]
SPECIALS = [0, -0x8000, 0x7FC1, -0x003F, 0x7E01, -1, 0x7F80, -0x0080, 0x7C00, 0x0001]   # +-0, NaN payloads, infs


def _bits(shape, gen) -> torch.Tensor:
    """Random int16 bit patterns; NaN payloads, infinities and +-0 of bf16 and fp16 spread through them."""
    x = torch.randint(-0x8000, 0x8000, shape, dtype=torch.int16, device="cuda", generator=gen)
    flat = x.view(-1)
    step = max(1, flat.numel() // 97)
    m = flat[::step].numel()
    flat[::step] = torch.tensor(SPECIALS, dtype=torch.int16, device="cuda").repeat(m // len(SPECIALS) + 1)[:m]
    return x


def _sentinel(shape, gen=None) -> torch.Tensor:
    return torch.full(shape, SENT16, dtype=torch.int16, device="cuda")


class Src:
    """A KV source or destination of one kind: the physical allocations (`storage`, compared whole, padding and unmapped
    paged rows included), the token-major views [rows, H, D] of its P * L planes (plane kv * L + l), the slot map of a
    paged KV, and the KvView the library gets."""

    def __init__(self, kind, L, H, D, T, fill, slot=None, plane_off2=False):
        from lmcache_b200.codec import KvView
        self.kind, self.T, self.plane_off2 = kind, T, plane_off2
        self.latent = kind.startswith("latent")
        self.P, self.L, self.H, self.D = (1 if self.latent else 2), L, (1 if self.latent else H), D
        H = self.H
        dt = torch.float16 if kind.endswith("hf") else torch.bfloat16
        self.slot = None
        if kind in ("blob_vllm", "blob_pad_d", "blob_pad_tok"):
            pad_d, pad_h = {"blob_vllm": (0, 0), "blob_pad_d": (8, 0), "blob_pad_tok": (0, 1)}[kind]
            phys = fill([L, 2, T, H + pad_h, D + pad_d])
            blob = phys[:, :, :, :H, :D]
            self.storage, self.planes = [phys], [blob[l, kv] for kv in range(2) for l in range(L)]
            self.view = KvView.from_blob(blob.view(dt), "vllm")
        elif kind == "blob_hf":
            phys = fill([L, 2, H, T, D])
            self.storage, self.planes = [phys], [phys[l, kv].transpose(0, 1) for kv in range(2) for l in range(L)]
            self.view = KvView.from_blob(phys.view(dt), "huggingface")
        elif kind in ("tuple_vllm", "tuple_hf"):
            shape = [T, H, D] if kind == "tuple_vllm" else [H, T, D]
            ts = [fill(shape) for _ in range(2 * L)]
            self.storage = list(ts)
            if plane_off2:     # plane 3 starts 2 bytes into its allocation
                self.storage[3] = fill([T * H * D + 1])
                ts[3] = self.storage[3][1:].view(shape)
            self.planes = ts if kind == "tuple_vllm" else [t.transpose(0, 1) for t in ts]
            self.view = KvView.from_tuple(tuple((ts[l].view(dt), ts[L + l].view(dt)) for l in range(L)),
                                          "vllm" if kind == "tuple_vllm" else "huggingface")
        elif kind in ("paged", "latent_paged"):
            bs = 16
            nb = (T + 29 + bs - 1) // bs
            if slot is None:    # a permutation of more rows than tokens: some rows are mapped by no token
                slot = torch.randperm(nb * bs, generator=torch.Generator().manual_seed(T))[:T].cuda()
            self.slot = slot
            shape = [nb, bs, D] if self.latent else [nb, bs, H, D]
            self.storage = [fill(shape) for _ in range(self.P * L)]
            self.planes = [c.view(nb * bs, H, D) for c in self.storage]
            cv = [c.view(dt) for c in self.storage]
            self.view = KvView.from_paged(cv if self.latent else [(cv[l], cv[L + l]) for l in range(L)], self.slot)
        elif kind == "latent_blob":
            phys = fill([L, T, D + 8])      # padded rows: sT = D + 8
            blob = phys[:, :, :D]
            self.storage, self.planes = [phys], [blob[l].unsqueeze(1) for l in range(L)]
            self.view = KvView.from_blob(blob.view(dt), "vllm")
        elif kind == "latent_tuple":
            self.storage = [fill([T, D]) for _ in range(L)]
            self.planes = [t.unsqueeze(1) for t in self.storage]
            self.view = KvView.from_tuple([t.view(dt) for t in self.storage], "vllm")
        else:
            raise ValueError(kind)

    def twin(self, fill):
        """Same kind and geometry (same slot map, same plane offsets), other contents."""
        return Src(self.kind, self.L, self.H, self.D, self.T, fill, slot=self.slot, plane_off2=self.plane_off2)

    def chunk_bytes(self, cs):
        return self.P * self.L * cs * self.H * self.D * 2

    def logical(self) -> torch.Tensor:
        """[L, P, T, H, D]: the tokens of the view, paged rows gathered through the slot map."""
        rows = [p if self.slot is None else p.index_select(0, self.slot) for p in self.planes]
        return torch.stack(rows).view(self.P, self.L, self.T, self.H, self.D).transpose(0, 1)

    def write(self, tok0, data):
        """Tokens [tok0, tok0 + n) of the view = data [L, P, n, H, D], through torch indexing."""
        n = data.shape[2]
        for kv in range(self.P):
            for l in range(self.L):
                p = self.planes[kv * self.L + l]
                if self.slot is None:
                    p[tok0:tok0 + n] = data[l, kv]
                else:
                    p[self.slot[tok0:tok0 + n]] = data[l, kv]


def _chunk_image(x, tb, nc, cs, last, hf, off, stride, size):
    """The chunk buffer a pack of x must produce: chunk j ([L,P,t,H,D], or [L,P,H,t,D] for hf) at off + j * stride,
    the sentinel everywhere else."""
    img = torch.full((size,), SENT8, dtype=torch.uint8, device="cuda")
    for j in range(nc):
        t = cs if j < nc - 1 else last
        b = x[:, :, tb + j * cs: tb + j * cs + t]
        if hf:
            b = b.permute(0, 1, 3, 2, 4)
        b = b.contiguous().view(-1).view(torch.uint8)
        img[off + j * stride: off + j * stride + b.numel()] = b
    return img


class _Chunks:
    """A sentinel-filled chunk buffer in device or mapped page-locked host memory; `ptr` is its device address + off."""

    def __init__(self, size, mem, off, pinned):
        self.mem = mem
        if mem == "dev":
            self.t = torch.full((size,), SENT8, dtype=torch.uint8, device="cuda")
            self.ptr = self.t.data_ptr() + off
        else:
            assert size <= pinned.nbytes
            self.t = torch.from_numpy(_host(pinned, size))
            self.t.fill_(SENT8)
            self.ptr = pinned.dev_ptr + off

    def read(self):
        return self.t.cuda()


def _pack_unpack(src, tb, nc, cs, last, hf, mem, pinned, stride_extra=0, off=0):
    """pack = the torch-made chunk image (gaps and tail keep the sentinel); unpack of it into a sentinel-filled twin =
    torch indexing of the covered tokens into another sentinel-filled twin, compared over every allocated element."""
    N = _N()
    lib = N.lib()
    x = src.logical()
    stride = src.chunk_bytes(cs) + stride_extra
    size = off + (nc - 1) * stride + src.chunk_bytes(last) + GUARD
    want = _chunk_image(x, tb, nc, cs, last, hf, off, stride, size)
    ch = _Chunks(size, mem, off, pinned)
    torch.cuda.synchronize()
    N.check(lib.b200kv_pack_chunks(ctypes.byref(src.view.desc), tb, nc, cs, last, hf, ch.ptr, stride, _s()), "pack")
    torch.cuda.synchronize()
    assert torch.equal(ch.read(), want), "pack"
    dst = src.twin(_sentinel)
    N.check(lib.b200kv_unpack_chunks(ch.ptr, stride, nc, cs, last, hf, ctypes.byref(dst.view.desc), tb, _s()), "unpack")
    exp = src.twin(_sentinel)
    n = (nc - 1) * cs + last
    exp.write(tb, x[:, :, tb:tb + n])
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(dst.storage, exp.storage)):
        assert torch.equal(a, b), f"unpack: allocation {i}"
    assert torch.equal(dst.logical()[:, :, tb:tb + n], x[:, :, tb:tb + n])


# (tok_begin, n_chunks, tokens of the last chunk) with chunks of 16 tokens
GEOMETRIES = [(0, 1, 16), (0, 1, 1), (37, 1, 15), (0, 3, 16), (37, 3, 1), (37, 3, 15)]


@pytest.mark.parametrize("D", [128, 20, 33])
@pytest.mark.parametrize("kind", KINDS)
def test_pack_unpack(kind, D, pinned):
    """Every KV kind against torch indexing, both chunk layouts, every geometry; chunks in device memory, in mapped
    page-locked host memory, and at a stride 48 bytes past the chunk.  D = 128 takes the vector path (8 halfs per
    access): every stride here is a multiple of 8 halfs, every plane and chunk address and the chunk stride multiples of
    16 bytes.  D = 20 and D = 33 are not multiples of 8 and take the scalar path."""
    gen = torch.Generator(device="cuda").manual_seed(1000 * KINDS.index(kind) + D)
    src = Src(kind, 3, 2, D, 100, lambda s: _bits(s, gen))
    for tb, nc, last in GEOMETRIES:
        for hf in (0, 1):
            for mem, extra in (("dev", 0), ("pinned", 0), ("dev", 48)):
                _pack_unpack(src, tb, nc, 16, last, hf, mem, pinned, stride_extra=extra)


@pytest.mark.parametrize("how", ["plane_off2", "chunks_off2", "stride_off2"])
def test_pack_unpack_forced_scalar(how, pinned):
    """D = 128, which would take the vector path, sent down the scalar path by each alignment check in turn: one plane
    tensor 2 bytes into its allocation, the chunk buffer 2 bytes past a 16-byte boundary, a chunk stride 2 bytes longer
    than the chunk (not a multiple of 16).  Every access stays 2-byte aligned, which is all the scalar path needs."""
    gen = torch.Generator(device="cuda").manual_seed(61)
    src = Src("tuple_vllm", 3, 2, 128, 100, lambda s: _bits(s, gen), plane_off2=how == "plane_off2")
    if how == "plane_off2":
        assert src.planes[3].data_ptr() % 16 == 2
    for tb, nc, last in GEOMETRIES:
        for hf in (0, 1):
            for mem in ("dev", "pinned"):
                _pack_unpack(src, tb, nc, 16, last, hf, mem, pinned, off=2 if how == "chunks_off2" else 0,
                             stride_extra=2 if how == "stride_off2" else 0)


@pytest.mark.parametrize("D,T,hf", [(128, 1024, 0), (20, 2048, 1)])
def test_pack_unpack_grid_stride(D, T, hf, pinned):
    """More units than the launch's grid holds (SMs x 32 CTAs x 256 threads), so every thread runs its grid-stride loop
    several times: L 32, H 8, D 128 on the vector path (8 halfs a unit), D 20 on the scalar path (1 half a unit)."""
    L, H, cs = 32, 8, 256
    units = 2 * L * T * H * (D // 8 if D % 8 == 0 else D)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert units > 2 * sms * 32 * 256
    gen = torch.Generator(device="cuda").manual_seed(62)
    src = Src("tuple_vllm", L, H, D, T + 40, lambda s: _bits(s, gen))
    _pack_unpack(src, 40, T // cs, cs, cs, hf, "dev", pinned)


def test_pack_unpack_refusals_write_nothing():
    """n_chunks 0, a last chunk of 0 or more than chunk_tokens, a chunk stride shorter than a chunk with several chunks,
    NULL chunks: refused (< 0), nothing written into the chunks or the KV."""
    N = _N()
    lib = N.lib()
    gen = torch.Generator(device="cuda").manual_seed(63)
    src = Src("tuple_vllm", 2, 2, 64, 64, lambda s: _bits(s, gen))
    dst = src.twin(_sentinel)
    cb = src.chunk_bytes(16)
    buf = torch.full((4 * cb,), SENT8, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    bad = [("n_chunks 0", p, cb, 0, 16, 16), ("last 0", p, cb, 2, 16, 0), ("last > chunk", p, cb, 2, 16, 17),
           ("chunk_tokens 0", p, cb, 1, 0, 1), ("stride too small", p, cb - 16, 2, 16, 16), ("NULL chunks", None, cb, 2, 16, 16)]
    for what, ptr, stride, nc, cs, last in bad:
        assert lib.b200kv_pack_chunks(ctypes.byref(src.view.desc), 0, nc, cs, last, 0, ptr, stride, _s()) < 0, what
        assert lib.b200kv_unpack_chunks(ptr, stride, nc, cs, last, 0, ctypes.byref(dst.view.desc), 0, _s()) < 0, what
    torch.cuda.synchronize()
    assert (buf.cpu().numpy() == SENT8).all()
    assert all((t == SENT16).all() for t in dst.storage)


# ==================================================================================================== copy_batch_async
def _batch(dsts, srcs, sizes, stream):
    d = np.asarray(dsts, np.uint64)
    s = np.asarray(srcs, np.uint64)
    z = np.asarray(sizes, np.int64)
    return _N().lib().b200kv_copy_batch_async(d.ctypes.data, s.ctypes.data, z.ctypes.data, len(z), stream)


@pytest.mark.parametrize("stream_kind", ["side", "default"])
@pytest.mark.parametrize("route", ["d2d", "d2h", "h2d"])
def test_copy_batch_odd_sizes(route, stream_kind, pinned):
    """~1000 copies of 1..4097 bytes at odd offsets, zero-size entries mixed in, into non-overlapping destinations
    with gaps: the destinations hold the source bytes, every other byte (the zero-size entries' destinations among
    them) keeps its sentinel.  Device -> device, device -> mapped page-locked host, page-locked host -> device; on a
    created stream (one batched driver call) and on the legacy default stream, which the batched call refuses (one
    call per copy there)."""
    rng = np.random.default_rng({"d2d": 1, "d2h": 2, "h2d": 3}[route])
    stream = torch.cuda.Stream() if stream_kind == "side" else torch.cuda.default_stream()
    assert (stream.cuda_stream == 0) == (stream_kind == "default")
    n = 1000
    sizes = rng.integers(1, 4098, n)
    sizes[::97] = 0
    src_len = (1 << 20) + 8192
    src_off = rng.integers(0, src_len - 4097, n) | 1
    dst_off, pos = np.empty(n, np.int64), 0
    for i in range(n):
        pos += int(rng.integers(1, 16))
        pos |= 1
        dst_off[i] = pos
        pos += int(sizes[i])
    dst_len = pos + GUARD
    src_np = rng.integers(0, 256, src_len, dtype=np.uint8)
    want = np.full(dst_len, SENT8, np.uint8)
    for i in range(n):
        want[dst_off[i]:dst_off[i] + sizes[i]] = src_np[src_off[i]:src_off[i] + sizes[i]]
    if route == "h2d":
        src_h = _host(pinned, src_len)
        src_h[:] = src_np
        src_base = pinned.host_ptr
    else:
        src_t = torch.from_numpy(src_np).cuda()
        src_base = src_t.data_ptr()
    if route == "d2h":
        dst_h = _host(pinned, dst_len)
        dst_h[:] = SENT8
        dst_base = pinned.host_ptr
    else:
        dst_t = torch.full((dst_len,), SENT8, dtype=torch.uint8, device="cuda")
        dst_base = dst_t.data_ptr()
    torch.cuda.synchronize()
    assert _batch(dst_base + dst_off, src_base + src_off, sizes, stream.cuda_stream) == 0, _N().last_error()
    torch.cuda.synchronize()
    got = dst_h.copy() if route == "d2h" else dst_t.cpu().numpy()
    assert np.array_equal(got, want)


def test_copy_batch_stream_order():
    """A batch is ordered on its stream both ways: kernels enqueued just before it (no synchronisation) write its
    sources, and a kernel enqueued just after it reads its destinations."""
    rng = np.random.default_rng(4)
    nbytes = 64 << 20
    src = torch.from_numpy(rng.integers(0, 256, nbytes, dtype=np.uint8)).cuda()
    expect_src = src + 16                      # uint8: wraps
    dst = torch.full((nbytes,), SENT8, dtype=torch.uint8, device="cuda")
    n = 200
    sizes = rng.integers(1, 1 << 16, n)        # one copy per 64 KB slot, 3 bytes in: no overlaps, nothing past the end
    off = np.sort(rng.choice(nbytes // (1 << 16) - 1, n, replace=False)) * (1 << 16) + 3
    torch.cuda.synchronize()
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        for _ in range(16):
            src.add_(1)
        rc = _batch(dst.data_ptr() + off, src.data_ptr() + off, sizes, stream.cuda_stream)
        after = dst.to(torch.int16)
    stream.synchronize()
    assert rc == 0, _N().last_error()
    want = torch.full((nbytes,), SENT8, dtype=torch.uint8, device="cuda")
    for o, z in zip(off.tolist(), sizes.tolist()):
        want[o:o + z] = expect_src[o:o + z]
    assert torch.equal(dst, want)
    assert torch.equal(after, want.to(torch.int16))


def test_copy_batch_empty_and_refusals():
    """n = 0 (NULL arrays) and batches of zero-size entries only are no-ops; a NULL pointer with a nonzero size, a
    negative size, or NULL arrays with n > 0 are refused, and then none of the batch's copies is made."""
    lib = _N().lib()
    src = torch.arange(256, dtype=torch.int32, device="cuda").to(torch.uint8)
    dst = torch.full((1024,), SENT8, dtype=torch.uint8, device="cuda")
    s, d = src.data_ptr(), dst.data_ptr()
    assert lib.b200kv_copy_batch_async(None, None, None, 0, _s()) == 0
    assert _batch([d, d + 10], [s, s], [0, 0], _s()) == 0
    assert _batch([d, 0, d + 300], [s, s, s], [100, 100, 100], _s()) < 0
    assert _batch([d, d + 300], [s, 0], [100, 100], _s()) < 0
    assert _batch([d, d + 300], [s, s], [100, -1], _s()) < 0
    assert lib.b200kv_copy_batch_async(None, None, None, 2, _s()) < 0
    torch.cuda.synchronize()
    assert (dst.cpu().numpy() == SENT8).all()
