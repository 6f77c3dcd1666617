"""Make tests/golden/cdf_edges.npz: the CDF-normaliser witness set (see tests/cdf_edges.py) with the CDF rows the
reference's own functions give them.

    python tests/golden/make_cdf_edges.py <path of an LMCache v0.1.2 tree>

The histograms come from cdf_edges.build_rows() (every two-part histogram and three-part composition for t <= 256, a
directed many-symbol family, and t in cdf_edges.BIG_T: exact ties, their neighbours, and the rows where a variant of
cdf_edges.VARIANTS differs from the spec).  Each is turned into a symbol column that has it and fed, one token count at a
time, to the reference's CacheGenEncoderImpl.compute_cdf (process_batch, cachegen_encoder.py:185-196) and
_convert_to_int_and_normalize (:95-126), imported from the reference tree with the three stubs of tests/_refstubs: no
reference arithmetic is restated here.

Keys:
  counts   uint16 [N, 33]  the histogram (symbols 0..30; entries 31, 32 are 0)
  t        int32  [N]      tokens
  cdf      int16  [N, 33]  the reference's CDF row
  kind     uint8  [N]      cdf_edges.K_* (tie, tie neighbour, witness, directed)
  domain   uint8  [N]      index into cdf_edges.DOMAINS: the search that produced the row
  tags     uint32 [N]      bit k <=> cdf_edges.VARIANTS[k] differs from the spec on the row
  found    int64  [4, V]   witnesses the search met, per domain and variant (0: equivalent to the spec in that domain)
  ties     int64  [4]      histograms with an exact tie the search met, per domain
  variants                 the variant names, in bit order

The archive is written with fixed member timestamps, so a rerun reproduces it byte for byte."""
import io
import os
import sys
import zipfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.join(HERE, "..", "_refstubs"), sys.argv[1], os.path.dirname(HERE),
                os.path.dirname(os.path.dirname(HERE))]

import numpy as np  # noqa: E402
import torch  # noqa: E402

torch.Tensor.cuda = lambda self, *a, **k: self  # the reference calls .cuda(); CPU-only here

from lmcache.storage_backend.serde.cachegen_encoder import (  # noqa: E402
    CacheGenEncoderImpl, _convert_to_int_and_normalize)

import cdf_edges as E  # noqa: E402


def reference_cdf(counts: np.ndarray, t: int) -> np.ndarray:
    """the reference's CDF rows of histograms [n, 33] that all have t tokens: one layer whose channels are the rows"""
    n = counts.shape[0]
    sym = np.stack([E.column(r) for r in counts], axis=1).astype(np.int8)           # [t, n]
    assert sym.shape == (t, n)
    fp = torch.zeros((1, t, n))
    impl = CacheGenEncoderImpl(fp_k=fp, fp_v=fp, config=None)
    impl.quantized_key = {0: torch.from_numpy(sym)}
    cdf = _convert_to_int_and_normalize(impl.compute_cdf(is_key=True), True)
    assert cdf.shape == (1, n, E.LP) and cdf.dtype == torch.int16
    return cdf[0].numpy().copy()


def save(path: str, arrays: dict):
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for name, a in arrays.items():
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.ascontiguousarray(a), allow_pickle=False)
            info = zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            info.external_attr = 0o644 << 16
            z.writestr(info, buf.getvalue())


def main():
    out = E.build_rows()
    cdf = np.zeros(out["counts"].shape, np.int16)
    for t in np.unique(out["t"]):
        s = out["t"] == t
        cdf[s] = reference_cdf(out["counts"][s], int(t))
    out["cdf"] = cdf
    save(E.FIXTURE, out)
    spec = np.concatenate([E.spec_cdf(out["counts"][i: i + 1], int(out["t"][i])) for i in range(cdf.shape[0])])
    print("rows", cdf.shape[0], "distinct t", np.unique(out["t"]).size, "bytes", os.path.getsize(E.FIXTURE),
          "rows where spec_cdf != reference:", int((spec != cdf).any(axis=1).sum()))
    for d, name in enumerate(E.DOMAINS):
        print(f"  {name:20s} ties {int(out['ties'][d]):6d} ", dict(zip(E.VARIANTS, out["found"][d].tolist())))
    print("torch", torch.__version__, "numpy", np.__version__)


if __name__ == "__main__":
    main()
