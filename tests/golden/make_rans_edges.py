"""Writes tests/golden/rans_edges.npz: the streams found by rans_edges.search() -- own-CDF columns (a histogram and an
order each) that reach every arithmetic and window edge of the rANS coder and tell every killable mutant from the
spec, the longest own-CDF stream the directed search found, and the chunk-wide-CDF columns.  Seeded and deterministic;
nothing but numpy and tests/cdf_edges.py is involved.  The file is kept because the search takes minutes.

    python tests/golden/make_rans_edges.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import rans_edges as R  # noqa: E402

if __name__ == "__main__":
    out = R.search()
    np.savez_compressed(R.FIXTURE, **out)
    print(f"{out['g'].size} own-CDF rows, longest stream {int(out['longest'])} halfwords (proven bound "
          f"{R.PROVEN_MAX_HALFWORDS}), {os.path.getsize(R.FIXTURE)} bytes")
