"""Writes tests/golden/ac_edges.npz: the streams found by ac_edges.search() -- own-CDF columns that reach every carry,
pending-run, shift, termination and decoder edge of the arithmetic coder (container version 1) and tell every
killable mutant from the spec, the longest own-CDF stream found, and the chunk-wide-CDF columns (among them chunks of
65505 tokens whose lone symbol has CDF width 1).  Seeded and deterministic; nothing but numpy and tests/cdf_edges.py
is involved.  The file is kept because the search takes minutes.

    python tests/golden/make_ac_edges.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import ac_edges as A  # noqa: E402

if __name__ == "__main__":
    out = A.search()
    np.savez_compressed(A.FIXTURE, **out)
    print(f"{out['g'].size} own-CDF rows, longest stream {int(out['longest'])} bytes (bound "
          f"{A.own_bound_bits() / 8:.2f}, row {4 * A.ROW_WORDS_OWN}), {os.path.getsize(A.FIXTURE)} bytes")
