"""The bound of a key turned twice, on top of the float64 statement of tests/rope_ref.py: a segment stored from inside
a longer prompt is turned by -s when it is stored and by s' when it is retrieved, each turn rounded once to the dtype."""
import numpy as np

from rope_ref import ulp


def tolerance_twice(ref_rounded, got, x, y, dtype_name):
    """what a key turned twice may differ from the float64 statement of one turn by s' - s, rounded (x, y: the pair's
    inputs, before either turn).  The first turn's error, at most one ulp of the pair's magnitude |(x, y)| plus its
    fp32 term on each element, is carried through the second rotation onto both elements: 2 ulp(|(x, y)|) + 2^-20
    (|x| + |y|).  The second turn adds one ulp of the result and its own fp32 term, at most 2^-21 sqrt(2) (|x| + |y|).
    In all: one ulp of the result + two ulps of |(x, y)| + 2^-19 (|x| + |y|)."""
    m = np.sqrt(np.asarray(x, dtype=np.float64) ** 2 + np.asarray(y, dtype=np.float64) ** 2)
    return (np.maximum(ulp(ref_rounded, dtype_name), ulp(got, dtype_name)) + 2 * ulp(m, dtype_name) +
            2.0 ** -19 * (np.abs(x) + np.abs(y)))
