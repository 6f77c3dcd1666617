"""Make tests/golden/quant_edges.npz: the quantiser / dequantiser witness set (see tests/quant_edges.py).

For bf16 and fp16 and every MAX 1..15, an exhaustive scan over every finite x with |x| <= m (both signs) against the
ladder of row maxima (quant_edges.ladder) finds
  * every exact tie (fp32 x * f + MAX == k + 0.5), stored with its +-1 ulp x neighbours;
  * every pair where a variant of quant_edges.MUTANTS differs from the spec, counted in full and stored up to
    quant_edges.WITNESS_CAP per (dtype, MAX, variant), spread evenly over the scan order;
and the set adds the special classes (quant_edges.special_pairs) and a seeded random sample.

Keys, per dtype prefix p in (bf16, fp16):
  p/x, p/m       uint16  the pairs' half bits (x, row maximum), deduplicated per MAX
  p/max          uint8   MAX of the pair
  p/kind         uint8   bit mask of quant_edges.K_* (tie, tie neighbour, witness, special, random)
  p/mut          uint16  bit mask over quant_edges.MUTANTS of the variants the pair is a stored witness of
  p/scan_count   int64 [15, len(MUTANTS)]  witnesses the scan found, per MAX and variant
  p/ties         int64 [15]                exact ties the scan found, per MAX
  mutants        the variant names, in bit order

Run from the repository root:  python tests/golden/make_quant_edges.py   (a few minutes on 8 cores)."""
import os
import sys
from multiprocessing import Pool

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import quant_edges as Q  # noqa: E402


def scan_one(args):
    dt, MAX = args
    tx, tm = [], []
    wx = {k: [] for k in Q.MUTANTS}
    wm = {k: [] for k in Q.MUTANTS}
    for blk in Q.blocks(Q.ladder(dt)):
        (a, b), wit = Q.scan_block(dt, MAX, blk)
        tx.append(a)
        tm.append(b)
        for k in Q.MUTANTS:
            wx[k].append(wit[k][0])
            wm[k].append(wit[k][1])
    tx, tm = np.concatenate(tx), np.concatenate(tm)
    counts, stored = [], {}
    for k in Q.MUTANTS:
        x, m = np.concatenate(wx[k]), np.concatenate(wm[k])
        counts.append(x.size)
        i = Q.cap_pick(x.size)
        stored[k] = (x[i], m[i])
    return dt, MAX, (tx, tm), stored, counts


def build_dtype(results, dt):
    xs, ms, mx, kind, mut = [], [], [], [], []
    scan = np.zeros((len(Q.MAXES), len(Q.MUTANTS)), np.int64)
    ties = np.zeros(len(Q.MAXES), np.int64)

    def add(x, m, MAX, k, mu=0):
        xs.append(np.asarray(x, np.uint16))
        ms.append(np.asarray(m, np.uint16))
        mx.append(np.full(len(x), MAX, np.uint8))
        kind.append(np.full(len(x), k, np.uint8))
        mut.append(np.full(len(x), mu, np.uint16))

    for d, MAX, (tx, tm), stored, counts in results:
        if d != dt:
            continue
        scan[MAX - 1] = counts
        ties[MAX - 1] = tx.size
        add(tx, tm, MAX, Q.K_TIE)
        nx, nm = Q.tie_neighbours(tx, tm)
        add(nx, nm, MAX, Q.K_TIE_NB)
        for bit, k in enumerate(Q.MUTANTS):
            add(stored[k][0], stored[k][1], MAX, Q.K_WITNESS, 1 << bit)
        sx, sm = Q.special_pairs(dt, MAX)
        add(sx, sm, MAX, Q.K_SPECIAL)
        rx, rm = Q.random_pairs(dt, MAX)
        add(rx, rm, MAX, Q.K_RANDOM)
    x, m, mx, kind, mut = (np.concatenate(a) for a in (xs, ms, mx, kind, mut))
    key = (mx.astype(np.uint64) << 32) | (m.astype(np.uint64) << 16) | x.astype(np.uint64)
    uk, inv = np.unique(key, return_inverse=True)
    k2 = np.zeros(uk.size, np.uint8)
    mu2 = np.zeros(uk.size, np.uint16)
    np.bitwise_or.at(k2, inv, kind)
    np.bitwise_or.at(mu2, inv, mut)
    p = Q.DT_NAME[dt]
    return {f"{p}/x": (uk & 0xFFFF).astype(np.uint16), f"{p}/m": ((uk >> 16) & 0xFFFF).astype(np.uint16),
            f"{p}/max": (uk >> 32).astype(np.uint8), f"{p}/kind": k2, f"{p}/mut": mu2, f"{p}/scan_count": scan,
            f"{p}/ties": ties}


def main():
    jobs = [(dt, M) for dt in Q.DTYPES for M in Q.MAXES]
    with Pool(min(8, os.cpu_count() or 1)) as pool:
        results = pool.map(scan_one, jobs, chunksize=1)
    out = {"mutants": np.array(Q.MUTANTS)}
    for dt in Q.DTYPES:
        out.update(build_dtype(results, dt))
    np.savez_compressed(Q.FIXTURE, **out)
    for dt in Q.DTYPES:
        p = Q.DT_NAME[dt]
        print(p, "pairs", out[f"{p}/x"].size, "ties per MAX", out[f"{p}/ties"].tolist())
        for i, k in enumerate(Q.MUTANTS):
            print(f"  {k:14s}", out[f"{p}/scan_count"][:, i].tolist())


if __name__ == "__main__":
    main()
