"""A Python restatement of the doc tile kernels' index arithmetic (fwd_sm90.cuh / bwd_sm90.cuh with kDoc, and the
argument normalisation of ba_fwd_chunk_doc / ba_bwd_chunk_doc), for the CPU tests.

``check_launch`` states, for one launch, what the kernels rely on:
* the forward: each row's key limits are exactly the row's visible keys, and every visible key lies in its warpgroup's
  tile range and in the CTA's;
* the backward: every visible pair lies in the key block's Q-block range, and the staged document offsets with the
  band give exactly the visible pairs;
* deterministic mode: for every Q block i, "key block x visits i" is exactly x_min(i) <= x <= x_max(i) -- the
  precondition of the turn order (x - x_min(i)) n_red + wg, without which a deterministic launch would wait forever.
``mutant`` names a deliberate fault, so that the tests can show each check rejects it.
"""
from __future__ import annotations

import bisect

BM, BN = 128, 128  # forward: rows per CTA, keys per tile
BWD_M, BWD_N = 64, 128  # backward: rows per Q block, keys per CTA


def normalise(Sq, Sk, causal, causal_off, lower):
    """check_chunk_args for the doc entries (csrc/host_common.cu): (causal_off, lo) as the kernels get them."""
    off = max(-Sq, min(Sk, causal_off)) if causal else causal_off
    if lower is None or lower <= 1 - Sq:
        lo = 1 - Sq  # masks nothing: row + 1 - Sq <= 0 <= key
    else:
        lo = min(lower, Sk)
    return off, lo


def doc_of(cu, x, mutant=None):
    if mutant == "search_lower_bound":  # the first d with cu[d] >= x instead of the last with cu[d] <= x
        return min(bisect.bisect_left(cu, x, 0, len(cu) - 1), len(cu) - 2)
    return bisect.bisect_right(cu, x, 0, len(cu) - 1) - 1


def view_index(x, pos0, ps, n):
    return 0 if x <= pos0 else min(n, (x - pos0 + ps - 1) // ps)


def interval(x, cu, pos0, ps, n, mutant=None):
    d = doc_of(cu, x, mutant)
    return view_index(cu[d], pos0, ps, n), view_index(cu[d + 1], pos0, ps, n)


class Launch:
    def __init__(self, Sq, Sk, causal, causal_off, lower, cu, q_pos0, k_pos0, ps):
        self.Sq, self.Sk, self.causal, self.cu = Sq, Sk, causal, list(cu)
        self.off, self.lo = normalise(Sq, Sk, causal, causal_off, lower)
        self.q_pos0, self.k_pos0, self.ps = q_pos0, k_pos0, ps

    def qpos(self, a):
        return self.q_pos0 + self.ps * a

    def kpos(self, c):
        return self.k_pos0 + self.ps * c

    def visible(self, a, c):
        """The oracle: band and same document, by positions."""
        if self.causal and c > a + self.off:
            return False
        if c < a + self.lo:
            return False
        return doc_of(self.cu, self.qpos(a)) == doc_of(self.cu, self.kpos(c))

    # ---- forward
    def trip(self, r0):
        if r0 >= self.Sq:
            return 0
        r_last = min(r0 + 63, self.Sq - 1)
        m = min(r_last + self.off, self.Sk - 1) if self.causal else self.Sk - 1
        return 0 if m < 0 else m // BN + 1

    def group_range(self, r0, mutant=None):
        """fwd_doc_range: the tiles [first, end) of the 64 rows from r0, (0, 0) when empty."""
        if r0 >= self.Sq:
            return 0, 0
        r_last = min(r0 + 63, self.Sq - 1)
        k_lo, _ = interval(self.qpos(r0), self.cu, self.k_pos0, self.ps, self.Sk, mutant)
        _, k_hi = interval(self.qpos(r0 if mutant == "range_first_row_only" else r_last), self.cu, self.k_pos0,
                           self.ps, self.Sk, mutant)
        f = max(max(0, r0 + self.lo) // BN, k_lo // BN)
        e = min(self.trip(r0), (k_hi + BN - 1) // BN)
        return (f, e) if e > f else (0, 0)

    def cta_range(self, row0, mutant=None):
        f0, e0 = self.group_range(row0, mutant)
        f1, e1 = self.group_range(row0 + 64, mutant)
        t0 = (min(f0, f1) if e1 > f1 else f0) if e0 > f0 else f1
        return t0, max(0, max(e0, e1) - t0)

    def row_limits(self, a, mutant=None):
        k_lo, k_hi = interval(self.qpos(a), self.cu, self.k_pos0, self.ps, self.Sk, mutant)
        if mutant == "fwd_edge_plus1":
            k_hi += 1
        elif mutant == "fwd_edge_minus1":
            k_hi -= 1
        limit = min(a + self.off, self.Sk - 1) if self.causal else self.Sk - 1
        return max(a + self.lo, k_lo), min(limit, k_hi - 1)

    # ---- backward
    def q_blocks(self, x, mutant=None):
        """[i_begin, i_end) of key block x."""
        k0 = x * BWD_N
        nQ = (self.Sq + BWD_M - 1) // BWD_M
        i_begin = max(0, k0 - self.off) // BWD_M if self.causal else 0
        q_last = min(k0 + BWD_N - 1, self.Sk - 1) - self.lo
        i_end = 0 if q_last < 0 else min(nQ, q_last // BWD_M + 1)
        r_lo, _ = interval(self.kpos(k0), self.cu, self.q_pos0, self.ps, self.Sq, mutant)
        last = k0 if mutant == "i_end_first_key" else min(k0 + BWD_N - 1, self.Sk - 1)
        _, r_hi = interval(self.kpos(last), self.cu, self.q_pos0, self.ps, self.Sq, mutant)
        return max(i_begin, r_lo // BWD_M), min(i_end, (r_hi + BWD_M - 1) // BWD_M)

    def staged(self, a, x, mutant=None):
        """The loader's (lo, hi) of row a relative to key block x."""
        k0 = x * BWD_N
        lo, hi = interval(self.qpos(a), self.cu, self.k_pos0, self.ps, self.Sk, mutant)
        if mutant == "bwd_edge_plus1":
            hi += 1
        elif mutant == "bwd_edge_minus1":
            hi -= 1
        return min(max(lo - k0, 0), BWD_N), min(max(hi - k0, 0), BWD_N)

    def x_min(self, i, mutant=None):
        q0 = i * BWD_M
        x = max(0, q0 + self.lo) // BWD_N
        if mutant != "x_min_band_only":
            k_lo, _ = interval(self.qpos(q0), self.cu, self.k_pos0, self.ps, self.Sk, mutant)
            x = max(x, k_lo // BWD_N)
        return x


def check_launch(L, mutant=None):
    """Assert the three properties of the module docstring for launch L (AssertionError names the first failure)."""
    nX = (L.Sk + BWD_N - 1) // BWD_N
    nQ = (L.Sq + BWD_M - 1) // BWD_M
    # forward
    for row0 in range(0, L.Sq, BM):
        t0, n = L.cta_range(row0, mutant)
        for wg in range(2):
            f, e = L.group_range(row0 + 64 * wg, mutant)
            for a in range(row0 + 64 * wg, min(row0 + 64 * wg + 64, L.Sq)):
                lo, hi = L.row_limits(a, mutant)
                for c in range(L.Sk):
                    vis = L.visible(a, c)
                    assert (lo <= c <= hi) == vis, ("fwd mask", a, c, vis)
                    if vis:
                        assert f <= c // BN < e and t0 <= c // BN < t0 + n, ("fwd tiles", a, c, (f, e), (t0, n))
    # backward
    visits = [set() for _ in range(nQ)]
    for x in range(nX):
        ib, ie = L.q_blocks(x, mutant)
        for i in range(ib, ie):
            visits[i].add(x)
        for c in range(x * BWD_N, min(x * BWD_N + BWD_N, L.Sk)):
            for a in range(L.Sq):
                vis = L.visible(a, c)
                if vis:
                    assert ib <= a // BWD_M < ie, ("bwd blocks", a, c, (ib, ie))
                if ib <= a // BWD_M < ie:
                    lo, hi = L.staged(a, x, mutant)
                    band = (not L.causal or c <= a + L.off) and c >= a + L.lo
                    assert (band and lo <= c - x * BWD_N < hi) == vis, ("bwd mask", a, c, vis)
    # deterministic turn order
    for i in range(nQ):
        if visits[i]:
            xs = sorted(visits[i])
            assert xs == list(range(L.x_min(i, mutant), xs[-1] + 1)), ("turns", i, xs, L.x_min(i, mutant))


def sweep():
    """Launches over document edges at tile phases 127/0/1 (128-row CTAs, 64-row blocks, 128-key tiles), several
    documents in one tile, documents spanning many tiles, zero-length documents, striped pstride 2-8, windows and
    causal offsets, and launches whose positions start inside a document."""
    out = []
    S = 520
    edges = [[0, 127, 128, 129, 255, 256, 257, 383, 384, 385, S], [0, 63, 64, 65, 191, 192, 193, S],
             [0, 5, 9, 9, 30, 31, 40, 41, 300, S], [0, S], [0, 0, 1, 200, 200, 519, S]]
    for cu in edges:
        for causal, off, lower in ((False, 0, None), (True, 0, None), (True, 0, -70), (False, 40, -40), (True, -3, -200)):
            out.append((S, S, causal, off, lower, cu, 0, 0, 1))
    # a launch inside a longer sequence: rows and keys from other positions, striped strides
    T = 4096
    cu = [0, 17, 300, 301, 1000, 1001, 1002, 2050, 2051, 3000, T]
    for ps in (1, 2, 3, 8):
        for q_pos0, k_pos0 in ((0, 0), (5, 0), (0, 7), (ps * 100, 1)):
            n = min(300, (T - 1 - max(q_pos0, k_pos0)) // ps + 1)
            out.append((n, n, True, (q_pos0 - k_pos0) // ps, None, cu, q_pos0, k_pos0, ps))
            out.append((n, n - 40, False, 0, None, cu, q_pos0, k_pos0, ps))
    return out


MUTANTS = ("fwd_edge_plus1", "bwd_edge_plus1", "fwd_edge_minus1", "bwd_edge_minus1", "range_first_row_only", "i_end_first_key", "search_lower_bound",
           "x_min_band_only")
