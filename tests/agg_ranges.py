"""The index walk of range_reduce (csrc/b2s_agg.cu) restated over numpy arrays of ranges, with no arithmetic on values (tests
only): which pieces of the range structure a row's range [lo, hi] reads, and the shape of its walk.

At each level L the walk either loops over elements [a, b] of one 32-wide block (or of the top level, L = n_levels), or reads
the suffix of a's block and the prefix of b's block and moves one level up to the whole blocks between them, (a >> 5) + 1 ..
(b >> 5) - 1, stopping there when there are none.  A walk's shapes are

    ("loop", L, length)             the final loop at level L over `length` elements (1 .. 32)
    ("split", L, a_on_start, b_on_end)   a suffix / prefix split at level L; whether the suffix starts on a block boundary
                                    (a % 32 == 0) and whether the prefix ends on one (b % 32 == 31)
    ("stop", L)                     the walk ends after its split at level L (no whole block between the two)

`possible(n)` lists every shape some range of n rows takes; `walk` reports the shapes a set of ranges takes and checks that
their pieces cover each range exactly once, in order."""

import numpy as np


def levels(n):
    """m[0] = n, m[L + 1] = ceil(m[L] / 32) while m[L] > 32; -> (n_levels, m)"""
    m = [n]
    while m[-1] > 32:
        m.append((m[-1] + 31) >> 5)
    return len(m) - 1, m


def _span(n, L, a, b):
    """first and last row under elements [a, b] of level L, and their count as leaves() computes it"""
    first = a << (5 * L)
    end = np.minimum((b + 1) << (5 * L), n)
    return first, end - 1, end - first


def walk(lo, hi, n):
    """ranges [lo, hi] (int64 arrays, 0 <= lo <= hi < n) -> (ok, shapes): ok[r] is True when the pieces range r reads are
    disjoint, in order and cover exactly lo .. hi, with leaves() counts that add up to hi - lo + 1; shapes is the set every
    range took"""
    n_levels, _m = levels(n)
    a, b = np.asarray(lo, np.int64).copy(), np.asarray(hi, np.int64).copy()
    left, right = a.copy(), b.copy()  # the next row the pieces from the left / right must start / end at
    counted = np.zeros(len(a), np.int64)
    ok = np.ones(len(a), bool)
    live = np.ones(len(a), bool)
    shapes = set()
    for L in range(n_levels + 1):
        if not live.any():
            break
        looping = live & ((L >= n_levels) | ((a >> 5) == (b >> 5)))
        if looping.any():
            first, last, cnt = _span(n, L, a[looping], b[looping])
            ok[looping] &= (first == left[looping]) & (last == right[looping])
            counted[looping] += cnt
            for length in np.unique(b[looping] - a[looping] + 1).tolist():
                shapes.add(("loop", L, length))
        split = live & ~looping
        if split.any():
            sa, sb = a[split], b[split]
            first, last, cnt = _span(n, L, sa, sa | 31)  # suffix of a's block
            ok[split] &= first == left[split]
            left[split] = last + 1
            counted[split] += cnt
            first, last, cnt = _span(n, L, sb & ~np.int64(31), sb)  # prefix of b's block
            ok[split] &= last == right[split]
            right[split] = first - 1
            counted[split] += cnt
            for code in np.unique(2 * (sa % 32 == 0) + (sb % 32 == 31)).tolist():
                shapes.add(("split", L, code >= 2, code % 2 == 1))
            a[split], b[split] = (sa >> 5) + 1, (sb >> 5) - 1
            stop = np.zeros(len(a), bool)
            stop[split] = a[split] > b[split]
            if stop.any():
                ok[stop] &= left[stop] == right[stop] + 1
                shapes.add(("stop", L))
            live = split & ~stop
        else:
            live = split
    assert not live.any()
    ok &= counted == np.asarray(hi, np.int64) - np.asarray(lo, np.int64) + 1
    return ok, shapes


def possible(n):
    """every shape some range [lo, hi] of n rows takes.  The walk reaches level 0 with any 0 <= a <= b < n and level L >= 1
    with any amin <= a <= b <= bmax, where amin = 1 and bmax = (bmax of level L - 1 >> 5) - 1: a pair there comes from the
    pair (32 (a - 1) + 31, 32 (b + 1)) one level down, which splits into it"""
    n_levels, _m = levels(n)
    out = set()
    amin, bmax = 0, n - 1
    for L in range(n_levels + 1):
        if amin > bmax:
            break
        if L == n_levels:
            out |= {("loop", L, k) for k in range(1, bmax - amin + 2)}
            break
        longest = max(min(32 * k + 31, bmax) - max(32 * k, amin) + 1 for k in {amin >> 5, (amin >> 5) + 1, bmax >> 5})
        out |= {("loop", L, k) for k in range(1, min(longest, 32) + 1)}
        a_on = -(-amin // 32) * 32        # the first suffix start on a block boundary
        a_off = amin if amin % 32 else amin + 1  # the first one off it
        for a_start, a in ((True, a_on), (False, a_off)):
            if 32 * ((a >> 5) + 1) <= bmax:
                out |= {("split", L, a_start, False), ("stop", L)}
            if 32 * ((a >> 5) + 1) + 31 <= bmax:
                out.add(("split", L, a_start, True))
        amin, bmax = 1, (bmax >> 5) - 1
    return out
