"""The Python restatement of the DEEP quotient (tests/opening_ref.py) against the oracle's accumulate_quotients, and its domain points
against the oracle's circle domain: the GPU tests of the opening phase use it as a second, independent referee."""
import numpy as np
import pytest

from oracle import pyoracle as orc
from tests import opening_ref as R
from tests import random_witness as rw

P = (1 << 31) - 1


@pytest.mark.parametrize("log_size", [1, 2, 3, 7, 12, 21])
def test_domain_points_match_the_oracle(log_size):
    rng = np.random.default_rng(log_size)
    n = 1 << log_size
    rows = sorted({0, n - 1, n // 2 - 1, n // 2} | {int(r) for r in rng.integers(0, n, 20)})
    for row in rows:
        want = orc.circle_domain_at(log_size, orc.bit_reverse_index(row, log_size))
        assert R.domain_point(log_size, row) == want, f"log {log_size} row {row}"


def test_oods_point_is_on_the_circle_and_shifts_by_a_domain_step():
    rng = np.random.default_rng(5)
    t = tuple(int(v) for v in rng.integers(0, P, 4))
    x, y = R.oods_point(t)
    assert R.F.qm31_add(R.F.qm31_mul(x, x), R.F.qm31_mul(y, y)) == R.ONE
    # 2^log steps of CanonicCoset(log) go once around its subgroup
    p = (x, y)
    for _ in range(1 << 3):
        p = R.shifted(p, 3, 1)
    assert p == (x, y)
    assert R.shifted(R.shifted((x, y), 10, 1), 10, -1) == (x, y)


def _rc(kind, rng):
    if kind == "one":
        return np.array([1, 0, 0, 0], np.uint32)
    if kind == "minus_one":
        return np.array([P - 1, 0, 0, 0], np.uint32)
    return rng.integers(0, P, 4, dtype=np.uint32)


def _case(log_size, counts, seed):
    """Columns from the edge mix (all P - 1, zero, an impulse at the last row, random_witness.mixed) and one sample batch per count, at
    an out-of-domain point and at shifts of it."""
    rng = np.random.default_rng(seed)
    n_cols = max(counts)
    n = 1 << log_size
    cols = np.empty((n_cols, n), np.uint32)
    for c in range(n_cols):
        kind = c % 4
        cols[c] = P - 1 if kind == 0 else 0
        if kind == 2:
            cols[c, n - 1] = rng.integers(1, P)
        elif kind == 3:
            cols[c] = rw.mixed(rng, n)
    base = R.oods_point(tuple(int(v) for v in rng.integers(0, P, 4)))
    batches = []
    for k, cnt in enumerate(counts):
        pt = R.point_words(R.shifted(base, max(log_size - 1, 1), k))
        batches.append((pt, [(int(c), rw.mixed(rng, 4)) for c in rng.permutation(n_cols)[:cnt]]))
    return rng, cols, batches


@pytest.mark.parametrize("rc_kind", ["one", "minus_one", "random"])
@pytest.mark.parametrize("log_size", [1, 2, 3, 6])
def test_deep_quotient_reference_matches_the_oracle_on_every_row(log_size, rc_kind):
    rng, cols, batches = _case(log_size, list(range(1, 10)), seed=10 * log_size + len(rc_kind))
    rc = _rc(rc_kind, rng)
    want = orc.accumulate_quotients(list(cols), rc, batches)
    got = R.deep_quotient_rows(lambda c, r: cols[c, r], log_size, batches, rc, range(1 << log_size))
    for row, v in got.items():
        assert v == tuple(int(x) for x in want[:, row]), f"row {row}"


def test_deep_quotient_reference_matches_the_oracle_at_2p12():
    """Every residue of the batch size mod 8, and rows on both sides of several 4-row groups."""
    log_size = 12
    rng, cols, batches = _case(log_size, [1, 2, 3, 8, 13, 14, 15, 20, 17], seed=12)
    rc = _rc("random", rng)
    want = orc.accumulate_quotients(list(cols), rc, batches)
    n = 1 << log_size
    rows = sorted({0, 1, 3, 4, 7, 8, n // 2 - 1, n // 2, n - 5, n - 4, n - 1} | {int(r) for r in rng.integers(0, n, 20)})
    got = R.deep_quotient_rows(lambda c, r: cols[c, r], log_size, batches, rc, rows)
    for row, v in got.items():
        assert v == tuple(int(x) for x in want[:, row]), f"row {row}"
