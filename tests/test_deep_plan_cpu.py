"""CPU-only: the host tables of the combined DEEP-quotient route (csrc/prove.cu deep_plan, nb200_deep_plan) against the plain restatement
of the quotient's coefficients in tests/opening_ref.py.

The route rests on one identity: per sample batch, accumulate_quotients' per-column coefficient alpha_k c equals alpha_k times the batch's
single c = conj(p.y) - p.y, so sum_k (alpha_k c) f_k = c G with G = sum_k alpha_k f_k.  The alphas must run over random_coeff^1, ^2, ...
in batch order, and A, B and random_coeff ^ count must be those accumulate_quotients sums."""
import numpy as np
import pytest

from nexus_zkvm_b200 import build as nb_build
from nexus_zkvm_b200 import field as F
from nexus_zkvm_b200 import prover as NP
from tests import opening_ref as R
from tests import random_witness as rw

P = (1 << 31) - 1


@pytest.fixture(scope="module", autouse=True)
def built():
    nb_build.build()


def _qm31(rng):
    return tuple(int(v) for v in rng.integers(0, P, 4))


def _batches(rng, counts):
    oods = R.oods_point(_qm31(rng))
    return [(R.point_words(R.shifted(oods, 10, k)), [(int(c), tuple(int(v) for v in rw.mixed(rng, 4))) for c in rng.permutation(40)[:cnt]])
            for k, cnt in enumerate(counts)]


@pytest.mark.parametrize("rc_kind", ["one", "minus_one", "random"])
@pytest.mark.parametrize("counts", [[1], [17], [40, 3, 4], list(range(1, 10))])
def test_plan_matches_the_restatement(counts, rc_kind):
    rng = np.random.default_rng(len(counts) * 100 + sum(counts))
    rc = {"one": (1, 0, 0, 0), "minus_one": (P - 1, 0, 0, 0)}.get(rc_kind) or _qm31(rng)
    batches = _batches(rng, counts)
    lines, alphas = NP.deep_plan(batches, rc)
    assert lines.shape == (len(batches), 24) and alphas.shape == (sum(counts), 4)
    e = 0
    for b, (point, entries) in enumerate(batches):
        px, py = tuple(point[:4]), tuple(point[4:])
        ln = [int(v) for v in lines[b]]
        assert ln[0:8] == [px[0], px[1], py[0], py[1], px[2], px[3], py[2], py[3]], f"batch {b}: point parts"
        c = F.qm31_sub(R.conj(py), py)
        assert tuple(ln[20:24]) == c, f"batch {b}: c"
        alpha, sa, sb = R.ONE, R.ZERO, R.ZERO
        for _col, value in entries:
            alpha = F.qm31_mul(alpha, rc)
            assert tuple(int(v) for v in alphas[e]) == alpha, f"batch {b} entry {e}: alpha"
            aa, ab, ac = R.line_coeffs(py, value, alpha)
            assert F.qm31_mul(alpha, c) == ac, f"batch {b} entry {e}: alpha c is the restatement's per-column coefficient"
            sa, sb = F.qm31_add(sa, aa), F.qm31_add(sb, ab)
            e += 1
        assert tuple(ln[8:12]) == sa and tuple(ln[12:16]) == sb, f"batch {b}: A / B"
        assert tuple(ln[16:20]) == alpha, f"batch {b}: random_coeff ^ count"


def test_plan_rejects_entries_out_of_order():
    rng = np.random.default_rng(3)
    sb, se, n_e = NP._sample_tables(_batches(rng, [2, 3]))
    sb[0].first_entry, sb[1].first_entry = 3, 0
    u32p = NP.C.POINTER(NP.C.c_uint32)
    lines, alphas = np.zeros((2, 24), np.uint32), np.zeros((n_e, 4), np.uint32)
    st = NP.lib().nb200_deep_plan(sb, NP.C.c_size_t(2), se, NP.C.c_size_t(n_e), NP._q(_qm31(rng)), lines.ctypes.data_as(u32p),
                                  alphas.ctypes.data_as(u32p))
    assert st != 0
