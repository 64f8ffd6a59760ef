"""Plain restatements, in Python integers, of the formulas the opening phase of a proof evaluates: circle-domain points, out-of-domain
sample points, and the DEEP quotient of QuotientOps::accumulate_quotients (stwo core/pcs/quotients.rs: complex_conjugate_line_coeffs,
column_line_coeffs, batch_random_coeffs, denominator_inverses, accumulate_row_quotients).

Nothing here shares code with the oracle (oracle/) or with the host-side hoisting of csrc/prove.cu (accumulate_quotients sums each
batch's line terms into one A y + B before the kernel runs; here every column's linear term is evaluated at every row).  It is slow, so
the tests evaluate it on a few dozen rows; tests/test_opening_ref_cpu.py pins it against the oracle."""
from nexus_zkvm_b200 import field as F

P = F.P
CIRCLE_GEN = (2, 1268011823)      # generator of the M31 circle group, of order 2^31
ONE = (1, 0, 0, 0)
ZERO = (0, 0, 0, 0)


# ---- the M31 circle group ------------------------------------------------------------------------------------------------------

def point_add(a, b):
    return ((a[0] * b[0] - a[1] * b[1]) % P, (a[0] * b[1] + a[1] * b[0]) % P)


def point_at_index(idx):
    """idx * CIRCLE_GEN (indices are taken mod 2^31)."""
    idx %= 1 << 31
    r, g = (1, 0), CIRCLE_GEN
    while idx:
        if idx & 1:
            r = point_add(r, g)
        g = point_add(g, g)
        idx >>= 1
    return r


def subgroup_gen_index(log_size):
    return (1 << (31 - log_size)) % (1 << 31)


def bit_reverse(i, log_size):
    return int(format(i, f"0{log_size}b")[::-1], 2) if log_size else 0


def domain_point(log_size, row):
    """The point of CanonicCoset(log_size).circle_domain() at bit-reversed position `row` (the committed order): the domain is the half
    coset half_odds(log_size - 1) = subgroup_gen(log_size + 1) + k subgroup_gen(log_size - 1) followed by its conjugates."""
    i = bit_reverse(row, log_size)
    half = 1 << (log_size - 1)
    k = i if i < half else i - half
    x, y = point_at_index(subgroup_gen_index(log_size + 1) + k * subgroup_gen_index(log_size - 1))
    return (x, y) if i < half else (x, (-y) % P)


# ---- points over QM31 ----------------------------------------------------------------------------------------------------------

def conj(q):
    """The complex conjugate over CM31: a + b u -> a - b u."""
    return (q[0], q[1], (-q[2]) % P, (-q[3]) % P)


def embed(v):
    return (v % P, 0, 0, 0)


def oods_point(t):
    """The circle point of parameter t, as sample_oods draws it: ((1 - t^2) / (1 + t^2), 2 t / (1 + t^2))."""
    t2 = F.qm31_mul(t, t)
    inv = F.qm31_inv(F.qm31_add(t2, ONE))
    return F.qm31_mul(F.qm31_sub(ONE, t2), inv), F.qm31_mul(F.qm31_add(t, t), inv)


def shifted(point, trace_log, offset):
    """point + offset steps of CanonicCoset(trace_log): the point a mask at a row offset samples."""
    sx, sy = point_at_index(offset * subgroup_gen_index(trace_log))
    x, y = point
    return (F.qm31_sub(F.qm31_mul_m31(x, sx), F.qm31_mul_m31(y, sy)), F.qm31_add(F.qm31_mul_m31(x, sy), F.qm31_mul_m31(y, sx)))


def point_words(point):
    """(x, y) -> the 8 words [x0..x3, y0..y3] of a sample point."""
    return [int(v) for v in point[0]] + [int(v) for v in point[1]]


# ---- the DEEP quotient ---------------------------------------------------------------------------------------------------------

def _cm31_of(q, k):
    return (q[2 * k], q[2 * k + 1])


def _mul_cm31(q, c):
    lo, hi = F.cm31_mul(_cm31_of(q, 0), c), F.cm31_mul(_cm31_of(q, 1), c)
    return (lo[0], lo[1], hi[0], hi[1])


def line_coeffs(point_y, value, alpha):
    """complex_conjugate_line_coeffs: (alpha a, alpha b, alpha c) of the line through (p, v) and its conjugate."""
    a = F.qm31_sub(conj(value), value)
    c = F.qm31_sub(conj(point_y), point_y)
    b = F.qm31_sub(F.qm31_mul(value, c), F.qm31_mul(a, point_y))
    return F.qm31_mul(alpha, a), F.qm31_mul(alpha, b), F.qm31_mul(alpha, c)


def deep_quotient_rows(column_at, log_size, batches, random_coeff, rows):
    """The DEEP quotient at the given rows of CanonicCoset(log_size).circle_domain() (bit-reversed order).
    column_at(col, row) -> the column's word; batches: [(point8, [(col, value4), ...]), ...] as NP.fri_quotients takes them.
    Returns {row: (c0, c1, c2, c3)}."""
    rc = tuple(int(v) for v in random_coeff)
    prepared = []
    for point, entries in batches:
        w = [int(v) % P for v in point]
        px, py = tuple(w[:4]), tuple(w[4:])
        alpha, coeffs = ONE, []
        for col, value in entries:                          # column_line_coeffs: alpha runs over rc, rc^2, ... within the batch
            alpha = F.qm31_mul(alpha, rc)
            coeffs.append((int(col), line_coeffs(py, tuple(int(v) for v in value), alpha)))
        batch_coeff = ONE
        for _ in entries:                                   # batch_random_coeffs: rc^(number of columns)
            batch_coeff = F.qm31_mul(batch_coeff, rc)
        prepared.append((px, py, coeffs, batch_coeff))
    out = {}
    for row in rows:
        x, y = domain_point(log_size, row)
        acc = ZERO
        for px, py, coeffs, batch_coeff in prepared:
            numer = ZERO
            for col, (a, b, c) in coeffs:
                value = F.qm31_mul_m31(c, int(column_at(col, row)))
                linear = F.qm31_add(F.qm31_mul_m31(a, y), b)
                numer = F.qm31_add(numer, F.qm31_sub(value, linear))
            # (prx - x) piy - (pry - y) pix over CM31
            prx, pix, pry, piy = _cm31_of(px, 0), _cm31_of(px, 1), _cm31_of(py, 0), _cm31_of(py, 1)
            den = F.cm31_sub(F.cm31_mul(((prx[0] - x) % P, prx[1]), piy), F.cm31_mul(((pry[0] - y) % P, pry[1]), pix))
            acc = F.qm31_add(F.qm31_mul(acc, batch_coeff), _mul_cm31(numer, F.cm31_inv(den)))
        out[row] = acc
    return out
