// The oracle's constraint check: stwo's assert_constraints_on_polys restated over the bytecode AIR with the oracle's own parser
// (orc::Air::parse) and interpreter (orc::run_program), for the tests of nb200_check_constraints.  Every row of the component's trace domain
// CanonicCoset(log_size) is visited in trace (coset) order; a mask at offset `off` reads the trace row (r + off) mod 2^log_size, which sits at
// bit_reverse(coset_index_to_circle_domain_index(.)) of the committed (bit-reversed circle-domain) column.  A constraint fails on a row when
// its value is not zero.  Compiled by tests/oracle_check.py against oracle/prove.h (test infrastructure only).
#include "prove.h"

using namespace orc;

extern "C" int orc_check_constraints(const uint32_t* words, size_t n_words, uint32_t comp, const uint32_t* const* const cols[3], const size_t n_cols[3],
                                     const uint32_t* params, size_t n_params, uint64_t* n_failing, uint64_t* first_row, size_t n) {
  try {
    const Air air = Air::parse(words, n_words);
    const Component& c = air.comps.at(comp);
    if (n != c.n_constraints) return 2;
    const size_t rows = (size_t)1 << c.log_size;
    std::vector<const uint32_t*> mcol(c.masks.size());
    for (size_t m = 0; m < c.masks.size(); ++m) {
      if (c.masks[m].tree > 2 || c.masks[m].col >= n_cols[c.masks[m].tree]) return 2;
      mcol[m] = cols[c.masks[m].tree][c.masks[m].col];
    }
    std::vector<QM31> prm(n_params);
    for (size_t i = 0; i < n_params; ++i) prm[i] = QM31::from_u32(params[4 * i], params[4 * i + 1], params[4 * i + 2], params[4 * i + 3]);
    for (size_t k = 0; k < n; ++k) { n_failing[k] = 0; first_row[k] = UINT64_MAX; }
    std::vector<M31> mask(c.masks.size());
    std::vector<M31> br(c.n_base_regs); std::vector<QM31> er(c.n_ext_regs);
    for (size_t r = 0; r < rows; ++r) {
      for (size_t m = 0; m < c.masks.size(); ++m) {
        const size_t at = (size_t)(((int64_t)r + c.masks[m].off) & (int64_t)(rows - 1));   // rem_euclid by a power of two
        mask[m] = M31::raw(mcol[m][bit_reverse_index(coset_index_to_circle_domain_index(at, c.log_size), c.log_size)]);
      }
      size_t k = 0;
      run_program<M31>(c.prog, mask.data(), prm, br, er, [&](QM31 v) {
        if (v != QM31::zero()) { if (!n_failing[k]++) first_row[k] = r; }
        ++k;
      }, [](QM31, QM31) {});
    }
    return 0;
  } catch (std::exception&) {
    return 2;
  }
}
