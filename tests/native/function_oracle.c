/* function_oracle.c -- test infrastructure: the row rule of the reference's FunctionOpIterator
 * (qip-iterators/src/iterators/qubit_iterators.rs:221-271), restated in plain C over a whole state so that
 * tests/test_function_cpu.py can pin the bit convention of qipb200_state_apply_function to it.
 *
 * The op acts on indices = in_qubits ++ out_qubits, indices[0] the most significant bit of its sub-row; qubit q is bit
 * n-1-q of a full index.  Sub-row (x, y) has exactly one non-zero column: x is kept, the function is called on the
 * bit-reversed x, its value is bit-reversed back into the y register and XORed there, and the entry is the complex
 * value the function returns with it (here e^{i theta}, or exactly one without theta).  Output row r of the state is
 * that entry times the input amplitude at the column.  Products and sums are taken one operation at a time in the
 * state's precision (built with -ffp-contract=off); without theta the amplitude is copied. */
#include <math.h>
#include <stdint.h>

static uint64_t flip_bits(uint64_t n, uint64_t v) {
  uint64_t r = 0;
  for (uint64_t i = 0; i < n; ++i) r |= ((v >> i) & 1u) << (n - 1 - i);
  return r;
}

/* The one column of full row `row`, and the argument of f and theta for that row. */
static uint64_t column_of(uint64_t n, const uint64_t *in_q, uint64_t n_in, const uint64_t *out_q, uint64_t n_out,
                          const uint64_t *f, uint64_t row, uint64_t *arg) {
  const uint64_t k = n_in + n_out;
  uint64_t sub = 0;
  for (uint64_t m = 0; m < k; ++m) {
    const uint64_t q = m < n_in ? in_q[m] : out_q[m - n_in];
    sub |= ((row >> (n - 1 - q)) & 1u) << (k - 1 - m);
  }
  const uint64_t x = sub >> n_out, y = sub & ((1ull << n_out) - 1);
  *arg = flip_bits(n_in, x);
  const uint64_t fx = f ? f[*arg] : 0;
  const uint64_t col_sub = (x << n_out) | (y ^ flip_bits(n_out, fx));
  uint64_t col = row;
  for (uint64_t m = 0; m < k; ++m) {
    const uint64_t q = m < n_in ? in_q[m] : out_q[m - n_in];
    const uint64_t b = n - 1 - q;
    col = (col & ~(1ull << b)) | (((col_sub >> (k - 1 - m)) & 1u) << b);
  }
  return col;
}

#define DEFINE_APPLY(NAME, R)                                                                                       \
  void NAME(uint64_t n, const uint64_t *in_q, uint64_t n_in, const uint64_t *out_q, uint64_t n_out,                 \
            const uint64_t *f, const double *theta, const R *psi, R *out) {                                          \
    for (uint64_t row = 0; row < (1ull << n); ++row) {                                                              \
      uint64_t arg = 0;                                                                                             \
      const uint64_t col = column_of(n, in_q, n_in, out_q, n_out, f, row, &arg);                                    \
      const R a = psi[2 * col], b = psi[2 * col + 1];                                                               \
      if (!theta) {                                                                                                 \
        out[2 * row] = a;                                                                                           \
        out[2 * row + 1] = b;                                                                                       \
        continue;                                                                                                   \
      }                                                                                                             \
      const R c = (R)cos(theta[arg]), s = (R)sin(theta[arg]);                                                       \
      const R ca = c * a, sb = s * b, cb = c * b, sa = s * a;                                                       \
      out[2 * row] = ca - sb;                                                                                       \
      out[2 * row + 1] = cb + sa;                                                                                   \
    }                                                                                                               \
  }

DEFINE_APPLY(fo_apply_function_f64, double)
DEFINE_APPLY(fo_apply_function_f32, float)
