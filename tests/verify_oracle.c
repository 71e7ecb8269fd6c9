/* The verifier's linear-time pieces restated for the C oracle -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Builds on oracle/oracle.c (included whole, unchanged) and adds the reference's loops run serially:
 *
 *   orc_r1cs_eval      multi_evaluate's evaluate_with_table (spartan/snark.rs:329-340) for one matrix:
 *                      sum over rows of sum over the row's entries of T_x[row] * T_y[col] * val
 *   orc_r1cs_eval_par  the same over rows split across threads (rayon's par_windows), one partial per thread
 *   orc_ipa_s          InnerProductArgument::verify's s (ipa_pc.rs:334-349) by the reference's recurrence,
 *                      s[0] = prod r^-1, s[i] = s[i - 2^pos] * r^2[L-1-pos], then times `scale` (NULL: 1)
 *
 * tests/verify_ref.py compiles it and wraps the entries.
 */
#include "../oracle/oracle.c"

typedef struct {
  const orc_field_t* F;
  const fe* D;
  const uint64_t* indices;
  const uint64_t* indptr;
  const fe* Tx;
  const fe* Ty;
  fe* partial;
} r1cs_ctx;

static void r1cs_rows(void* v, size_t lo, size_t hi, int tid) {
  r1cs_ctx* c = (r1cs_ctx*)v;
  fe acc;
  memset(&acc, 0, 32);
  for (size_t r = lo; r < hi; r++)
    for (uint64_t e = c->indptr[r]; e < c->indptr[r + 1]; e++) {
      fe t;
      fe_mul(c->F, &t, &c->Tx[r], &c->Ty[c->indices[e]]);
      fe_mul(c->F, &t, &t, &c->D[e]);
      fe_add(c->F, &acc, &acc, &t);
    }
  c->partial[tid] = acc;
}

EXPORT int orc_r1cs_eval_par(int fid, const void* data, const uint64_t* indices, const uint64_t* indptr, size_t rows,
                             const void* Tx, const void* Ty, void* out, int nthreads) {
  if (fid < 0 || fid > 3) return 1;
  if (nthreads < 1) nthreads = 1;
  fe* partial = (fe*)calloc((size_t)nthreads, sizeof(fe));
  if (!partial) return 6;
  r1cs_ctx c = {&ORC_FIELDS[fid], (const fe*)data, indices, indptr, (const fe*)Tx, (const fe*)Ty, partial};
  par_chunks(rows, nthreads, r1cs_rows, &c);
  fe acc;
  memset(&acc, 0, 32);
  for (int t = 0; t < nthreads; t++) fe_add(c.F, &acc, &acc, &partial[t]);
  free(partial);
  *(fe*)out = acc;
  return 0;
}

EXPORT int orc_r1cs_eval(int fid, const void* data, const uint64_t* indices, const uint64_t* indptr, size_t rows,
                         const void* Tx, const void* Ty, void* out) {
  return orc_r1cs_eval_par(fid, data, indices, indptr, rows, Tx, Ty, out, 1);
}

EXPORT int orc_ipa_s(int fid, const void* r_inv, const void* r_sq, int L, const void* scale_or_null, void* out) {
  if (fid < 0 || fid > 3 || L < 0 || L > 31) return 1;
  const orc_field_t* F = &ORC_FIELDS[fid];
  const fe* ri = (const fe*)r_inv;
  const fe* rs = (const fe*)r_sq;
  fe* s = (fe*)out;
  const size_t n = (size_t)1 << L;
  fe_one(F, &s[0]);
  for (int j = 0; j < L; j++) fe_mul(F, &s[0], &s[0], &ri[j]);
  for (size_t i = 1; i < n; i++) {
    int pos = 63 - __builtin_clzll((unsigned long long)i);
    fe_mul(F, &s[i], &s[i - ((size_t)1 << pos)], &rs[L - 1 - pos]);
  }
  if (scale_or_null)
    for (size_t i = 0; i < n; i++) fe_mul(F, &s[i], &s[i], (const fe*)scale_or_null);
  return 0;
}
