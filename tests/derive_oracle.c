/* ck_derive_by_address restated for the C oracle -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Builds on oracle/oracle.c (included whole, unchanged) and adds one entry, the reference's loop
 * (traits/commitment.rs:177-194, pedersen.rs:360-382, hyperkzg.rs:731-749) run serially:
 *
 *   bases = ck_to_group_elements(ck)              panics if any generator is the identity
 *   addresses.len() > ck.len()                    -> InvalidCommitmentKeyLength
 *   addresses[i] >= table_size                    -> InvalidIndex
 *   derived[addresses[i]] += bases[i]             one projective (XYZZ) mixed addition per address
 *   normalize                                     identity -> (0, 0)
 *
 * tests/derive_ref.py compiles it and wraps the entry.
 */
#include "../oracle/oracle.c"

/* returns 0, or 2 (an identity generator: the reference's panic), 3 (m > n), 4 (an address >= table_size, the
 * smallest such position in *first_bad); *first_bad is also the identity generator's index for 2.  5: bad curve id,
 * 6: out of memory. */
EXPORT int orc_ck_derive_by_address(int curve, const void* bases, size_t n, const uint64_t* addresses, size_t m,
                                    size_t table_size, void* out_affine, size_t* first_bad) {
  curve_t cv;
  if (get_curve(curve, &cv)) return 5;
  const orc_field_t* F = cv.base;
  const aff* b = (const aff*)bases;
  *first_bad = (size_t)-1;
  for (size_t i = 0; i < n; i++)
    if (aff_is_identity(&b[i])) { *first_bad = i; return 2; }
  if (m > n) return 3;
  for (size_t i = 0; i < m; i++)
    if (addresses[i] >= table_size) { *first_bad = i; return 4; }
  xyzz* acc = (xyzz*)malloc((table_size ? table_size : 1) * sizeof(xyzz));
  if (!acc) return 6;
  for (size_t j = 0; j < table_size; j++) xyzz_zero(F, &acc[j]);
  for (size_t i = 0; i < m; i++) xyzz_add_affine(F, &acc[addresses[i]], &b[i]);
  for (size_t j = 0; j < table_size; j++) xyzz_to_affine(F, &((aff*)out_affine)[j], &acc[j]);
  free(acc);
  return 0;
}
