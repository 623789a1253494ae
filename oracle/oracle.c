/*
 * ORACLE (test infrastructure, NOT product code; only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs may load this library).
 *
 * CPU restatement, in plain C, of the reference algorithms on Boojum's polynomial-commitment
 * hot path.  Every function cites the reference lines (relative to the era-boojum repository root) it follows.
 * Parallelisation mirrors the reference's rayon chunking (one serial NTT per column spread over
 * threads; row-chunked hashing) via OpenMP so it can double as the "restated reference" CPU baseline.
 *
 * Parity status: Poseidon2 / sponge / Merkle layout / transcript / DEEP / FRI fold are pinned by the
 * reference's own golden fixture proof.json (tests/test_oracle_golden.py, fixture extracted by
 * tools/make_golden.py).  The NTT has no numeric golden vector in the reference tree (all its NTT
 * tests draw from thread_rng); it is pinned by definition: equality with the O(n^2) DFT in bit-reversed
 * order with and without coset 7, exactly the identity the reference's tests assert
 * (src/fft/mod.rs:1344-1384, 1591-1634), plus the FRI final-monomial check in proof.json which
 * exercises iNTT indirectly.
 */
#include "gl64.h"
#include "poseidon_rc.h"
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------------------------------
 * scalar helpers exported for tests
 * ---------------------------------------------------------------------------------------------- */
API uint64_t orc_add(uint64_t a, uint64_t b) { return gl_add(gl_canon(a), gl_canon(b)); }
API uint64_t orc_sub(uint64_t a, uint64_t b) { return gl_sub(gl_canon(a), gl_canon(b)); }
API uint64_t orc_mul(uint64_t a, uint64_t b) { return gl_mul(gl_canon(a), gl_canon(b)); }
API uint64_t orc_mul_slow(uint64_t a, uint64_t b) { return gl_mul_slow(gl_canon(a), gl_canon(b)); }
API uint64_t orc_inv(uint64_t a) { return gl_inv(gl_canon(a)); }
API uint64_t orc_pow(uint64_t a, uint64_t e) { return gl_pow(gl_canon(a), e); }
API uint64_t orc_omega(unsigned log_n) { return gl_omega(log_n); }
API void orc_ext_mul(const uint64_t a[2], const uint64_t b[2], uint64_t out[2]) {
  gl2_t r = gl2_mul((gl2_t){gl_canon(a[0]), gl_canon(a[1])}, (gl2_t){gl_canon(b[0]), gl_canon(b[1])});
  out[0] = r.c0;
  out[1] = r.c1;
}
API void orc_ext_inv(const uint64_t a[2], uint64_t out[2]) {
  gl2_t r = gl2_inv((gl2_t){gl_canon(a[0]), gl_canon(a[1])});
  out[0] = r.c0;
  out[1] = r.c1;
}
API int orc_num_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}
API void orc_set_threads(int n) {
#ifdef _OPENMP
  if (n > 0) omp_set_num_threads(n);
#else
  (void)n;
#endif
}

/* ------------------------------------------------------------------------------------------------
 * NTT family
 * ---------------------------------------------------------------------------------------------- */

/* bitreverse_enumeration_inplace                         src/fft/mod.rs:41-155 (semantics only) */
API void orc_bitreverse(uint64_t *a, unsigned log_n) {
  size_t n = (size_t)1 << log_n;
  for (size_t i = 0; i < n; i++) {
    size_t j = gl_bitrev(i, log_n);
    if (i < j) {
      uint64_t t = a[i];
      a[i] = a[j];
      a[j] = t;
    }
  }
}

/* precompute_twiddles_for_fft: tab[i] = w^bitrev_{n/2}(i), i < n/2, w = omega_n or its inverse.
 *                                                         src/cs/implementations/utils.rs:88-125
 * (the reference's O(n) primitivity assert loop :107-110 is optional here: with_assert) */
API void orc_twiddles(uint64_t *tab, unsigned log_n, int inverse, int with_assert) {
  size_t n = (size_t)1 << log_n;
  uint64_t w = gl_omega(log_n);
  if (inverse) w = gl_inv(w);
  if (with_assert) {
    volatile uint64_t sink = 0;
    for (size_t i = 1; i < n; i++) sink ^= gl_pow(w, i); /* assert_ne!(omega^i, 1) */
    (void)sink;
  }
  size_t half = n / 2;
  if (half == 0) return;
  uint64_t cur = 1;
  for (size_t i = 0; i < half; i++) {
    tab[i] = cur;
    cur = gl_mul(cur, w);
  }
  if (log_n >= 2) orc_bitreverse(tab, log_n - 1);
}

/* serial_ct_ntt_natural_to_bitreversed                    src/fft/mod.rs:659-734 */
static void ntt_network(uint64_t *a, unsigned log_n, const uint64_t *tab) {
  size_t n = (size_t)1 << log_n;
  if (n == 1) return;
  size_t pairs = n / 2, groups = 1, dist = n / 2;
  while (groups < n) {
    for (size_t k = 0; k < groups; k++) {
      size_t i1 = k * pairs * 2, i2 = i1 + pairs;
      uint64_t s = tab[k];
      for (size_t j = i1; j < i2; j++) {
        uint64_t u = a[j], v = gl_mul(a[j + dist], s);
        a[j + dist] = gl_sub(u, v);
        a[j] = gl_add(u, v);
      }
    }
    pairs /= 2;
    groups *= 2;
    dist /= 2;
  }
}

/* distribute_powers: a[i] *= c^i                           src/fft/mod.rs:308-317 */
static void distribute_powers(uint64_t *a, size_t n, uint64_t c) {
  uint64_t s = 1;
  for (size_t i = 0; i < n; i++) {
    a[i] = gl_mul(a[i], s);
    s = gl_mul(s, c);
  }
}

static void canon_vec(uint64_t *a, size_t n) {
  for (size_t i = 0; i < n; i++) a[i] = gl_canon(a[i]);
}

/* fft_natural_to_bitreversed                               src/fft/mod.rs:398-411 */
API void orc_ntt_n2b_tab(uint64_t *a, unsigned log_n, uint64_t coset, const uint64_t *tab) {
  size_t n = (size_t)1 << log_n;
  canon_vec(a, n);
  coset = gl_canon(coset);
  if (coset != 1) distribute_powers(a, n, coset);
  ntt_network(a, log_n, tab);
}

/* ifft_natural_to_natural                                  src/fft/mod.rs:464-491 */
API void orc_intt_n2n_tab(uint64_t *a, unsigned log_n, uint64_t coset, const uint64_t *inv_tab) {
  size_t n = (size_t)1 << log_n;
  canon_vec(a, n);
  coset = gl_canon(coset);
  ntt_network(a, log_n, inv_tab);
  orc_bitreverse(a, log_n);
  if (coset != 1) distribute_powers(a, n, gl_inv(coset));
  if (n > 1) {
    uint64_t ninv = gl_inv((uint64_t)n % GL_P);
    for (size_t i = 0; i < n; i++) a[i] = gl_mul(a[i], ninv);
  }
}

/* batched drivers: n_cols columns of n elements, column c at a + c*stride.
 * One serial NTT per column, columns spread across threads (src/cs/implementations/utils.rs:295-304) */
API void orc_ntt_n2b(uint64_t *a, unsigned log_n, size_t n_cols, size_t stride, uint64_t coset) {
  size_t n = (size_t)1 << log_n;
  uint64_t *tab = (uint64_t *)malloc(sizeof(uint64_t) * (n / 2 + 1));
  orc_twiddles(tab, log_n, 0, 0);
#pragma omp parallel for schedule(static)
  for (long c = 0; c < (long)n_cols; c++) orc_ntt_n2b_tab(a + (size_t)c * stride, log_n, coset, tab);
  free(tab);
}
API void orc_intt_n2n(uint64_t *a, unsigned log_n, size_t n_cols, size_t stride, uint64_t coset) {
  size_t n = (size_t)1 << log_n;
  uint64_t *tab = (uint64_t *)malloc(sizeof(uint64_t) * (n / 2 + 1));
  orc_twiddles(tab, log_n, 1, 0);
#pragma omp parallel for schedule(static)
  for (long c = 0; c < (long)n_cols; c++) orc_intt_n2n_tab(a + (size_t)c * stride, log_n, coset, tab);
  free(tab);
}

/* transform_raw_storages_to_lde + transform_monomials_to_lde
 *                                                          src/cs/implementations/utils.rs:270-403
 * in : n_cols columns of n Lagrange values (natural order), column c at in + c*n
 * out: [col][coset j][n] with coset shift 7 * omega_{nL}^{bitrev_L(j)}, values bit-reversed in the coset.
 * from_monomials != 0 skips the iNTT (transform_monomials_to_lde). */
API void orc_lde(const uint64_t *in, uint64_t *out, unsigned log_n, unsigned log_lde, size_t n_cols,
                 int from_monomials) {
  size_t n = (size_t)1 << log_n, L = (size_t)1 << log_lde;
  uint64_t *ftab = (uint64_t *)malloc(sizeof(uint64_t) * (n / 2 + 1));
  uint64_t *itab = (uint64_t *)malloc(sizeof(uint64_t) * (n / 2 + 1));
  orc_twiddles(ftab, log_n, 0, 0);
  orc_twiddles(itab, log_n, 1, 0);
  uint64_t w_big = gl_omega(log_n + log_lde);
  uint64_t *mono = (uint64_t *)malloc(sizeof(uint64_t) * n * n_cols);
  memcpy(mono, in, sizeof(uint64_t) * n * n_cols);
#pragma omp parallel for schedule(static)
  for (long c = 0; c < (long)n_cols; c++) {
    if (!from_monomials) orc_intt_n2n_tab(mono + (size_t)c * n, log_n, 1, itab);
    else canon_vec(mono + (size_t)c * n, n);
  }
#pragma omp parallel for schedule(static)
  for (long job = 0; job < (long)(n_cols * L); job++) {
    size_t j = (size_t)job / n_cols, c = (size_t)job % n_cols; /* coset-major jobs, utils.rs:363-379 */
    uint64_t shift = gl_mul(GL_MULT_GEN, gl_pow(w_big, gl_bitrev(j, log_lde)));
    uint64_t *dst = out + (c * L + j) * n;
    memcpy(dst, mono + c * n, sizeof(uint64_t) * n);
    orc_ntt_n2b_tab(dst, log_n, shift, ftab);
  }
  free(mono);
  free(ftab);
  free(itab);
}

/* O(n^2) definition: out[bitrev(k)] = sum_i a_i (c w^k)^i  (what the reference tests compare against,
 * src/fft/mod.rs:1344-1384) */
API void orc_naive_dft_bitreversed(const uint64_t *a, uint64_t *out, unsigned log_n, uint64_t coset) {
  size_t n = (size_t)1 << log_n;
  uint64_t w = gl_omega(log_n);
  coset = gl_canon(coset);
  for (size_t k = 0; k < n; k++) {
    uint64_t x = gl_mul(coset, gl_pow(w, k)), acc = 0;
    for (size_t i = n; i-- > 0;) acc = gl_add(gl_mul(acc, x), gl_canon(a[i]));
    out[gl_bitrev(k, log_n)] = acc;
  }
}

/* ------------------------------------------------------------------------------------------------
 * Poseidon2 (t = 12, x^7, 4 + 22 + 4 rounds) and the overwrite-mode sponge
 * ---------------------------------------------------------------------------------------------- */

/* M4 block of the external matrix                         src/implementations/suggested_mds.rs:19-56 */
static inline void p2_block(uint64_t *x) {
  uint64_t t0 = gl_add(x[0], x[1]);
  uint64_t t1 = gl_add(x[2], x[3]);
  uint64_t t2 = gl_add(gl_dbl(x[1]), t1);
  uint64_t t3 = gl_add(gl_dbl(x[3]), t0);
  uint64_t t4 = gl_add(gl_dbl(gl_dbl(t1)), t3);
  uint64_t t5 = gl_add(gl_dbl(gl_dbl(t0)), t2);
  x[0] = gl_add(t3, t5);
  x[1] = t5;
  x[2] = gl_add(t2, t4);
  x[3] = t4;
}
/* M_E = circ(2 M4, M4, M4)                                 src/implementations/suggested_mds.rs:59-97 */
static inline void p2_external(uint64_t *s) {
  p2_block(s);
  p2_block(s + 4);
  p2_block(s + 8);
  for (int i = 0; i < 4; i++) {
    uint64_t sum = gl_add(gl_add(s[i], s[4 + i]), s[8 + i]);
    s[i] = gl_add(s[i], sum);
    s[4 + i] = gl_add(s[4 + i], sum);
    s[8 + i] = gl_add(s[8 + i], sum);
  }
}
static inline uint64_t p2_pow7(uint64_t x) {
  uint64_t x2 = gl_sqr(x), x3 = gl_mul(x2, x), x4 = gl_sqr(x2);
  return gl_mul(x4, x3);
}
/* internal matrix diag(2^s_i) + J                          state_generic_impl.rs:69-82, 171-200 */
static const unsigned P2_DIAG_SHIFT[12] = {4, 14, 11, 8, 0, 5, 2, 9, 13, 6, 3, 12};
static inline void p2_internal(uint64_t *s) {
  uint64_t sum = 0;
  for (int i = 0; i < 12; i++) sum = gl_add(sum, s[i]);
  for (int i = 0; i < 12; i++) s[i] = gl_add(gl_mul(s[i], (uint64_t)1 << P2_DIAG_SHIFT[i]), sum);
}
/* poseidon2_permutation: one global round counter 0..29    state_generic_impl.rs:158-233 */
API void orc_poseidon2_permutation(uint64_t *s) {
  for (int i = 0; i < 12; i++) s[i] = gl_canon(s[i]);
  p2_external(s);
  int r = 0;
  for (int k = 0; k < 4; k++, r++) {
    for (int i = 0; i < 12; i++) s[i] = p2_pow7(gl_add(s[i], ORACLE_POSEIDON_RC[r * 12 + i]));
    p2_external(s);
  }
  for (int k = 0; k < 22; k++, r++) {
    s[0] = p2_pow7(gl_add(s[0], ORACLE_POSEIDON_RC[r * 12]));
    p2_internal(s);
  }
  for (int k = 0; k < 4; k++, r++) {
    for (int i = 0; i < 12; i++) s[i] = p2_pow7(gl_add(s[i], ORACLE_POSEIDON_RC[r * 12 + i]));
    p2_external(s);
  }
}

/* GoldilocksPoseidon2Sponge<AbsorptionModeOverwrite>::hash_into_leaf
 *   src/cs/oracle/mod.rs:141-151, src/algebraic_props/sponge.rs:224-239 (absorb), :300-323 (finalize) */
API void orc_poseidon2_hash_leaf(const uint64_t *els, size_t n, uint64_t out[4]) {
  uint64_t st[12] = {0};
  size_t i = 0;
  for (; i + 8 <= n; i += 8) {
    for (int k = 0; k < 8; k++) st[k] = gl_canon(els[i + k]);
    orc_poseidon2_permutation(st);
  }
  if (i < n) {
    size_t f = n - i;
    for (size_t k = 0; k < f; k++) st[k] = gl_canon(els[i + k]);
    for (size_t k = f; k < 8; k++) st[k] = 0;
    orc_poseidon2_permutation(st);
  }
  memcpy(out, st, 4 * sizeof(uint64_t));
}
/* hash_into_node(l, r) = sponge over l || r = one permutation   src/cs/oracle/mod.rs:162-168 */
API void orc_poseidon2_hash_node(const uint64_t l[4], const uint64_t r[4], uint64_t out[4]) {
  uint64_t st[12] = {0};
  for (int k = 0; k < 4; k++) {
    st[k] = gl_canon(l[k]);
    st[4 + k] = gl_canon(r[k]);
  }
  orc_poseidon2_permutation(st);
  memcpy(out, st, 4 * sizeof(uint64_t));
}

/* Leaf hashing for MerkleTreeWithCap::construct (elems_per_leaf == 1, merkle_tree.rs:78-172) and
 * construct_by_chunking / _from_flat_sources (elems_per_leaf == 2^k, :176-386):
 * leaf m = concat over sources s (in order) of source_s[m*k .. (m+1)*k).
 * sources: n_src pointers to flat arrays of n_leaves*k u64 (a column's cosets flattened coset-major). */
API void orc_merkle_leaf_hashes(const uint64_t *const *sources, size_t n_src, size_t n_leaves,
                                size_t elems_per_leaf, uint64_t *leaf_hashes) {
#pragma omp parallel
  {
    uint64_t *buf = (uint64_t *)malloc(sizeof(uint64_t) * n_src * elems_per_leaf);
#pragma omp for schedule(static)
    for (long m = 0; m < (long)n_leaves; m++) {
      size_t w = 0;
      for (size_t s = 0; s < n_src; s++)
        for (size_t e = 0; e < elems_per_leaf; e++) buf[w++] = sources[s][(size_t)m * elems_per_leaf + e];
      orc_poseidon2_hash_leaf(buf, w, leaf_hashes + 4 * (size_t)m);
    }
    free(buf);
  }
}

/* continue_from_leaf_hashes: level by level until cap_size nodes remain  merkle_tree.rs:388-449
 * nodes: concatenated levels (n_leaves/2, n_leaves/4, ..., cap_size digests); returns #digests written.
 * The cap is the last level (or the leaf hashes themselves if n_leaves == cap_size). */
API size_t orc_merkle_nodes(const uint64_t *leaf_hashes, size_t n_leaves, size_t cap_size, uint64_t *nodes) {
  const uint64_t *prev = leaf_hashes;
  size_t cnt = n_leaves, written = 0;
  while (cnt > cap_size) {
    size_t next = cnt / 2;
    uint64_t *dst = nodes + 4 * written;
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)next; i++)
      orc_poseidon2_hash_node(prev + 8 * (size_t)i, prev + 8 * (size_t)i + 4, dst + 4 * (size_t)i);
    prev = dst;
    written += next;
    cnt = next;
  }
  return written;
}

/* verify_proof_over_cap                                     merkle_tree.rs:482-504 */
API int orc_merkle_verify(const uint64_t leaf_hash[4], const uint64_t *path, size_t path_len,
                          const uint64_t *cap, size_t cap_size, size_t idx) {
  uint64_t cur[4];
  memcpy(cur, leaf_hash, sizeof cur);
  for (size_t d = 0; d < path_len; d++) {
    const uint64_t *sib = path + 4 * d;
    uint64_t nxt[4];
    if (idx & 1) orc_poseidon2_hash_node(sib, cur, nxt);
    else orc_poseidon2_hash_node(cur, sib, nxt);
    memcpy(cur, nxt, sizeof cur);
    idx >>= 1;
  }
  if (idx >= cap_size) return 0;
  for (int k = 0; k < 4; k++)
    if (gl_canon(cap[4 * idx + k]) != cur[k]) return 0;
  return 1;
}

/* ------------------------------------------------------------------------------------------------
 * FRI fold                                                   src/cs/implementations/fri/mod.rs:362-474
 * out[i] = (f[2i] + f[2i+1]) + alpha * (f[2i] - f[2i+1]) * roots[i] * coset_inv   (Fp2, no 1/2)
 * roots = inverse twiddle table of the FULL LDE domain (prefix reused every level, :509, :612)
 * ---------------------------------------------------------------------------------------------- */
API void orc_fri_fold(const uint64_t *c0, const uint64_t *c1, size_t m, const uint64_t alpha[2],
                      const uint64_t *roots, uint64_t coset_inv, uint64_t *o0, uint64_t *o1) {
  gl2_t al = {gl_canon(alpha[0]), gl_canon(alpha[1])};
  coset_inv = gl_canon(coset_inv);
#pragma omp parallel for schedule(static)
  for (long i = 0; i < (long)(m / 2); i++) {
    uint64_t a0 = gl_canon(c0[2 * i]), b0 = gl_canon(c0[2 * i + 1]);
    uint64_t a1 = gl_canon(c1[2 * i]), b1 = gl_canon(c1[2 * i + 1]);
    uint64_t r = gl_mul(gl_canon(roots[i]), coset_inv);
    gl2_t diff = {gl_mul(gl_sub(a0, b0), r), gl_mul(gl_sub(a1, b1), r)};
    gl2_t t = gl2_mul(diff, al);
    o0[i] = gl_add(gl_add(t.c0, a0), b0);
    o1[i] = gl_add(gl_add(t.c1, a1), b1);
  }
}

/* ------------------------------------------------------------------------------------------------
 * batch inverse (Montgomery trick)                           src/cs/implementations/utils.rs:405-600
 * zeros are not expected by the reference (it would panic on inverse of 0); here 0 -> 0 is NOT
 * special-cased either: callers must pass non-zero values.
 * ---------------------------------------------------------------------------------------------- */
API void orc_batch_inverse(uint64_t *a, size_t n) {
  if (n == 0) return;
  uint64_t *pre = (uint64_t *)malloc(sizeof(uint64_t) * n);
  uint64_t acc = 1;
  for (size_t i = 0; i < n; i++) {
    pre[i] = acc;
    acc = gl_mul(acc, gl_canon(a[i]));
  }
  uint64_t inv = gl_inv(acc);
  for (size_t i = n; i-- > 0;) {
    uint64_t ai = gl_canon(a[i]);
    a[i] = gl_mul(inv, pre[i]);
    inv = gl_mul(inv, ai);
  }
  free(pre);
}
API void orc_batch_inverse_ext(uint64_t *c0, uint64_t *c1, size_t n) {
  if (n == 0) return;
  gl2_t *pre = (gl2_t *)malloc(sizeof(gl2_t) * n);
  gl2_t acc = {1, 0};
  for (size_t i = 0; i < n; i++) {
    pre[i] = acc;
    acc = gl2_mul(acc, (gl2_t){gl_canon(c0[i]), gl_canon(c1[i])});
  }
  gl2_t inv = gl2_inv(acc);
  for (size_t i = n; i-- > 0;) {
    gl2_t ai = {gl_canon(c0[i]), gl_canon(c1[i])};
    gl2_t r = gl2_mul(inv, pre[i]);
    c0[i] = r.c0;
    c1[i] = r.c1;
    inv = gl2_mul(inv, ai);
  }
  free(pre);
}

/* ------------------------------------------------------------------------------------------------
 * DEEP quotening on one (coset,row):                         src/cs/implementations/prover.rs:2523-2706,
 * verifier-side statement src/cs/implementations/verifier.rs:2526-2565.
 * acc += (1/(x - at)) * sum_i ch_i * (f_i(x) - v_i), f_i in Fp2 given as (c0,c1).
 * ---------------------------------------------------------------------------------------------- */
API void orc_deep_point(uint64_t acc[2], const uint64_t *f_c0, const uint64_t *f_c1, const uint64_t *v_c0,
                        const uint64_t *v_c1, const uint64_t *ch_c0, const uint64_t *ch_c1, size_t n,
                        uint64_t x, const uint64_t at[2]) {
  gl2_t den = gl2_sub((gl2_t){gl_canon(x), 0}, (gl2_t){gl_canon(at[0]), gl_canon(at[1])});
  den = gl2_inv(den);
  gl2_t s = {0, 0};
  for (size_t i = 0; i < n; i++) {
    gl2_t d = gl2_sub((gl2_t){gl_canon(f_c0[i]), gl_canon(f_c1[i])}, (gl2_t){gl_canon(v_c0[i]), gl_canon(v_c1[i])});
    s = gl2_add(s, gl2_mul((gl2_t){gl_canon(ch_c0[i]), gl_canon(ch_c1[i])}, d));
  }
  s = gl2_mul(s, den);
  gl2_t r = gl2_add((gl2_t){gl_canon(acc[0]), gl_canon(acc[1])}, s);
  acc[0] = r.c0;
  acc[1] = r.c1;
}

/* DEEP accumulation over the whole LDE domain for one opening point (prover-side driver of the sum above):
 * quotening_operation_in_extension                              src/cs/implementations/prover.rs:2523-2706
 * for t in 0..2^log_rows: x = 7 * w_{nL}^{bitrev(t)};  acc[t] += sum_i ch_i (f_i[t] - v_i) / (x - at)
 * src_c1[i] == NULL marks a base-field polynomial. */
API void orc_deep_group(uint64_t *acc0, uint64_t *acc1, const uint64_t *const *src_c0, const uint64_t *const *src_c1,
                        size_t n_src, const uint64_t *values_at, const uint64_t *challenges, const uint64_t at[2],
                        unsigned log_rows) {
  size_t rows = (size_t)1 << log_rows;
  uint64_t w = gl_omega(log_rows);
  gl2_t a = {gl_canon(at[0]), gl_canon(at[1])};
#pragma omp parallel for schedule(static)
  for (long t = 0; t < (long)rows; t++) {
    uint64_t x = gl_mul(GL_MULT_GEN, gl_pow(w, gl_bitrev((size_t)t, log_rows)));
    gl2_t den = gl2_inv(gl2_sub((gl2_t){x, 0}, a));
    gl2_t s = {0, 0};
    for (size_t i = 0; i < n_src; i++) {
      gl2_t f = {gl_canon(src_c0[i][t]), src_c1[i] ? gl_canon(src_c1[i][t]) : 0};
      gl2_t v = {gl_canon(values_at[2 * i]), gl_canon(values_at[2 * i + 1])};
      gl2_t c = {gl_canon(challenges[2 * i]), gl_canon(challenges[2 * i + 1])};
      s = gl2_add(s, gl2_mul(c, gl2_sub(f, v)));
    }
    s = gl2_mul(s, den);
    acc0[t] = gl_add(gl_canon(acc0[t]), s.c0);
    acc1[t] = gl_add(gl_canon(acc1[t]), s.c1);
  }
}

/* ------------------------------------------------------------------------------------------------
 * Copy-permutation argument (stage 2 and its quotient terms)
 * Fp2 values are (c0, c1) column pairs; k_j are the non-residues of make_non_residues
 * (src/cs/implementations/utils.rs:636-688), passed in by the caller.
 * ---------------------------------------------------------------------------------------------- */
static inline gl2_t gl2_of(const uint64_t *c0, const uint64_t *c1, size_t i) {
  return (gl2_t){gl_canon(c0[i]), gl_canon(c1[i])};
}
static inline gl2_t gl2_canon2(const uint64_t v[2]) { return (gl2_t){gl_canon(v[0]), gl_canon(v[1])}; }

/* w + beta * s + gamma for base-field w and s */
static inline gl2_t cp_factor(uint64_t w, uint64_t s, gl2_t beta, gl2_t gamma) {
  return gl2_add(gl2_add(gl2_mul_base(beta, gl_canon(s)), (gl2_t){gl_canon(w), 0}), gamma);
}

/* R_c(x_i) = prod_{j in chunk c} (w_j + beta k_j x_i + gamma) / (w_j + beta sigma_j + gamma),  x_i = omega_n^i
 *                                                      pointwise_rational_in_extension, copy_permutation.rs:114-248 */
static gl2_t cp_ratio(const uint64_t *const *vars, const uint64_t *const *sigmas, const uint64_t *ks, size_t c0, size_t c1,
                      size_t i, uint64_t x, gl2_t beta, gl2_t gamma) {
  gl2_t num = {1, 0}, den = {1, 0};
  for (size_t j = c0; j < c1; j++) {
    num = gl2_mul(num, cp_factor(vars[j][i], gl_mul(gl_canon(ks[j]), x), beta, gamma));
    den = gl2_mul(den, cp_factor(vars[j][i], sigmas[j][i], beta, gamma));
  }
  return gl2_mul(num, gl2_inv(den));
}

/* compute_partial_products_in_extension                 src/cs/implementations/copy_permutation.rs:649-766
 * z[i] = prod_{t < i} prod_c R_c[t] (shifted_grand_product_in_extension, :425-510), p_c = z * R_0 * ... * R_c for every
 * chunk but the last.  Chunks are `chunk` consecutive columns.  partials: [n_chunks - 1][2][n] (may be NULL for one chunk).
 * grand[2] receives prod over all rows of prod_c R_c (one for a satisfied copy permutation). */
API void orc_cp_stage2(const uint64_t *const *vars, const uint64_t *const *sigmas, size_t n_cols, const uint64_t *ks,
                       const uint64_t beta_in[2], const uint64_t gamma_in[2], unsigned log_n, size_t chunk, uint64_t *z0,
                       uint64_t *z1, uint64_t *partials, uint64_t grand[2]) {
  size_t n = (size_t)1 << log_n, n_chunks = (n_cols + chunk - 1) / chunk;
  gl2_t beta = gl2_canon2(beta_in), gamma = gl2_canon2(gamma_in);
  uint64_t w = gl_omega(log_n);
  /* almost_z[i] = prod_c R_c[i], into z */
#pragma omp parallel for schedule(static)
  for (long i = 0; i < (long)n; i++) {
    uint64_t x = gl_pow(w, (uint64_t)i);
    gl2_t az = {1, 0};
    for (size_t c = 0; c < n_chunks; c++) {
      size_t e = (c + 1) * chunk < n_cols ? (c + 1) * chunk : n_cols;
      az = gl2_mul(az, cp_ratio(vars, sigmas, ks, c * chunk, e, (size_t)i, x, beta, gamma));
    }
    z0[i] = az.c0;
    z1[i] = az.c1;
  }
  /* exclusive prefix product, serially */
  gl2_t run = {1, 0};
  for (size_t i = 0; i < n; i++) {
    gl2_t a = {z0[i], z1[i]};
    z0[i] = run.c0;
    z1[i] = run.c1;
    run = gl2_mul(run, a);
  }
  grand[0] = run.c0;
  grand[1] = run.c1;
  if (n_chunks < 2) return;
#pragma omp parallel for schedule(static)
  for (long i = 0; i < (long)n; i++) {
    uint64_t x = gl_pow(w, (uint64_t)i);
    gl2_t p = {z0[i], z1[i]};
    for (size_t c = 0; c + 1 < n_chunks; c++) {
      p = gl2_mul(p, cp_ratio(vars, sigmas, ks, c * chunk, (c + 1) * chunk, (size_t)i, x, beta, gamma));
      partials[(2 * c) * n + (size_t)i] = p.c0;
      partials[(2 * c + 1) * n + (size_t)i] = p.c1;
    }
  }
}

/* x(t) = 7 * omega_{2^bits}^{bitrev_bits(t)}: the point of flat LDE index t (coset-major, bit-reversed inside a coset) */
static inline uint64_t lde_point(size_t t, unsigned bits) { return gl_mul(GL_MULT_GEN, gl_pow(gl_omega(bits), gl_bitrev(t, bits))); }

/* Quotient terms of the copy permutation at the flat LDE indices t < 2^(log_n + log_q), ADDED to q:
 *   alpha_0 (z - 1) (x^n - 1) / (x - 1)                                 prover.rs:1189-1227 (z(1) = 1)
 *   alpha_{c+1} (lhs_c prod_j (w_j + beta sigma_j + gamma) - rhs_c prod_j (w_j + beta k_j x + gamma))
 *     lhs = p_0, ..., p_{m-2}, z(omega x);  rhs = z, p_0, ..., p_{m-2}    copy_permutation.rs:1000-1249
 *   z(omega x) at bitrev(bitrev(i) + 1) of the same coset                utils.rs:1245-1271
 * var_ldes, sigma_ldes, z, partials (c0, c1 of each, 2 * (n_chunks - 1) pointers): flat LDEs of factor 2^log_lde. */
API void orc_cp_quotient(const uint64_t *const *var_ldes, const uint64_t *const *sigma_ldes, size_t n_cols, const uint64_t *ks,
                         const uint64_t *z0, const uint64_t *z1, const uint64_t *const *partials, const uint64_t beta_in[2],
                         const uint64_t gamma_in[2], const uint64_t *alphas, unsigned log_n, unsigned log_lde, unsigned log_q,
                         size_t chunk, uint64_t *q0, uint64_t *q1) {
  size_t n = (size_t)1 << log_n, n_chunks = (n_cols + chunk - 1) / chunk;
  size_t n_points = n << log_q;
  gl2_t beta = gl2_canon2(beta_in), gamma = gl2_canon2(gamma_in);
#pragma omp parallel for schedule(static)
  for (long tl = 0; tl < (long)n_points; tl++) {
    size_t t = (size_t)tl, coset = t >> log_n, i = t & (n - 1);
    uint64_t x = lde_point(t, log_n + log_lde);
    size_t tsh = (coset << log_n) | gl_bitrev((gl_bitrev(i, log_n) + 1) & (n - 1), log_n);
    gl2_t z = gl2_of(z0, z1, t);
    uint64_t l1 = gl_mul(gl_sub(gl_pow(x, n), 1), gl_inv(gl_sub(x, 1)));
    gl2_t q = gl2_mul(gl2_mul_base(gl2_sub(z, (gl2_t){1, 0}), l1), gl2_canon2(alphas));
    for (size_t c = 0; c < n_chunks; c++) {
      gl2_t lhs = c + 1 < n_chunks ? gl2_of(partials[2 * c], partials[2 * c + 1], t) : gl2_of(z0, z1, tsh);
      gl2_t rhs = c == 0 ? z : gl2_of(partials[2 * (c - 1)], partials[2 * (c - 1) + 1], t);
      size_t e = (c + 1) * chunk < n_cols ? (c + 1) * chunk : n_cols;
      for (size_t j = c * chunk; j < e; j++) {
        lhs = gl2_mul(lhs, cp_factor(var_ldes[j][t], sigma_ldes[j][t], beta, gamma));
        rhs = gl2_mul(rhs, cp_factor(var_ldes[j][t], gl_mul(gl_canon(ks[j]), x), beta, gamma));
      }
      q = gl2_add(q, gl2_mul(gl2_sub(lhs, rhs), gl2_canon2(alphas + 2 * (c + 1))));
    }
    q0[t] = gl_add(gl_canon(q0[t]), q.c0);
    q1[t] = gl_add(gl_canon(q1[t]), q.c1);
  }
}

/* divide_by_vanishing_for_bitreversed_coset_enumeration      utils.rs:770-817
 * q[t] /= x^n - 1 on the first 2^log_q cosets of the size-n*2^log_q domain (one constant per coset) */
API void orc_divide_by_vanishing(uint64_t *q0, uint64_t *q1, unsigned log_n, unsigned log_q) {
  size_t n = (size_t)1 << log_n, Q = (size_t)1 << log_q;
  for (size_t j = 0; j < Q; j++) {
    uint64_t shift = gl_mul(GL_MULT_GEN, gl_pow(gl_omega(log_n + log_q), gl_bitrev(j, log_q)));
    uint64_t m = gl_inv(gl_sub(gl_pow(shift, n), 1));
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)n; i++) {
      size_t t = j * n + (size_t)i;
      q0[t] = gl_mul(gl_canon(q0[t]), m);
      q1[t] = gl_mul(gl_canon(q1[t]), m);
    }
  }
}

/* ------------------------------------------------------------------------------------------------
 * Log-derivative lookup argument over specialised columns       src/cs/implementations/lookup_argument_in_ext.rs
 * A sub-argument's tuple is `width` lookup columns, then the table id column if there is one; the table has
 * n_table_cols = width (+ 1) columns.  agg(cols) = beta + sum_j gamma^j cols[j].
 * ---------------------------------------------------------------------------------------------- */
static gl2_t lookup_agg(const uint64_t *const *cols, size_t n, const uint64_t *extra, size_t r, gl2_t beta, gl2_t gamma) {
  gl2_t acc = beta, g = {1, 0};
  for (size_t j = 0; j < n; j++) {
    acc = gl2_add(acc, gl2_mul_base(g, gl_canon(cols[j][r])));
    g = gl2_mul(g, gamma);
  }
  if (extra) acc = gl2_add(acc, gl2_mul_base(g, gl_canon(extra[r])));
  return acc;
}

/* compute_lookup_poly_pairs_specialized                   :320-947
 * out [n_sub + 1][2][n]: A_i = 1 / agg(tuple_i), then B = m / agg(table) */
API void orc_lookup_polys(const uint64_t *const *lookup_cols, size_t n_sub, size_t width, const uint64_t *table_id,
                          const uint64_t *const *table_cols, size_t n_table_cols, const uint64_t *mult, const uint64_t beta_in[2],
                          const uint64_t gamma_in[2], size_t n, uint64_t *out) {
  gl2_t beta = gl2_canon2(beta_in), gamma = gl2_canon2(gamma_in);
#pragma omp parallel for schedule(static)
  for (long rl = 0; rl < (long)n; rl++) {
    size_t r = (size_t)rl;
    for (size_t i = 0; i < n_sub; i++) {
      gl2_t a = gl2_inv(lookup_agg(lookup_cols + i * width, width, table_id, r, beta, gamma));
      out[(2 * i) * n + r] = a.c0;
      out[(2 * i + 1) * n + r] = a.c1;
    }
    gl2_t b = gl2_mul_base(gl2_inv(lookup_agg(table_cols, n_table_cols, NULL, r, beta, gamma)), gl_canon(mult[r]));
    out[(2 * n_sub) * n + r] = b.c0;
    out[(2 * n_sub + 1) * n + r] = b.c1;
  }
}

/* compute_quotient_terms_for_lookup_specialized           :949-1319, ADDED to q at points t < n_points:
 *   alpha_i (A_i agg(tuple_i) - 1) for each sub-argument, alpha_{n_sub} (B agg(table) - m)
 * a_ldes: 2 * n_sub pointers (c0, c1 of each A_i) */
API void orc_lookup_quotient(const uint64_t *const *lookup_ldes, size_t n_sub, size_t width, const uint64_t *table_id,
                             const uint64_t *const *table_ldes, size_t n_table_cols, const uint64_t *mult,
                             const uint64_t *const *a_ldes, const uint64_t *b0, const uint64_t *b1, const uint64_t beta_in[2],
                             const uint64_t gamma_in[2], const uint64_t *alphas, size_t n_points, uint64_t *q0, uint64_t *q1) {
  gl2_t beta = gl2_canon2(beta_in), gamma = gl2_canon2(gamma_in);
#pragma omp parallel for schedule(static)
  for (long tl = 0; tl < (long)n_points; tl++) {
    size_t t = (size_t)tl;
    gl2_t q = {0, 0};
    for (size_t i = 0; i < n_sub; i++) {
      gl2_t d = lookup_agg(lookup_ldes + i * width, width, table_id, t, beta, gamma);
      gl2_t v = gl2_sub(gl2_mul(d, gl2_of(a_ldes[2 * i], a_ldes[2 * i + 1], t)), (gl2_t){1, 0});
      q = gl2_add(q, gl2_mul(v, gl2_canon2(alphas + 2 * i)));
    }
    gl2_t d = lookup_agg(table_ldes, n_table_cols, NULL, t, beta, gamma);
    gl2_t v = gl2_sub(gl2_mul(d, gl2_of(b0, b1, t)), (gl2_t){gl_canon(mult[t]), 0});
    q = gl2_add(q, gl2_mul(v, gl2_canon2(alphas + 2 * n_sub)));
    q0[t] = gl_add(gl_canon(q0[t]), q.c0);
    q1[t] = gl_add(gl_canon(q1[t]), q.c1);
  }
}

/* ------------------------------------------------------------------------------------------------
 * f(at) by Horner for base-field coefficient columns (low degree first) at an Fp2 point: with orc_intt_n2n, the
 * definition that barycentric_evaluate_*_at_extension (utils.rs:907-1243) computes in another way.
 * out: [n_cols][2]
 * ---------------------------------------------------------------------------------------------- */
API void orc_horner_ext(const uint64_t *mono, size_t n_cols, size_t n, const uint64_t at_in[2], uint64_t *out) {
  gl2_t at = gl2_canon2(at_in);
#pragma omp parallel for schedule(static)
  for (long c = 0; c < (long)n_cols; c++) {
    const uint64_t *m = mono + (size_t)c * n;
    gl2_t acc = {0, 0};
    for (size_t i = n; i-- > 0;) acc = gl2_add(gl2_mul(acc, at), (gl2_t){gl_canon(m[i]), 0});
    out[2 * c] = acc.c0;
    out[2 * c + 1] = acc.c1;
  }
}

/* ------------------------------------------------------------------------------------------------
 * Gate programs: the recorded SSA programs (bj_gate_desc, include/boojum_b200.h) interpreted directly, one relation at a
 * time, with canonical values - no peephole, no slot allocation, no step encoding - so these restate what
 * bj_quotient_gates_general_purpose and the gate half of bj_check_satisfied compute independently of the compiler they run.
 *   RowwiseEvaluator (repetitions, PerChunkOffset)     src/cs/traits/evaluator.rs:376-397
 *   push_evaluation_result / proceed_to_next_gate      src/cs/implementations/buffering_source.rs:158-221, 304-362
 *   compute_selector_subpath                           src/cs/implementations/prover.rs:2775-2916
 *   check_if_satisfied (gates)                         src/cs/implementations/satisfiability_test.rs:15-353
 * Flat arguments:
 *   gates  [n_gates][ORC_GD_WORDS]: the descriptor fields below (path_bits: bit i = path[i]);
 *   rels   [*][6]: op, dst temporary, a.kind, a.value, b.kind, b.value (BJ_REL_*, BJ_IDX_*), indexed from ORC_GD_REL_BEGIN;
 *   writes [*][2]: kind, value, indexed from ORC_GD_WRITE_BEGIN;
 *   cols: [variables | witnesses | constants], lazy u64 values.  The selector reads constant columns 0 .. path_len - 1.
 * Inverse of 0 is 0.
 * ---------------------------------------------------------------------------------------------- */
enum {
  ORC_GD_REL_BEGIN, ORC_GD_N_REL, ORC_GD_WRITE_BEGIN, ORC_GD_N_WRITES, ORC_GD_REPS, ORC_GD_VAR_OFF, ORC_GD_WIT_OFF,
  ORC_GD_CONST_OFF, ORC_GD_CONST_PLACE, ORC_GD_PATH_LEN, ORC_GD_PATH_BITS, ORC_GD_VAR_INIT, ORC_GD_WIT_INIT, ORC_GD_WORDS
};

typedef struct {
  const uint64_t *gates, *rels, *writes;
  size_t n_gates;
  const uint64_t *const *cols;
  uint64_t n_vars, n_wits;
  size_t n_tmp, max_writes; /* temporaries any program names, terms per repetition at most */
} orc_gate_set;

static orc_gate_set gate_set(const uint64_t *gates, size_t n_gates, const uint64_t *rels, const uint64_t *writes,
                             const uint64_t *const *cols, uint32_t n_vars, uint32_t n_wits) {
  orc_gate_set s = {gates, rels, writes, n_gates, cols, n_vars, n_wits, 1, 1};
  for (size_t g = 0; g < n_gates; g++) {
    const uint64_t *d = gates + g * ORC_GD_WORDS;
    for (uint64_t i = 0; i < d[ORC_GD_N_REL]; i++)
      if (rels[6 * (d[ORC_GD_REL_BEGIN] + i) + 1] + 1 > s.n_tmp) s.n_tmp = rels[6 * (d[ORC_GD_REL_BEGIN] + i) + 1] + 1;
    if (d[ORC_GD_N_WRITES] > s.max_writes) s.max_writes = d[ORC_GD_N_WRITES];
  }
  return s;
}

static uint64_t gate_operand(const orc_gate_set *s, const uint64_t *d, uint64_t kind, uint64_t v, uint64_t rep, size_t t,
                             const uint64_t *tmp) {
  const uint64_t consts = s->n_vars + s->n_wits;
  switch (kind) {
    case 0: return gl_canon(s->cols[d[ORC_GD_VAR_INIT] + v + rep * d[ORC_GD_VAR_OFF]][t]);
    case 1: return gl_canon(s->cols[s->n_vars + d[ORC_GD_WIT_INIT] + v + rep * d[ORC_GD_WIT_OFF]][t]);
    case 2: return gl_canon(s->cols[consts + d[ORC_GD_CONST_PLACE] + v + rep * d[ORC_GD_CONST_OFF]][t]);
    case 3: return tmp[v];
    case 4: return gl_canon(v);
    default: return gl_canon(s->cols[consts + d[ORC_GD_CONST_PLACE] + v][t]); /* row-shared constant: read at repetition 0 */
  }
}

/* the terms of repetition `rep` of gate d at point t, in write order */
static void gate_terms(const orc_gate_set *s, const uint64_t *d, uint64_t rep, size_t t, uint64_t *tmp, uint64_t *terms) {
  for (uint64_t i = 0; i < d[ORC_GD_N_REL]; i++) {
    const uint64_t *r = s->rels + 6 * (d[ORC_GD_REL_BEGIN] + i);
    const uint64_t a = gate_operand(s, d, r[2], r[3], rep, t, tmp);
    const int binary = r[0] == 0 || r[0] == 2 || r[0] == 4;
    const uint64_t b = binary ? gate_operand(s, d, r[4], r[5], rep, t, tmp) : 0;
    uint64_t v;
    switch (r[0]) {
      case 0: v = gl_add(a, b); break;
      case 1: v = gl_dbl(a); break;
      case 2: v = gl_sub(a, b); break;
      case 3: v = gl_neg(a); break;
      case 4: v = gl_mul(a, b); break;
      case 5: v = gl_sqr(a); break;
      default: v = gl_inv(a); break; /* 0 -> 0 */
    }
    tmp[r[1]] = v;
  }
  for (uint64_t k = 0; k < d[ORC_GD_N_WRITES]; k++) {
    const uint64_t *w = s->writes + 2 * (d[ORC_GD_WRITE_BEGIN] + k);
    terms[k] = gate_operand(s, d, w[0], w[1], rep, t, tmp);
  }
}

static uint64_t gate_selector(const orc_gate_set *s, const uint64_t *d, size_t t) {
  uint64_t sel = 1;
  for (uint64_t i = 0; i < d[ORC_GD_PATH_LEN]; i++) {
    const uint64_t c = gl_canon(s->cols[s->n_vars + s->n_wits + i][t]);
    sel = gl_mul(sel, ((d[ORC_GD_PATH_BITS] >> i) & 1) ? c : gl_sub(1, c));
  }
  return sel;
}

/* q[t] += sum_g sel_g(t) * sum_k alpha[k] * term_k(t), k running on across gates and repetitions; alphas (c0, c1) per term */
API void orc_gates_quotient(const uint64_t *gates, size_t n_gates, const uint64_t *rels, const uint64_t *writes,
                            const uint64_t *const *cols, uint32_t n_vars, uint32_t n_wits, const uint64_t *alphas,
                            size_t n_points, uint64_t *q0, uint64_t *q1) {
  const orc_gate_set s = gate_set(gates, n_gates, rels, writes, cols, n_vars, n_wits);
#pragma omp parallel
  {
    uint64_t *tmp = calloc(s.n_tmp, sizeof(uint64_t)), *terms = calloc(s.max_writes, sizeof(uint64_t));
#pragma omp for schedule(static)
    for (long tl = 0; tl < (long)n_points; tl++) {
      const size_t t = (size_t)tl;
      uint64_t r0 = gl_canon(q0[t]), r1 = gl_canon(q1[t]);
      size_t k = 0;
      for (size_t g = 0; g < n_gates; g++) {
        const uint64_t *d = gates + g * ORC_GD_WORDS;
        uint64_t a0 = 0, a1 = 0;
        for (uint64_t rep = 0; rep < d[ORC_GD_REPS]; rep++) {
          gate_terms(&s, d, rep, t, tmp, terms);
          for (uint64_t j = 0; j < d[ORC_GD_N_WRITES]; j++, k++) {
            a0 = gl_add(a0, gl_mul(terms[j], gl_canon(alphas[2 * k])));
            a1 = gl_add(a1, gl_mul(terms[j], gl_canon(alphas[2 * k + 1])));
          }
        }
        const uint64_t sel = gate_selector(&s, d, t);
        r0 = gl_add(r0, gl_mul(sel, a0));
        r1 = gl_add(r1, gl_mul(sel, a1));
      }
      q0[t] = r0;
      q1[t] = r1;
    }
    free(tmp);
    free(terms);
  }
}

/* Check mode over n_rows rows: every term of every repetition of a gate must be 0 where the gate's selector is nonzero.
 * out[0] = failing (row, gate, repetition) instances, out[1] = the first failing row, out[2] = its first failing global term
 * index (term base of the gate + rep * n_writes + term) in (gate, repetition, term) order; first_value / first_selector [n_rows]
 * = that term's value and its gate's selector on every failing row, 0 on the others.  out[1], out[2] are 0 without failures. */
API void orc_gates_check(const uint64_t *gates, size_t n_gates, const uint64_t *rels, const uint64_t *writes,
                         const uint64_t *const *cols, uint32_t n_vars, size_t n_rows, uint64_t *first_value,
                         uint64_t *first_selector, uint64_t out[3]) {
  const orc_gate_set s = gate_set(gates, n_gates, rels, writes, cols, n_vars, 0);
  uint64_t failures = 0, first_key = UINT64_MAX;
#pragma omp parallel reduction(+ : failures) reduction(min : first_key)
  {
    uint64_t *tmp = calloc(s.n_tmp, sizeof(uint64_t)), *terms = calloc(s.max_writes, sizeof(uint64_t));
#pragma omp for schedule(static)
    for (long tl = 0; tl < (long)n_rows; tl++) {
      const size_t t = (size_t)tl;
      uint64_t term_base = 0, row_term = UINT64_MAX;
      first_value[t] = first_selector[t] = 0;
      for (size_t g = 0; g < n_gates; g++) {
        const uint64_t *d = gates + g * ORC_GD_WORDS;
        const uint64_t sel = gate_selector(&s, d, t);
        for (uint64_t rep = 0; sel && rep < d[ORC_GD_REPS]; rep++) {
          gate_terms(&s, d, rep, t, tmp, terms);
          for (uint64_t j = 0; j < d[ORC_GD_N_WRITES]; j++) {
            if (!terms[j]) continue;
            failures++;
            if (row_term == UINT64_MAX) {
              row_term = term_base + rep * d[ORC_GD_N_WRITES] + j;
              first_value[t] = terms[j];
              first_selector[t] = sel;
            }
            break;
          }
        }
        term_base += d[ORC_GD_REPS] * d[ORC_GD_N_WRITES];
      }
      if (row_term != UINT64_MAX && (((uint64_t)t << 32) | row_term) < first_key) first_key = ((uint64_t)t << 32) | row_term;
    }
    free(tmp);
    free(terms);
  }
  out[0] = failures;
  out[1] = failures ? first_key >> 32 : 0;
  out[2] = failures ? first_key & 0xffffffffu : 0;
}

/* ------------------------------------------------------------------------------------------------
 * setup / witness materialisation (oracle/setup_oracle.py is the line-by-line Python restatement these are pinned to)
 * ---------------------------------------------------------------------------------------------- */
#define ORC_PLACEHOLDER_BIT (1ull << 63) /* Variable::placeholder       src/cs/mod.rs:44 */
#define ORC_LOW_U48 ((1ull << 48) - 1)   /* LOW_U48_MASK                src/cs/mod.rs:47 */

/* materialize_variables_polynomials_from_dense_hint        src/cs/implementations/witness.rs:325-385
 * out [n_cols][2^log_n]: out[c][row] = all_values[hint[c][row]] mod p for row < hint_rows, 0 for placeholders and the rows
 * past the hint.  The index is the Variable's low 48 bits (the reference indexes with the whole word, which is the same for
 * every Variable it creates).  Returns the number of non-placeholder cells whose index is >= n_values (those stay 0). */
API uint64_t orc_materialize_columns(const uint64_t *values, size_t n_values, const uint64_t *hint, size_t n_cols, size_t hint_rows,
                                     unsigned log_n, uint64_t *out) {
  const size_t n = (size_t)1 << log_n;
  uint64_t bad = 0;
#pragma omp parallel for schedule(static) reduction(+ : bad)
  for (long cl = 0; cl < (long)n_cols; cl++) {
    const size_t c = (size_t)cl;
    for (size_t row = 0; row < n; row++) {
      uint64_t v = 0;
      if (row < hint_rows) {
        const uint64_t h = hint[c * hint_rows + row];
        if (!(h & ORC_PLACEHOLDER_BIT)) {
          if ((h & ORC_LOW_U48) < n_values) v = gl_canon(values[h & ORC_LOW_U48]);
          else bad++;
        }
      }
      out[c * n + row] = v;
    }
  }
  return bad;
}

/* the per-variable scratch of create_permutation_polys, a HashMap<Variable, (F, (usize, usize))> in the reference: open
 * addressing with linear probing, keyed by the variable index (an empty slot holds ~0, which no 48-bit index equals).  One
 * entry holds all a visit touches, so a visit costs one cache miss, and the walk prefetches the entries of the cells ahead. */
typedef struct {
  uint64_t key, value, first; /* variable index, the value it carries, the flat cell of its first occurrence */
} orc_scratch_entry;

typedef struct {
  orc_scratch_entry *e;
  size_t cap, count;
} orc_scratch;

static inline size_t scratch_home(const orc_scratch *s, uint64_t key) {
  return (size_t)((key * 0x9E3779B97F4A7C15ull) >> 20) & (s->cap - 1);
}

static size_t scratch_slot(const orc_scratch *s, uint64_t key) {
  size_t i = scratch_home(s, key);
  while (s->e[i].key != ~0ull && s->e[i].key != key) i = (i + 1) & (s->cap - 1);
  return i;
}

static int scratch_alloc(orc_scratch *s, size_t cap) {
  s->cap = cap;
  s->count = 0;
  s->e = malloc(sizeof(orc_scratch_entry) * cap);
  if (!s->e) return -1;
#pragma omp parallel for schedule(static)
  for (long i = 0; i < (long)cap; i++) s->e[i].key = ~0ull;
  return 0;
}

/* doubles the table once it is three quarters full */
static int scratch_grow(orc_scratch *s) {
  orc_scratch t;
  if (scratch_alloc(&t, s->cap * 2)) return -1;
  for (size_t i = 0; i < s->cap; i++)
    if (s->e[i].key != ~0ull) t.e[scratch_slot(&t, s->e[i].key)] = s->e[i];
  t.count = s->count;
  free(s->e);
  *s = t;
  return 0;
}

/* create_permutation_polys                                 src/cs/implementations/setup.rs:419-502
 * placement [n_cols][2^log_n] Variables (copy_permutation_data), non_residues [n_cols] (non_residues_for_copy_permutation),
 * out [n_cols][2^log_n] the sigma columns.  out starts as the identity k_c * w^row (materialize_x_by_non_residue_polys);
 * the cells are visited column by column, row by row, and each occurrence of a variable swaps its value with the variable's
 * scratch value (:446-473); at the end every variable's scratch value goes to its first occurrence (:476-489).  Returns 0,
 * or -1 when the scratch table cannot be allocated. */
API int orc_create_permutation_polys(const uint64_t *placement, size_t n_cols, unsigned log_n, const uint64_t *non_residues,
                                     uint64_t *out) {
  const size_t n = (size_t)1 << log_n, cells = n * n_cols;
  const uint64_t w = gl_omega(log_n);
  uint64_t *pows = malloc(sizeof(uint64_t) * n);
  if (!pows) return -1;
#pragma omp parallel for schedule(static)
  for (long rl = 0; rl < (long)n; rl += 4096) {
    uint64_t x = gl_pow(w, (uint64_t)rl);
    for (size_t row = (size_t)rl; row < (size_t)rl + 4096 && row < n; row++) {
      pows[row] = x;
      x = gl_mul(x, w);
    }
  }
#pragma omp parallel for schedule(static)
  for (long cl = 0; cl < (long)n_cols; cl++) {
    const size_t c = (size_t)cl;
    const uint64_t k = gl_canon(non_residues[c]);
    for (size_t row = 0; row < n; row++) out[c * n + row] = gl_mul(k, pows[row]);
  }
  free(pows);
  /* sized for a variable per two cells, about what a circuit has; the table grows past that */
  size_t cap = 1 << 16;
  while (cap < cells / 2) cap *= 2;
  orc_scratch s;
  if (scratch_alloc(&s, cap)) return -1;
  enum { AHEAD = 16 };
  for (size_t cell = 0; cell < cells; cell++) {
    if (cell + AHEAD < cells) __builtin_prefetch(&s.e[scratch_home(&s, placement[cell + AHEAD] & ORC_LOW_U48)], 1);
    const uint64_t var = placement[cell];
    if (var & ORC_PLACEHOLDER_BIT) continue;
    const uint64_t idx = var & ORC_LOW_U48;
    size_t i = scratch_slot(&s, idx);
    if (s.e[i].key == idx) {
      const uint64_t t = s.e[i].value;
      s.e[i].value = out[cell];
      out[cell] = t;
      continue;
    }
    if (4 * (s.count + 1) > 3 * s.cap) {
      if (scratch_grow(&s)) {
        free(s.e);
        return -1;
      }
      i = scratch_slot(&s, idx);
    }
    s.e[i] = (orc_scratch_entry){idx, out[cell], cell};
    s.count++;
  }
  for (size_t i = 0; i < s.cap; i++)
    if (s.e[i].key != ~0ull) out[s.e[i].first] = s.e[i].value;
  free(s.e);
  return 0;
}
