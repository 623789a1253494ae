// Quotient-side kernels other than the gate evaluator: copy-permutation relations, the z(1) = 1 term, division by the
// vanishing polynomial.  All run over the first Q cosets of the LDE (flat index t = coset * n + i, values bit-reversed
// inside a coset), x(t) = 7 * w_{nL}^{bitrev(t)} = 7 * (-1)^(t&1) * tab[t >> 1].
//   z(1) = 1 term                                  src/cs/implementations/prover.rs:1189-1227  (z - 1) * (x^n - 1)/(x - 1) * alpha
//     unnormalized_l1_inverse                      src/cs/implementations/utils.rs:1585-1665
//   compute_quotient_terms_in_extension            src/cs/implementations/copy_permutation.rs:1000-1249
//     relation c: alpha_c * ( lhs_c * prod_{j in chunk c}(w_j + beta sigma_j + gamma) - rhs_c * prod_j (w_j + beta k_j x + gamma) ),
//     lhs = partial_0, ..., partial_{m-2}, z(omega x) ; rhs = z, partial_0, ..., partial_{m-2}
//     z(omega x): shift_by_omega_assuming_bitreversed utils.rs:1245-1271 (index bitrev(bitrev(i) + 1) in the same coset)
//   divide_by_vanishing_for_bitreversed_coset_enumeration   utils.rs:770-817 (one constant per coset)
#include <vector>
#include "ctx.hpp"

namespace bj {

struct QCopyPermParams {
  const u64* const* vars;    // LDE columns (flat [L][n])
  const u64* const* sigmas;
  const u64* non_residues;
  u32 n_cols, chunk, n_chunks;
  const u64* z_c0;
  const u64* z_c1;
  const u64* z_next_c0;        // z(omega x) on the same points (split domain shard), or nullptr: read z at bitrev(bitrev(i) + 1)
  const u64* z_next_c1;
  const u64* const* partials;  // 2 * (n_chunks - 1) pointers: c0, c1 of each partial product LDE
  gl::e2 beta, gamma;
  const u64* alphas;           // (n_chunks + 1) Fp2: z(1)=1 term first, then one per relation
  const u64* tab;              // forward twiddles of the full LDE domain
  const u64* coset_xn_minus_1; // per coset: x^n - 1
  int log_n;
  u64 n_points;                // (local cosets among the first Q) * n
  CosetShard shard;
  u64* q_c0;
  u64* q_c1;
};

template <bool kZNext>
__global__ void __launch_bounds__(128) quotient_copy_perm_kernel(const QCopyPermParams p) {
  const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= p.n_points) return;
  const u64 n = 1ull << p.log_n;
  const u64 coset = t >> p.log_n, i = t & (n - 1);   // local coset slot
  const u64 tg = p.shard.global_index(t, p.log_n);   // index in the whole LDE domain
  u64 x = gl::mul(__ldg(p.tab + (tg >> 1)), gl::MULT_GEN);
  if (tg & 1) x = gl::neg(x);
  const gl::e2 z = {p.z_c0[t], p.z_c1[t]};
  gl::e2 q = {0, 0};
  {
    // alpha_0 * (z - 1) * (x^n - 1) / (x - 1)
    const u64 l1 = gl::mul(__ldg(p.coset_xn_minus_1 + (tg >> p.log_n)), gl_inv_chain(gl::canon(gl::sub(x, 1))));
    gl::e2 v = {gl::mul(gl::sub(z.c0, 1), l1), gl::mul(z.c1, l1)};
    q = gl::e2_mul(v, {__ldg(p.alphas), __ldg(p.alphas + 1)});
  }
  // z(omega x): same coset, position bitrev(bitrev(i) + 1); a row block of a split shard does not hold that row, so there
  // z(omega x) comes as its own LDE columns
  u64 ish = 0;
  if (!kZNext && p.log_n) {
    const u64 nat = (__brevll(i) >> (64 - p.log_n)) + 1;
    ish = __brevll(nat & (n - 1)) >> (64 - p.log_n);
  }
  const u64 tsh = (coset << p.log_n) | ish;
  const gl::e2 bx = {gl::mul(p.beta.c0, x), gl::mul(p.beta.c1, x)};
  u32 col = 0;
  for (u32 c = 0; c < p.n_chunks; c++) {
    gl::e2 lhs, rhs;
    if (c + 1 < p.n_chunks) lhs = {p.partials[2 * c][t], p.partials[2 * c + 1][t]};
    else if (kZNext) lhs = {p.z_next_c0[t], p.z_next_c1[t]};
    else lhs = {p.z_c0[tsh], p.z_c1[tsh]};
    if (c == 0) rhs = z;
    else rhs = {p.partials[2 * (c - 1)][t], p.partials[2 * (c - 1) + 1][t]};
    lhs = {gl::canon(lhs.c0), gl::canon(lhs.c1)};
    rhs = {gl::canon(rhs.c0), gl::canon(rhs.c1)};
    for (u32 j = 0; j < p.chunk && col < p.n_cols; j++, col++) {
      const u64 w = p.vars[col][t];
      const u64 s = p.sigmas[col][t];
      const u64 k = __ldg(p.non_residues + col);
      const u64 wg = gl::add_lazy(p.gamma.c0, w);                      // w + gamma.c0 (lazy), shared by both factors
      // w + beta sigma + gamma: the addend rides in the product's 128 bits (one reduction per component)
      const gl::e2 b = {gl::fma_lazy(p.beta.c0, s, wg), gl::fma_lazy(p.beta.c1, s, p.gamma.c1)};
      lhs = gl::e2_mul_lazy(lhs, b);
      // w + (beta x) k + gamma: the non-residues are small integers (make_non_residues counts up from 2, utils.rs:636-688), so
      // the product is a 64 x 32 bit one kept in 96 bits together with the addend; full product for an unexpectedly large k
      gl::e2 a;
      if (k >> 31) {
        a = {gl::fma_lazy(bx.c0, k, wg), gl::fma_lazy(bx.c1, k, p.gamma.c1)};
      } else {
        a = {gl::w96_reduce(gl::w96_add64(gl::mul_u32_wide(bx.c0, (u32)k), wg)),
             gl::w96_reduce(gl::w96_add64(gl::mul_u32_wide(bx.c1, (u32)k), p.gamma.c1))};
      }
      rhs = gl::e2_mul_lazy(rhs, a);
    }
    gl::e2 d = {gl::canon(gl::sub_lazy(lhs.c0, rhs.c0)), gl::canon(gl::sub_lazy(lhs.c1, rhs.c1))};
    d = gl::e2_mul(d, {__ldg(p.alphas + 2 * (c + 1)), __ldg(p.alphas + 2 * (c + 1) + 1)});
    q = {gl::canon(gl::add(q.c0, d.c0)), gl::canon(gl::add(q.c1, d.c1))};
  }
  p.q_c0[t] = gl::canon(gl::add(p.q_c0[t], q.c0));
  p.q_c1[t] = gl::canon(gl::add(p.q_c1[t], q.c1));
}

__global__ void __launch_bounds__(256) scale_by_coset_constant_kernel(u64* __restrict__ c0, u64* __restrict__ c1, int log_n,
                                                                       u64 n_points, const u64* __restrict__ per_coset, CosetShard shard) {
  const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_points) return;
  const u64 m = __ldg(per_coset + (shard.global_index(t, log_n) >> log_n));
  c0[t] = gl::mul(c0[t], m);
  c1[t] = gl::mul(c1[t], m);
}

// host: (7 * w_{nQ}^{bitrev_Q(j)})^n - 1 for j < Q
static void coset_vanishing_values(u32 log_n, u32 log_q, std::vector<u64>& out) {
  const u64 Q = 1ull << log_q;
  const u64 w = gl::omega(log_n + log_q);
  out.resize(Q);
  for (u64 j = 0; j < Q; j++) {
    u64 jr = 0;
    for (u32 b = 0; b < log_q; b++) jr |= ((j >> b) & 1) << (log_q - 1 - b);
    const u64 shift = gl::mul(gl::MULT_GEN, gl::pow(w, jr));
    out[j] = gl::canon(gl::sub(gl::pow(shift, 1ull << log_n), 1));
  }
}

static int32_t quotient_copy_permutation(bj_ctx* ctx, const uint64_t* const* h_variable_ldes, const uint64_t* const* h_sigma_ldes,
                                         uint32_t n_cols, const uint64_t* h_non_residues, const uint64_t* d_z_c0, const uint64_t* d_z_c1,
                                         const uint64_t* d_z_next_c0, const uint64_t* d_z_next_c1, const uint64_t* const* h_partial_ldes,
                                         const uint64_t h_beta[2], const uint64_t h_gamma[2], const uint64_t* h_alphas, uint32_t log_n,
                                         uint32_t log_lde, uint32_t log_quotient_degree, uint32_t chunk_size, uint64_t* d_q_c0, uint64_t* d_q_c1) {
  if (!ctx || !h_variable_ldes || !h_sigma_ldes || !h_non_residues || !d_z_c0 || !d_z_c1 || !h_beta || !h_gamma || !h_alphas ||
      !d_q_c0 || !d_q_c1 || n_cols == 0 || chunk_size == 0 || log_quotient_degree > log_lde || log_n + log_lde > 32)
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_quotient_copy_permutation: bad argument");
  if (!d_z_next_c0 != !d_z_next_c1) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_quotient_copy_permutation: z(omega x) needs both components");
  if (ctx->shard.log_split && !d_z_next_c0)
    BJ_FAIL(ctx, BJ_ERR_UNSUPPORTED,
            "bj_quotient_copy_permutation: a row block of a split domain shard does not hold z(omega x) - use bj_quotient_copy_permutation_with_z_next");
  const u32 n_chunks = (n_cols + chunk_size - 1) / chunk_size;
  if (n_chunks > 1 && !h_partial_ldes) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_quotient_copy_permutation: partial products missing");
  BJ_TRY(ensure_twiddles(ctx, (int)(log_n + log_lde)));
  QCopyPermParams p{};
  void* d;
  BJ_TRY(param_upload(ctx, h_variable_ldes, sizeof(u64*) * n_cols, &d));
  p.vars = (const u64* const*)d;
  BJ_TRY(param_upload(ctx, h_sigma_ldes, sizeof(u64*) * n_cols, &d));
  p.sigmas = (const u64* const*)d;
  std::vector<u64> nr(n_cols);
  for (u32 i = 0; i < n_cols; i++) nr[i] = gl::canon(h_non_residues[i]);
  BJ_TRY(param_upload(ctx, nr.data(), sizeof(u64) * n_cols, &d));
  p.non_residues = (const u64*)d;
  static const u64* const null_ptr = nullptr;
  BJ_TRY(param_upload(ctx, n_chunks > 1 ? (const void*)h_partial_ldes : (const void*)&null_ptr,
                      sizeof(u64*) * std::max(2 * (n_chunks - 1), 1u), &d));
  p.partials = (const u64* const*)d;
  std::vector<u64> al(2 * (size_t)(n_chunks + 1));
  for (size_t i = 0; i < al.size(); i++) al[i] = gl::canon(h_alphas[i]);
  BJ_TRY(param_upload(ctx, al.data(), sizeof(u64) * al.size(), &d));
  p.alphas = (const u64*)d;
  std::vector<u64> van;
  coset_vanishing_values(log_n, log_quotient_degree, van);
  BJ_TRY(param_upload(ctx, van.data(), sizeof(u64) * van.size(), &d));
  p.coset_xn_minus_1 = (const u64*)d;
  p.n_cols = n_cols;
  p.chunk = chunk_size;
  p.n_chunks = n_chunks;
  p.z_c0 = (const u64*)d_z_c0;
  p.z_c1 = (const u64*)d_z_c1;
  p.z_next_c0 = (const u64*)d_z_next_c0;
  p.z_next_c1 = (const u64*)d_z_next_c1;
  p.beta = {gl::canon(h_beta[0]), gl::canon(h_beta[1])};
  p.gamma = {gl::canon(h_gamma[0]), gl::canon(h_gamma[1])};
  p.tab = ctx->tw_fwd;
  p.log_n = (int)log_n;
  p.shard = ctx->shard;
  p.n_points = ctx->shard.local_points(1ull << log_quotient_degree, (int)log_n);
  if (p.n_points == 0) return BJ_OK;  // this shard owns none of the quotient cosets
  p.q_c0 = (u64*)d_q_c0;
  p.q_c1 = (u64*)d_q_c1;
  if (d_z_next_c0) quotient_copy_perm_kernel<true><<<(unsigned)((p.n_points + 127) / 128), 128, 0, ctx->stream>>>(p);
  else quotient_copy_perm_kernel<false><<<(unsigned)((p.n_points + 127) / 128), 128, 0, ctx->stream>>>(p);
  BJ_LAUNCH_CHECK(ctx);
  return BJ_OK;
}

}  // namespace bj

using namespace bj;

extern "C" {

int32_t bj_quotient_copy_permutation(bj_ctx* ctx, const uint64_t* const* h_variable_ldes, const uint64_t* const* h_sigma_ldes,
                                     uint32_t n_cols, const uint64_t* h_non_residues, const uint64_t* d_z_c0,
                                     const uint64_t* d_z_c1, const uint64_t* const* h_partial_ldes, const uint64_t h_beta[2],
                                     const uint64_t h_gamma[2], const uint64_t* h_alphas, uint32_t log_n, uint32_t log_lde,
                                     uint32_t log_quotient_degree, uint32_t chunk_size, uint64_t* d_q_c0, uint64_t* d_q_c1) {
  bj::DeviceGuard device_guard(ctx);
  return quotient_copy_permutation(ctx, h_variable_ldes, h_sigma_ldes, n_cols, h_non_residues, d_z_c0, d_z_c1, nullptr, nullptr,
                                   h_partial_ldes, h_beta, h_gamma, h_alphas, log_n, log_lde, log_quotient_degree, chunk_size, d_q_c0, d_q_c1);
}

int32_t bj_quotient_copy_permutation_with_z_next(bj_ctx* ctx, const uint64_t* const* h_variable_ldes, const uint64_t* const* h_sigma_ldes,
                                                 uint32_t n_cols, const uint64_t* h_non_residues, const uint64_t* d_z_c0,
                                                 const uint64_t* d_z_c1, const uint64_t* d_z_next_c0, const uint64_t* d_z_next_c1,
                                                 const uint64_t* const* h_partial_ldes, const uint64_t h_beta[2], const uint64_t h_gamma[2],
                                                 const uint64_t* h_alphas, uint32_t log_n, uint32_t log_lde, uint32_t log_quotient_degree,
                                                 uint32_t chunk_size, uint64_t* d_q_c0, uint64_t* d_q_c1) {
  bj::DeviceGuard device_guard(ctx);
  if (ctx && (!d_z_next_c0 || !d_z_next_c1))
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_quotient_copy_permutation_with_z_next: z(omega x) columns missing");
  return quotient_copy_permutation(ctx, h_variable_ldes, h_sigma_ldes, n_cols, h_non_residues, d_z_c0, d_z_c1, d_z_next_c0, d_z_next_c1,
                                   h_partial_ldes, h_beta, h_gamma, h_alphas, log_n, log_lde, log_quotient_degree, chunk_size, d_q_c0, d_q_c1);
}

int32_t bj_quotient_divide_by_vanishing(bj_ctx* ctx, uint64_t* d_q_c0, uint64_t* d_q_c1, uint32_t log_n,
                                        uint32_t log_quotient_degree) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || !d_q_c0 || !d_q_c1 || log_n + log_quotient_degree > 32)
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_quotient_divide_by_vanishing: bad argument");
  std::vector<u64> van;
  coset_vanishing_values(log_n, log_quotient_degree, van);
  for (auto& v : van) v = gl::inv(v);
  void* d;
  BJ_TRY(param_upload(ctx, van.data(), sizeof(u64) * van.size(), &d));
  const u64 n_points = ctx->shard.local_points(1ull << log_quotient_degree, (int)log_n);
  if (n_points == 0) return BJ_OK;
  scale_by_coset_constant_kernel<<<(unsigned)((n_points + 255) / 256), 256, 0, ctx->stream>>>((u64*)d_q_c0, (u64*)d_q_c1, (int)log_n, n_points,
                                                                                              (const u64*)d, ctx->shard);
  BJ_LAUNCH_CHECK(ctx);
  return BJ_OK;
}

}  // extern "C"
