// FRI fold kernel.  Reference: fold_multiple (src/cs/implementations/fri/mod.rs:362-474) driven by
// interpolate_independent_cosets / interpolate_flattened_cosets (:476-678): one oracle step is K in {1,2,3}
// successive fold-by-2 of the flat (coset-major, bit-reversed) Fp2 codeword:
//     out[i] = (f[2i] + f[2i+1]) + alpha_l * (f[2i] - f[2i+1]) * R[i] * kappa_l
// with R = the inverse twiddle table (prefix reused at every level), kappa_0 = running coset inverse, squared per
// fold, alpha_l = alpha^(2^l).  The reference runs K passes over memory; here one thread folds its 2^K inputs in
// registers, so a step moves 16*(2^K + 1) bytes per output instead of 48 per fold.
#include "ctx.hpp"

namespace bj {

struct FoldParams {
  gl::e2 alpha[3];
  u64 kappa[3];
  CosetShard shard;   // coset shard of a multi-GPU prover: local pair indices are mapped to global ones for the roots
  int log_coset_out;  // log2 of the coset length of the OUTPUT vector
};

template <int K>
__global__ void __launch_bounds__(256) fri_fold_kernel(const u64* __restrict__ c0, const u64* __restrict__ c1,
                                                        u64 n_out, const u64* __restrict__ roots, FoldParams fp,
                                                        u64* __restrict__ o0, u64* __restrict__ o1) {
  const u64 o = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= n_out) return;
  constexpr int N = 1 << K;
  u64 a0[N], a1[N];
  const ulonglong2* p0 = reinterpret_cast<const ulonglong2*>(c0 + o * N);
  const ulonglong2* p1 = reinterpret_cast<const ulonglong2*>(c1 + o * N);
#pragma unroll
  for (int i = 0; i < N / 2; i++) {
    const ulonglong2 v0 = p0[i], v1 = p1[i];
    a0[2 * i] = gl::canon(v0.x);
    a0[2 * i + 1] = gl::canon(v0.y);
    a1[2 * i] = gl::canon(v1.x);
    a1[2 * i + 1] = gl::canon(v1.y);
  }
#pragma unroll
  for (int l = 0; l < K; l++) {
    const int cnt = N >> (l + 1);  // outputs of this level held by the thread
#pragma unroll
    for (int j = 0; j < cnt; j++) {
      // pair index at this level: the level's output vector has cosets of 2^(log_coset_out + log2(cnt)) elements
      const u64 gidx = fp.shard.global_index(o * cnt + j, fp.log_coset_out + (K - 1 - l));
      const u64 r = gl::mul(__ldg(roots + gidx), fp.kappa[l]);
      const u64 x0 = a0[2 * j], y0 = a0[2 * j + 1], x1 = a1[2 * j], y1 = a1[2 * j + 1];
      gl::e2 d = {gl::mul(gl::sub(x0, y0), r), gl::mul(gl::sub(x1, y1), r)};
      d = gl::e2_mul(d, fp.alpha[l]);
      a0[j] = gl::canon(gl::add(gl::add(d.c0, x0), y0));
      a1[j] = gl::canon(gl::add(gl::add(d.c1, x1), y1));
    }
  }
  o0[o] = a0[0];
  o1[o] = a1[0];
}

}  // namespace bj

using namespace bj;

extern "C" int32_t bj_fri_fold(bj_ctx* ctx, const uint64_t* d_c0, const uint64_t* d_c1, uint32_t log_m,
                               uint32_t log_fold, const uint64_t h_alpha[2], uint64_t* h_coset_inv_io,
                               uint64_t* d_out_c0, uint64_t* d_out_c1) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || !d_c0 || !d_c1 || !h_alpha || !h_coset_inv_io || !d_out_c0 || !d_out_c1)
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_fri_fold: NULL argument");
  if (log_fold < 1 || log_fold > 3 || log_fold > log_m || log_m > 32)
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_fri_fold: log_fold must be 1..3 and <= log_m");
  if (((uintptr_t)d_c0 | (uintptr_t)d_c1) & 15) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_fri_fold: inputs must be 16-byte aligned");
  FoldParams fp;
  gl::e2 a = {gl::canon(h_alpha[0]), gl::canon(h_alpha[1])};
  u64 kappa = gl::canon(*h_coset_inv_io);
  for (uint32_t l = 0; l < 3; l++) {
    fp.alpha[l] = a;
    fp.kappa[l] = kappa;
    if (l < log_fold) {
      a = gl::e2_sqr(a);
      kappa = gl::sqr(kappa);
    }
  }
  u64 n_out = 1ull << (log_m - log_fold);
  fp.shard = ctx->shard;
  fp.log_coset_out = 0;
  if (ctx->shard.log_stride) {
    // local vectors hold the owned units only; a fold never crosses a unit while the folded unit is >= 1 element
    if (log_m < ctx->shard_log_lde + ctx->shard.log_split + log_fold)
      BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_fri_fold: fold would cross units of the shard");
    fp.log_coset_out = (int)(log_m - log_fold - ctx->shard_log_lde);
    n_out = ctx->shard.local_points(1ull << ctx->shard_log_lde, fp.log_coset_out);
  }
  BJ_TRY(ensure_twiddles(ctx, (int)log_m));
  const unsigned blocks = (unsigned)((n_out + 255) / 256);
  const u64* roots = ctx->tw_inv;
  switch (log_fold) {
    case 1: fri_fold_kernel<1><<<blocks, 256, 0, ctx->stream>>>((const u64*)d_c0, (const u64*)d_c1, n_out, roots, fp, (u64*)d_out_c0, (u64*)d_out_c1); break;
    case 2: fri_fold_kernel<2><<<blocks, 256, 0, ctx->stream>>>((const u64*)d_c0, (const u64*)d_c1, n_out, roots, fp, (u64*)d_out_c0, (u64*)d_out_c1); break;
    default: fri_fold_kernel<3><<<blocks, 256, 0, ctx->stream>>>((const u64*)d_c0, (const u64*)d_c1, n_out, roots, fp, (u64*)d_out_c0, (u64*)d_out_c1); break;
  }
  BJ_LAUNCH_CHECK(ctx);
  *h_coset_inv_io = kappa;
  return BJ_OK;
}
