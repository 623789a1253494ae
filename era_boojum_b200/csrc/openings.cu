// Openings: evaluate committed polynomials at an Fp2 point from their values on the first LDE coset this context holds.
// Reference: precompute_for_barycentric_evaluation_in_extension + barycentric_evaluate_*_at_extension_for_bitreversed_parallel
// (src/cs/implementations/utils.rs:907-1243), driven from prove_cpu_basic (prover.rs:1519-1802).  f(at) is a field
// element fixed by f alone, so only the value matters:  with x_i = 7 w_n^{bitrev(i)} (coset 0 of the LDE, bit-reversed),
//   f(at) = (at^n - 7^n) / (n 7^n) * sum_i f(x_i) * x_i / (at - x_i).
// Fp2-valued polynomials are stored as two base columns and are evaluated column by column (f = f0 + u f1).
// On a coset-sharded context (multi-GPU) local slot 0 is the global coset j = rank with shift c = 7 w_{nL}^{bitrev_L(j)}
// instead of 7: the same formula with c in place of 7 gives the same f(at), so every rank can open any column from the
// coset it owns and the columns are split over the ranks.  On a split domain shard local slot 0 is one row block of coset
// j: the sum runs over that block's rows with the whole coset's scale and the result is the block's CONTRIBUTION; the B
// contributions of the ranks holding coset j add up to f(at).
#include <vector>
#include "ctx.hpp"

namespace bj {

// den[i] = at - x_i  (Fp2), and xs[i] = x_i
__global__ void __launch_bounds__(256) bary_denominators_kernel(const u64* __restrict__ tab, u64 n, gl::e2 at, u64 shift, u64* __restrict__ d0,
                                                                 u64* __restrict__ d1, u64* __restrict__ xs) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  u64 x = gl::mul(n > 1 ? __ldg(tab + (i >> 1)) : 1, shift);
  if (i & 1) x = gl::neg(x);
  xs[i] = x;
  d0[i] = gl::canon(gl::sub(at.c0, x));
  d1[i] = at.c1;
}

// w[i] = scale * x_i * inv[i]
__global__ void __launch_bounds__(256) bary_weights_kernel(u64* __restrict__ w0, u64* __restrict__ w1, const u64* __restrict__ xs, u64 n,
                                                            gl::e2 scale) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const gl::e2 v = gl::e2_mul(gl::e2_mul_base({w0[i], w1[i]}, xs[i]), scale);
  w0[i] = v.c0;
  w1[i] = v.c1;
}

constexpr int DOT_COLS = 8;
constexpr int DOT_T = 256;

// partial[block][col] = sum over the block's rows of f_col[i] * w[i]
__global__ void __launch_bounds__(DOT_T) bary_dot_kernel(const u64* const* __restrict__ cols, u32 n_cols, u64 n, const u64* __restrict__ w0,
                                                          const u64* __restrict__ w1, u64* __restrict__ partial) {
  __shared__ u64 red[DOT_T / 32][DOT_COLS][2];
  const u32 cbase = blockIdx.y * DOT_COLS;
  gl::e2 acc[DOT_COLS];
#pragma unroll
  for (int c = 0; c < DOT_COLS; c++) acc[c] = {0, 0};
  for (u64 i = (u64)blockIdx.x * DOT_T + threadIdx.x; i < n; i += (u64)gridDim.x * DOT_T) {
    const u64 a0 = w0[i], a1 = w1[i];
#pragma unroll
    for (int c = 0; c < DOT_COLS; c++) {
      if (cbase + c < n_cols) {
        const u64 f = cols[cbase + c][i];
        acc[c].c0 = gl::add(acc[c].c0, gl::mul(f, a0));
        acc[c].c1 = gl::add(acc[c].c1, gl::mul(f, a1));
      }
    }
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int c = 0; c < DOT_COLS; c++) {
    u64 v0 = gl::canon(acc[c].c0), v1 = gl::canon(acc[c].c1);
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) {
      v0 = gl::canon(gl::add(v0, __shfl_down_sync(0xffffffffu, v0, d)));
      v1 = gl::canon(gl::add(v1, __shfl_down_sync(0xffffffffu, v1, d)));
    }
    if (lane == 0) {
      red[wid][c][0] = v0;
      red[wid][c][1] = v1;
    }
  }
  __syncthreads();
  if (threadIdx.x < DOT_COLS * 2) {
    const int c = threadIdx.x >> 1, k = threadIdx.x & 1;
    u64 s = 0;
    for (int wv = 0; wv < DOT_T / 32; wv++) s = gl::canon(gl::add(s, red[wv][c][k]));
    if (cbase + c < n_cols) partial[((u64)blockIdx.x * n_cols + cbase + c) * 2 + k] = s;
  }
}

}  // namespace bj

using namespace bj;

extern "C" int32_t bj_barycentric_evaluate(bj_ctx* ctx, const uint64_t* const* h_cols, uint32_t n_cols, uint32_t log_n,
                                           const uint64_t h_at[2], uint64_t* h_out) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || !h_cols || !h_at || !h_out || n_cols == 0 || log_n > 32)
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_barycentric_evaluate: bad argument");
  const u64 n = 1ull << log_n;
  // shift of the unit in local slot 0 (the global unit `first`): 7 * w_{nL}^{bitrev_L(j)} for a whole coset (7 itself without a
  // shard / on rank 0), times w_n^{bitrev_s(p)} for row block p of a split shard, which sums over its n / B rows only
  const u32 split = ctx->shard.log_split;
  if (split >= log_n && split) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_barycentric_evaluate: fewer rows than row blocks of the domain shard");
  const u64 rows = n >> split;
  u64 shift = gl::MULT_GEN;
  if (ctx->shard.first) shift = ctx->shard.unit_shift(ctx->shard.first, log_n, ctx->shard_log_lde);
  BJ_TRY(ensure_twiddles(ctx, (int)log_n));
  const gl::e2 at = {gl::canon(h_at[0]), gl::canon(h_at[1])};
  // scale = (at^n - c^n) / (n * c^n), c = the coset's shift (c^n = shift^n: the row-block factor is an n-th root of unity)
  gl::e2 atn = at;
  for (u32 i = 0; i < log_n; i++) atn = gl::e2_sqr(atn);
  const u64 cn = gl::pow(shift, n);
  gl::e2 scale = {gl::canon(gl::sub(atn.c0, cn)), atn.c1};
  scale = gl::e2_mul_base(scale, gl::inv(gl::mul(gl::canon(n % gl::P), cn)));
  const u32 gx = (u32)std::min<u64>((rows + DOT_T - 1) / DOT_T, 4 * (u64)ctx->sm_count);
  const size_t need = sizeof(u64) * (3 * rows + (size_t)gx * n_cols * 2);
  BJ_TRY(ensure_scratch(ctx, need));
  u64* w0 = (u64*)ctx->scratch;
  u64* w1 = w0 + rows;
  u64* xs = w1 + rows;
  u64* partial = xs + rows;
  const unsigned blocks = (unsigned)((rows + 255) / 256);
  bary_denominators_kernel<<<blocks, 256, 0, ctx->stream>>>(ctx->tw_fwd, rows, at, shift, w0, w1, xs);
  BJ_LAUNCH_CHECK(ctx);
  BJ_TRY(bj_batch_inverse_ext(ctx, (uint64_t*)w0, (uint64_t*)w1, rows));
  bary_weights_kernel<<<blocks, 256, 0, ctx->stream>>>(w0, w1, xs, rows, scale);
  BJ_LAUNCH_CHECK(ctx);
  void* d;
  BJ_TRY(param_upload(ctx, h_cols, sizeof(u64*) * n_cols, &d));
  dim3 grid(gx, (n_cols + DOT_COLS - 1) / DOT_COLS);
  bary_dot_kernel<<<grid, DOT_T, 0, ctx->stream>>>((const u64* const*)d, n_cols, rows, w0, w1, partial);
  BJ_LAUNCH_CHECK(ctx);
  std::vector<u64> hp((size_t)gx * n_cols * 2);
  BJ_CUDA(ctx, cudaMemcpyAsync(hp.data(), partial, sizeof(u64) * hp.size(), cudaMemcpyDeviceToHost, ctx->stream));
  BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  for (u32 c = 0; c < n_cols; c++) {
    u64 s0 = 0, s1 = 0;
    for (u32 b = 0; b < gx; b++) {
      s0 = gl::canon(gl::add(s0, hp[((size_t)b * n_cols + c) * 2]));
      s1 = gl::canon(gl::add(s1, hp[((size_t)b * n_cols + c) * 2 + 1]));
    }
    h_out[2 * c] = s0;
    h_out[2 * c + 1] = s1;
  }
  return BJ_OK;
}
