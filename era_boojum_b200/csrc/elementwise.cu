// Element-wise field kernels on the hot path: Montgomery batch inversion (base and Fp2) and the DEEP quotening.
// References:
//   batch_inverse_inplace / batch_inverse_inplace_in_extension   src/cs/implementations/utils.rs:405-600
//   quotening_operation_in_extension (DEEP)                       src/cs/implementations/prover.rs:2523-2706
//     verifier-side statement of the same sum                     src/cs/implementations/verifier.rs:2526-2565
#include "ctx.hpp"

namespace bj {

// x^(p-2) with 64 squarings + 10 multiplications: p - 2 = (2^31 - 1) * 2^33 + (2^32 - 1)
__device__ __forceinline__ u64 gl_inv_chain(u64 x) {
  auto sqn = [](u64 v, int n) {
    for (int i = 0; i < n; i++) v = gl::sqr(v);
    return v;
  };
  const u64 a1 = x;
  const u64 a2 = gl::mul(gl::sqr(a1), a1);          // 2^2 - 1
  const u64 a4 = gl::mul(sqn(a2, 2), a2);           // 2^4 - 1
  const u64 a8 = gl::mul(sqn(a4, 4), a4);           // 2^8 - 1
  const u64 a16 = gl::mul(sqn(a8, 8), a8);          // 2^16 - 1
  const u64 a24 = gl::mul(sqn(a16, 8), a8);         // 2^24 - 1
  const u64 a28 = gl::mul(sqn(a24, 4), a4);         // 2^28 - 1
  const u64 a30 = gl::mul(sqn(a28, 2), a2);         // 2^30 - 1
  const u64 a31 = gl::mul(gl::sqr(a30), a1);        // 2^31 - 1
  const u64 a32 = gl::mul(gl::sqr(a31), a1);        // 2^32 - 1
  return gl::mul(sqn(a31, 33), a32);
}

__device__ __forceinline__ gl::e2 e2_inv_chain(gl::e2 a) {
  const u64 n = gl::canon(gl::sub(gl::sqr(a.c0), gl::mul7(gl::sqr(a.c1))));
  const u64 ni = gl_inv_chain(n);
  return {gl::mul(a.c0, ni), gl::mul(gl::neg(a.c1), ni)};
}

constexpr int BI_K = 8;  // elements per thread (strided by the grid so that loads stay coalesced)

// in place; zeros are mapped to zeros (the reference panics on them, utils.rs:425-427)
__global__ void __launch_bounds__(256) batch_inverse_kernel(u64* __restrict__ a, u64 n) {
  const u64 stride = (u64)gridDim.x * blockDim.x;
  const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  u64 pre[BI_K];
  u64 acc = 1;
#pragma unroll
  for (int j = 0; j < BI_K; j++) {
    const u64 i = t + j * stride;
    pre[j] = acc;
    if (i < n) {
      const u64 v = gl::canon(a[i]);
      if (v) acc = gl::mul(acc, v);
    }
  }
  u64 inv = gl_inv_chain(acc);
#pragma unroll
  for (int j = BI_K - 1; j >= 0; j--) {
    const u64 i = t + j * stride;
    if (i < n) {
      const u64 v = gl::canon(a[i]);
      if (v) {
        a[i] = gl::mul(inv, pre[j]);
        inv = gl::mul(inv, v);
      } else {
        a[i] = 0;
      }
    }
  }
}

__global__ void __launch_bounds__(256) batch_inverse_ext_kernel(u64* __restrict__ c0, u64* __restrict__ c1, u64 n) {
  const u64 stride = (u64)gridDim.x * blockDim.x;
  const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  gl::e2 pre[BI_K];
  gl::e2 acc = {1, 0};
#pragma unroll
  for (int j = 0; j < BI_K; j++) {
    const u64 i = t + j * stride;
    pre[j] = acc;
    if (i < n) {
      const gl::e2 v = {gl::canon(c0[i]), gl::canon(c1[i])};
      if (v.c0 | v.c1) acc = gl::e2_mul(acc, v);
    }
  }
  gl::e2 inv = e2_inv_chain(acc);
#pragma unroll
  for (int j = BI_K - 1; j >= 0; j--) {
    const u64 i = t + j * stride;
    if (i < n) {
      const gl::e2 v = {gl::canon(c0[i]), gl::canon(c1[i])};
      if (v.c0 | v.c1) {
        const gl::e2 r = gl::e2_mul(inv, pre[j]);
        c0[i] = r.c0;
        c1[i] = r.c1;
        inv = gl::e2_mul(inv, v);
      } else {
        c0[i] = 0;
        c1[i] = 0;
      }
    }
  }
}

// DEEP group: acc[t] += (sum_i ch_i * f_i(t) - K) / (x(t) - at), t over the whole LDE domain (coset-major, bit-reversed
// in coset), x(t) = 7 * w_{nL}^{bitrev(t)} = 7 * (-1)^(t & 1) * tab[t >> 1] with the forward twiddle table.
// Each thread owns DEEP_R rows strided by the grid; the Fp2 denominators of its rows share one inversion.
constexpr int DEEP_R = 4;

// one base-field column of the DEEP sum with its two coefficients: acc.c0 += k0 * f, acc.c1 += k1 * f.  An Fp2 polynomial
// (f0, f1) with challenge (c0, c1) is two such columns: f0 with (c0, c1) and f1 with (7 c1, c0)   (u^2 = 7).
struct DeepColumn {
  const u64* f;
  u64 k0, k1;
};

struct DeepParams {
  const DeepColumn* cols;
  u32 n_cols;
  u64 n_rows;                // local points: (local units) * (rows per unit)
  int log_n;                 // coset length (locates the coset bits when the context holds a coset shard)
  CosetShard shard;
  const u64* tab;            // forward twiddles of the whole LDE domain
  gl::e2 at;
  gl::e2 k_const;            // sum_i ch_i * value_at_i  (precomputed on the host)
  u64* acc_c0;
  u64* acc_c1;
  u64 first;                 // RANGE kernel: global index of point 0 (the buffers hold points [first, first + n_rows))
};

// Unreduced accumulator for sums of 64x64-bit products: 128 bits + an overflow word (exact for < 2^32 terms).  One
// reduction per accumulator at the end instead of one per product: the DEEP sum has ~270 terms per row.
struct Acc160 {
  u64 lo, hi;
  u32 ov;
};
__device__ __forceinline__ void acc_mad(Acc160& a, u64 x, u64 y) {
  const u64 pl = x * y, ph = __umul64hi(x, y);
  asm("add.cc.u64 %0, %0, %3;\n\taddc.cc.u64 %1, %1, %4;\n\taddc.u32 %2, %2, 0;" : "+l"(a.lo), "+l"(a.hi), "+r"(a.ov) : "l"(pl), "l"(ph));
}
__device__ __forceinline__ u64 acc_reduce(const Acc160& a) {
  // lo + 2^64 hi + 2^128 ov,  2^128 = -2^32 (mod p)
  const u64 r = gl::reduce128(a.lo, a.hi);
  return gl::canon(gl::sub(r, gl::mul((u64)a.ov, 1ull << 32)));
}

constexpr int DEEP_U = 4;  // columns whose loads are issued together (memory-level parallelism: the kernel streams ~70 GB)

// RANGE = false: the whole domain of this context (x(t) through the shard's global index).  RANGE = true: an unsharded run of
// n_rows consecutive points starting at the global index p.first (a few cosets of the domain, e.g. one recomputed coset).
template <bool RANGE>
__global__ void __launch_bounds__(256) deep_group_kernel(const DeepParams p) {
  const u64 stride = (u64)gridDim.x * blockDim.x;
  const u64 t0 = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  Acc160 a0[DEEP_R], a1[DEEP_R];
#pragma unroll
  for (int r = 0; r < DEEP_R; r++) a0[r] = a1[r] = {0, 0, 0};
  u32 i = 0;
  for (; i + DEEP_U <= p.n_cols; i += DEEP_U) {
    DeepColumn c[DEEP_U];
    u64 v[DEEP_U][DEEP_R];
#pragma unroll
    for (int u = 0; u < DEEP_U; u++) {
      c[u].f = p.cols[i + u].f;
      c[u].k0 = __ldg(&p.cols[i + u].k0);
      c[u].k1 = __ldg(&p.cols[i + u].k1);
    }
#pragma unroll
    for (int u = 0; u < DEEP_U; u++)
#pragma unroll
      for (int r = 0; r < DEEP_R; r++) {
        const u64 t = t0 + r * stride;
        v[u][r] = t < p.n_rows ? __ldcs(c[u].f + t) : 0;  // streamed once: evict first
      }
#pragma unroll
    for (int u = 0; u < DEEP_U; u++)
#pragma unroll
      for (int r = 0; r < DEEP_R; r++) {
        acc_mad(a0[r], c[u].k0, v[u][r]);
        acc_mad(a1[r], c[u].k1, v[u][r]);
      }
  }
  for (; i < p.n_cols; i++) {
    const DeepColumn c = p.cols[i];
#pragma unroll
    for (int r = 0; r < DEEP_R; r++) {
      const u64 t = t0 + r * stride;
      const u64 v = t < p.n_rows ? __ldcs(c.f + t) : 0;
      acc_mad(a0[r], c.k0, v);
      acc_mad(a1[r], c.k1, v);
    }
  }
  gl::e2 s[DEEP_R];
#pragma unroll
  for (int r = 0; r < DEEP_R; r++) s[r] = {acc_reduce(a0[r]), acc_reduce(a1[r])};
  // denominators x - at for the thread's rows, inverted together
  gl::e2 den[DEEP_R], pre[DEEP_R];
  gl::e2 acc = {1, 0};
  const u64 neg_at1 = gl::neg(p.at.c1);
#pragma unroll
  for (int r = 0; r < DEEP_R; r++) {
    const u64 t = t0 + r * stride;
    pre[r] = acc;
    if (t < p.n_rows) {
      const u64 tg = RANGE ? p.first + t : p.shard.global_index(t, p.log_n);
      u64 x = gl::mul(__ldg(p.tab + (tg >> 1)), gl::MULT_GEN);
      if (tg & 1) x = gl::neg(x);
      den[r] = {gl::canon(gl::sub(x, p.at.c0)), neg_at1};
      acc = gl::e2_mul(acc, den[r]);
    }
  }
  gl::e2 inv = e2_inv_chain(acc);
#pragma unroll
  for (int r = DEEP_R - 1; r >= 0; r--) {
    const u64 t = t0 + r * stride;
    if (t < p.n_rows) {
      const gl::e2 dinv = gl::e2_mul(inv, pre[r]);
      inv = gl::e2_mul(inv, den[r]);
      gl::e2 num = {gl::canon(gl::sub(s[r].c0, p.k_const.c0)), gl::canon(gl::sub(s[r].c1, p.k_const.c1))};
      const gl::e2 q = gl::e2_mul(num, dinv);
      p.acc_c0[t] = gl::canon(gl::add(p.acc_c0[t], q.c0));
      p.acc_c1[t] = gl::canon(gl::add(p.acc_c1[t], q.c1));
    }
  }
}

// small parameter arena on the device (pointer tables, challenge vectors): bump allocation, sync on wrap
int32_t param_upload(bj_ctx* ctx, const void* host, size_t bytes, void** d_out) {
  // Bump arena for the small parameter blocks of a call (pointer tables, challenge lists, gate programs).  A wrap restarts at
  // offset 0 after the stream has drained; blocks are capped at ARENA / 32 and no entry point uploads more than 16 blocks, so
  // the blocks a call places after a wrap (<= ARENA / 2 from the start) cannot reach the ones it placed before it (which lie
  // in the upper half: the wrap happened because the arena was full).
  const size_t ARENA = 8 << 20;
  if (bytes > ARENA / 32) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "parameter block too large (256 KiB limit)");
  if (!ctx->param_arena) {
    BJ_CUDA(ctx, cudaMalloc(&ctx->param_arena, ARENA));
    ctx->param_off = 0;
  }
  const size_t need = (bytes + 255) & ~(size_t)255;
  if (ctx->param_off + need > ARENA) {
    BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // everything that read older slices is done
    ctx->param_off = 0;
  }
  void* d = (char*)ctx->param_arena + ctx->param_off;
  ctx->param_off += need;
  BJ_CUDA(ctx, cudaMemcpyAsync(d, host, bytes, cudaMemcpyHostToDevice, ctx->stream));
  *d_out = d;
  return BJ_OK;
}

}  // namespace bj

using namespace bj;

extern "C" {

int32_t bj_batch_inverse(bj_ctx* ctx, uint64_t* d_data, uint64_t n) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || (!d_data && n)) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_batch_inverse: bad argument");
  if (n == 0) return BJ_OK;
  const u64 threads = (n + BI_K - 1) / BI_K;
  batch_inverse_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, ctx->stream>>>((u64*)d_data, n);
  BJ_LAUNCH_CHECK(ctx);
  return BJ_OK;
}

int32_t bj_batch_inverse_ext(bj_ctx* ctx, uint64_t* d_c0, uint64_t* d_c1, uint64_t n) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || ((!d_c0 || !d_c1) && n)) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_batch_inverse_ext: bad argument");
  if (n == 0) return BJ_OK;
  const u64 threads = (n + BI_K - 1) / BI_K;
  batch_inverse_ext_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, ctx->stream>>>((u64*)d_c0, (u64*)d_c1, n);
  BJ_LAUNCH_CHECK(ctx);
  return BJ_OK;
}

int32_t bj_deep_quotient_group(bj_ctx* ctx, const uint64_t* const* h_src_c0, const uint64_t* const* h_src_c1,
                               uint32_t n_src, const uint64_t* h_values_at, const uint64_t* h_challenges,
                               const uint64_t h_at[2], uint32_t log_rows, uint64_t* d_acc_c0, uint64_t* d_acc_c1) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || !h_src_c0 || !h_src_c1 || !h_values_at || !h_challenges || !h_at || !d_acc_c0 || !d_acc_c1 || n_src == 0 ||
      log_rows < 1 || log_rows > 32)
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_deep_quotient_group: bad argument");
  BJ_TRY(ensure_twiddles(ctx, (int)log_rows));
  DeepParams p;
  // canonical challenges, K = sum ch_i * v_i on the host, and the flattened column list
  std::vector<DeepColumn> cols;
  cols.reserve(2 * (size_t)n_src);
  gl::e2 k = {0, 0};
  for (uint32_t i = 0; i < n_src; i++) {
    const gl::e2 c = {gl::canon(h_challenges[2 * i]), gl::canon(h_challenges[2 * i + 1])};
    const gl::e2 v = {gl::canon(h_values_at[2 * i]), gl::canon(h_values_at[2 * i + 1])};
    if (!h_src_c0[i]) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_deep_quotient_group: NULL source column");
    cols.push_back({(const u64*)h_src_c0[i], c.c0, c.c1});
    if (h_src_c1[i]) cols.push_back({(const u64*)h_src_c1[i], gl::mul7(c.c1), c.c0});
    const gl::e2 m = gl::e2_mul(c, v);
    k = {gl::canon(gl::add(k.c0, m.c0)), gl::canon(gl::add(k.c1, m.c1))};
  }
  void* dcols;
  BJ_TRY(param_upload(ctx, cols.data(), sizeof(DeepColumn) * cols.size(), &dcols));
  p.cols = (const DeepColumn*)dcols;
  p.n_cols = (u32)cols.size();
  p.n_rows = 1ull << log_rows;
  p.log_n = (int)log_rows;
  p.shard = ctx->shard;
  if (ctx->shard.log_stride) {
    if (log_rows < ctx->shard_log_lde + ctx->shard.log_split + 1)
      BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_deep_quotient_group: domain smaller than the units of the shard");
    p.log_n = (int)(log_rows - ctx->shard_log_lde);
    p.n_rows = ctx->shard.local_points(1ull << ctx->shard_log_lde, p.log_n);
  }
  p.tab = ctx->tw_fwd;
  p.at = {gl::canon(h_at[0]), gl::canon(h_at[1])};
  p.k_const = k;
  p.acc_c0 = (u64*)d_acc_c0;
  p.acc_c1 = (u64*)d_acc_c1;
  const u64 threads = (p.n_rows + DEEP_R - 1) / DEEP_R;
  deep_group_kernel<false><<<(unsigned)((threads + 255) / 256), 256, 0, ctx->stream>>>(p);
  BJ_LAUNCH_CHECK(ctx);
  return BJ_OK;
}

int32_t bj_deep_quotient_range(bj_ctx* ctx, const uint64_t* const* h_src_c0, const uint64_t* const* h_src_c1, uint32_t n_src,
                               const uint64_t* h_values_at, const uint64_t* h_challenges, const uint64_t h_at[2], uint32_t log_rows,
                               uint64_t first_point, uint64_t n_points, uint64_t* d_acc_c0, uint64_t* d_acc_c1) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || !h_src_c0 || !h_src_c1 || !h_values_at || !h_challenges || !h_at || !d_acc_c0 || !d_acc_c1 || n_src == 0 ||
      log_rows < 1 || log_rows > 32 || n_points == 0 || first_point + n_points > (1ull << log_rows))
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_deep_quotient_range: bad argument");
  if (ctx->shard.log_stride) BJ_FAIL(ctx, BJ_ERR_UNSUPPORTED, "bj_deep_quotient_range: not on a sharded context");
  BJ_TRY(ensure_twiddles(ctx, (int)log_rows));
  DeepParams p;
  std::vector<DeepColumn> cols;
  cols.reserve(2 * (size_t)n_src);
  gl::e2 k = {0, 0};
  for (uint32_t i = 0; i < n_src; i++) {
    const gl::e2 c = {gl::canon(h_challenges[2 * i]), gl::canon(h_challenges[2 * i + 1])};
    const gl::e2 v = {gl::canon(h_values_at[2 * i]), gl::canon(h_values_at[2 * i + 1])};
    if (!h_src_c0[i]) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_deep_quotient_range: NULL source column");
    cols.push_back({(const u64*)h_src_c0[i], c.c0, c.c1});
    if (h_src_c1[i]) cols.push_back({(const u64*)h_src_c1[i], gl::mul7(c.c1), c.c0});
    const gl::e2 m = gl::e2_mul(c, v);
    k = {gl::canon(gl::add(k.c0, m.c0)), gl::canon(gl::add(k.c1, m.c1))};
  }
  void* dcols;
  BJ_TRY(param_upload(ctx, cols.data(), sizeof(DeepColumn) * cols.size(), &dcols));
  p.cols = (const DeepColumn*)dcols;
  p.n_cols = (u32)cols.size();
  p.n_rows = n_points;
  p.log_n = (int)log_rows;
  p.tab = ctx->tw_fwd;
  p.at = {gl::canon(h_at[0]), gl::canon(h_at[1])};
  p.k_const = k;
  p.acc_c0 = (u64*)d_acc_c0;
  p.acc_c1 = (u64*)d_acc_c1;
  p.first = first_point;
  const u64 threads = (p.n_rows + DEEP_R - 1) / DEEP_R;
  deep_group_kernel<true><<<(unsigned)((threads + 255) / 256), 256, 0, ctx->stream>>>(p);
  BJ_LAUNCH_CHECK(ctx);
  return BJ_OK;
}

}  // extern "C"
