// Goldilocks NTT / iNTT / LDE kernels and drivers (sm_90a).  See ntt.cuh for what is computed and where the
// reference defines it.  Layout of one pass:
//
//   tile = 2^t "rows" x 2^w "columns" of one polynomial, element (row, col) at  base + row * S + col
//   (S = distance between rows).  The pass runs reference rounds [r0, r0+t): butterflies pair rows, columns are
//   independent.  Rounds are executed as radix-16 register stages (4 rounds per stage, 16 values per thread),
//   values travel HBM -> smem once, smem <-> registers once per stage, smem -> HBM once.
//   Twiddle of reference round rho, group k is tab[k] (bit-reversed table); for a thread it is
//   tab[(PFX << q) | (j >> (4 - q))] with PFX = index bits above the thread's 16 values.
//
//   PASS_TILE           : store position == load position (in-place order, bit-reversed frequencies)
//   PASS_TRANSPOSE_LAST : last pass of a natural -> natural transform: the tile's columns are 2^w consecutive
//                         low frequency indices k1 (each a contiguous block of 2^t values, block = bitrev(k1)),
//                         outputs are written to k1 + kappa * 2^r0 (natural order) - the four-step transpose
//                         folded into the store; must be out of place unless r0 == 0.
#include <algorithm>
#include <cstdlib>
#include "ctx.hpp"
#include "ntt.cuh"
#include "ntt_v2.cuh"

namespace bj {

using gl::u32;

__device__ __forceinline__ int phys(int e) { return e + (e >> 4); }  // 1 pad word per 16: conflict-free stages

__device__ __forceinline__ u64 scale_factor(const NttPass& p, u64 idx) {
  if (p.scale_mode == SCALE_CONST) return p.scale_const;
  if (p.scale_mode == SCALE_FULL) return __ldg(p.pw_full + idx);
  u64 lo = __ldg(p.pw_lo + (idx & ((1ull << p.pw_split) - 1)));
  u64 hi = __ldg(p.pw_hi + (idx >> p.pw_split));
  return gl::mul(lo, hi);
}

// RS reference rounds on the top RS bits of the local index j (bit 3 first)
template <int RS>
__device__ __forceinline__ void stage_compute(u64 (&x)[16], const u64* __restrict__ tab, u32 pfx) {
#pragma unroll
  for (int q = 0; q < RS; q++) {
    const int bit = 1 << (3 - q);
#pragma unroll
    for (int j0 = 0; j0 < 16; j0++) {
      if (j0 & bit) continue;
      const int j1 = j0 | bit;
      const u32 k = (pfx << q) | (u32)(j0 >> (4 - q));
      const u64 s = __ldg(tab + k);
      const u64 v = gl::mul(x[j1], s);  // canonical
      x[j1] = gl::sub(x[j0], v);
      x[j0] = gl::add(x[j0], v);
    }
  }
}

__global__ void __launch_bounds__(512) ntt_pass_kernel(const NttPass p) {
  extern __shared__ u64 sm[];
  const int t = p.t, w = p.w, LOG_E = t + w;
  const int E = 1 << LOG_E, W = 1 << w;
  const int tid = threadIdx.x, nthr = blockDim.x;
  const u64 tile = blockIdx.x;
  const u64* __restrict__ src = p.src + (u64)blockIdx.y * p.src_col_stride;
  u64* __restrict__ dst = p.dst + (u64)blockIdx.y * p.dst_col_stride;
  const int m = p.log_n, r0 = p.r0;
  const bool do_scale = p.scale_mode != SCALE_NONE;

  u64 base = 0, S = 1;
  u32 hi = 0;
  if (p.kind == PASS_TILE) {
    const int lo_bits = m - r0 - t;
    const int groups_log = lo_bits - w;
    S = 1ull << lo_bits;
    hi = (u32)(tile >> groups_log);
    const u64 lo0 = (tile & ((1ull << groups_log) - 1)) << w;
    base = ((u64)hi << (m - r0)) + lo0;
    for (int e = tid; e < E; e += nthr) {
      const int row = e >> w, col = e & (W - 1);
      const u64 gi = base + (u64)row * S + col;
      u64 v = src[gi];
      if (do_scale && p.scale_on_load) v = gl::mul(v, scale_factor(p, gi));
      sm[phys(e)] = v;
    }
  } else {
    for (int idx = tid; idx < E; idx += nthr) {
      const int col = idx >> t, row = idx & ((1 << t) - 1);
      const u32 k1 = (u32)(tile << w) + col;
      const u32 blk = r0 ? (__brev(k1) >> (32 - r0)) : 0u;
      const u64 gi = ((u64)blk << t) + row;
      u64 v = src[gi];
      if (do_scale && p.scale_on_load) v = gl::mul(v, scale_factor(p, gi));
      sm[phys(row * W + col)] = v;
    }
  }
  __syncthreads();

  int done = 0;
  int rs = t & 3;
  if (rs == 0) rs = 4;
  const int nvt = E >> 4;  // virtual threads (16 values each)
  while (done < t) {
    const int b_lo = t - done - rs;
    const int pp = b_lo + w - (4 - rs);  // position of the 4 thread-local index bits
    for (int q = tid; q < nvt; q += nthr) {
      const int e0 = ((q >> pp) << (pp + 4)) | (q & ((1 << pp) - 1));
      u32 hq = hi | p.tw_prefix;  // twisted table: round rho's twiddles start at tab + 2^rho (ntt.cuh)
      if (p.kind != PASS_TILE) {
        const u32 k1 = (u32)(tile << w) + (e0 & (W - 1));
        hq = r0 ? (__brev(k1) >> (32 - r0)) : 0u;
      }
      const u32 pfx = (hq << (LOG_E - pp - 4)) | (u32)(q >> pp);
      u64 x[16];
#pragma unroll
      for (int j = 0; j < 16; j++) x[j] = sm[phys(e0 | (j << pp))];
      switch (rs) {
        case 1: stage_compute<1>(x, p.tab, pfx); break;
        case 2: stage_compute<2>(x, p.tab, pfx); break;
        case 3: stage_compute<3>(x, p.tab, pfx); break;
        default: stage_compute<4>(x, p.tab, pfx); break;
      }
#pragma unroll
      for (int j = 0; j < 16; j++) sm[phys(e0 | (j << pp))] = x[j];
    }
    __syncthreads();
    done += rs;
    rs = 4;
  }

  if (p.kind == PASS_TILE) {
    for (int e = tid; e < E; e += nthr) {
      const int row = e >> w, col = e & (W - 1);
      const u64 gi = base + (u64)row * S + col;
      u64 v = sm[phys(e)];
      if (do_scale && !p.scale_on_load) v = gl::mul(v, scale_factor(p, gi));
      if (p.canon_out) v = gl::canon(v);
      dst[gi] = v;
    }
  } else {
    for (int idx = tid; idx < E; idx += nthr) {
      const int col = idx & (W - 1);
      const u32 kappa = (u32)(idx >> w);
      const u32 rho = t ? (__brev(kappa) >> (32 - t)) : 0u;
      u64 v = sm[phys((int)rho * W + col)];
      const u64 k1 = (tile << w) + col;
      const u64 go = k1 + ((u64)kappa << r0);
      if (do_scale && !p.scale_on_load) v = gl::mul(v, scale_factor(p, go));
      if (p.canon_out) v = gl::canon(v);
      dst[go] = v;
    }
  }
}

// Serial fallback for tiny transforms (log_n < 4): one thread per column, the reference network verbatim.
__global__ void ntt_small_kernel(u64* data, u64 col_stride, u32 n_cols, int log_n, const u64* __restrict__ tab,
                                 u64 coset_or_inv, u64 n_inv, int inverse) {
  const u32 c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_cols) return;
  u64* a = data + (u64)c * col_stride;
  const int n = 1 << log_n;
  u64 x[8];
  for (int i = 0; i < n; i++) x[i] = gl::canon(a[i]);
  if (!inverse && coset_or_inv != 1) {
    u64 s = 1;
    for (int i = 0; i < n; i++) {
      x[i] = gl::mul(x[i], s);
      s = gl::mul(s, coset_or_inv);
    }
  }
  int pairs = n / 2, groups = 1, dist = n / 2;
  while (groups < n) {
    for (int k = 0; k < groups; k++) {
      const u64 s = tab[k];
      for (int j = k * pairs * 2; j < k * pairs * 2 + pairs; j++) {
        const u64 u = x[j], v = gl::mul(x[j + dist], s);
        x[j + dist] = gl::canon(gl::sub(u, v));
        x[j] = gl::canon(gl::add(u, v));
      }
    }
    pairs /= 2;
    groups *= 2;
    dist /= 2;
  }
  if (inverse) {
    u64 y[8];
    for (int i = 0; i < n; i++) y[log_n ? (__brev((u32)i) >> (32 - log_n)) : 0] = x[i];
    u64 s = n_inv;
    for (int i = 0; i < n; i++) {
      x[i] = gl::mul(y[i], s);
      s = gl::mul(s, coset_or_inv);  // coset^-1
    }
  }
  for (int i = 0; i < n; i++) a[i] = gl::canon(x[i]);
}

struct PowSquares {
  u64 sq[33];  // sq[b] = w^(2^b)
};

// tab[k] = w^bitrev_bits(k)
__global__ void twiddle_table_kernel(u64* tab, u32 count, int bits, PowSquares ps) {
  const u32 k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= count) return;
  const u32 e = bits ? (__brev(k) >> (32 - bits)) : 0u;
  u64 r = 1;
  for (int b = 0; b < bits; b++)
    if ((e >> b) & 1) r = gl::mul(r, ps.sq[b]);
  tab[k] = gl::canon(r);
}

// out[i] = scale * base^i
__global__ void pow_table_kernel(u64* out, u32 count, int bits, PowSquares ps, u64 scale) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  u64 r = scale;
  for (int b = 0; b < bits; b++)
    if ((i >> b) & 1) r = gl::mul(r, ps.sq[b]);
  out[i] = gl::canon(r);
}

// tw[2^r + G] = tab[G] * c^(2^(log_n - r - 1)) for r < log_n, G < 2^r (tw[0] is not read); ps.sq[b] = c^(2^b)
__global__ void twist_table_kernel(u64* tw, u32 count, int log_n, const u64* __restrict__ tab, PowSquares ps) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  if (i == 0) {
    tw[0] = 0;
    return;
  }
  const int r = 31 - __clz(i);
  tw[i] = gl::canon(gl::mul(__ldg(tab + (i - (1u << r))), ps.sq[log_n - r - 1]));
}

__global__ void bitreverse_kernel(u64* data, u64 col_stride, int log_n) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (1ull << log_n)) return;
  u64* a = data + (u64)blockIdx.y * col_stride;
  const u64 j = __brevll(i) >> (64 - log_n);
  if (i < j) {
    const u64 t = a[i];
    a[i] = a[j];
    a[j] = t;
  }
}

// ------------------------------------------------------------------------------------------------ host side

int32_t ensure_scratch(bj_ctx* ctx, size_t bytes) {
  if (ctx->scratch_bytes >= bytes) return BJ_OK;
  if (ctx->scratch) {
    BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    BJ_CUDA(ctx, cudaFree(ctx->scratch));
    ctx->scratch = nullptr;
    ctx->scratch_bytes = 0;
  }
  cudaError_t e = cudaMalloc(&ctx->scratch, bytes);
  if (e != cudaSuccess) {
    cudaGetLastError();
    BJ_FAIL(ctx, BJ_ERR_OOM, "scratch allocation failed");
  }
  ctx->scratch_bytes = bytes;
  return BJ_OK;
}

static PowSquares make_squares(u64 w) {
  PowSquares ps;
  for (int b = 0; b < 33; b++) {
    ps.sq[b] = w;
    w = gl::sqr(w);
  }
  return ps;
}

// bytes of the n-entry tables the owner's caches hold: the expanded coset powers of pow_cache and the twisted tables
static size_t cached_full_bytes(const bj_ctx* owner) {
  size_t b = 0;
  for (const auto& e : owner->pow_cache)
    if (e.full) b += sizeof(u64) << e.log_n;
  for (const auto& e : owner->twist_cache) b += sizeof(u64) << e.log_n;
  return b;
}

// a parent whose lanes are all gone frees the tables it retired while they lived.  Called on the parent's own thread under its
// tables_mu, after its stream has drained: no lane is left to read them (bj_ctx_destroy synchronised each lane's stream) and
// the parent's earlier kernels are done.  The full-table budget is then recounted from the caches.
static int32_t release_retired(bj_ctx* owner) {
  if (owner->tables_retired.empty() || owner->lanes.load() > 0) return BJ_OK;
  BJ_CUDA(owner, cudaStreamSynchronize(owner->stream));
  for (void* p : owner->tables_retired) cudaFree(p);
  owner->tables_retired.clear();
  owner->pow_full_bytes = cached_full_bytes(owner);
  return BJ_OK;
}

int32_t ensure_twiddles(bj_ctx* ctx, int log_n) {
  if (log_n < 1) log_n = 1;
  if (log_n > 32) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "log_n > 32 (two-adicity of the field)");
  if (ctx->tw_log >= log_n) return BJ_OK;
  if (ctx->parent && !ctx->own_twiddles) {  // a lane: view the parent's pair if it is long enough (ctx.hpp)
    bj_ctx* p = ctx->parent;
    std::lock_guard<std::mutex> lock(p->tables_mu);
    if (p->tw_log >= log_n) {
      ctx->tw_fwd = p->tw_fwd;
      ctx->tw_inv = p->tw_inv;
      ctx->tw_log = p->tw_log;
      return BJ_OK;
    }
    ctx->tw_fwd = ctx->tw_inv = nullptr;  // else a private pair below
    ctx->tw_log = 0;
    ctx->own_twiddles = true;
  }
  std::unique_lock<std::mutex> lock(ctx->tables_mu, std::defer_lock);
  if (!ctx->parent) {  // lanes read the pair under this lock
    lock.lock();
    BJ_TRY(release_retired(ctx));
  }
  // grow: tables of 2^(log_n-1) entries, tab[k] = w_{2^log_n}^{bitrev_{log_n-1}(k)} (prefix-stable)
  if (ctx->tw_fwd) {
    BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (ctx->lanes.load() > 0) {  // a lane may still read the old pair
      ctx->tables_retired.push_back(ctx->tw_fwd);
      ctx->tables_retired.push_back(ctx->tw_inv);
    } else {
      cudaFree(ctx->tw_fwd);
      cudaFree(ctx->tw_inv);
    }
    ctx->tw_fwd = ctx->tw_inv = nullptr;
    ctx->tw_log = 0;
  }
  const u32 count = 1u << (log_n - 1);
  u64 *fwd = nullptr, *inv = nullptr;
  BJ_CUDA(ctx, cudaMalloc(&fwd, sizeof(u64) * count));
  BJ_CUDA(ctx, cudaMalloc(&inv, sizeof(u64) * count));
  const u64 w = gl::omega(log_n);
  const u32 blocks = (count + 255) / 256;
  twiddle_table_kernel<<<blocks, 256, 0, ctx->stream>>>(fwd, count, log_n - 1, make_squares(w));
  BJ_LAUNCH_CHECK(ctx);
  twiddle_table_kernel<<<blocks, 256, 0, ctx->stream>>>(inv, count, log_n - 1, make_squares(gl::inv(w)));
  BJ_LAUNCH_CHECK(ctx);
  if (ctx->lanes.load() > 0) BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // complete before a lane can view it
  ctx->tw_fwd = fwd;
  ctx->tw_inv = inv;
  ctx->tw_log = log_n;
  return BJ_OK;
}

// full[i] = lo[i & mask] * hi[i >> split]
__global__ void __launch_bounds__(256) pow_full_kernel(u64* __restrict__ full, u64 n, const u64* __restrict__ lo,
                                                        const u64* __restrict__ hi, int split) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  full[i] = gl::mul(__ldg(lo + (i & ((1ull << split) - 1))), __ldg(hi + (i >> split)));
}

// c^i tables for i < 2^log_n: c^i = lo[i & mask] * hi[i >> split], hi pre-multiplied by `scale`; plus the expanded table
// `full` (one load + one multiplication per element in the pass kernels instead of two + two) while the context's
// budget lasts - the pass kernels are meant to be ALU-bound rather than HBM-bound, so 8 more bytes per element of
// (mostly L2-resident, shared by all columns) traffic are cheaper than 25 more instructions.
static constexpr size_t POW_FULL_BUDGET = (size_t)3 << 30;
static int32_t get_pow_tables(bj_ctx* ctx, u64 c, int log_n, u64 scale, PowTab* out) {
  // a lane's tables are its parent's cache, built by whichever context misses first (ctx.hpp); the kernels run on ctx's stream
  bj_ctx* owner = ctx->parent ? ctx->parent : ctx;
  std::lock_guard<std::mutex> lock(owner->tables_mu);
  if (owner == ctx) BJ_TRY(release_retired(ctx));
  for (auto& e : owner->pow_cache)
    if (e.coset == c && e.log_n == log_n && e.scale == scale) {
      *out = e;
      return BJ_OK;
    }
  const bool shared = owner->lanes.load() > 0;
  if (owner->pow_cache.size() >= 64) {  // bounded cache: drop everything (tables are cheap to rebuild)
    BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (auto& e : owner->pow_cache) {
      if (shared) {  // a lane may still read them
        owner->tables_retired.insert(owner->tables_retired.end(), {(void*)e.lo, (void*)e.hi});
        if (e.full) owner->tables_retired.push_back(e.full);
        continue;
      }
      cudaFree(e.lo);
      cudaFree(e.hi);
      if (e.full) cudaFree(e.full);
    }
    owner->pow_cache.clear();
    if (!shared) owner->pow_full_bytes = cached_full_bytes(owner);  // retired full tables count against the budget until release_retired
  }
  PowTab pt;
  pt.coset = c;
  pt.log_n = log_n;
  pt.scale = scale;
  pt.split = log_n / 2;
  const u32 nlo = 1u << pt.split, nhi = 1u << (log_n - pt.split);
  BJ_CUDA(ctx, cudaMalloc(&pt.lo, sizeof(u64) * nlo));
  BJ_CUDA(ctx, cudaMalloc(&pt.hi, sizeof(u64) * nhi));
  pow_table_kernel<<<(nlo + 255) / 256, 256, 0, ctx->stream>>>(pt.lo, nlo, pt.split, make_squares(c), 1);
  BJ_LAUNCH_CHECK(ctx);
  const u64 chi = gl::pow(c, 1ull << pt.split);
  pow_table_kernel<<<(nhi + 255) / 256, 256, 0, ctx->stream>>>(pt.hi, nhi, log_n - pt.split, make_squares(chi),
                                                                gl::canon(scale));
  BJ_LAUNCH_CHECK(ctx);
  pt.full = nullptr;
  const size_t full_bytes = sizeof(u64) << log_n;
  if (ctx->ntt_full_pow && log_n >= 8 && owner->pow_full_bytes + full_bytes <= POW_FULL_BUDGET &&
      cudaMalloc(&pt.full, full_bytes) == cudaSuccess) {
    const u64 n = 1ull << log_n;
    pow_full_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(pt.full, n, pt.lo, pt.hi, pt.split);
    BJ_LAUNCH_CHECK(ctx);
    owner->pow_full_bytes += full_bytes;
  } else {
    cudaGetLastError();
    pt.full = nullptr;
  }
  if (shared) BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // complete before another stream can read it
  owner->pow_cache.push_back(pt);
  *out = pt;
  return BJ_OK;
}

int32_t get_pow_tables_public(bj_ctx* ctx, u64 c, int log_n, u64 scale, PowTab* out) { return get_pow_tables(ctx, c, log_n, scale, out); }

// The forward transform on the coset c w^k evaluates a mod (X^n - c^n): round r splits X^(n/2^r) - c^(n/2^r) w_G into
// X^(n/2^(r+1)) -+ c^(n/2^(r+1)) tab[G], so the coset folds into the twiddles, tab_c[2^r + G] = tab[G] c^(2^(log_n - r - 1)),
// and the outputs are the same points in the same bit-reversed order with no per-element scaling.  One table of 2^log_n
// entries per (c, log_n), cached on the owner context with the rules of the coset-power tables (ctx.hpp) and counted against
// their budget; *out = nullptr when the budget is spent, and the caller scales on load instead.  ctx's twiddles must cover
// log_n (ensure_twiddles).
// The price is the front pass's FIRST stage (group 0's twiddle is no longer 1): 0.5-0.94 multiplications per element against
// the 1 multiplication and 8-byte table read of the scale.  From 2^13 on (multi-pass plans) that pays; a one-pass transform
// up to 2^12 keeps scaling on load, where the two are about even and a table per (coset, size) would only fill the cache.
static constexpr int TWIST_MIN_LOG = 13;
static int32_t get_twist_table(bj_ctx* ctx, u64 c, int log_n, const u64** out) {
  *out = nullptr;
  bj_ctx* owner = ctx->parent ? ctx->parent : ctx;
  std::lock_guard<std::mutex> lock(owner->tables_mu);
  if (owner == ctx) BJ_TRY(release_retired(ctx));
  for (const auto& e : owner->twist_cache)
    if (e.coset == c && e.log_n == log_n) {
      *out = e.tab;
      return BJ_OK;
    }
  const bool shared = owner->lanes.load() > 0;
  if (owner->twist_cache.size() >= 64) {  // bounded cache, as get_pow_tables
    BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (auto& e : owner->twist_cache) {
      if (shared) owner->tables_retired.push_back(e.tab);
      else cudaFree(e.tab);
    }
    owner->twist_cache.clear();
    if (!shared) owner->pow_full_bytes = cached_full_bytes(owner);
  }
  const size_t bytes = sizeof(u64) << log_n;
  TwistTab tt{c, log_n, nullptr};
  if (owner->pow_full_bytes + bytes > POW_FULL_BUDGET || cudaMalloc(&tt.tab, bytes) != cudaSuccess) {
    cudaGetLastError();
    return BJ_OK;
  }
  const u32 count = 1u << log_n;
  twist_table_kernel<<<(count + 255) / 256, 256, 0, ctx->stream>>>(tt.tab, count, log_n, ctx->tw_fwd, make_squares(c));
  BJ_LAUNCH_CHECK(ctx);
  owner->pow_full_bytes += bytes;
  if (shared) BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // complete before another stream can read it
  owner->twist_cache.push_back(tt);
  *out = tt.tab;
  return BJ_OK;
}

// The largest plan of any allowed tile setting (BJ_NTT_MAX_TILE_LOG 8..14) up to log_n = 32: an inverse of 2^31 or 2^32
// with 2^8-value tiles takes 6 passes (tools/ntt_model.py enumerates them).
static constexpr int NTT_MAX_PASSES = 6;

struct Plan {
  int n_pass;
  int t[NTT_MAX_PASSES];
  int w[NTT_MAX_PASSES];
};

// false when the plan would need more than NTT_MAX_PASSES passes (pl->n_pass is set, the arrays are not)
static bool make_plan(const bj_ctx* ctx, int m, bool transpose_last, Plan* out) {
  Plan& pl = *out;
  pl = Plan{};
  const int MAXE = ctx->ntt_max_tile_log;
  if (m <= 12) {
    pl.n_pass = 1;
    pl.t[0] = m;
    pl.w[0] = 0;
    return true;
  }
  // tiles of at most 2^MAXE values (default 2^13 = 68 KB of shared memory -> 3 CTAs per SM); the transposing last pass
  // keeps at least 4 columns so that its stores are 32-byte segments
  const int TL = transpose_last ? MAXE - 2 : MAXE;
  const int TM = MAXE - 2;
  int t_last = std::min(TL, std::max((m + 1) / 2, m - 10));
  int rest = m - t_last;
  int n_front = (rest + TM - 1) / TM;
  pl.n_pass = n_front + 1;
  if (pl.n_pass > NTT_MAX_PASSES) return false;
  int r0 = 0;
  for (int i = 0; i < n_front; i++) {
    int ti = rest / (n_front - i);
    rest -= ti;
    int wi = ctx->ntt_pass1_w >= 0 ? ctx->ntt_pass1_w : std::max(2, std::min(5, MAXE - ti));
    wi = std::min(wi, MAXE - ti);
    wi = std::min(wi, m - r0 - ti);
    if (ti + wi < 4) wi = 4 - ti;
    pl.t[i] = ti;
    pl.w[i] = wi;
    r0 += ti;
  }
  pl.t[n_front] = t_last;
  pl.w[n_front] = transpose_last ? std::min(std::min(MAXE - t_last, 5), r0) : 0;
  return true;
}

// grid.y limit: a batch of more columns is launched in slices of at most this many columns
static constexpr u32 MAX_GRID_Y = 65535;

// Launches `fn` over the batch in column slices of at most MAX_GRID_Y columns, each slice with src / dst moved to its
// first column.  Even strides keep the 16-byte alignment the specialised kernels need.
template <typename F>
static int32_t launch_column_slices(bj_ctx* ctx, const NttPass& p, u32 n_cols, F&& fn) {
  for (u32 c0 = 0; c0 < n_cols; c0 += std::min(MAX_GRID_Y, n_cols - c0)) {
    NttPass ps = p;
    ps.src = p.src + (u64)c0 * p.src_col_stride;
    ps.dst = p.dst + (u64)c0 * p.dst_col_stride;
    fn(ps, std::min(MAX_GRID_Y, n_cols - c0));
    BJ_LAUNCH_CHECK(ctx);
  }
  return BJ_OK;
}

static int32_t launch_pass(bj_ctx* ctx, const NttPass& p, u32 n_cols) {
  const int LOG_E = p.t + p.w;
  const u64 tiles = p.kind == PASS_TILE ? (1ull << (p.log_n - p.t - p.w)) : (1ull << (p.r0 - p.w));
  if (tiles > 0x7fffffffull) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "grid too large");
  // specialised kernel when one is instantiated for this tile shape and the buffers allow 128-bit accesses
  V2Launch v2;
  const bool aligned = ((((uintptr_t)p.src | (uintptr_t)p.dst) & 15) == 0) && ((p.src_col_stride | p.dst_col_stride) & 1) == 0;
  // the specialised one-column tiles (w = 0) move pairs of adjacent rows, so they serve contiguous (last) passes only; a
  // front pass with w = 0 (BJ_NTT_PASS1_W=0) has strided rows and takes the generic kernel
  const bool v2_shape_ok = !(p.kind == PASS_TILE && p.w == 0 && p.log_n - p.r0 - p.t != 0);
  // experiment: bulk-copy (TMA) staged contiguous pass, BJ_NTT_BULK=1 (ntt_v2.cuh)
  const bool bulk_ok = ctx->ntt_bulk && aligned && p.kind == PASS_TILE && p.w == 0 && p.scale_mode == SCALE_NONE &&
                       p.log_n - p.r0 - p.t == 0 && ((p.src_col_stride | p.dst_col_stride) & 15) == 0;
  const bool bulk = ctx->ntt_use_v2 && aligned && v2_shape_ok && bulk_ok && v2_bulk_lookup(p.t, &v2);
  if (bulk || (ctx->ntt_use_v2 && aligned && v2_shape_ok && v2_lookup(p.t, p.w, p.kind, &v2))) {
    bool known = false;
    for (void* f : ctx->attr_done) known |= (f == (void*)v2.fn);
    if (!known) {
      BJ_CUDA(ctx, cudaFuncSetAttribute((const void*)v2.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
      BJ_CUDA(ctx, cudaFuncSetAttribute((const void*)v2.fn, cudaFuncAttributePreferredSharedMemoryCarveout,
                                        cudaSharedmemCarveoutMaxShared));
      ctx->attr_done.push_back((void*)v2.fn);
    }
    // Column-fastest order: block w is tile w / n_cols of column w % n_cols, so the same tile of every column runs back to
    // back and the tile's slices of the twiddle and coset-power tables come from DRAM once per batch instead of once per
    // column.  By default the contiguous last passes take it (twiddle slices, 1-2 % faster), and the front passes whose
    // coset-power table is larger than the L2 set-aside that pins it (from 2^22 on the H100, 6-9 % faster).  A front pass
    // whose table stays in L2 keeps the tile-fastest order: there neighbouring tiles of one column, which share DRAM pages,
    // running together is worth more (5-14 % slower otherwise).  BJ_NTT_COL_FASTEST = bit 0 front, bit 1 last forces it.
    const bool is_last = p.log_n - p.r0 - p.t == 0;
    bool col_fastest;
    if (ctx->ntt_col_fastest >= 0) {
      col_fastest = (ctx->ntt_col_fastest >> (is_last ? 1 : 0)) & 1;
    } else {
      const bool big_table = p.scale_mode == SCALE_FULL && (sizeof(u64) << p.log_n) > ctx->l2_persist_bytes;
      col_fastest = is_last || big_table;
    }
    if (p.kind == PASS_TILE && !bulk && col_fastest && tiles * n_cols <= 0x7fffffffull) {
      NttPass ps = p;
      ps.n_cols = n_cols;
      v2.fn<<<(unsigned)(tiles * n_cols), v2.threads, v2.smem, ctx->stream>>>(ps);
      BJ_LAUNCH_CHECK(ctx);
      return BJ_OK;
    }
    return launch_column_slices(ctx, p, n_cols, [&](const NttPass& ps, u32 cols) {
      v2.fn<<<dim3((unsigned)tiles, cols, 1), v2.threads, v2.smem, ctx->stream>>>(ps);
    });
  }
  const int threads = std::max(32, std::min(512, (1 << LOG_E) >> 4));
  const size_t smem = sizeof(u64) * ((size_t)(1 << LOG_E) + ((size_t)(1 << LOG_E) >> 4) + 1);
  if (!ctx->ntt_attr_set) {
    BJ_CUDA(ctx, cudaFuncSetAttribute(ntt_pass_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    BJ_CUDA(ctx, cudaFuncSetAttribute(ntt_pass_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                                      cudaSharedmemCarveoutMaxShared));
    ctx->ntt_attr_set = true;
  }
  return launch_column_slices(ctx, p, n_cols, [&](const NttPass& ps, u32 cols) {
    ntt_pass_kernel<<<dim3((unsigned)tiles, cols, 1), threads, smem, ctx->stream>>>(ps);
  });
}

// One batched transform.  src may equal dst for forward; the natural->natural inverse with more than one
// pass needs `scratch` (n_cols * n elements) because its last pass cannot run in place.
//   forward: the coset's twisted twiddles (get_twist_table), or where there are none coset scaling on load of the first
//   pass; inverse: n^-1 coset^-i on the store of the last pass.
static int32_t run_transform(bj_ctx* ctx, const u64* src, u64 src_stride, u64* dst, u64 dst_stride, int m,
                             u32 n_cols, u64 coset, bool inverse, u64* scratch, u64 scratch_stride) {
  BJ_TRY(ensure_twiddles(ctx, m));
  const u64* tab = inverse ? ctx->tw_inv : ctx->tw_fwd;
  coset = gl::canon(coset);
  if (m < 4) {
    if (src != dst || src_stride != dst_stride) {
      for (u32 c = 0; c < n_cols; c++)
        BJ_CUDA(ctx, cudaMemcpyAsync(dst + c * dst_stride, src + c * src_stride, sizeof(u64) << m,
                                     cudaMemcpyDeviceToDevice, ctx->stream));
    }
    const u64 n_inv = gl::inv((u64)1 << m);  // n == 1: identity, as in the reference (fft/mod.rs:478)
    ntt_small_kernel<<<(n_cols + 63) / 64, 64, 0, ctx->stream>>>(dst, dst_stride, n_cols, m, tab,
                                                                 inverse ? gl::inv(coset) : coset, n_inv, inverse);
    BJ_LAUNCH_CHECK(ctx);
    return BJ_OK;
  }
  Plan pl;
  if (!make_plan(ctx, m, inverse, &pl)) BJ_FAIL(ctx, BJ_ERR_UNSUPPORTED, "NTT plan needs more passes than NTT_MAX_PASSES");
  PowTab pt{};
  int scale_mode = SCALE_NONE;
  u64 scale_const = 1;
  const u64* twist = nullptr;
  if (!inverse) {
    // a coset from 2^TWIST_MIN_LOG on: the coset's twisted twiddles (get_twist_table), no scaling; while their budget lasts
    if (coset != 1 && ctx->ntt_twist && ctx->ntt_full_pow && m >= TWIST_MIN_LOG) BJ_TRY(get_twist_table(ctx, coset, m, &twist));
    if (coset != 1 && !twist) {
      BJ_TRY(get_pow_tables(ctx, coset, m, 1, &pt));
      scale_mode = SCALE_POW;
    }
  } else {
    const u64 n_inv = gl::inv((u64)1 << m);
    if (coset != 1) {
      BJ_TRY(get_pow_tables(ctx, gl::inv(coset), m, n_inv, &pt));
      scale_mode = SCALE_POW;
    } else {
      scale_mode = SCALE_CONST;
      scale_const = n_inv;
    }
  }
  const u64* cur_src = src;
  u64 cur_src_stride = src_stride;
  int r0 = 0;
  for (int i = 0; i < pl.n_pass; i++) {
    const bool first = i == 0, last = i == pl.n_pass - 1;
    NttPass p{};
    p.tab = twist ? twist : tab;
    p.tw_prefix = twist ? 1u << r0 : 0u;
    p.log_n = m;
    p.r0 = r0;
    p.t = pl.t[i];
    p.w = pl.w[i];
    p.kind = (inverse && last) ? PASS_TRANSPOSE_LAST : PASS_TILE;
    p.src = cur_src;
    p.src_col_stride = cur_src_stride;
    if (inverse && pl.n_pass > 1) {
      // ping-pong so that the (out-of-place) last pass lands in dst
      const int remaining = pl.n_pass - 1 - i;  // passes after this one
      const bool to_dst = (remaining % 2) == 0;
      p.dst = to_dst ? dst : scratch;
      p.dst_col_stride = to_dst ? dst_stride : scratch_stride;
      if (last && p.dst == p.src) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "internal: in-place transpose pass");
    } else {
      p.dst = dst;
      p.dst_col_stride = dst_stride;
    }
    p.scale_mode = SCALE_NONE;
    if (!inverse && first && scale_mode != SCALE_NONE) {
      p.scale_mode = scale_mode;
      p.scale_on_load = 1;
    }
    if (inverse && last) {
      p.scale_mode = scale_mode;
      p.scale_on_load = 0;
      p.scale_const = scale_const;
    }
    p.pw_lo = pt.lo;
    p.pw_hi = pt.hi;
    p.pw_split = pt.split;
    p.pw_full = pt.full;
    if (p.scale_mode == SCALE_POW && pt.full) p.scale_mode = SCALE_FULL;
    p.canon_out = last ? 1 : 0;
    // the coset-power table (8 bytes per element of one column, shared by every column of the batch) is the one operand of the
    // scaled pass that is re-read: pin it in L2 (persisting access-policy window) while the streamed data is marked streaming,
    // so that the batch does not evict it and the first pass reads it from DRAM once.  BJ_NTT_L2_PERSIST=0 disables.
    // A table larger than the set-aside is pinned in part (hitRatio = set-aside / window), so that it does not thrash.
    const bool pin = ctx->ntt_l2_persist && p.scale_mode == SCALE_FULL && n_cols > 1 && ctx->l2_persist_bytes && ctx->l2_window_max;
    if (pin) {
      if (!ctx->l2_limit_set) {
        cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, ctx->l2_persist_bytes);
        cudaGetLastError();
        ctx->l2_limit_set = true;
      }
      cudaStreamAttrValue av = {};
      av.accessPolicyWindow.base_ptr = (void*)p.pw_full;
      av.accessPolicyWindow.num_bytes = std::min<size_t>(sizeof(u64) << m, ctx->l2_window_max);
      av.accessPolicyWindow.hitRatio = std::min(1.0f, (float)ctx->l2_persist_bytes / (float)av.accessPolicyWindow.num_bytes);
      av.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
      av.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
      if (cudaStreamSetAttribute(ctx->stream, cudaStreamAttributeAccessPolicyWindow, &av) != cudaSuccess) cudaGetLastError();
    }
    const int32_t st_pass = launch_pass(ctx, p, n_cols);
    if (pin) {
      cudaStreamAttrValue av = {};
      av.accessPolicyWindow.num_bytes = 0;
      if (cudaStreamSetAttribute(ctx->stream, cudaStreamAttributeAccessPolicyWindow, &av) != cudaSuccess) cudaGetLastError();
    }
    BJ_TRY(st_pass);
    cur_src = p.dst;
    cur_src_stride = p.dst_col_stride;
    r0 += pl.t[i];
  }
  return BJ_OK;
}

static bool inverse_needs_scratch(const bj_ctx* ctx, int m) {
  Plan pl;
  make_plan(ctx, m, true, &pl);  // n_pass is set even when the plan is refused; run_transform reports that
  return m >= 4 && pl.n_pass > 1;
}

}  // namespace bj

using namespace bj;

extern "C" {

int32_t bj_twiddles(bj_ctx* ctx, uint32_t log_n, int32_t inverse, uint64_t* d_out) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || !d_out || log_n < 1 || log_n > 32) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_twiddles: bad argument");
  BJ_TRY(ensure_twiddles(ctx, (int)log_n));
  BJ_CUDA(ctx, cudaMemcpyAsync(d_out, inverse ? ctx->tw_inv : ctx->tw_fwd, sizeof(u64) << (log_n - 1),
                               cudaMemcpyDeviceToDevice, ctx->stream));
  return BJ_OK;
}

int32_t bj_ntt_natural_to_bitreversed(bj_ctx* ctx, uint64_t* d_data, uint32_t log_n, uint32_t n_cols,
                                      uint64_t col_stride, uint64_t coset) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || !d_data || log_n > 32 || col_stride < (1ull << log_n))
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_ntt_natural_to_bitreversed: bad argument");
  if (n_cols == 0) return BJ_OK;
  return run_transform(ctx, (const u64*)d_data, col_stride, (u64*)d_data, col_stride, (int)log_n, n_cols, coset,
                       false, nullptr, 0);
}

int32_t bj_intt_natural_to_natural(bj_ctx* ctx, uint64_t* d_data, uint32_t log_n, uint32_t n_cols,
                                   uint64_t col_stride, uint64_t coset) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || !d_data || log_n > 32 || col_stride < (1ull << log_n))
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_intt_natural_to_natural: bad argument");
  if (n_cols == 0) return BJ_OK;
  if (gl::canon(coset) == 0) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "coset must be invertible");
  const u64 n = 1ull << log_n;
  if (!inverse_needs_scratch(ctx, (int)log_n))
    return run_transform(ctx, (const u64*)d_data, col_stride, (u64*)d_data, col_stride, (int)log_n, n_cols, coset,
                         true, nullptr, 0);
  // chunk the batch so the scratch stays bounded (<= 1 GiB)
  u32 chunk = (u32)std::max<u64>(1, std::min<u64>(n_cols, (1ull << 27) / n));
  BJ_TRY(ensure_scratch(ctx, sizeof(u64) * n * chunk));
  for (u32 c0 = 0; c0 < n_cols; c0 += chunk) {
    const u32 cnt = std::min(chunk, n_cols - c0);
    u64* d = (u64*)d_data + (u64)c0 * col_stride;
    BJ_TRY(run_transform(ctx, d, col_stride, d, col_stride, (int)log_n, cnt, coset, true, (u64*)ctx->scratch, n));
  }
  return BJ_OK;
}

int32_t bj_bitreverse(bj_ctx* ctx, uint64_t* d_data, uint32_t log_n, uint32_t n_cols, uint64_t col_stride) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || !d_data || log_n > 40) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_bitreverse: bad argument");
  if (n_cols == 0 || log_n == 0) return BJ_OK;
  const u64 n = 1ull << log_n;
  if ((n + 255) / 256 > 0x7fffffffull) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_bitreverse: grid too large");
  for (u32 c0 = 0; c0 < n_cols; c0 += std::min(MAX_GRID_Y, n_cols - c0)) {  // grid.y slices, as in launch_pass
    dim3 grid((unsigned)((n + 255) / 256), std::min(MAX_GRID_Y, n_cols - c0));
    bitreverse_kernel<<<grid, 256, 0, ctx->stream>>>((u64*)d_data + (u64)c0 * col_stride, col_stride, (int)log_n);
    BJ_LAUNCH_CHECK(ctx);
  }
  return BJ_OK;
}

}  // extern "C"

namespace bj {

struct UnitPowers {
  u64 v[8];  // sigma^(m * n / B), m < B
};

// Fold of a coefficient vector onto a row block: on the points of a unit with shift sigma, x^(n/B) = sigma^(n/B), so
// f(x) = sum_{k < n/B} b_k x^k with b_k = sum_{m < B} sigma^(m n / B) a_{k + m n / B}.
// b[c][k] for c < cnt columns (a: column stride a_stride, b: column stride b_stride).
__global__ void __launch_bounds__(256) lde_unit_fold_kernel(const u64* __restrict__ a, u64 a_stride, u64* __restrict__ b, u64 b_stride,
                                                             int log_nb, u32 n_blocks, u64 total, UnitPowers pw) {
  const u64 idx = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const u64 c = idx >> log_nb, k = idx & ((1ull << log_nb) - 1);
  const u64* src = a + c * a_stride + k;
  u64 acc = gl::canon(src[0]);
  for (u32 m = 1; m < n_blocks; m++) acc = gl::add(acc, gl::canon(gl::mul(src[(u64)m << log_nb], pw.v[m])));  // any u64 input
  b[c * b_stride + k] = gl::canon(acc);
}

// bj_lde, and with next_row the LDE of f(w_n x) (every unit shift times w_n, same row order).  cosets = {k0, k1} on an
// unsharded context: only the cosets [k0, k1) (bj_lde_cosets), d_out [col][k1 - k0][row]
struct CosetRange {
  u64 k0, k1;
};
static int32_t lde_impl(bj_ctx* ctx, const uint64_t* d_in, uint64_t in_col_stride, uint64_t* d_out, uint32_t log_n, uint32_t log_lde,
                        uint32_t n_cols, int32_t from_monomials, bool next_row, const CosetRange* cosets = nullptr) {
  if (!ctx || !d_in || !d_out || log_n + log_lde > 32 || in_col_stride < (1ull << log_n))
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_lde: bad argument");
  if (n_cols == 0) return BJ_OK;
  const u64 n = 1ull << log_n, L = 1ull << log_lde;
  // a shard owns the units u = first (mod world) of ANY factor with at least `world` units (the first L cosets of a larger
  // domain are the factor-L domain), so the quotient's wider evaluation domain shards the same way as the committed one
  const u32 s = ctx->shard.log_split;
  if (ctx->shard.log_stride > log_lde + s)
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_lde: LDE factor smaller than the number of shards");
  if (s && log_n <= s) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_lde: fewer than 2 rows per row block of the domain shard");
  const u64 w_row = next_row ? gl::omega(log_n) : 1;
  if (s) {
    // split shard: per owned unit, fold the monomials onto the row block (straight into the unit's output slot), then one
    // in-place forward transform of size n / B on the unit's shift
    const int mb = (int)(log_n - s);
    const u64 nb = 1ull << mb, U_loc = ctx->shard.local_units(L);
    u32 chunk = (u32)std::max<u64>(1, std::min<u64>(n_cols, (1ull << 26) / n));
    const bool two_bufs = !from_monomials && inverse_needs_scratch(ctx, (int)log_n);
    for (u32 c0 = 0; c0 < n_cols; c0 += chunk) {
      const u32 cnt = std::min(chunk, n_cols - c0);
      const u64* mono = (const u64*)d_in + (u64)c0 * in_col_stride;
      u64 mono_stride = in_col_stride;
      if (!from_monomials) {
        BJ_TRY(ensure_scratch(ctx, sizeof(u64) * n * chunk * (two_bufs ? 2 : 1)));
        u64* mbuf = (u64*)ctx->scratch;
        BJ_TRY(run_transform(ctx, mono, in_col_stride, mbuf, n, (int)log_n, cnt, 1, true, two_bufs ? mbuf + n * chunk : nullptr, n));
        mono = mbuf;
        mono_stride = n;
      }
      for (u64 k = 0; k < U_loc; k++) {
        const u64 sigma = gl::mul(ctx->shard.unit_shift(ctx->shard.global_unit(k), log_n, log_lde), w_row);
        UnitPowers pw{};
        const u64 sb = gl::pow(sigma, nb);
        pw.v[0] = 1;
        for (u32 i = 1; i < (1u << s); i++) pw.v[i] = gl::mul(pw.v[i - 1], sb);
        u64* out = (u64*)d_out + ((u64)c0 * U_loc + k) * nb;
        const u64 total = (u64)cnt << mb;
        lde_unit_fold_kernel<<<(unsigned)((total + 255) / 256), 256, 0, ctx->stream>>>(mono, mono_stride, out, nb * U_loc, mb, 1u << s, total, pw);
        BJ_LAUNCH_CHECK(ctx);
        BJ_TRY(run_transform(ctx, out, nb * U_loc, out, nb * U_loc, mb, cnt, sigma, false, nullptr, 0));
      }
    }
    return BJ_OK;
  }
  const u64 L_loc = ctx->shard.local_units(L);  // cosets owned by this context (all of them without a shard)
  const u64 k0 = cosets ? cosets->k0 : 0, k1 = cosets ? cosets->k1 : L_loc, n_out = k1 - k0;
  const int m = (int)log_n;
  // per chunk of columns: monomials (natural order) in scratch, then one forward transform per coset that
  // reads the monomials and writes straight into the coset's slot of d_out.
  const bool two_bufs = !from_monomials && inverse_needs_scratch(ctx, m);
  u32 chunk = (u32)std::max<u64>(1, std::min<u64>(n_cols, (1ull << 26) / n));
  for (u32 c0 = 0; c0 < n_cols; c0 += chunk) {
    const u32 cnt = std::min(chunk, n_cols - c0);
    const u64* in = (const u64*)d_in + (u64)c0 * in_col_stride;
    const u64* mono = in;
    u64 mono_stride = in_col_stride;
    if (!from_monomials) {
      BJ_TRY(ensure_scratch(ctx, sizeof(u64) * n * chunk * (two_bufs ? 2 : 1)));
      u64* mbuf = (u64*)ctx->scratch;
      u64* tmp = two_bufs ? mbuf + n * chunk : nullptr;
      BJ_TRY(run_transform(ctx, in, in_col_stride, mbuf, n, m, cnt, 1, true, tmp, n));
      mono = mbuf;
      mono_stride = n;
    }
    for (u64 k = k0; k < k1; k++) {
      u64 shift = ctx->shard.unit_shift(ctx->shard.global_unit(k), log_n, log_lde);  // the coset of local slot k
      if (next_row) shift = gl::mul(shift, w_row);
      u64* out = (u64*)d_out + ((u64)c0 * n_out + (k - k0)) * n;
      BJ_TRY(run_transform(ctx, mono, mono_stride, out, n * n_out, m, cnt, shift, false, nullptr, 0));
    }
  }
  return BJ_OK;
}

}  // namespace bj

extern "C" {

int32_t bj_lde(bj_ctx* ctx, const uint64_t* d_in, uint64_t in_col_stride, uint64_t* d_out, uint32_t log_n,
               uint32_t log_lde, uint32_t n_cols, int32_t from_monomials) {
  bj::DeviceGuard device_guard(ctx);
  return lde_impl(ctx, d_in, in_col_stride, d_out, log_n, log_lde, n_cols, from_monomials, false);
}

int32_t bj_lde_next_row(bj_ctx* ctx, const uint64_t* d_in, uint64_t in_col_stride, uint64_t* d_out, uint32_t log_n,
                        uint32_t log_lde, uint32_t n_cols, int32_t from_monomials) {
  bj::DeviceGuard device_guard(ctx);
  return lde_impl(ctx, d_in, in_col_stride, d_out, log_n, log_lde, n_cols, from_monomials, true);
}

// LDE onto the cosets [coset_begin, coset_end) of the factor-2^log_lde domain only (unsharded contexts): the same coset
// transforms as bj_lde, so every value is bit-identical to the matching slot of the full LDE.
int32_t bj_lde_cosets(bj_ctx* ctx, const uint64_t* d_in, uint64_t in_col_stride, uint64_t* d_out, uint32_t log_n, uint32_t log_lde,
                      uint32_t coset_begin, uint32_t coset_end, uint32_t n_cols, int32_t from_monomials) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || coset_begin >= coset_end || log_lde > 32 || coset_end > (1ull << log_lde)) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_lde_cosets: bad argument");
  if (ctx->shard.log_stride) BJ_FAIL(ctx, BJ_ERR_UNSUPPORTED, "bj_lde_cosets: not on a sharded context");
  const CosetRange r{coset_begin, coset_end};
  return lde_impl(ctx, d_in, in_col_stride, d_out, log_n, log_lde, n_cols, from_monomials, false, &r);
}

// Host-buffer entry points: the batch is cut into column chunks that flow through a 3-slot device ring, upload of chunk
// k+1, transform of chunk k and download of chunk k-1 overlapping on three streams (copy engines are full duplex).
// Overlap needs pinned host memory (bj_alloc_host_pinned / cudaHostRegister); pageable memory still works, serialised.
static int32_t host_pipeline(bj_ctx* ctx, uint64_t* h_data, uint32_t log_n, uint32_t n_cols, uint64_t coset, bool inverse) {
  if (!ctx || !h_data || log_n > 32) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "host transform: bad argument");
  if (n_cols == 0) return BJ_OK;
  const u64 n = 1ull << log_n;
  const size_t col_bytes = sizeof(u64) * n;
  // chunks of ~ntt_chunk_mb MiB (BJ_NTT_CHUNK_MB), at least one column: small enough that the un-overlapped first upload
  // and last download of a call stay short, large enough to keep the copy engines and the pass kernels efficient
  const u64 chunk_bytes = (u64)(ctx->ntt_chunk_mb > 0 ? ctx->ntt_chunk_mb : 64) << 20;
  u32 chunk_cols = (u32)std::max<u64>(1, std::min<u64>(n_cols, chunk_bytes / col_bytes));
  const u32 n_chunks = (n_cols + chunk_cols - 1) / chunk_cols;
  const int SLOTS = 3;
  if (!ctx->copy_streams_ready) {
    BJ_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->h2d_stream, cudaStreamNonBlocking));
    BJ_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->d2h_stream, cudaStreamNonBlocking));
    for (int i = 0; i < 3; i++) {
      BJ_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_up[i], cudaEventDisableTiming));
      BJ_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_done[i], cudaEventDisableTiming));
      BJ_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_down[i], cudaEventDisableTiming));
    }
    ctx->copy_streams_ready = true;
  }
  const size_t slot_bytes = col_bytes * chunk_cols;
  if (ctx->host_ring_bytes < slot_bytes * SLOTS) {
    if (ctx->host_ring) {
      BJ_CUDA(ctx, cudaDeviceSynchronize());
      cudaFree(ctx->host_ring);
      ctx->host_ring = nullptr;
      ctx->host_ring_bytes = 0;
    }
    if (cudaMalloc(&ctx->host_ring, slot_bytes * SLOTS) != cudaSuccess) {
      cudaGetLastError();
      BJ_FAIL(ctx, BJ_ERR_OOM, "host transform: device staging allocation failed");
    }
    ctx->host_ring_bytes = slot_bytes * SLOTS;
  }
  // the ring may still be in use by a previous call's downloads
  BJ_CUDA(ctx, cudaStreamSynchronize(ctx->d2h_stream));
  BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  int32_t st = BJ_OK;
  for (u32 k = 0; k < n_chunks && st == BJ_OK; k++) {
    const int slot = k % SLOTS;
    const u32 c0 = k * chunk_cols, cnt = std::min(chunk_cols, n_cols - c0);
    uint64_t* d = (uint64_t*)((char*)ctx->host_ring + slot_bytes * slot);
    uint64_t* h = h_data + (u64)c0 * n;
    if (k >= (u32)SLOTS) BJ_CUDA(ctx, cudaStreamWaitEvent(ctx->h2d_stream, ctx->ev_down[slot], 0));  // slot drained
    BJ_CUDA(ctx, cudaMemcpyAsync(d, h, col_bytes * cnt, cudaMemcpyHostToDevice, ctx->h2d_stream));
    BJ_CUDA(ctx, cudaEventRecord(ctx->ev_up[slot], ctx->h2d_stream));
    BJ_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_up[slot], 0));
    st = inverse ? bj_intt_natural_to_natural(ctx, d, log_n, cnt, n, coset)
                 : bj_ntt_natural_to_bitreversed(ctx, d, log_n, cnt, n, coset);
    if (st != BJ_OK) break;
    BJ_CUDA(ctx, cudaEventRecord(ctx->ev_done[slot], ctx->stream));
    BJ_CUDA(ctx, cudaStreamWaitEvent(ctx->d2h_stream, ctx->ev_done[slot], 0));
    BJ_CUDA(ctx, cudaMemcpyAsync(h, d, col_bytes * cnt, cudaMemcpyDeviceToHost, ctx->d2h_stream));
    BJ_CUDA(ctx, cudaEventRecord(ctx->ev_down[slot], ctx->d2h_stream));
  }
  cudaError_t e1 = cudaStreamSynchronize(ctx->d2h_stream);
  cudaError_t e2 = cudaStreamSynchronize(ctx->stream);
  if (st == BJ_OK && (e1 != cudaSuccess || e2 != cudaSuccess)) {
    ctx->last_error = std::string("host transform: ") + cudaGetErrorString(e1 != cudaSuccess ? e1 : e2);
    st = BJ_ERR_CUDA;
  }
  return st;
}

int32_t bj_ntt_natural_to_bitreversed_host(bj_ctx* ctx, uint64_t* h_data, uint32_t log_n, uint32_t n_cols,
                                           uint64_t coset) {
  bj::DeviceGuard device_guard(ctx);
  return host_pipeline(ctx, h_data, log_n, n_cols, coset, false);
}

int32_t bj_intt_natural_to_natural_host(bj_ctx* ctx, uint64_t* h_data, uint32_t log_n, uint32_t n_cols,
                                        uint64_t coset) {
  bj::DeviceGuard device_guard(ctx);
  if (ctx && gl::canon(coset) == 0) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "coset must be invertible");
  return host_pipeline(ctx, h_data, log_n, n_cols, coset, true);
}

}  // extern "C"
