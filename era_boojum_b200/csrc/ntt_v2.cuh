// Compile-time specialised NTT pass kernel (same algorithm and tile geometry as ntt_pass_kernel in ntt.cu, see the
// comment there): tile shape (T rows bits, W column bits) and pass kind are template parameters, so every
// shared-memory offset, stage width and stage position folds into immediates; global traffic uses 128-bit accesses;
// the 2^q twiddles of round q are fetched as 128-bit vectors.  Selected by launch_pass() when an instantiation exists
// and the buffers are 16-byte aligned with even strides; otherwise the generic kernel runs.
#pragma once
#include "ntt.cuh"

// Pipe balance of the butterfly (A/B builds):
//   BJ_NTT_ADD_ALU = 1: the sum's wrap correction on the ALU pipe (gl::add_alu) instead of the FMA pipe (gl::add); 0 is the
//                       default;
//   BJ_NTT_SUB_FMA = 1: the difference's borrow correction as multiply-adds (gl::sub_fma) instead of the sub chain (gl::sub).
#ifndef BJ_NTT_ADD_ALU
#define BJ_NTT_ADD_ALU 0
#endif
#ifndef BJ_NTT_SUB_FMA
#define BJ_NTT_SUB_FMA 0
#endif

namespace bj {

using gl::u32;

template <int T, int W>
struct V2Cfg {
  static constexpr int LOG_E = T + W;
  static constexpr int E = 1 << LOG_E;
  static constexpr int NVT = E >> 4;  // virtual threads of 16 values
  static constexpr int THREADS = NVT < 32 ? 32 : (NVT > 256 ? 256 : NVT);
  static constexpr int RS0 = (T & 3) ? (T & 3) : 4;  // bits of the first (short) stage
  static constexpr int NSTAGES = (T + 3) / 4;
  static constexpr size_t SMEM = sizeof(u64) * (size_t)(E + (E >> 4) + 2);
  // (12,0) is the only shape ptxas takes past 64 registers (66 -> 3 instead of 4 CTAs per SM); the others sit at 63-64
  static constexpr bool CAP_REGS = (T == 12 && W == 0);
};

__device__ __forceinline__ int v2_phys(int e) { return e + (e >> 4); }

__device__ __forceinline__ u64 v2_scale(const NttPass& p, u64 idx) {
  if (p.scale_mode == SCALE_CONST) return p.scale_const;
  if (p.scale_mode == SCALE_FULL) return __ldg(p.pw_full + idx);
  const u64 lo = __ldg(p.pw_lo + (idx & ((1ull << p.pw_split) - 1)));
  const u64 hi = __ldg(p.pw_hi + (idx >> p.pw_split));
  return gl::mul(lo, hi);
}

// factors of the adjacent positions idx (even) and idx + 1
__device__ __forceinline__ void v2_scale2(const NttPass& p, u64 idx, u64& s0, u64& s1) {
  if (p.scale_mode == SCALE_FULL) {
    const ulonglong2 v = __ldg(reinterpret_cast<const ulonglong2*>(p.pw_full + idx));
    s0 = v.x;
    s1 = v.y;
  } else {
    s0 = v2_scale(p, idx);
    s1 = v2_scale(p, idx + 1);
  }
}

// FIRST: the stage starts the whole transform (no round done before it, prefix 0), so the twiddle of group 0 of every
// round is tab[0] = 1 and 15 of the 32 multiplications of a radix-16 stage disappear.
template <int RS, int Q, bool FIRST>
__device__ __forceinline__ void v2_round(u64 (&x)[16], const u64* __restrict__ tab, u32 pfx) {
  constexpr int NG = 1 << Q;       // twiddles of this round
  constexpr int BIT = 1 << (3 - Q);
  u64 tw[NG];
  const u64* tp = tab + ((size_t)pfx << Q);
  if constexpr (NG == 1) {
    tw[0] = __ldg(tp);
  } else {
    const ulonglong2* tv = reinterpret_cast<const ulonglong2*>(tp);
#pragma unroll
    for (int g = 0; g < NG / 2; g++) {
      const ulonglong2 v = __ldg(tv + g);
      tw[2 * g] = v.x;
      tw[2 * g + 1] = v.y;
    }
  }
#pragma unroll
  for (int j0 = 0; j0 < 16; j0++) {
    if (j0 & BIT) continue;
    const int j1 = j0 | BIT;
    u64 v;
    if (FIRST && (j0 >> (4 - Q)) == 0) v = gl::canon(x[j1]);
    else v = gl::mul(x[j1], tw[j0 >> (4 - Q)]);
#if BJ_NTT_SUB_FMA
    x[j1] = gl::sub_fma(x[j0], v);
#else
    x[j1] = gl::sub(x[j0], v);
#endif
#if BJ_NTT_ADD_ALU
    x[j0] = gl::add_alu(x[j0], v);
#else
    x[j0] = gl::add(x[j0], v);
#endif
  }
}

template <int RS, bool FIRST>
__device__ __forceinline__ void v2_stage_compute(u64 (&x)[16], const u64* __restrict__ tab, u32 pfx) {
  v2_round<RS, 0, FIRST>(x, tab, pfx);
  if constexpr (RS > 1) v2_round<RS, 1, FIRST>(x, tab, pfx);
  if constexpr (RS > 2) v2_round<RS, 2, FIRST>(x, tab, pfx);
  if constexpr (RS > 3) v2_round<RS, 3, FIRST>(x, tab, pfx);
}

template <int T, int W, int KIND, int STAGE, bool FIRST = false>
__device__ __forceinline__ void v2_stage(u64* __restrict__ sm, const u64* __restrict__ tab, int tid, u32 hi, u32 tile,
                                         int r0) {
  using C = V2Cfg<T, W>;
  constexpr int RS = STAGE == 0 ? C::RS0 : 4;
  constexpr int DONE = STAGE == 0 ? 0 : C::RS0 + 4 * (STAGE - 1);
  constexpr int B_LO = T - DONE - RS;
  constexpr int PP = B_LO + W - (4 - RS);
  static_assert(PP >= 0, "tile too small for 16-value threads");
#pragma unroll 1
  for (int q = tid; q < C::NVT; q += C::THREADS) {
    const int e0 = ((q >> PP) << (PP + 4)) | (q & ((1 << PP) - 1));
    u32 hq = hi;
    if constexpr (KIND == PASS_TRANSPOSE_LAST) {
      const u32 k1 = (tile << W) + (u32)(e0 & ((1 << W) - 1));
      hq = r0 ? (__brev(k1) >> (32 - r0)) : 0u;
    }
    const u32 pfx = (hq << (C::LOG_E - PP - 4)) | (u32)(q >> PP);
    u64* base = sm + v2_phys(e0);
    u64 x[16];
#pragma unroll
    for (int j = 0; j < 16; j++) x[j] = base[(j << PP) + ((j << PP) >> 4)];
    v2_stage_compute<RS, FIRST>(x, tab, pfx);
#pragma unroll
    for (int j = 0; j < 16; j++) base[(j << PP) + ((j << PP) >> 4)] = x[j];
  }
  __syncthreads();
  if constexpr (STAGE + 1 < C::NSTAGES) v2_stage<T, W, KIND, STAGE + 1>(sm, tab, tid, hi, tile, r0);
}

template <int T, int W, int KIND>
__device__ __forceinline__ void ntt_pass_v2_body(const NttPass& p) {
  using C = V2Cfg<T, W>;
  extern __shared__ u64 sm[];
  constexpr int WM = (1 << W) - 1;
  const int tid = threadIdx.x;
  u32 tile = blockIdx.x, column = blockIdx.y;
  if (KIND == PASS_TILE && p.n_cols) {
    tile = blockIdx.x / p.n_cols;
    column = blockIdx.x - tile * p.n_cols;
  }
  const u64* __restrict__ src = p.src + (u64)column * p.src_col_stride;
  u64* __restrict__ dst = p.dst + (u64)column * p.dst_col_stride;
  const int m = p.log_n, r0 = p.r0;
  const bool scale_load = p.scale_mode != SCALE_NONE && p.scale_on_load;
  const bool scale_store = p.scale_mode != SCALE_NONE && !p.scale_on_load;

  u64 base = 0;
  int lo_bits = 0;
  u32 hi = 0;
  if constexpr (KIND == PASS_TILE) {
    lo_bits = m - r0 - T;
    const int groups_log = lo_bits - W;
    hi = tile >> groups_log;
    const u64 lo0 = (u64)(tile & ((1u << groups_log) - 1)) << W;
    base = ((u64)hi << (m - r0)) + lo0;
#pragma unroll 4
    for (int pi = tid; pi < C::E / 2; pi += C::THREADS) {
      const int e = 2 * pi;
      const int row = e >> W, col = e & WM;
      const u64 gi = base + ((u64)row << lo_bits) + col;
      ulonglong2 v;
      if constexpr (W == 0) {
        // contiguous tile (lo_bits == 0): e and e+1 are adjacent rows
        v = *reinterpret_cast<const ulonglong2*>(src + base + e);
      } else {
        v = *reinterpret_cast<const ulonglong2*>(src + gi);
      }
      if (scale_load) {
        const u64 g0 = (W == 0) ? base + e : gi;
        u64 s0, s1;
        v2_scale2(p, g0, s0, s1);
        v.x = gl::mul(v.x, s0);
        v.y = gl::mul(v.y, s1);
      }
      const int pe = v2_phys(e);
      sm[pe] = v.x;
      sm[pe + 1] = v.y;
    }
  } else {
#pragma unroll 4
    for (int pi = tid; pi < C::E / 2; pi += C::THREADS) {
      const int col = pi >> (T - 1), row = (pi & ((1 << (T - 1)) - 1)) * 2;
      const u32 k1 = (tile << W) + col;
      const u32 blk = r0 ? (__brev(k1) >> (32 - r0)) : 0u;
      const u64 gi = ((u64)blk << T) + row;
      ulonglong2 v = *reinterpret_cast<const ulonglong2*>(src + gi);
      if (scale_load) {
        u64 s0, s1;
        v2_scale2(p, gi, s0, s1);
        v.x = gl::mul(v.x, s0);
        v.y = gl::mul(v.y, s1);
      }
      sm[v2_phys((row << W) + col)] = v.x;
      sm[v2_phys(((row + 1) << W) + col)] = v.y;
    }
  }
  __syncthreads();

  // a twisted table (PASS_TILE): the tile's twiddle prefix gets the leading 1 that selects round rho's slice tab + 2^rho, and
  // group 0's twiddle is a coset power, not 1, so the FIRST stage does not apply
  const u32 tw_prefix = KIND == PASS_TILE ? p.tw_prefix : 0u;
  const u32 hs = hi | tw_prefix;
  if ((r0 | tw_prefix) == 0) v2_stage<T, W, KIND, 0, true>(sm, p.tab, tid, hs, tile, r0);
  else v2_stage<T, W, KIND, 0, false>(sm, p.tab, tid, hs, tile, r0);

  if constexpr (KIND == PASS_TILE) {
#pragma unroll 4
    for (int pi = tid; pi < C::E / 2; pi += C::THREADS) {
      const int e = 2 * pi;
      const int row = e >> W, col = e & WM;
      const u64 gi = (W == 0) ? base + e : base + ((u64)row << lo_bits) + col;
      const int pe = v2_phys(e);
      ulonglong2 v;
      v.x = sm[pe];
      v.y = sm[pe + 1];
      if (scale_store) {
        u64 s0, s1;
        v2_scale2(p, gi, s0, s1);
        v.x = gl::mul(v.x, s0);
        v.y = gl::mul(v.y, s1);
      }
      if (p.canon_out) {
        v.x = gl::canon(v.x);
        v.y = gl::canon(v.y);
      }
      *reinterpret_cast<ulonglong2*>(dst + gi) = v;
    }
  } else if constexpr (W == 0) {
    // single tile per column (r0 == 0): natural-order store dst[kappa] = value at row bitrev(kappa)
#pragma unroll 4
    for (int kappa = tid; kappa < C::E; kappa += C::THREADS) {
      const u32 rho = __brev((u32)kappa) >> (32 - T);
      u64 v = sm[v2_phys((int)rho)];
      const u64 go = (u64)tile + ((u64)kappa << r0);
      if (scale_store) v = gl::mul(v, v2_scale(p, go));
      if (p.canon_out) v = gl::canon(v);
      dst[go] = v;
    }
  } else {
#pragma unroll 4
    for (int pi = tid; pi < C::E / 2; pi += C::THREADS) {
      const int col = (pi & (WM >> 1)) * 2;
      const u32 kappa = (u32)(pi >> (W - 1));
      const u32 rho = __brev(kappa) >> (32 - T);
      const int pe = v2_phys(((int)rho << W) + col);  // col even: both values sit in one 16-group
      ulonglong2 v;
      v.x = sm[pe];
      v.y = sm[pe + 1];
      const u64 go = ((u64)tile << W) + col + ((u64)kappa << r0);
      if (scale_store) {
        u64 s0, s1;
        v2_scale2(p, go, s0, s1);
        v.x = gl::mul(v.x, s0);
        v.y = gl::mul(v.y, s1);
      }
      if (p.canon_out) {
        v.x = gl::canon(v.x);
        v.y = gl::canon(v.y);
      }
      *reinterpret_cast<ulonglong2*>(dst + go) = v;
    }
  }
}

template <int T, int W, int KIND>
__global__ void __launch_bounds__(V2Cfg<T, W>::THREADS) ntt_pass_v2_kernel(const NttPass p) {
  ntt_pass_v2_body<T, W, KIND>(p);
}
// 2^13-value tiles: shared memory admits 3 CTAs per SM, so up to 85 registers per thread cost no occupancy
template <int T, int W, int KIND>
__global__ void __launch_bounds__(V2Cfg<T, W>::THREADS, 3) ntt_pass_v2_kernel_r85(const NttPass p) {
  ntt_pass_v2_body<T, W, KIND>(p);
}
// same body with the register cap that keeps 4 CTAs (of 256 threads) per SM
template <int T, int W, int KIND>
__global__ void __launch_bounds__(V2Cfg<T, W>::THREADS, 4) ntt_pass_v2_kernel_r64(const NttPass p) {
  ntt_pass_v2_body<T, W, KIND>(p);
}

// ---- experiment (north_star: "TMA bulk copies into shared memory for the butterfly tiles"): the contiguous pass (W = 0, no
// scaling) with its tile moved by the bulk-copy engine instead of through registers.  One elected thread arms an mbarrier with
// the tile's byte count and issues ONE cp.async.bulk (global -> shared, UBLKCP in SASS); the tile lands densely in a staging
// buffer, is re-laid into the padded layout the conflict-free register stages need (the bulk engine cannot produce the 17/16
// padding), and after the stages it is packed back and leaves with one cp.async.bulk (shared -> global).  BJ_NTT_BULK=1 selects
// it.
__device__ __forceinline__ u32 smem_u32(const void* p) { return (u32)__cvta_generic_to_shared(p); }

template <int T>
__global__ void __launch_bounds__(V2Cfg<T, 0>::THREADS) ntt_pass_bulk_kernel(const NttPass p) {
  using C = V2Cfg<T, 0>;
  extern __shared__ __align__(128) u64 sm[];
  constexpr int PADDED = (C::E + (C::E >> 4) + 2 + 15) & ~15;   // staging starts 128-byte aligned
  u64* stage = sm + PADDED;
  __shared__ __align__(8) unsigned long long bar;
  const int tid = threadIdx.x;
  const u32 tile = blockIdx.x;
  const u64* __restrict__ src = p.src + (u64)blockIdx.y * p.src_col_stride + ((u64)tile << T);
  u64* __restrict__ dst = p.dst + (u64)blockIdx.y * p.dst_col_stride + ((u64)tile << T);
  constexpr u32 BYTES = (u32)(sizeof(u64) << T);
  if (tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&bar)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&bar)), "r"(BYTES) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(stage)), "l"(src),
                 "r"(BYTES), "r"(smem_u32(&bar))
                 : "memory");
  }
  {  // every thread waits for the bytes (phase 0)
    u32 done = 0;
    while (!done)
      asm volatile("{\n\t.reg .pred q;\n\tmbarrier.try_wait.parity.shared::cta.b64 q, [%1], 0;\n\tselp.u32 %0, 1, 0, q;\n\t}" : "=r"(done) : "r"(smem_u32(&bar)) : "memory");
  }
#pragma unroll 4
  for (int pi = tid; pi < C::E / 2; pi += C::THREADS) {
    const ulonglong2 v = reinterpret_cast<const ulonglong2*>(stage)[pi];
    const int pe = v2_phys(2 * pi);
    sm[pe] = v.x;
    sm[pe + 1] = v.y;
  }
  __syncthreads();
  if ((p.r0 | p.tw_prefix) == 0) v2_stage<T, 0, PASS_TILE, 0, true>(sm, p.tab, tid, tile, tile, p.r0);
  else v2_stage<T, 0, PASS_TILE, 0, false>(sm, p.tab, tid, tile | p.tw_prefix, tile, p.r0);
#pragma unroll 4
  for (int pi = tid; pi < C::E / 2; pi += C::THREADS) {
    const int pe = v2_phys(2 * pi);
    ulonglong2 v;
    v.x = sm[pe];
    v.y = sm[pe + 1];
    if (p.canon_out) {
      v.x = gl::canon(v.x);
      v.y = gl::canon(v.y);
    }
    reinterpret_cast<ulonglong2*>(stage)[pi] = v;
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes visible to the bulk-copy (async) proxy
  __syncthreads();
  if (tid == 0) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_u32(stage)), "r"(BYTES) : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // the staging buffer must outlive the copy's reads
  }
}

template <int T>
struct V2BulkCfg {
  static constexpr size_t SMEM = sizeof(u64) * (size_t)(((V2Cfg<T, 0>::E + (V2Cfg<T, 0>::E >> 4) + 2 + 15) & ~15) + V2Cfg<T, 0>::E);
};

typedef void (*V2KernelPtr)(const NttPass);

template <int T, int W, int KIND>
struct V2Entry {
  static V2KernelPtr get() {
    if constexpr (V2Cfg<T, W>::CAP_REGS) return ntt_pass_v2_kernel_r64<T, W, KIND>;
    else if constexpr (T + W == 13) return ntt_pass_v2_kernel_r85<T, W, KIND>;
    else return ntt_pass_v2_kernel<T, W, KIND>;
  }
};

struct V2Launch {
  V2KernelPtr fn;
  int threads;
  size_t smem;
};

#define BJ_V2_CASE(TT, WW)                                                                   \
  if (t == TT && w == WW) {                                                                  \
    out->fn = kind == PASS_TILE ? V2Entry<TT, WW, PASS_TILE>::get()                          \
                                : V2Entry<TT, WW, PASS_TRANSPOSE_LAST>::get();                \
    out->threads = V2Cfg<TT, WW>::THREADS;                                                   \
    out->smem = V2Cfg<TT, WW>::SMEM;                                                         \
    return true;                                                                             \
  }

static bool v2_bulk_lookup(int t, V2Launch* out) {
#define BJ_V2_BULK_CASE(TT)                        \
  if (t == TT) {                                   \
    out->fn = ntt_pass_bulk_kernel<TT>;            \
    out->threads = V2Cfg<TT, 0>::THREADS;          \
    out->smem = V2BulkCfg<TT>::SMEM;               \
    return true;                                   \
  }
  BJ_V2_BULK_CASE(10) BJ_V2_BULK_CASE(11) BJ_V2_BULK_CASE(12) BJ_V2_BULK_CASE(13)
#undef BJ_V2_BULK_CASE
  return false;
}

// instantiation menu (see make_plan): contiguous last passes, strided front passes, transposed last passes
static bool v2_lookup(int t, int w, int kind, V2Launch* out) {
  BJ_V2_CASE(4, 0) BJ_V2_CASE(5, 0) BJ_V2_CASE(6, 0) BJ_V2_CASE(7, 0) BJ_V2_CASE(8, 0) BJ_V2_CASE(9, 0)
  BJ_V2_CASE(10, 0) BJ_V2_CASE(11, 0) BJ_V2_CASE(12, 0) BJ_V2_CASE(13, 0) BJ_V2_CASE(14, 0)
  BJ_V2_CASE(11, 2)
  BJ_V2_CASE(8, 3) BJ_V2_CASE(9, 3) BJ_V2_CASE(10, 3) BJ_V2_CASE(11, 3)
  BJ_V2_CASE(8, 4) BJ_V2_CASE(9, 4) BJ_V2_CASE(10, 4)
  BJ_V2_CASE(6, 5) BJ_V2_CASE(7, 5) BJ_V2_CASE(8, 5) BJ_V2_CASE(9, 5)
  return false;
}

}  // namespace bj
