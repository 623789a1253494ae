// Blake2s-256 Merkle tree hasher (the TreeHasher of run_sha256_prover_non_recursive, BASELINE config 4).
// Reference: impl TreeHasher<F> for blake2::Blake2s256, src/cs/oracle/mod.rs:179-245 - a leaf is Blake2s-256 (RFC 7693,
// unkeyed, 32-byte digest; crate blake2 = "0.10", Cargo.toml:33) over the little-endian bytes of the REDUCED u64 of every
// element in preimage order; a node is Blake2s-256(left || right).  Digests are 32 bytes, stored here as 4 little-endian
// u64 so that trees share the [n][4] u64 layout of the Poseidon2 trees (byte-identical to [u8; 32]).
#include <cstring>
#include "ctx.hpp"

namespace bj {

using gl::u32;

__constant__ u32 c_blake2s_iv[8] = {0x6A09E667u, 0xBB67AE85u, 0x3C6EF372u, 0xA54FF53Au, 0x510E527Fu, 0x9B05688Cu, 0x1F83D9ABu, 0x5BE0CD19u};
__device__ __forceinline__ u32 rotr32(u32 x, int r) { return __funnelshift_r(x, x, r); }

// Pipe balance: the G function is xor / rotate / add only, all of which ptxas issues on the ALU pipe (LOP3, SHF, IADD3)
// except half of the adds.  An addition is also a multiply-add by 1, which runs on the FMA pipe; ptxas folds a literal 1 back
// into IADD3, so the 1 arrives as a kernel parameter (`one`) it cannot see through.  All six two-input additions of a G then
// issue as IMAD, off the ALU pipe.
__device__ __forceinline__ u32 add_fma(u32 a, u32 b, u32 one) { return a * one + b; }

#define BJ_B2S_G(a, b, c, d, x, y)                  \
  a = add_fma(b, add_fma(x, a, one), one);          \
  d = rotr32(d ^ a, 16);                            \
  c = add_fma(d, c, one);                           \
  b = rotr32(b ^ c, 12);                            \
  a = add_fma(b, add_fma(y, a, one), one);          \
  d = rotr32(d ^ a, 8);                             \
  c = add_fma(d, c, one);                           \
  b = rotr32(b ^ c, 7);

// one compression: h updated in place; m = 16 message words, t = byte counter (low 32 bits suffice up to 4 GiB), last flag;
// one == 1 (opaque to the compiler, see above)
__device__ __forceinline__ void blake2s_compress(u32 (&h)[8], const u32 (&m)[16], u32 t_lo, u32 t_hi, bool last, u32 one = 1) {
  u32 v0 = h[0], v1 = h[1], v2 = h[2], v3 = h[3], v4 = h[4], v5 = h[5], v6 = h[6], v7 = h[7];
  u32 v8 = c_blake2s_iv[0], v9 = c_blake2s_iv[1], v10 = c_blake2s_iv[2], v11 = c_blake2s_iv[3];
  u32 v12 = c_blake2s_iv[4] ^ t_lo, v13 = c_blake2s_iv[5] ^ t_hi;
  u32 v14 = last ? ~c_blake2s_iv[6] : c_blake2s_iv[6], v15 = c_blake2s_iv[7];
#pragma unroll
  for (int r = 0; r < 10; r++) {
    // sigma is compile-time after unrolling; the table below is only read through constant indices
    constexpr unsigned char S[10][16] = {
        {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3},
        {11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4}, {7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8},
        {9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13}, {2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9},
        {12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11}, {13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10},
        {6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5}, {10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0}};
    BJ_B2S_G(v0, v4, v8, v12, m[S[r][0]], m[S[r][1]])
    BJ_B2S_G(v1, v5, v9, v13, m[S[r][2]], m[S[r][3]])
    BJ_B2S_G(v2, v6, v10, v14, m[S[r][4]], m[S[r][5]])
    BJ_B2S_G(v3, v7, v11, v15, m[S[r][6]], m[S[r][7]])
    BJ_B2S_G(v0, v5, v10, v15, m[S[r][8]], m[S[r][9]])
    BJ_B2S_G(v1, v6, v11, v12, m[S[r][10]], m[S[r][11]])
    BJ_B2S_G(v2, v7, v8, v13, m[S[r][12]], m[S[r][13]])
    BJ_B2S_G(v3, v4, v9, v14, m[S[r][14]], m[S[r][15]])
  }
  h[0] ^= v0 ^ v8;
  h[1] ^= v1 ^ v9;
  h[2] ^= v2 ^ v10;
  h[3] ^= v3 ^ v11;
  h[4] ^= v4 ^ v12;
  h[5] ^= v5 ^ v13;
  h[6] ^= v6 ^ v14;
  h[7] ^= v7 ^ v15;
}

__device__ __forceinline__ void blake2s_init(u32 (&h)[8]) {
#pragma unroll
  for (int i = 0; i < 8; i++) h[i] = c_blake2s_iv[i];
  h[0] ^= 0x01010020u;  // digest length 32, no key, fanout 1, depth 1
}

__device__ __forceinline__ void blake2s_store(const u32 (&h)[8], u64* out) {
#pragma unroll
  for (int k = 0; k < 4; k++) out[k] = (u64)h[2 * k] | ((u64)h[2 * k + 1] << 32);
}

// leaf m absorbs source_s[m*epl + e] (8 LE bytes of the canonical value each), s = 0..n_src-1, e = 0..epl-1
__global__ void __launch_bounds__(128) blake2s_leaf_kernel(const u64* const* __restrict__ srcs, u32 n_src, u64 n_leaves, int log_epl,
                                                            u64* __restrict__ digests, u32 one) {
  const u64 leaf = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (leaf >= n_leaves) return;
  u32 h[8];
  blake2s_init(h);
  const u64 total = (u64)n_src << log_epl;  // elements; 8 per 64-byte block
  const u64 epl_mask = (1ull << log_epl) - 1;
  const u64 row0 = leaf << log_epl;
  const u64 n_blocks = total == 0 ? 1 : (total + 7) / 8;
  for (u64 blk = 0; blk < n_blocks; blk++) {
    u32 m[16];
#pragma unroll
    for (int k = 0; k < 8; k++) {
      const u64 idx = blk * 8 + k;
      u64 v = 0;
      if (idx < total) v = gl::canon(srcs[idx >> log_epl][row0 + (idx & epl_mask)]);
      m[2 * k] = (u32)v;
      m[2 * k + 1] = (u32)(v >> 32);
    }
    const bool last = blk + 1 == n_blocks;
    const u64 t = last ? total * 8 : (blk + 1) * 64;
    blake2s_compress(h, m, (u32)t, (u32)(t >> 32), last, one);
  }
  blake2s_store(h, digests + 4 * leaf);
}

__global__ void __launch_bounds__(128) blake2s_node_kernel(const u64* __restrict__ prev, u64 n_out, u64* __restrict__ next, u32 one) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_out) return;
  u32 h[8], m[16];
  blake2s_init(h);
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const u64 v = prev[8 * i + k];
    m[2 * k] = (u32)v;
    m[2 * k + 1] = (u32)(v >> 32);
  }
  blake2s_compress(h, m, 64u, 0u, true, one);
  blake2s_store(h, next + 4 * i);
}

// the node levels of a tree over existing leaf hashes (the leaves may have been hashed a slice at a time)
int32_t merkle_nodes_blake2s(bj_ctx* ctx, const u64* d_leaf_hashes, u64 n_leaves, u32 cap_size, u64* d_nodes) {
  const u64* prev = d_leaf_hashes;
  u64 cnt = n_leaves, written = 0;
  while (cnt > cap_size) {
    const u64 next = cnt / 2;
    u64* dst = d_nodes + 4 * written;
    blake2s_node_kernel<<<(unsigned)((next + 127) / 128), 128, 0, ctx->stream>>>(prev, next, dst, ctx->one);
    BJ_LAUNCH_CHECK(ctx);
    prev = dst;
    written += next;
    cnt = next;
  }
  return BJ_OK;
}

}  // namespace bj

using namespace bj;

extern "C" int32_t bj_merkle_build_blake2s(bj_ctx* ctx, const uint64_t* const* h_sources, uint32_t n_sources, uint64_t n_leaves,
                                           uint32_t elems_per_leaf, uint32_t cap_size, uint64_t* d_leaf_hashes, uint64_t* d_nodes) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || !h_sources || !d_leaf_hashes || n_sources == 0 || n_leaves == 0)
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_merkle_build_blake2s: bad argument");
  if ((n_leaves & (n_leaves - 1)) || (cap_size & (cap_size - 1)) || cap_size == 0 || cap_size > n_leaves ||
      (elems_per_leaf & (elems_per_leaf - 1)) || elems_per_leaf == 0)
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_merkle_build_blake2s: sizes must be powers of two, cap <= leaves");
  if (n_leaves > cap_size && !d_nodes) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_merkle_build_blake2s: d_nodes is NULL");
  void* d_src;
  BJ_TRY(param_upload(ctx, h_sources, sizeof(u64*) * n_sources, &d_src));
  int log_epl = 0;
  while ((1u << log_epl) < elems_per_leaf) log_epl++;
  blake2s_leaf_kernel<<<(unsigned)((n_leaves + 127) / 128), 128, 0, ctx->stream>>>((const u64* const*)d_src, n_sources, n_leaves, log_epl,
                                                                                   (u64*)d_leaf_hashes, ctx->one);
  BJ_LAUNCH_CHECK(ctx);
  if (n_leaves > cap_size) BJ_TRY(merkle_nodes_blake2s(ctx, (const u64*)d_leaf_hashes, n_leaves, cap_size, (u64*)d_nodes));
  return BJ_OK;
}

// ---- proof of work: impl PoWRunner for Blake2s256 (src/cs/implementations/pow.rs:52-147): find a u64 `challenge` such that
// the first 8 bytes (LE) of Blake2s-256(seed || challenge.to_le_bytes()) have >= pow_bits trailing zero bits.  One thread per
// candidate, 2^24 candidates per launch, the smallest hit of the first successful batch is returned (the reference's serial
// search for <= 16 bits returns the smallest overall; its parallel search returns whichever worker wins).
namespace bj {

__global__ void __launch_bounds__(256) blake2s_pow_kernel(const u32* __restrict__ seed_words, u32 seed_len, u64 base, u32 pow_bits,
                                                           unsigned long long* __restrict__ best) {
  const u64 nonce = base + (u64)blockIdx.x * blockDim.x + threadIdx.x;
  // message = seed (seed_len <= 56 bytes, zero padded in seed_words) || nonce: always one 64-byte block
  u32 m[16];
#pragma unroll
  for (int i = 0; i < 16; i++) m[i] = seed_words[i];
  const u32 off = seed_len;  // byte offset of the nonce
  const u64 lo_shift = (off & 3) * 8;
  // place the 8 nonce bytes at byte offset `off` (unaligned in general)
  u32 w = off >> 2;
  u64 carry = nonce;
  if (lo_shift == 0) {
    m[w] = (u32)carry;
    m[w + 1] = (u32)(carry >> 32);
  } else {
    m[w] |= (u32)(carry << lo_shift);
    m[w + 1] = (u32)(carry >> (32 - lo_shift));
    m[w + 2] |= (u32)(carry >> (64 - lo_shift));
  }
  u32 h[8];
  blake2s_init(h);
  blake2s_compress(h, m, seed_len + 8, 0u, true);
  const u64 first = (u64)h[0] | ((u64)h[1] << 32);
  const bool ok = pow_bits == 0 || (first << (64 - pow_bits)) == 0;  // trailing_zeros >= pow_bits (pow_bits <= 32)
  if (ok) atomicMin(best, (unsigned long long)nonce);
}

}  // namespace bj

extern "C" int32_t bj_pow_blake2s(bj_ctx* ctx, const uint8_t* h_seed, uint32_t seed_len, uint32_t pow_bits, uint64_t* h_challenge) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || (!h_seed && seed_len) || !h_challenge || pow_bits > 32 || seed_len > 52)
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_pow_blake2s: bad argument (pow_bits <= 32, seed <= 52 bytes)");
  u32 words[16] = {0};
  memcpy(words, h_seed, seed_len);
  void* d_seed;
  BJ_TRY(param_upload(ctx, words, sizeof(words), &d_seed));
  // one word per context, kept: a proof on a lane must not cudaMalloc / cudaFree (both synchronise the whole device)
  if (!ctx->pow_best) BJ_CUDA(ctx, cudaMalloc(&ctx->pow_best, sizeof(unsigned long long)));
  unsigned long long* d_best = ctx->pow_best;
  const unsigned long long none = ~0ull;
  const u64 batch = 1ull << 24;
  int32_t st = BJ_OK;
  unsigned long long best = none;
  for (u64 base = 0; best == none; base += batch) {
    if (base >= (1ull << 40)) {  // 2^40 candidates without a hit for <= 32 bits does not happen; do not spin forever
      st = BJ_ERR_UNSUPPORTED;
      break;
    }
    if (cudaMemcpyAsync(d_best, &none, sizeof(none), cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) st = BJ_ERR_CUDA;
    blake2s_pow_kernel<<<(unsigned)(batch / 256), 256, 0, ctx->stream>>>((const u32*)d_seed, seed_len, base, pow_bits, d_best);
    ctx->launches++;
    if (cudaMemcpyAsync(&best, d_best, sizeof(best), cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
        cudaStreamSynchronize(ctx->stream) != cudaSuccess)
      st = BJ_ERR_CUDA;
    if (st != BJ_OK) break;
  }
  if (st == BJ_ERR_CUDA) BJ_FAIL(ctx, BJ_ERR_CUDA, "bj_pow_blake2s: CUDA error");
  if (st != BJ_OK) BJ_FAIL(ctx, st, "bj_pow_blake2s: no solution found");
  *h_challenge = best;
  return BJ_OK;
}
