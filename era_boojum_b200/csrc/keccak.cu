// Keccak-256 Merkle tree hasher: impl TreeHasher<F> for sha3::Keccak256 (src/cs/oracle/mod.rs:247-313) - a leaf is
// Keccak-256 over the little-endian bytes of the REDUCED u64 of every element in preimage order, a node is
// Keccak-256(left || right).  Digests are 32 bytes, stored as 4 little-endian u64 (the [n][4] u64 layout of the other trees).
// One thread per leaf / node; an element is exactly one 64-bit lane, so absorbing is an XOR into the state.
#include "ctx.hpp"
#include "keccak.cuh"

namespace bj {

__global__ void __launch_bounds__(128) keccak_leaf_kernel(const u64* const* __restrict__ srcs, u32 n_src, u64 n_leaves, int log_epl,
                                                           u64* __restrict__ digests) {
  const u64 leaf = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (leaf >= n_leaves) return;
  uint64_t st[25];
#pragma unroll
  for (int i = 0; i < 25; i++) st[i] = 0;
  const u64 total = (u64)n_src << log_epl;
  const u64 epl_mask = (1ull << log_epl) - 1;
  const u64 row0 = leaf << log_epl;
  u64 idx = 0;
  // full rate blocks of 17 lanes
  for (; idx + 17 <= total; idx += 17) {
#pragma unroll
    for (int k = 0; k < 17; k++) {
      const u64 e = idx + k;
      st[k] ^= gl::canon(srcs[e >> log_epl][row0 + (e & epl_mask)]);
    }
    keccak_f1600(st);
  }
  // last (partial, possibly empty) block + padding 0x01 ... 0x80
  const u32 rem = (u32)(total - idx);
#pragma unroll
  for (int k = 0; k < 17; k++) {
    uint64_t w = 0;
    if ((u32)k < rem) {
      const u64 e = idx + k;
      w = gl::canon(srcs[e >> log_epl][row0 + (e & epl_mask)]);
    } else if ((u32)k == rem) {
      w = 0x01;
    }
    if (k == 16) w ^= 0x8000000000000000ull;
    st[k] ^= w;
  }
  keccak_f1600(st);
#pragma unroll
  for (int k = 0; k < 4; k++) digests[4 * leaf + k] = st[k];
}

__global__ void __launch_bounds__(128) keccak_node_kernel(const u64* __restrict__ prev, u64 n_out, u64* __restrict__ next) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_out) return;
  uint64_t st[25];
#pragma unroll
  for (int k = 0; k < 25; k++) st[k] = 0;
#pragma unroll
  for (int k = 0; k < 8; k++) st[k] = prev[8 * i + k];
  st[8] = 0x01;
  st[16] = 0x8000000000000000ull;
  keccak_f1600(st);
#pragma unroll
  for (int k = 0; k < 4; k++) next[4 * i + k] = st[k];
}

// the node levels of a tree over existing leaf hashes (the leaves may have been hashed a slice at a time)
int32_t merkle_nodes_keccak256(bj_ctx* ctx, const u64* d_leaf_hashes, u64 n_leaves, u32 cap_size, u64* d_nodes) {
  const u64* prev = d_leaf_hashes;
  u64 cnt = n_leaves, written = 0;
  while (cnt > cap_size) {
    const u64 next = cnt / 2;
    u64* dst = d_nodes + 4 * written;
    keccak_node_kernel<<<(unsigned)((next + 127) / 128), 128, 0, ctx->stream>>>(prev, next, dst);
    BJ_LAUNCH_CHECK(ctx);
    prev = dst;
    written += next;
    cnt = next;
  }
  return BJ_OK;
}

}  // namespace bj

using namespace bj;

extern "C" {

int32_t bj_merkle_build_keccak256(bj_ctx* ctx, const uint64_t* const* h_sources, uint32_t n_sources, uint64_t n_leaves,
                                  uint32_t elems_per_leaf, uint32_t cap_size, uint64_t* d_leaf_hashes, uint64_t* d_nodes) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || !h_sources || !d_leaf_hashes || n_sources == 0 || n_leaves == 0)
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_merkle_build_keccak256: bad argument");
  if ((n_leaves & (n_leaves - 1)) || (cap_size & (cap_size - 1)) || cap_size == 0 || cap_size > n_leaves ||
      (elems_per_leaf & (elems_per_leaf - 1)) || elems_per_leaf == 0)
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_merkle_build_keccak256: sizes must be powers of two, cap <= leaves");
  if (n_leaves > cap_size && !d_nodes) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_merkle_build_keccak256: d_nodes is NULL");
  void* d_src;
  BJ_TRY(param_upload(ctx, h_sources, sizeof(u64*) * n_sources, &d_src));
  int log_epl = 0;
  while ((1u << log_epl) < elems_per_leaf) log_epl++;
  keccak_leaf_kernel<<<(unsigned)((n_leaves + 127) / 128), 128, 0, ctx->stream>>>((const u64* const*)d_src, n_sources, n_leaves, log_epl,
                                                                                  (u64*)d_leaf_hashes);
  BJ_LAUNCH_CHECK(ctx);
  if (n_leaves > cap_size) BJ_TRY(merkle_nodes_keccak256(ctx, (const u64*)d_leaf_hashes, n_leaves, cap_size, (u64*)d_nodes));
  return BJ_OK;
}

void bj_host_keccak256(const uint8_t* data, size_t n, uint8_t out[32]) {
  HostKeccak256 h;
  if (n) h.update(data, n);
  h.finalize_reset(out);
}

// ---- proof of work: impl PoWRunner for Keccak256 (src/cs/implementations/pow.rs:140-230): find a u64 `challenge` such that the
// first 8 bytes (LE) of Keccak-256(seed || challenge.to_le_bytes()) have >= pow_bits trailing zero bits.  Same scheme as the
// Blake2s runner (bj_pow_blake2s): one thread per candidate, 2^24 candidates per launch, the smallest hit of the first
// successful batch is returned.  seed || nonce (<= 120 bytes) is a single rate block.
}  // extern "C"

namespace bj {
__global__ void __launch_bounds__(256) keccak_pow_kernel(const uint8_t* __restrict__ seed, u32 seed_len, u64 base, u32 pow_bits,
                                                          unsigned long long* __restrict__ best) {
  const u64 nonce = base + (u64)blockIdx.x * blockDim.x + threadIdx.x;
  uint8_t msg[136];
#pragma unroll 1
  for (int i = 0; i < 136; i++) msg[i] = 0;
  for (u32 i = 0; i < seed_len; i++) msg[i] = seed[i];
  for (int k = 0; k < 8; k++) msg[seed_len + k] = (uint8_t)(nonce >> (8 * k));
  msg[seed_len + 8] |= 0x01;
  msg[135] |= 0x80;
  uint64_t st[25];
#pragma unroll
  for (int i = 0; i < 25; i++) st[i] = 0;
  for (int i = 0; i < 17; i++) {
    uint64_t w = 0;
    for (int k = 0; k < 8; k++) w |= (uint64_t)msg[8 * i + k] << (8 * k);
    st[i] = w;
  }
  keccak_f1600(st);
  const bool ok = pow_bits == 0 || (st[0] << (64 - pow_bits)) == 0;
  if (ok) atomicMin(best, (unsigned long long)nonce);
}
}  // namespace bj

extern "C" int32_t bj_pow_keccak256(bj_ctx* ctx, const uint8_t* h_seed, uint32_t seed_len, uint32_t pow_bits, uint64_t* h_challenge) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || (!h_seed && seed_len) || !h_challenge || pow_bits > 32 || seed_len > 120)
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_pow_keccak256: bad argument (pow_bits <= 32, seed <= 120 bytes)");
  uint8_t padded[128] = {0};
  memcpy(padded, h_seed, seed_len);
  void* d_seed;
  BJ_TRY(param_upload(ctx, padded, sizeof(padded), &d_seed));
  struct Best {
    unsigned long long* d = nullptr;
    ~Best() {
      if (d) cudaFree(d);
    }
  } best_buf;
  BJ_CUDA(ctx, cudaMalloc(&best_buf.d, sizeof(unsigned long long)));
  const unsigned long long none = ~0ull;
  const u64 batch = 1ull << 24;
  unsigned long long best = none;
  for (u64 base = 0; best == none; base += batch) {
    if (base >= (1ull << 40)) BJ_FAIL(ctx, BJ_ERR_UNSUPPORTED, "bj_pow_keccak256: no solution found");
    BJ_CUDA(ctx, cudaMemcpyAsync(best_buf.d, &none, sizeof(none), cudaMemcpyHostToDevice, ctx->stream));
    keccak_pow_kernel<<<(unsigned)(batch / 256), 256, 0, ctx->stream>>>((const uint8_t*)d_seed, seed_len, base, pow_bits, best_buf.d);
    BJ_LAUNCH_CHECK(ctx);
    BJ_CUDA(ctx, cudaMemcpyAsync(&best, best_buf.d, sizeof(best), cudaMemcpyDeviceToHost, ctx->stream));
    BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  *h_challenge = best;
  return BJ_OK;
}
