// FRI commit phase driver and query answering (host C++ over the device kernels).
//   do_fri                                   src/cs/implementations/fri/mod.rs:49-357
//   OracleQuery::construct / get_proof       src/cs/implementations/proof.rs:65-97, src/cs/oracle/merkle_tree.rs:462-480
// The transcript stays on the host: every oracle cap is downloaded (32 * cap bytes) and absorbed, the two challenge
// elements are drawn, and the next fold is launched - exactly the interleaving of the reference.
#include <cstring>
#include <memory>
#include <vector>
#include "ctx.hpp"

struct bj_transcript;
extern "C" void bj_transcript_witness_field_elements(bj_transcript* t, const uint64_t* els, size_t n);
extern "C" void bj_transcript_witness_merkle_tree_cap(bj_transcript* t, const uint64_t* cap, size_t n_digests);
extern "C" uint64_t bj_transcript_get_challenge(bj_transcript* t);

namespace bj {

// out[q][s * epl + e] = src_s[idx_q * epl + e]
__global__ void gather_leaves_kernel(const u64* const* __restrict__ srcs, u32 n_src, u32 epl, const u64* __restrict__ idx,
                                     u32 n_idx, u64* __restrict__ out) {
  const u32 row_len = n_src * epl;
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (u64)n_idx * row_len) return;
  const u32 q = (u32)(i / row_len), w = (u32)(i % row_len);
  const u32 s = w / epl, e = w % epl;
  out[i] = gl::canon(srcs[s][idx[q] * epl + e]);
}

// out[q][d] = sibling digest of leaf idx_q at depth d (bottom-up, cap level excluded)
__global__ void gather_paths_kernel(const u64* __restrict__ leaf_hashes, const u64* __restrict__ nodes, u64 n_leaves,
                                    u32 depth, const u64* __restrict__ idx, u32 n_idx, u64* __restrict__ out) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_idx * depth * 4) return;
  const u32 k = i & 3, d = (i >> 2) % depth, q = (i >> 2) / depth;
  u64 pos = idx[q] >> d;
  const u64* layer = leaf_hashes;
  u64 cnt = n_leaves;
  for (u32 l = 0; l < d; l++) {
    layer = (l == 0) ? nodes : layer + 4 * cnt;  // level l+1 starts after level l (levels are concatenated)
    cnt >>= 1;
  }
  out[i] = gl::canon(layer[4 * (pos ^ 1) + k]);
}

// device buffer from the context's stream-ordered pool (no device-wide synchronisation on allocation or release)
struct DevBuf {
  void* p = nullptr;
  bj_ctx* owner = nullptr;
  ~DevBuf() {
    if (!p) return;
    if (owner && owner->pool) cudaFreeAsync(p, owner->stream);
    else cudaFree(p);
  }
  int32_t alloc(bj_ctx* ctx, size_t bytes) {
    owner = ctx;
    const cudaError_t e = ctx->pool ? cudaMallocFromPoolAsync(&p, bytes ? bytes : 8, ctx->pool, ctx->stream) : cudaMalloc(&p, bytes ? bytes : 8);
    if (e != cudaSuccess) {
      cudaGetLastError();
      p = nullptr;
      BJ_FAIL(ctx, BJ_ERR_OOM, "FRI: device allocation failed");
    }
    return BJ_OK;
  }
  u64* u() const { return (u64*)p; }
};

struct FriLevel {
  u32 log_size = 0;       // elements in c0 / c1
  u32 log_fold = 0;       // elements per leaf = 2^log_fold
  bool owns_source = false;
  const u64 *c0 = nullptr, *c1 = nullptr;  // the step's input (the base level borrows the caller's codeword)
  std::unique_ptr<DevBuf> own0, own1, leaf_hashes, nodes;
  std::vector<u64> cap;   // host copy, cap_size digests
};

}  // namespace bj

struct bj_fri_oracles {
  bj_ctx* ctx = nullptr;
  uint32_t cap_size = 0;
  std::vector<bj::FriLevel> levels;      // base oracle + intermediate oracles
  std::vector<uint64_t> mono_c0, mono_c1;  // final monomial forms
  std::vector<uint64_t> challenges;        // (c0, c1) of the first challenge of every step (for tests / debugging)
};

using namespace bj;

extern "C" {

int32_t bj_query_leaf_elements(bj_ctx* ctx, const uint64_t* const* h_sources, uint32_t n_sources, uint32_t elems_per_leaf,
                               uint64_t n_leaves, const uint64_t* h_indices, uint32_t n_indices, uint64_t* h_out) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || !h_sources || !h_indices || !h_out || n_sources == 0 || elems_per_leaf == 0)
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_query_leaf_elements: bad argument");
  if (n_indices == 0) return BJ_OK;
  for (uint32_t i = 0; i < n_indices; i++)
    if (h_indices[i] >= n_leaves) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_query_leaf_elements: leaf index out of range");
  for (uint32_t i = 0; i < n_sources; i++)
    if (!h_sources[i]) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_query_leaf_elements: NULL source column");
  void *d_src, *d_idx;
  BJ_TRY(param_upload(ctx, h_sources, sizeof(u64*) * n_sources, &d_src));
  BJ_TRY(param_upload(ctx, h_indices, sizeof(u64) * n_indices, &d_idx));
  const size_t total = (size_t)n_indices * n_sources * elems_per_leaf;
  DevBuf out;
  BJ_TRY(out.alloc(ctx, sizeof(u64) * total));
  gather_leaves_kernel<<<(unsigned)((total + 255) / 256), 256, 0, ctx->stream>>>((const u64* const*)d_src, n_sources, elems_per_leaf,
                                                                                 (const u64*)d_idx, n_indices, out.u());
  BJ_LAUNCH_CHECK(ctx);
  BJ_CUDA(ctx, cudaMemcpyAsync(h_out, out.p, sizeof(u64) * total, cudaMemcpyDeviceToHost, ctx->stream));
  BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return BJ_OK;
}

int32_t bj_merkle_paths(bj_ctx* ctx, const uint64_t* d_leaf_hashes, const uint64_t* d_nodes, uint64_t n_leaves,
                        uint32_t cap_size, const uint64_t* h_indices, uint32_t n_indices, uint64_t* h_out) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || !d_leaf_hashes || !h_indices || (!h_out && n_indices) || cap_size == 0 || n_leaves < cap_size)
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_merkle_paths: bad argument");
  u32 depth = 0;
  while ((n_leaves >> depth) > cap_size) depth++;
  for (uint32_t i = 0; i < n_indices; i++)
    if (h_indices[i] >= n_leaves) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_merkle_paths: leaf index out of range");
  if (n_indices == 0 || depth == 0) return BJ_OK;
  if (!d_nodes) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_merkle_paths: d_nodes is NULL");
  void* d_idx;
  BJ_TRY(param_upload(ctx, h_indices, sizeof(u64) * n_indices, &d_idx));
  const size_t total = (size_t)n_indices * depth * 4;
  DevBuf out;
  BJ_TRY(out.alloc(ctx, sizeof(u64) * total));
  gather_paths_kernel<<<(unsigned)((total + 255) / 256), 256, 0, ctx->stream>>>((const u64*)d_leaf_hashes, (const u64*)d_nodes, n_leaves,
                                                                                depth, (const u64*)d_idx, n_indices, out.u());
  BJ_LAUNCH_CHECK(ctx);
  BJ_CUDA(ctx, cudaMemcpyAsync(h_out, out.p, sizeof(u64) * total, cudaMemcpyDeviceToHost, ctx->stream));
  BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return BJ_OK;
}

void bj_fri_oracles_free(bj_fri_oracles* o) {
  if (!o) return;
  bj::DeviceGuard device_guard(o->ctx);
  if (o->ctx) cudaStreamSynchronize(o->ctx->stream);
  delete o;
}

int32_t bj_do_fri(bj_ctx* ctx, bj_transcript* transcript, const uint64_t* d_c0, const uint64_t* d_c1, uint32_t log_full_size,
                  const uint32_t* schedule, uint32_t n_schedule, uint32_t log_lde, uint32_t cap_size,
                  bj_fri_oracles** out) {
  bj::DeviceGuard device_guard(ctx);
  return bj_do_fri_with_hasher(ctx, transcript, d_c0, d_c1, log_full_size, schedule, n_schedule, log_lde, cap_size, BJ_HASHER_POSEIDON2, out);
}

int32_t bj_do_fri_with_hasher(bj_ctx* ctx, bj_transcript* transcript, const uint64_t* d_c0, const uint64_t* d_c1, uint32_t log_full_size,
                              const uint32_t* schedule, uint32_t n_schedule, uint32_t log_lde, uint32_t cap_size, uint32_t hasher,
                              bj_fri_oracles** out) {
  bj::DeviceGuard device_guard(ctx);
  if (hasher > BJ_HASHER_KECCAK256) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_do_fri: unknown tree hasher");
  if (!ctx || !transcript || !d_c0 || !d_c1 || !schedule || n_schedule == 0 || !out || cap_size == 0 ||
      (cap_size & (cap_size - 1)) || log_full_size > 32 || log_lde > log_full_size)
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_do_fri: bad argument");
  *out = nullptr;
  u32 total_fold = 0;
  for (u32 i = 0; i < n_schedule; i++) {
    if (schedule[i] < 1 || schedule[i] > 3) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_do_fri: folds must be 1..3 (fri/mod.rs:205-206)");
    total_fold += schedule[i];
  }
  if (total_fold + log_lde > log_full_size) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_do_fri: final degree would be zero");
  std::unique_ptr<bj_fri_oracles> fo(new bj_fri_oracles());
  fo->ctx = ctx;
  fo->cap_size = cap_size;
  u64 kappa = gl::INV7;  // coset_inverse = multiplicative_generator^-1 (fri/mod.rs:194)
  const u64* cur0 = (const u64*)d_c0;
  const u64* cur1 = (const u64*)d_c1;
  u32 log_m = log_full_size;
  // sharded context: the codewords hold this rank's units only ([local unit][row], 1 / world of every vector); folds and
  // oracle subtrees are local (a fold of 2^k neighbours never leaves a unit), caps are assembled across the ranks so that all
  // of them draw the same challenges, and the last codeword (a few hundred elements) is gathered and interpolated everywhere
  const u32 world = comm_world(ctx);
  u32 log_world = 0;
  while ((1u << log_world) < world) log_world++;
  if (world > 1 && (log_lde != ctx->shard_log_lde || cap_size < std::max(1u << log_lde, world)))
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_do_fri: sharded FRI needs cap_size >= max(LDE factor, world) and the LDE factor of the shard");
  const u32 cap_local = cap_size / world;
  for (u32 i = 0; i < n_schedule; i++) {
    const u32 k = schedule[i];
    fo->levels.emplace_back();
    FriLevel& lv = fo->levels.back();
    lv.log_size = log_m - log_world;  // LOCAL size: queries address the local [coset][row] layout
    lv.log_fold = k;
    lv.c0 = cur0;
    lv.c1 = cur1;
    // oracle over the step's input: 2^k consecutive c0 values then the same 2^k c1 values per leaf (fri/mod.rs:173-187, 252-268)
    const u64 n_leaves = (1ull << (log_m - k)) / world;
    if (n_leaves < cap_local || cap_local == 0) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_do_fri: oracle smaller than the cap (schedule / cap mismatch)");
    lv.leaf_hashes.reset(new DevBuf());
    lv.nodes.reset(new DevBuf());
    BJ_TRY(lv.leaf_hashes->alloc(ctx, sizeof(u64) * 4 * n_leaves));
    BJ_TRY(lv.nodes->alloc(ctx, sizeof(u64) * 4 * (n_leaves - cap_local)));
    const uint64_t* srcs[2] = {(const uint64_t*)cur0, (const uint64_t*)cur1};
    BJ_TRY((hasher == BJ_HASHER_BLAKE2S ? bj_merkle_build_blake2s : hasher == BJ_HASHER_KECCAK256 ? bj_merkle_build_keccak256 : bj_merkle_build_poseidon2)(
        ctx, srcs, 2, n_leaves, 1u << k, cap_local, (uint64_t*)lv.leaf_hashes->p, (uint64_t*)lv.nodes->p));
    lv.cap.resize(4 * (size_t)cap_size);
    {
      std::vector<u64> local_cap(4 * (size_t)cap_local);
      const u64* cap_src = n_leaves == cap_local ? lv.leaf_hashes->u() : lv.nodes->u() + 4 * (n_leaves - 2 * (u64)cap_local);
      BJ_CUDA(ctx, cudaMemcpyAsync(local_cap.data(), cap_src, sizeof(u64) * 4 * cap_local, cudaMemcpyDeviceToHost, ctx->stream));
      BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
      BJ_TRY(comm_assemble_cap(ctx, local_cap.data(), cap_size, 1u << log_lde, lv.cap.data()));
    }
    bj_transcript_witness_merkle_tree_cap(transcript, (const uint64_t*)lv.cap.data(), cap_size);
    uint64_t alpha[2];
    alpha[0] = bj_transcript_get_challenge(transcript);
    alpha[1] = bj_transcript_get_challenge(transcript);
    fo->challenges.push_back(alpha[0]);
    fo->challenges.push_back(alpha[1]);
    // fold k times (interpolate_independent_cosets / interpolate_flattened_cosets)
    std::unique_ptr<DevBuf> n0(new DevBuf()), n1(new DevBuf());
    BJ_TRY(n0->alloc(ctx, (sizeof(u64) << (log_m - k)) / world));
    BJ_TRY(n1->alloc(ctx, (sizeof(u64) << (log_m - k)) / world));
    uint64_t kap = kappa;
    BJ_TRY(bj_fri_fold(ctx, (const uint64_t*)cur0, (const uint64_t*)cur1, log_m, k, alpha, &kap, (uint64_t*)n0->p, (uint64_t*)n1->p));
    kappa = kap;
    log_m -= k;
    cur0 = n0->u();
    cur1 = n1->u();
    // the folded vectors are the next level's source (or the final vector); keep them alive in the structure
    if (i + 1 < n_schedule) {
      // ownership moves to the next level when it is created; stash in this level for now
    }
    lv.own0 = std::move(n0);  // NOTE: own0/own1 of level i hold the OUTPUT of step i (input of step i+1)
    lv.own1 = std::move(n1);
  }
  // final vector -> monomials: bitreverse, iNTT on coset kappa^-1 (fri/mod.rs:312-321)
  const u64 fft_size = 1ull << log_m;
  DevBuf f0, f1;
  BJ_TRY(f0.alloc(ctx, sizeof(u64) * fft_size));
  BJ_TRY(f1.alloc(ctx, sizeof(u64) * fft_size));
  if (world == 1) {
    BJ_CUDA(ctx, cudaMemcpyAsync(f0.p, cur0, sizeof(u64) * fft_size, cudaMemcpyDeviceToDevice, ctx->stream));
    BJ_CUDA(ctx, cudaMemcpyAsync(f1.p, cur1, sizeof(u64) * fft_size, cudaMemcpyDeviceToDevice, ctx->stream));
  } else {
    // local [units / world][mc] (c0 | c1) from every rank -> global [units][mc]: unit slot kk of rank r is unit j below
    const u64 units = (1ull << log_lde) << ctx->shard.log_split;
    const u64 loc = fft_size / world, mc = fft_size / units, u_loc = units / world;
    if (mc == 0) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_do_fri: the last codeword is shorter than the units of the shard");
    DevBuf snd, rcv;
    BJ_TRY(snd.alloc(ctx, sizeof(u64) * 2 * loc));
    BJ_TRY(rcv.alloc(ctx, sizeof(u64) * 2 * fft_size));
    BJ_CUDA(ctx, cudaMemcpyAsync(snd.u(), cur0, sizeof(u64) * loc, cudaMemcpyDeviceToDevice, ctx->stream));
    BJ_CUDA(ctx, cudaMemcpyAsync(snd.u() + loc, cur1, sizeof(u64) * loc, cudaMemcpyDeviceToDevice, ctx->stream));
    BJ_TRY(comm_all_gather(ctx->comm, snd.u(), rcv.u(), 2 * loc));
    for (u32 r = 0; r < world; r++)
      for (u64 kk = 0; kk < u_loc; kk++) {
        const u64 j = ctx->shard.unit_of(r, kk);
        BJ_CUDA(ctx, cudaMemcpyAsync((u64*)f0.p + j * mc, rcv.u() + (u64)r * 2 * loc + kk * mc, sizeof(u64) * mc, cudaMemcpyDeviceToDevice, ctx->stream));
        BJ_CUDA(ctx, cudaMemcpyAsync((u64*)f1.p + j * mc, rcv.u() + (u64)r * 2 * loc + loc + kk * mc, sizeof(u64) * mc, cudaMemcpyDeviceToDevice, ctx->stream));
      }
    BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // snd / rcv are released below
  }
  const u64 coset = gl::inv(kappa);
  BJ_TRY(bj_bitreverse(ctx, (uint64_t*)f0.p, log_m, 1, fft_size));
  BJ_TRY(bj_bitreverse(ctx, (uint64_t*)f1.p, log_m, 1, fft_size));
  BJ_TRY(bj_intt_natural_to_natural(ctx, (uint64_t*)f0.p, log_m, 1, fft_size, coset));
  BJ_TRY(bj_intt_natural_to_natural(ctx, (uint64_t*)f1.p, log_m, 1, fft_size, coset));
  std::vector<uint64_t> h0(fft_size), h1(fft_size);
  BJ_CUDA(ctx, cudaMemcpyAsync(h0.data(), f0.p, sizeof(u64) * fft_size, cudaMemcpyDeviceToHost, ctx->stream));
  BJ_CUDA(ctx, cudaMemcpyAsync(h1.data(), f1.p, sizeof(u64) * fft_size, cudaMemcpyDeviceToHost, ctx->stream));
  BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  const u64 final_degree = fft_size >> log_lde;
  for (u64 i = final_degree; i < fft_size; i++)
    if (h0[i] != 0 || h1[i] != 0)  // the reference's self-check (fri/mod.rs:326-334) panics here
      BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_do_fri: folded codeword is not of low degree (input was not an LDE of a degree < n polynomial)");
  bj_transcript_witness_field_elements(transcript, h0.data(), final_degree);
  bj_transcript_witness_field_elements(transcript, h1.data(), final_degree);
  fo->mono_c0.assign(h0.begin(), h0.begin() + final_degree);
  fo->mono_c1.assign(h1.begin(), h1.begin() + final_degree);
  *out = fo.release();
  return BJ_OK;
}

uint32_t bj_fri_oracles_num_oracles(const bj_fri_oracles* o) { return o ? (uint32_t)o->levels.size() : 0; }
uint32_t bj_fri_oracles_num_monomials(const bj_fri_oracles* o) { return o ? (uint32_t)o->mono_c0.size() : 0; }

int32_t bj_fri_oracles_get_cap(const bj_fri_oracles* o, uint32_t oracle_idx, uint64_t* h_out) {
  if (!o || oracle_idx >= o->levels.size() || !h_out) return BJ_ERR_INVALID_ARG;
  memcpy(h_out, o->levels[oracle_idx].cap.data(), sizeof(uint64_t) * o->levels[oracle_idx].cap.size());
  return BJ_OK;
}
int32_t bj_fri_oracles_get_monomials(const bj_fri_oracles* o, uint64_t* h_c0, uint64_t* h_c1) {
  if (!o || !h_c0 || !h_c1) return BJ_ERR_INVALID_ARG;
  memcpy(h_c0, o->mono_c0.data(), sizeof(uint64_t) * o->mono_c0.size());
  memcpy(h_c1, o->mono_c1.data(), sizeof(uint64_t) * o->mono_c1.size());
  return BJ_OK;
}
int32_t bj_fri_oracles_get_challenges(const bj_fri_oracles* o, uint64_t* h_out) {
  if (!o || !h_out) return BJ_ERR_INVALID_ARG;
  memcpy(h_out, o->challenges.data(), sizeof(uint64_t) * o->challenges.size());
  return BJ_OK;
}

// OracleQuery for FRI oracle `oracle_idx` at base-tree index `base_index` (the index is shifted by the folds of the
// earlier steps exactly as in prover.rs:2236-2262): leaf elements (2 * 2^k u64) and the Merkle path.
int32_t bj_fri_oracles_query(bj_fri_oracles* o, uint32_t oracle_idx, uint64_t leaf_index, uint64_t* h_leaf_elements,
                             uint64_t* h_path, uint32_t* path_len) {
  return bj_fri_oracles_query_batch(o, oracle_idx, &leaf_index, 1, h_leaf_elements, h_path, path_len);
}

// the same for n leaves of one oracle with two device round trips in total: h_leaf_elements [n][2 * 2^k], h_paths [n][depth][4]
int32_t bj_fri_oracles_query_batch(bj_fri_oracles* o, uint32_t oracle_idx, const uint64_t* h_leaf_indices, uint32_t n_indices,
                                   uint64_t* h_leaf_elements, uint64_t* h_paths, uint32_t* path_len) {
  if (!o || oracle_idx >= o->levels.size() || !h_leaf_indices || !h_leaf_elements || !h_paths || !path_len) return BJ_ERR_INVALID_ARG;
  bj_ctx* ctx = o->ctx;
  bj::DeviceGuard device_guard(ctx);
  const FriLevel& lv = o->levels[oracle_idx];
  const u64 n_leaves = 1ull << (lv.log_size - lv.log_fold);
  const uint64_t* srcs[2] = {(const uint64_t*)lv.c0, (const uint64_t*)lv.c1};
  BJ_TRY(bj_query_leaf_elements(ctx, srcs, 2, 1u << lv.log_fold, n_leaves, h_leaf_indices, n_indices, h_leaf_elements));
  const u32 cap_local = o->cap_size / comm_world(ctx);  // the level's tree covers this rank's cosets
  u32 depth = 0;
  while ((n_leaves >> depth) > cap_local) depth++;
  *path_len = depth;
  return bj_merkle_paths(ctx, (const uint64_t*)lv.leaf_hashes->p, (const uint64_t*)lv.nodes->p, n_leaves, cap_local, h_leaf_indices, n_indices, h_paths);
}

}  // extern "C"
