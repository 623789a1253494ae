// Library context: one device + one stream, cached twiddle / coset-power tables, scratch arena.
// Replaces the reference's Worker (src/worker/mod.rs:5-87) as the "data-parallel executor" handle and caches
// what the reference recomputes on every stage (precompute_twiddles_for_fft, utils.rs:88-125).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <algorithm>
#include <atomic>
#include <mutex>
#include <string>
#include <vector>
#include "../../include/boojum_b200.h"
#include "gl64.cuh"

namespace bj {
using gl::u64;
using gl::u32;

struct PowTab {
  u64 coset;
  int log_n;
  u64 scale;
  int split;
  u64* lo;
  u64* hi;
  u64* full;  // s * c^i for all i < 2^log_n, or nullptr (built while the per-context budget lasts)
};

// a forward coset transform's twiddles with the coset folded in (ntt.cu get_twist_table): tab[2^r + G], 2^log_n entries
struct TwistTab {
  u64 coset;
  int log_n;
  u64* tab;
};

// Domain shard of a multi-GPU prover, the one owner of the layout rule.  The LDE domain is cut into UNITS u = j * B + p,
// B = 2^log_split: row block p (rows [p n / B, (p + 1) n / B) of the coset's bit-reversed row order) of coset j, so the flat
// index of a domain point is t = u * (n / B) + i'.  LDE-domain buffers of this context hold only the units
// u = first + k * 2^log_stride (k = 0, 1, ...), stored [local unit k][n / B rows]: a local flat index [k | i'] maps to the
// global index [k | first | i'].  log_split = 0 is the coset shard (a unit is a whole coset).  The first L * B units of any
// factor D >= L are the factor-L domain, so the quotient's wider domain shards the same way as the committed one.
struct CosetShard {
  uint32_t first = 0;
  uint32_t log_stride = 0;  // log2(world)
  uint32_t log_split = 0;   // log2(B), row blocks per coset
  __host__ __device__ __forceinline__ u64 global_index(u64 t_loc, int log_coset_len) const {
    if (log_stride == 0) return t_loc;
    const int lu = log_coset_len - (int)log_split;
    const u64 i = t_loc & ((1ull << lu) - 1);
    const u64 k = t_loc >> lu;
    return ((((k << log_stride) | first)) << lu) | i;
  }
  // global unit held by `rank` in its local slot k
  __host__ __device__ __forceinline__ u64 unit_of(u64 rank, u64 k) const { return (k << log_stride) | rank; }
  __host__ __device__ __forceinline__ u64 global_unit(u64 k) const { return unit_of(first, k); }
  // how many units of the first `cosets` (power of two) global cosets are local
  __host__ __device__ __forceinline__ u64 local_units(u64 cosets) const {
    const u64 stride = 1ull << log_stride, group = cosets << log_split;
    if (group >= stride) return group >> log_stride;
    return first < group ? 1 : 0;
  }
  // local points of the first `cosets` cosets of 2^log_coset_len rows
  __host__ __device__ __forceinline__ u64 local_points(u64 cosets, int log_coset_len) const {
    return local_units(cosets) << (log_coset_len - (int)log_split);
  }
  // rank that holds the global flat index t, and t's index in that rank's local layout
  __host__ __device__ __forceinline__ u32 owner(u64 t, int log_coset_len) const {
    return (u32)((t >> (log_coset_len - (int)log_split)) & ((1ull << log_stride) - 1));
  }
  __host__ __device__ __forceinline__ u64 owner_index(u64 t, int log_coset_len) const {
    const int lu = log_coset_len - (int)log_split;
    return (((t >> lu) >> log_stride) << lu) | (t & ((1ull << lu) - 1));
  }
  // shift sigma of global unit u on the factor-2^log_lde LDE of 2^log_n rows: its points are sigma * w_{n/B}^{bitrev(i')},
  // sigma = c_j * w_n^{bitrev_s(p)} with c_j = 7 * w_{nL}^{bitrev_L(j)} the shift of coset j
  __host__ u64 unit_shift(u64 u, u32 log_n, u32 log_lde) const {
    const u64 j = u >> log_split, p = u & ((1ull << log_split) - 1);
    u64 jr = 0, pr = 0;
    for (u32 b = 0; b < log_lde; b++) jr |= ((j >> b) & 1) << (log_lde - 1 - b);
    for (u32 b = 0; b < log_split; b++) pr |= ((p >> b) & 1) << (log_split - 1 - b);
    u64 s = gl::mul(gl::MULT_GEN, gl::pow(gl::omega(log_n + log_lde), jr));
    if (log_split) s = gl::mul(s, gl::pow(gl::omega(log_n), pr));
    return s;
  }
  // the window of one coset j of 2^log_cosets: a buffer that holds coset j alone is the local layout of rank j in a coset
  // shard of world 2^log_cosets, so the row-local kernels reading it get global_index(t) = j * n + t, the coset's x(t) and
  // vanishing constant, and z(omega x) inside the same coset, exactly as on the whole domain.  With log_split > 0 the window
  // is of one unit u of 2^log_units (a row block of a coset): the layout of rank u in a split shard of world 2^log_units, so
  // bj_lde evaluates that unit alone (the split shard's fold + row-block transform) and the kernels see its global indices.
  __host__ static CosetShard window(uint32_t log_units, uint32_t u, uint32_t log_split = 0) {
    CosetShard w;
    w.first = u;
    w.log_stride = log_units;
    w.log_split = log_split;
    return w;
  }
};

}  // namespace bj

struct bj_comm;

struct bj_ctx {
  int device = 0;
  bj_comm* comm = nullptr;  // communicator of a coset-sharded multi-GPU prover (comm.cu); nullptr = single GPU
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  std::string last_error;
  // bit-reversed twiddle tables tab[k] = w^bitrev(k); prefix property makes one table serve all sizes
  bj::u64* tw_fwd = nullptr;
  bj::u64* tw_inv = nullptr;
  int tw_log = 0;  // tables hold 2^(tw_log-1) entries
  std::vector<bj::PowTab> pow_cache;
  std::vector<bj::TwistTab> twist_cache;
  size_t pow_full_bytes = 0;  // bytes held by the full power tables of pow_cache and the tables of twist_cache
  void* scratch = nullptr;
  size_t scratch_bytes = 0;
  void* ptr_table = nullptr;  // device copy of host pointer arrays (Merkle sources)
  size_t ptr_table_bytes = 0;
  // host-buffer entry points: auxiliary copy streams + device staging ring (created on first use)
  bool copy_streams_ready = false;
  cudaStream_t h2d_stream = nullptr, d2h_stream = nullptr;
  cudaEvent_t ev_up[3] = {}, ev_done[3] = {}, ev_down[3] = {};
  void* host_ring = nullptr;
  size_t host_ring_bytes = 0;
  // witness slot sets (witness_stream.cu): the copy stream their uploads run on, created by the first slot set (a lane's by
  // its first slot set, destroyed with the lane)
  cudaStream_t witness_stream = nullptr;
  // slot sets alive on this context and the pool bytes they count: a parent's sets their full bj_witness_slots_bytes, a
  // lane's sets out[0] of bj_witness_slots_bytes_split.  On a parent, lane_witness_* sums the sets of all its lanes.  A lane's
  // fields and its parent's lane_witness_* are read and written under the parent's tables_mu.
  uint32_t witness_sets = 0;
  uint64_t witness_set_bytes = 0;
  uint32_t lane_witness_sets = 0;
  uint64_t lane_witness_set_bytes = 0;
  void* param_arena = nullptr;  // bump arena for small per-call parameter blocks
  size_t param_off = 0;
  uint64_t launches = 0;  // kernels launched by this library through this context
  int sm_count = 132;
  bool ntt_attr_set = false;
  std::vector<void*> attr_done;  // kernels whose smem attributes are set on this device
  int ntt_use_v2 = 1;            // BJ_NTT_V2=0 forces the generic pass kernel
  int ntt_col_fastest = -1;      // BJ_NTT_COL_FASTEST: tile passes run column-fastest, -1 by the rule of launch_pass, else bit 0 front, bit 1 last
  int ntt_max_tile_log = 13;  // tunables (env BJ_NTT_*)
  int ntt_pass1_w = -1;
  int ntt_chunk_mb = 0;
  int ntt_full_pow = 1;          // BJ_NTT_FULL_POW=0 keeps the two-level coset power tables only (no expanded, no twisted table)
  int ntt_twist = 1;             // BJ_NTT_TWIST=0: forward coset transforms scale on load instead of using twisted twiddles
  uint32_t one = 1;              // a 1 the compiler cannot see (passed as a kernel parameter): additions written as multiply-adds by it issue on the FMA pipe (blake2s.cu)
  int gate_peephole = 15;          // BJ_GATE_PEEPHOLE: bit 0 = alias x*1 / x+0 / x*0, 1 = multiply-add fusion, 2 = linear combinations, 3 = pushing steps (gates.cu)
  int gate_points_per_thread = 0;  // BJ_GATE_POINTS_PER_THREAD=1|2|4: force the gate interpreter's points per thread (0: by size)
  int ntt_l2_persist = 1;        // BJ_NTT_L2_PERSIST=0: do not pin the coset-power table in L2 during the scaled pass
  bool l2_limit_set = false;
  size_t l2_persist_bytes = 0;   // L2 set aside for that table: 3/8 of the device's L2, within its persisting maximum
  size_t l2_window_max = 0;      // largest access-policy window the device accepts
  int ntt_bulk = 0;              // BJ_NTT_BULK=1: experiment, bulk-copy (TMA) staged contiguous pass (ntt_v2.cuh)
  cudaMemPool_t pool = nullptr;  // private stream-ordered pool of the prover driver (keeps freed blocks: no OS round trips per proof)
  bj::CosetShard shard;  // bj_ctx_set_coset_shard / bj_ctx_set_domain_shard; default = the whole domain
  uint32_t shard_log_lde = 0;  // LDE factor the shard was declared for (locates the coset bits of flat indices)
  uint64_t memory_limit = 0;   // bj_ctx_set_memory_limit: device bytes a proof may use (0: what is free when the setup is created)
  bool allow_recompute_plan = false;  // bj_ctx_allow_recompute_plan: bj_setup_create may fall back to the recompute plan (one GPU)
  bool allow_sharded_recompute_plan = false;  // bj_ctx_allow_sharded_recompute_plan: the same on a context with a communicator
  uint32_t max_row_blocks = 1;  // bj_ctx_set_max_row_blocks: row blocks per coset the one-GPU recompute plan may cut its units into
  unsigned long long* pow_best = nullptr;  // bj_pow_blake2s's one-word result, allocated on first use
  void* gate_program = nullptr;            // a long gate program's device copy (gates.cu), grown on demand, kept
  size_t gate_program_bytes = 0;
  // ---- lanes (bj_ctx_create_lane): contexts on the parent's device that prove against the parent's setups concurrently ----
  // One rule per piece of state, so that distinct lanes of one parent may run bj_prove from different host threads at once:
  //  - twiddles: the parent's.  A lane's tw_* view the parent's pair, read under the parent's tables_mu; a transform longer
  //    than that pair makes the lane build a private pair (own_twiddles, freed with the lane).  A lane never grows the
  //    parent's pair.  The parent grows its own pair under tables_mu and, while it has lanes, retires the replaced pair
  //    (tables_retired, freed with the parent) instead of freeing it, so a lane's view stays valid.
  //  - coset-power and twisted twiddle tables: the parent's pow_cache and twist_cache, shared.  Every lookup and insert, the parent's too, holds the parent's
  //    tables_mu.  A missing table is built on the caller's stream and, when a lane could read it, that stream is
  //    synchronised before the table is published, so a published table is complete.  While the parent has lanes its cache
  //    is never flushed: the 64-entry flush retires the tables instead.  The 3 GiB budget of full tables is the parent's.
  //  - scratch, parameter arena, long gate program buffer, pointer table, launch counter, kernel-attribute bookkeeping,
  //    stream, pool, proof-of-work word and last_error: the lane's own, touched by the lane's thread only.  All of them
  //    only grow, so after its first proof a lane allocates nothing outside its pool.
  //  - the persisting-L2 window: the device's carve-out is sized for the one coset-power table of one stream, so lanes do
  //    not pin (ntt_l2_persist = 0); N streams pinning N tables into one carve-out would only evict one another.
  //  - Poseidon2 round constants: device constant memory written once by bj_ctx_create; a lane does not rewrite them.
  //  - the setups of the parent are read only; bj_prove on a lane first waits for the setup's ready event.
  //  - witness slot sets created on a lane (witness_stream.cu) and the lane's witness_stream: the lane's own, touched by the
  //    lane's thread only.  Their buffers and pinned staging ring belong to the set and come from the lane's pool; a
  //    WitnessVec gather on the lane's copy stream reads the setup's u32 hint (the parent's pool), which
  //    bj_setup_attach_variables_hint refuses to replace while a lane's set is alive.  The counts of live sets (witness_sets,
  //    the parent's lane_witness_*) are kept under the parent's tables_mu, for the memory checks of the parent's thread.
  // Teardown: bj_ctx_destroy refuses a context with lanes alive, and a lane with slot sets alive; sets go first, then lanes.
  bj_ctx* parent = nullptr;       // a lane's parent (nullptr: a context of bj_ctx_create)
  std::atomic<uint32_t> lanes{0};  // lanes of this context alive
  std::mutex tables_mu;            // guards tw_*, pow_cache, twist_cache, pow_full_bytes, tables_retired, setups and the set counts (see above)
  std::vector<void*> tables_retired;
  bool own_twiddles = true;        // false while a lane's tw_* view the parent's pair
  std::vector<const bj_setup*> setups;  // setups alive on this context: bj_ctx_create_lane plans against them
};

#define BJ_FAIL(ctx, code, msg)          \
  do {                                   \
    if (ctx) (ctx)->last_error = (msg);  \
    return (code);                       \
  } while (0)

#define BJ_CUDA(ctx, expr)                                                                      \
  do {                                                                                          \
    cudaError_t _e = (expr);                                                                    \
    if (_e != cudaSuccess) {                                                                    \
      if (ctx) (ctx)->last_error = std::string(#expr) + ": " + cudaGetErrorString(_e);          \
      return BJ_ERR_CUDA;                                                                       \
    }                                                                                           \
  } while (0)

#define BJ_TRY(expr)                 \
  do {                               \
    int32_t _s = (expr);             \
    if (_s != BJ_OK) return _s;      \
  } while (0)

#define BJ_LAUNCH_CHECK(ctx)                                                              \
  do {                                                                                    \
    (ctx)->launches++;                                                                    \
    cudaError_t _e = cudaGetLastError();                                                  \
    if (_e != cudaSuccess) {                                                              \
      (ctx)->last_error = std::string("kernel launch: ") + cudaGetErrorString(_e);        \
      return BJ_ERR_CUDA;                                                                 \
    }                                                                                     \
  } while (0)

namespace bj {
// Every extern "C" entry that takes a context runs on THAT context's device whatever the caller's current device is (a
// process may hold contexts on several GPUs, or switch devices between calls); the caller's current device is restored.
struct DeviceGuard {
  int prev = -1;
  bool switched = false;
  explicit DeviceGuard(const bj_ctx* ctx) {
    if (!ctx) return;
    if (cudaGetDevice(&prev) != cudaSuccess) {
      cudaGetLastError();
      prev = -1;
    }
    if (prev != ctx->device) switched = cudaSetDevice(ctx->device) == cudaSuccess && prev >= 0;
  }
  ~DeviceGuard() {
    if (switched) cudaSetDevice(prev);
  }
  DeviceGuard(const DeviceGuard&) = delete;
  DeviceGuard& operator=(const DeviceGuard&) = delete;
};
int32_t ensure_scratch(bj_ctx* ctx, size_t bytes);
// collectives of the sharded prover (comm.cu); all no-ops / plain copies for a world of one
int32_t comm_all_gather(bj_comm* c, const u64* d_send, u64* d_recv, u64 n);
int32_t comm_all_gather_host(bj_comm* c, const u64* h_send, u64* h_recv, u64 n);
int32_t comm_all_gather_overlapped(bj_comm* c, const u64* d_send, u64* d_recv, u64 n, cudaEvent_t* done);
int32_t comm_wait(bj_comm* c, cudaEvent_t done);
int32_t comm_broadcast_host(bj_comm* c, u64* h_buf, u64 n, uint32_t root);
uint32_t comm_world(const bj_ctx* ctx);
uint32_t comm_rank(const bj_ctx* ctx);
// global cap (cap_size digests) of an oracle whose local tree (this rank's units [k][row]) ends in cap_size / world digests:
// cap node c of the global tree belongs to unit c / (cap_size / (L * B)) (leaf index = coset * n + row, proof.rs:89-91)
int32_t comm_assemble_cap(bj_ctx* ctx, const u64* h_local_cap, uint32_t cap_size, uint32_t lde_factor, u64* h_global_cap);
int32_t ensure_twiddles(bj_ctx* ctx, int log_n);
int32_t param_upload(bj_ctx* ctx, const void* host, size_t bytes, void** d_out);
}  // namespace bj
