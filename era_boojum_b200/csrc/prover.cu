// Host driver of the five-round IOP: the role of CSReferenceAssembly::prove_cpu_basic
// (src/cs/implementations/prover.rs:153-2269) and of the setup materialisation that feeds it (setup.rs:1093-1255), for
// circuits whose gates live on general-purpose columns, with the optional log-derivative lookup argument over specialised
// columns (table id in a constant column).  Plain host C++ over the device entry points of this library: every heavy step
// is one of the bj_* kernels; the transcript, the FRI schedule, query-index derivation and proof assembly stay on the host
// exactly as in the reference.  The proof is handed back in the reference's serde_json shape (proof.rs:57-143), so that a
// Rust shim can `serde_json::from_str::<Proof<..>>` it.
//
// Round structure (prover.rs line numbers):
//   1  witness LDE + oracle                      :313-353        4  openings at z, z*omega, 0             :1501-1802
//   2  copy-permutation / lookup polys + oracle  :360-554        5  DEEP combination + FRI                :1828-2102
//   3  quotient, interpolation, chunks + oracle  :560-1495       6  queries                               :2161-2266
#include <chrono>
#include <cstring>
#include <functional>
#include <memory>
#include <string>
#include <vector>
#include "ctx.hpp"

namespace bj {

// stream-ordered device buffer
struct DevMem {
  bj_ctx* ctx = nullptr;
  u64* p = nullptr;
  DevMem() = default;
  DevMem(const DevMem&) = delete;
  DevMem& operator=(const DevMem&) = delete;
  ~DevMem() { release(); }
  void release() {
    if (p) cudaFreeAsync(p, ctx->stream);
    p = nullptr;
  }
  int32_t alloc(bj_ctx* c, size_t n_u64) {
    release();
    ctx = c;
    const size_t bytes = sizeof(u64) * (n_u64 ? n_u64 : 1);
    const cudaError_t e = c->pool ? cudaMallocFromPoolAsync((void**)&p, bytes, c->pool, c->stream) : cudaMallocAsync((void**)&p, bytes, c->stream);
    if (e != cudaSuccess) {
      cudaGetLastError();
      p = nullptr;
      uint64_t used = 0;
      if (c->pool) cudaMemPoolGetAttribute(c->pool, cudaMemPoolAttrUsedMemCurrent, &used);
      BJ_FAIL(c, BJ_ERR_OOM, "prover: device allocation of " + std::to_string(bytes) + " bytes failed (" + std::to_string(used) + " bytes of the pool in use)");
    }
    return BJ_OK;
  }
};

// a Merkle oracle over LDE columns
struct Oracle {
  std::vector<const uint64_t*> cols;
  DevMem leaf_hashes, nodes;
  u64 n_leaves = 0;
  u32 cap_size = 0;
  std::vector<u64> cap;  // host, 4 * cap_size
};

int32_t merkle_nodes_poseidon2(bj_ctx* ctx, const u64* d_leaf_hashes, u64 n_leaves, u32 cap_size, u64* d_nodes);  // poseidon2.cu
int32_t merkle_nodes_blake2s(bj_ctx* ctx, const u64* d_leaf_hashes, u64 n_leaves, u32 cap_size, u64* d_nodes);    // blake2s.cu
int32_t merkle_nodes_keccak256(bj_ctx* ctx, const u64* d_leaf_hashes, u64 n_leaves, u32 cap_size, u64* d_nodes);  // keccak.cu

// the tree hasher's whole build (leaves, then node levels down to the cap) and its node phase alone
using MerkleBuild = int32_t (*)(bj_ctx*, const uint64_t* const*, uint32_t, uint64_t, uint32_t, uint32_t, uint64_t*, uint64_t*);
using MerkleNodes = int32_t (*)(bj_ctx*, const u64*, u64, u32, u64*);
static MerkleBuild merkle_build(u32 hasher) {
  return hasher == BJ_HASHER_BLAKE2S ? bj_merkle_build_blake2s : hasher == BJ_HASHER_KECCAK256 ? bj_merkle_build_keccak256 : bj_merkle_build_poseidon2;
}
static MerkleNodes merkle_nodes(u32 hasher) {
  return hasher == BJ_HASHER_BLAKE2S ? merkle_nodes_blake2s : hasher == BJ_HASHER_KECCAK256 ? merkle_nodes_keccak256 : merkle_nodes_poseidon2;
}

// the cap of a built tree, assembled over the ranks of a sharded context
static int32_t oracle_cap(bj_ctx* ctx, Oracle& o, u32 cap_global, u32 lde_factor) {
  const u64 n_leaves = o.n_leaves;
  const u32 cap_size = o.cap_size;
  std::vector<u64> local(4 * (size_t)cap_size);
  const u64* src = n_leaves == cap_size ? o.leaf_hashes.p : o.nodes.p + 4 * (n_leaves - 2 * (u64)cap_size);
  BJ_CUDA(ctx, cudaMemcpyAsync(local.data(), src, sizeof(u64) * 4 * cap_size, cudaMemcpyDeviceToHost, ctx->stream));
  BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  o.cap.resize(4 * (size_t)cap_global);
  return comm_assemble_cap(ctx, local.data(), cap_global, lde_factor, o.cap.data());
}

// n_leaves / cap_size are GLOBAL; on a coset-sharded context the tree covers this rank's cosets (n_leaves / world leaves,
// cap_size / world local cap nodes - same depth), and o.cap is the assembled global cap (lde_factor locates the cosets).
static int32_t oracle_build(bj_ctx* ctx, Oracle& o, u64 n_leaves, u32 cap_size, u32 hasher, u32 lde_factor) {
  const u32 world = comm_world(ctx);
  const u32 cap_global = cap_size;
  n_leaves /= world;
  cap_size /= world;
  o.n_leaves = n_leaves;
  o.cap_size = cap_size;
  if (cap_size == 0 || n_leaves < cap_size) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "prover: oracle smaller than the cap");
  BJ_TRY(o.leaf_hashes.alloc(ctx, 4 * n_leaves));
  BJ_TRY(o.nodes.alloc(ctx, 4 * (n_leaves - cap_size)));
  BJ_TRY(merkle_build(hasher)(ctx, o.cols.data(), (u32)o.cols.size(), n_leaves, 1, cap_size, (uint64_t*)o.leaf_hashes.p, (uint64_t*)o.nodes.p));
  return oracle_cap(ctx, o, cap_global, lde_factor);
}

// natural-order columns of stride n: `cnt` of them from `p`
struct NatSpan {
  const uint64_t* p;
  u32 cnt;
};

// streamed and recompute plans: while the kernels of unit u run on a buffer that holds unit u alone, the context's shard is
// the window of unit u; the caller's shard comes back on every exit path
struct ShardWindow {
  bj_ctx* ctx;
  CosetShard saved;
  ShardWindow(bj_ctx* c, u32 log_units, u32 u, u32 log_split) : ctx(c), saved(c->shard) { c->shard = CosetShard::window(log_units, u, log_split); }
  ~ShardWindow() { ctx->shard = saved; }
  ShardWindow(const ShardWindow&) = delete;
  ShardWindow& operator=(const ShardWindow&) = delete;
};

// recompute plan: `cnt` columns of `in` (stride n; natural order, or monomials with from_monomials) evaluated on local unit k of
// the committed domain alone into `out` (stride n >> split, the unit's rows).  One GPU: coset k (bj_lde_cosets), or, with
// 2^rb row blocks per coset, row block k % 2^rb of coset k >> rb.  Sharded (rb = 0): the rank's global unit k.  A row block
// or a sharded unit goes through bj_lde under the unit's window - the same coset transform, or fold + row-block transform,
// as the resident sharded plan's LDE writes into local slot k, so every value is bit-identical to the resident plan's.
static int32_t lde_unit(bj_ctx* ctx, const uint64_t* in, uint64_t* out, u32 log_n, u32 log_l, u32 cnt, u64 k, int32_t from_monomials, u32 rb = 0) {
  if (cnt == 0) return BJ_OK;
  const u32 split = ctx->shard.log_split + rb;
  if (comm_world(ctx) == 1 && split == 0) return bj_lde_cosets(ctx, in, 1ull << log_n, out, log_n, log_l, (u32)k, (u32)k + 1, cnt, from_monomials);
  ShardWindow window(ctx, log_l + split, (u32)ctx->shard.global_unit(k), split);  // one GPU: global_unit(k) = k
  return bj_lde(ctx, in, 1ull << log_n, out, log_n, log_l, cnt, from_monomials);
}

// recompute plan: the tree of oracle_build over the LDE at factor L of the spans' columns, built one committed unit at a time
// (a coset on one GPU or a coset shard, a row block of nb = n / B rows on a split shard or, with rb > 0, on one GPU cutting
// each coset into B = 2^rb row blocks).  Local unit k is leaves [k nb, (k + 1) nb) of this context's tree: its columns are
// evaluated into an nb-row scratch per column (lde_unit), its leaves hashed into their slice, and the node levels are built
// once the leaf array is complete.  A unit is a whole subtree, so the tree, its local cap and the cap exchange are those of
// oracle_build.  o.cols are the natural columns.
static int32_t oracle_build_by_coset(bj_ctx* ctx, Oracle& o, const std::vector<NatSpan>& spans, u32 log_n, u32 log_l, u32 cap_size, u32 hasher,
                                     u32 rb) {
  const u32 world = comm_world(ctx);
  const u64 n = 1ull << log_n, nb = n >> (ctx->shard.log_split + rb), units = ctx->shard.local_units(1ull << log_l) << rb, n_leaves = units * nb;
  o.cols.clear();
  for (const NatSpan& sp : spans)
    for (u32 i = 0; i < sp.cnt; i++) o.cols.push_back(sp.p + (size_t)i * n);
  o.n_leaves = n_leaves;
  o.cap_size = cap_size / world;
  if (o.cap_size == 0 || n_leaves < o.cap_size) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "prover: oracle smaller than the cap");
  BJ_TRY(o.leaf_hashes.alloc(ctx, 4 * n_leaves));
  {
    DevMem ev;
    BJ_TRY(ev.alloc(ctx, o.cols.size() * nb));
    std::vector<const uint64_t*> on_unit(o.cols.size());
    for (size_t i = 0; i < on_unit.size(); i++) on_unit[i] = (const uint64_t*)ev.p + i * nb;
    for (u64 k = 0; k < units; k++) {
      size_t c0 = 0;
      for (const NatSpan& sp : spans) {
        BJ_TRY(lde_unit(ctx, sp.p, (uint64_t*)ev.p + c0 * nb, log_n, log_l, sp.cnt, k, 0, rb));
        c0 += sp.cnt;
      }
      // the leaf phase alone: a tree of nb leaves whose cap is its leaves
      BJ_TRY(merkle_build(hasher)(ctx, on_unit.data(), (u32)on_unit.size(), nb, 1, (u32)nb, (uint64_t*)o.leaf_hashes.p + 4 * (size_t)k * nb, nullptr));
    }
  }
  BJ_TRY(o.nodes.alloc(ctx, 4 * (n_leaves - o.cap_size)));
  BJ_TRY(merkle_nodes(hasher)(ctx, o.leaf_hashes.p, n_leaves, o.cap_size, o.nodes.p));
  return oracle_cap(ctx, o, cap_size, 1u << log_l);
}

// LDE of trace-domain columns (Lagrange values, natural order) onto this context's cosets.  One GPU: bj_lde.  Sharded: the
// two natural partitions meet here (SURVEY.md 8e) - the iNTT is independent per COLUMN, so rank r interpolates the block of
// columns [r * per, (r + 1) * per) only, ONE all-gather hands every rank all the monomials (8 * n * n_cols bytes in total), and
// each rank then evaluates them on its own cosets.  Without it every rank would repeat all the iNTTs (1/9 of the LDE work,
// which stops scaling).  Columns must be contiguous (stride n).
static int32_t lde_columns(bj_ctx* ctx, const uint64_t* d_in, uint64_t* d_out, u32 log_n, u32 log_l, u32 n_cols) {
  const u32 world = comm_world(ctx), rank = comm_rank(ctx);
  const u64 n = 1ull << log_n;
  if (world == 1 || n_cols < 2) return bj_lde(ctx, d_in, n, d_out, log_n, log_l, n_cols, 0);
  // software pipeline over groups of columns: while the all-gather of group g travels over NVLink (auxiliary stream), this
  // rank interpolates its share of group g + 1 and evaluates group g - 1 on its cosets
  const u64 out_stride = (n << log_l) / world;
  const u32 group = std::max<u32>(world, ((n_cols + 3) / 4 + world - 1) / world * world);  // <= 4 groups, a multiple of world
  struct Group {
    u32 c0, cnt, per;
    DevMem mono;
    cudaEvent_t gathered = nullptr;
  };
  std::vector<std::unique_ptr<Group>> groups;
  for (u32 c0 = 0; c0 < n_cols; c0 += group) {
    groups.emplace_back(new Group());
    groups.back()->c0 = c0;
    groups.back()->cnt = std::min(group, n_cols - c0);
    groups.back()->per = (groups.back()->cnt + world - 1) / world;
  }
  auto start = [&](Group& g) -> int32_t {
    BJ_TRY(g.mono.alloc(ctx, (size_t)world * g.per * n));
    const u32 first = std::min(rank * g.per, g.cnt), cnt = std::min(g.per, g.cnt - first);
    u64* mine = g.mono.p + (size_t)rank * g.per * n;
    if (cnt) {
      BJ_CUDA(ctx, cudaMemcpyAsync(mine, d_in + (size_t)(g.c0 + first) * n, sizeof(u64) * cnt * n, cudaMemcpyDeviceToDevice, ctx->stream));
      BJ_TRY(bj_intt_natural_to_natural(ctx, (uint64_t*)mine, log_n, cnt, n, 1));
    }
    if (cnt < g.per) BJ_CUDA(ctx, cudaMemsetAsync(mine + (size_t)cnt * n, 0, sizeof(u64) * (g.per - cnt) * n, ctx->stream));
    // in place: my block is my slot of the gathered array
    return comm_all_gather_overlapped(ctx->comm, mine, g.mono.p, (u64)g.per * n, &g.gathered);
  };
  auto finish = [&](Group& g) -> int32_t {
    BJ_TRY(comm_wait(ctx->comm, g.gathered));
    BJ_TRY(bj_lde(ctx, (const uint64_t*)g.mono.p, n, d_out + (size_t)g.c0 * out_stride, log_n, log_l, g.cnt, 1));
    g.mono.release();
    return BJ_OK;
  };
  for (size_t i = 0; i < groups.size(); i++) {
    BJ_TRY(start(*groups[i]));
    if (i) BJ_TRY(finish(*groups[i - 1]));
  }
  return finish(*groups.back());
}

int32_t copy_permutation_stage2_sharded(bj_ctx* ctx, const uint64_t* const* h_variable_cols, const uint64_t* const* h_sigma_cols, u32 n_cols,
                                        const uint64_t* h_non_residues, gl::e2 beta, gl::e2 gamma, u32 log_n, u32 chunk_size, u64* d_out);  // stage2.cu

struct GateCopy {
  std::vector<bj_gate_relation> relations;
  std::vector<bj_gate_index> writes;
  std::vector<uint8_t> path;
};

static inline void json_u64(std::string& s, u64 v) {  // decimal digits straight into the string (std::to_string allocates)
  char buf[24];
  int k = 24;
  do {
    buf[--k] = (char)('0' + v % 10);
    v /= 10;
  } while (v);
  s.append(buf + k, 24 - k);
}
static void json_u64_list(std::string& s, const u64* v, size_t n) {
  s += '[';
  for (size_t i = 0; i < n; i++) {
    if (i) s += ',';
    json_u64(s, v[i]);
  }
  s += ']';
}
// TreeHasher::Output in serde form: Poseidon2 digests are [GoldilocksField; 4] = 4 numbers; Blake2s256 / Keccak256 digests are
// [u8; 32] = 32 numbers (src/cs/oracle/mod.rs:180, 245).  Internally every digest is kept as 4 little-endian u64.
static void json_digests(std::string& s, const u64* v, size_t n_digests, bool as_bytes) {
  s += '[';
  for (size_t i = 0; i < n_digests; i++) {
    if (i) s += ',';
    if (!as_bytes) {
      json_u64_list(s, v + 4 * i, 4);
      continue;
    }
    s += '[';
    for (int b = 0; b < 32; b++) {
      if (b) s += ',';
      json_u64(s, (v[4 * i + b / 8] >> (8 * (b % 8))) & 0xff);
    }
    s += ']';
  }
  s += ']';
}
static void json_ext_list(std::string& s, const std::vector<gl::e2>& v) {
  s += '[';
  for (size_t i = 0; i < v.size(); i++) {
    if (i) s += ',';
    s += "{\"coeffs\":[";
    json_u64(s, v[i].c0);
    s += ',';
    json_u64(s, v[i].c1);
    s += "],\"_marker\":null}";
  }
  s += ']';
}

struct QueryAnswer {
  std::vector<u64> leaf_elements;
  std::vector<u64> path;  // 4 * depth
};

// ---- memory plan: the one owner of what bj_setup_create + bj_prove hold on the device at their peak ----
// Three plans.  RESIDENT keeps every LDE column on all D = max(L, Q) cosets until the proof is done.  COMPACT (one GPU, Q < L)
// keeps only the first Q cosets of the setup, witness and stage-2 columns once their trees are built: the quotient reads
// cosets [0, Q) and the openings coset 0, so cosets [Q, L) are read by DEEP and the query answers only, and those two
// recompute them from the natural-order columns, a chunk of columns and one coset at a time.  The quotient oracle stays
// resident.  STREAMED (Q > L) evaluates the setup, witness and stage-2 columns on the committed cosets [0, L) only:
// cosets [L, Q) are read by the quotient alone, which evaluates every column it reads onto one such coset at a time into a
// coset-sized scratch, from the natural-order columns (the stage-2 ones are kept for it).  On a sharded context each rank
// keeps its units of the committed cosets and evaluates its own units of cosets [L, Q), one unit (a coset, or a row block
// of one on a split shard, with its z(omega x) columns) at a time into a unit-sized scratch.  RECOMPUTE (one GPU, any Q and
// L, opt-in; one GPU or sharded) keeps no coset of the setup, witness and stage-2 columns at all: their trees are built one committed coset at a
// time (oracle_build_by_coset), the quotient runs the streamed plan's unit loop with no kept unit, the openings rebuild coset
// 0 and DEEP and the queries cosets [0, L), all from the natural-order columns a chunk at a time.  On a sharded context
// (opt-in of its own) every rank does the same on its own units: its committed units for the trees, DEEP and the queries it
// answers, its local slot 0 for the openings, its quotient units for the quotient.  On one GPU the recompute plan may cut
// every coset into B = 2^rb row blocks (bj_ctx_set_max_row_blocks): the trees and the quotient then walk the L * B and Q * B
// row-block units the way a split shard walks its own, so their scratch is a row block of every column instead of a coset;
// the openings, DEEP and the queries rebuild whole cosets a chunk of columns at a time as before.  The plan replays the
// driver's stream-ordered pool allocations in order (pool_peak) and adds what the library keeps outside the pool
// (library_reserve): twiddles, coset-power tables and the NTT scratch.
enum MemoryPlan : u32 {
  PLAN_RESIDENT = BJ_PLAN_RESIDENT,
  PLAN_COMPACT = BJ_PLAN_COMPACT,
  PLAN_STREAMED = BJ_PLAN_STREAMED,
  PLAN_RECOMPUTE = BJ_PLAN_RECOMPUTE
};
struct ProofShape {
  u32 V, C, T, W, n_s2, Q, L, log_n, log_l, log_d, log_q, world, split, cap, n_queries, sched_len;
  u32 rb = 0;  // one GPU, recompute plan: log2 of the row blocks per coset its trees and quotient are built in
  u32 sched[32];
  u64 n;
  bool lk;
  u32 nat_cols() const { return V + C + T + W + n_s2; }  // natural-order columns a compact / streamed / recompute proof recomputes from
};

static int32_t proof_shape(const bj_circuit& c, u32 world, ProofShape* s) {
  auto lg = [](u32 x) { u32 l = 0; while ((1u << l) < x) l++; return l; };
  s->V = c.num_variables;
  s->C = c.num_constants;
  s->lk = c.lookup_width != 0;
  s->T = s->lk ? c.lookup_width + 1 : 0;
  s->W = s->V + (s->lk ? 1 : 0);
  s->Q = c.quotient_degree;
  s->L = c.fri_lde_factor;
  const u32 n_partial = (s->V + s->Q - 1) / s->Q - 1;
  s->n_s2 = 2 + 2 * n_partial + (s->lk ? 2 * (c.lookup_num_repetitions + 1) : 0);
  s->log_n = c.log_n;
  s->log_l = lg(s->L);
  s->log_q = lg(s->Q);
  s->log_d = std::max(s->log_l, s->log_q);
  s->world = world;
  s->split = world > s->L ? lg(world) - s->log_l : 0;
  s->cap = c.merkle_tree_cap_size;
  s->n = 1ull << c.log_n;
  u32 new_pow = 0, fd = 0;
  return bj_compute_fri_schedule(c.security_level, c.merkle_tree_cap_size, c.pow_bits, s->log_l, c.log_n, &new_pow, &s->n_queries, s->sched,
                                 &s->sched_len, &fd);
}

// bytes the context's pool counts as used for one allocation of n u64 (the requested size: DevMem asks for at least one)
static inline u64 pool_bytes(u64 n_u64) { return sizeof(u64) * std::max<u64>(n_u64, 1); }

struct Ledger {
  u64 cur = 0, peak = 0;
  void add(u64 n_u64) {
    cur += pool_bytes(n_u64);
    peak = std::max(peak, cur);
  }
  void sub(u64 n_u64) { cur -= pool_bytes(n_u64); }
  void tree(const ProofShape& s) {  // oracle_build: leaf hashes, then the nodes
    const u64 leaves = (s.n << s.log_l) / s.world;
    add(4 * leaves);
    add(4 * (leaves - s.cap / s.world));
  }
  void tree_by_coset(const ProofShape& s, u64 cols) {  // oracle_build_by_coset: leaf hashes, one unit of the columns, then the nodes
    const u64 leaves = (s.n << s.log_l) / s.world, unit_rows = s.n >> (s.split + s.rb);
    add(4 * leaves);
    add(cols * unit_rows);
    sub(cols * unit_rows);
    add(4 * (leaves - s.cap / s.world));
  }
  void lde_groups(const ProofShape& s, u32 cols) {  // lde_columns on a sharded context: at most two column groups of monomials at once
    const u64 w = s.world;
    if (w == 1 || cols < 2) return;
    const u64 group = std::max<u64>(w, ((cols + 3) / 4 + w - 1) / w * w), mono = w * ((group + w - 1) / w) * s.n;
    const int alive = cols > group ? 2 : 1;
    for (int i = 0; i < alive; i++) add(mono);
    for (int i = 0; i < alive; i++) sub(mono);
  }
};

// Every DevMem of bj_setup_create and bj_prove (and the FRI / query buffers of fri_driver.cu) is replayed by pool_peak in the
// same order: the committed column sets' steps by ColumnSet::replay, beside them, the rest by pool_peak itself.  A new
// allocation on either side must be added on the other, or the plan no longer bounds the pool (tests/test_gpu_memory_budget.py
// pins the pool's high-water mark to the plan).

// What one committed oracle (the setup, the witness or stage 2) keeps under the memory plan: its natural-order columns
// (`nat`, stride n, in the oracle's column order), the LDE the plan keeps of them and the tree.  tree.cols are the kept LDE
// columns (this context's units of the D cosets, of the L committed ones on the streamed plan, of cosets [0, Q) once the
// compact plan has repacked them; stride `stride`) or, on the recompute plan, the natural-order columns themselves.  The LDE
// is held in one allocation for all the spans (the setup) or one per span (the witness's variables and multiplicities, stage
// 2), cut into column groups on the compact plan so that the repack to cosets [0, Q) frees each group as soon as it is copied
// (the transient is one group's kept columns, not the oracle's).
struct ColumnSet {
  MemoryPlan plan = PLAN_RESIDENT;
  std::vector<NatSpan> nat;
  bool one_allocation = false;
  u32 log_n = 0, log_l = 0, log_d = 0, Q = 0, rb = 0;
  std::vector<std::unique_ptr<DevMem>> full, kept;  // the LDE's allocations, and on the compact plan their repacked copies
  std::vector<u32> alloc_cols;                      // columns of each allocation
  u64 stride = 0;
  Oracle tree;

  struct Piece {
    u32 span, first, cnt;
  };
  static constexpr u32 COMPACT_GROUPS = 4;
  // the LDE's allocations in order, each as the runs of span columns it holds
  static std::vector<std::vector<Piece>> allocations(const std::vector<u32>& span_cols, bool one_allocation, MemoryPlan plan) {
    std::vector<std::vector<Piece>> a;
    for (u32 i = 0; i < span_cols.size(); i++) {
      const u32 cnt = span_cols[i], per = plan == PLAN_COMPACT && !one_allocation ? (cnt + COMPACT_GROUPS - 1) / COMPACT_GROUPS : cnt;
      for (u32 c0 = 0; c0 < cnt; c0 += per) {
        if (a.empty() || !one_allocation) a.emplace_back();
        a.back().push_back({i, c0, std::min(per, cnt - c0)});
      }
    }
    return a;
  }
  static u64 cols_of(const std::vector<Piece>& a) {
    u64 cols = 0;
    for (const Piece& p : a) cols += p.cnt;
    return cols;
  }
  // stride of an LDE column as first evaluated: D cosets, or on the streamed plan the L committed ones
  static u64 evaluated_stride(MemoryPlan plan, u64 n, u32 log_l, u32 log_d, u32 world) { return (n << (plan == PLAN_STREAMED ? log_l : log_d)) / world; }

  void init(MemoryPlan p, const ProofShape& s, std::vector<NatSpan> spans, bool one) {
    plan = p;
    nat = std::move(spans);
    one_allocation = one;
    log_n = s.log_n;
    log_l = s.log_l;
    log_d = s.log_d;
    Q = s.Q;
    rb = s.rb;
  }
  u32 size() const {
    u32 cols = 0;
    for (const NatSpan& sp : nat) cols += sp.cnt;
    return cols;
  }
  const uint64_t* nat_col(u32 j) const {
    for (const NatSpan& sp : nat) {
      if (j < sp.cnt) return sp.p + ((size_t)j << log_n);
      j -= sp.cnt;
    }
    return nullptr;
  }
  std::vector<u32> span_cols() const {
    std::vector<u32> cols;
    for (const NatSpan& sp : nat) cols.push_back(sp.cnt);
    return cols;
  }

  // the LDE of the natural columns onto the cosets the plan evaluates (none on the recompute plan: its tree evaluates them
  // a unit at a time)
  int32_t evaluate(bj_ctx* ctx) {
    if (plan == PLAN_RECOMPUTE) return BJ_OK;
    const u32 log_kept = plan == PLAN_STREAMED ? log_l : log_d;
    const u64 n = 1ull << log_n;
    stride = evaluated_stride(plan, n, log_l, log_d, comm_world(ctx));
    for (const auto& a : allocations(span_cols(), one_allocation, plan)) {
      full.emplace_back(new DevMem());
      alloc_cols.push_back((u32)cols_of(a));
      BJ_TRY(full.back()->alloc(ctx, (size_t)alloc_cols.back() * stride));
      uint64_t* out = (uint64_t*)full.back()->p;
      for (const Piece& p : a) {
        BJ_TRY(lde_columns(ctx, nat[p.span].p + (size_t)p.first * n, out, log_n, log_kept, p.cnt));
        out += (size_t)p.cnt * stride;
      }
      for (u32 j = 0; j < alloc_cols.back(); j++) tree.cols.push_back((const uint64_t*)full.back()->p + (size_t)j * stride);
    }
    return BJ_OK;
  }
  int32_t build_tree(bj_ctx* ctx, u32 cap, u32 hasher) {
    if (plan == PLAN_RECOMPUTE) return oracle_build_by_coset(ctx, tree, nat, log_n, log_l, cap, hasher, rb);
    return oracle_build(ctx, tree, (1ull << log_n) << log_l, cap, hasher, 1u << log_l);
  }
  // compact plan: the first Q cosets of every column repacked with stride Q n, an allocation at a time; tree.cols repointed
  int32_t keep_first_cosets(bj_ctx* ctx) {
    if (plan != PLAN_COMPACT) return BJ_OK;
    const u64 qn = (u64)Q << log_n;
    size_t c0 = 0;
    for (size_t k = 0; k < full.size(); k++) {
      kept.emplace_back(new DevMem());
      BJ_TRY(kept.back()->alloc(ctx, (size_t)alloc_cols[k] * qn));
      for (u32 j = 0; j < alloc_cols[k]; j++) {
        BJ_CUDA(ctx, cudaMemcpyAsync(kept.back()->p + (size_t)j * qn, tree.cols[c0 + j], sizeof(u64) * qn, cudaMemcpyDeviceToDevice, ctx->stream));
        tree.cols[c0 + j] = (const uint64_t*)kept.back()->p + (size_t)j * qn;
      }
      full[k]->release();
      c0 += alloc_cols[k];
    }
    stride = qn;
    return BJ_OK;
  }
  // the kept stride matches a context of `world` ranks
  bool built_for(u32 world) const {
    const u64 n = 1ull << log_n;
    return stride == (plan == PLAN_COMPACT ? (u64)Q * n : plan == PLAN_RECOMPUTE ? 0 : evaluated_stride(plan, n, log_l, log_d, world));
  }
  // the kept columns hold every local point of the quotient's cosets [0, Q)
  bool keeps_quotient_cosets() const { return plan == PLAN_RESIDENT || plan == PLAN_COMPACT; }
  // the natural columns are read again once the tree is built: the compact plan recomputes cosets [Q, L) from them, the
  // streamed [L, Q), the recompute plan every coset
  bool reads_natural() const { return plan != PLAN_RESIDENT; }
  // the first of the `units` local committed units that DEEP and the queries rebuild from the natural columns (the compact
  // plan keeps cosets [0, Q), the recompute plan none); `units` when every one is kept
  u64 first_rebuilt(u64 units) const { return plan == PLAN_COMPACT ? Q : plan == PLAN_RECOMPUTE ? 0 : units; }
  // the columns on local quotient unit k of `shard` (units of n >> shard.log_split rows; the caller sets the unit's window):
  // on the streamed plan a unit of the committed cosets [0, L) is read from the kept columns, any other unit is evaluated
  // from the natural columns into the next slots of `scratch` (bj_lde under the window: the same coset transform, or fold +
  // row-block transform, as the resident plan's LDE)
  int32_t quotient_unit(bj_ctx* ctx, const CosetShard& shard, u64 k, uint64_t*& scratch, std::vector<const uint64_t*>& out) const {
    const u64 n = 1ull << log_n, ub = n >> shard.log_split;
    out.clear();
    if (plan == PLAN_STREAMED && k < shard.local_units(1ull << log_l)) {
      for (const uint64_t* p : tree.cols) out.push_back(p + (size_t)k * ub);
      return BJ_OK;
    }
    for (const NatSpan& sp : nat) {
      if (sp.cnt) BJ_TRY(bj_lde(ctx, sp.p, n, scratch, log_n, log_d, sp.cnt, 0));
      for (u32 i = 0; i < sp.cnt; i++) out.push_back(scratch + (size_t)i * ub);
      scratch += (size_t)sp.cnt * ub;
    }
    return BJ_OK;
  }

  // pool_peak's replay of evaluate, build_tree and keep_first_cosets for a set of spans of span_cols columns; before_tree
  // replays what the driver allocates or frees between evaluate and build_tree
  static void replay(Ledger& m, const ProofShape& s, MemoryPlan plan, const std::vector<u32>& span_cols, bool one_allocation,
                     const std::function<void()>& before_tree = nullptr) {
    const auto allocs = allocations(span_cols, one_allocation, plan);
    const u64 nE = plan == PLAN_RECOMPUTE ? 0 : evaluated_stride(plan, s.n, s.log_l, s.log_d, s.world);
    if (plan != PLAN_RECOMPUTE)
      for (const auto& a : allocs) {
        m.add(cols_of(a) * nE);
        for (const Piece& p : a) m.lde_groups(s, p.cnt);
      }
    if (before_tree) before_tree();
    if (plan == PLAN_RECOMPUTE) {
      u64 cols = 0;
      for (u32 c : span_cols) cols += c;
      m.tree_by_coset(s, cols);
    } else {
      m.tree(s);
    }
    if (plan == PLAN_COMPACT)
      for (const auto& a : allocs) {
        m.add(cols_of(a) * s.n * s.Q);
        m.sub(cols_of(a) * nE);
      }
  }
};

// peak pool bytes of bj_setup_create followed by bj_prove; `chunk`: columns recomputed at a time (compact and recompute plans);
// `setup_held`: the pool bytes the setup holds once bj_setup_create has returned
static u64 pool_peak(const ProofShape& s, MemoryPlan plan, u32 chunk, u64* setup_held = nullptr) {
  Ledger m;
  const bool compact = plan == PLAN_COMPACT, streamed = plan == PLAN_STREAMED, recompute = plan == PLAN_RECOMPUTE;
  const u64 n = s.n, w = s.world, nL = (n << s.log_l) / w, nQ = n << s.log_q;
  const u64 nD = (n << s.log_d) / w;
  const u64 unit_rows = n >> (s.split + s.rb);  // rows of a quotient unit on the recompute plan
  const u64 leaves = (n << s.log_l) / w, capl = s.cap / w;
  auto rebuild_chunks = [&]() {  // for_chunks: the monomials and one unit (a coset, or a row block) of a chunk of natural columns
    m.add((u64)chunk * n);
    m.add((u64)chunk * (n >> s.split));
    m.sub((u64)chunk * (n >> s.split));
    m.sub((u64)chunk * n);
  };
  const u64 S = s.V + s.C + s.T;
  // bj_setup_create
  ColumnSet::replay(m, s, plan, {s.V, s.C, s.T}, true);
  if (setup_held) *setup_held = m.cur;
  // round 1
  ColumnSet::replay(m, s, plan, {s.V, s.lk ? 1u : 0u}, false);
  // round 2: the natural stage-2 columns, then their set, with z(omega x) on a split shard of the resident plan (the streamed
  // and recompute plans evaluate it per unit, into their scratch) between evaluation and tree
  m.add(s.n_s2 * n);
  const u64 zn = s.split && !streamed && !recompute ? 2 * nD : 0;
  ColumnSet::replay(m, s, plan, {s.n_s2}, false, [&]() {
    if (zn) m.add(zn);
    // the compact plan keeps the natural stage-2 columns for DEEP and the queries, the streamed plan for the quotient, the
    // recompute plan for both
    if (!compact && !streamed && !recompute) m.sub(s.n_s2 * n);
  });
  // round 3
  m.add(2 * nQ);
  const u64 nQl = ((u64)s.Q << s.split) >= w ? nQ / w : n >> s.split;
  if (w > 1) m.add(2 * std::max<u64>(nQl, 1));
  if (streamed || recompute) {  // one unit of every column the quotient reads (and of z(omega x) on a row block)
    const u64 unit = (u64)(s.nat_cols() + (s.split + s.rb ? 2 : 0)) * unit_rows;
    m.add(unit);
    m.sub(unit);
  }
  if (zn) m.sub(zn);
  if (w > 1) {
    const u64 per = std::max<u64>(1, ((u64)s.Q << s.split) / w), nb = n >> s.split;
    m.add(per * 2 * nb);
    m.add(w * per * 2 * nb);
    m.sub(w * per * 2 * nb);
    m.sub(per * 2 * nb);
    m.sub(2 * std::max<u64>(nQl, 1));
  }
  m.add(2 * nQ);  // chunks
  m.sub(2 * nQ);  // qq
  m.add(2 * (u64)s.Q * nL);
  m.sub(2 * nQ);  // chunks
  m.tree(s);
  // round 4: the recompute plan opens the natural columns on coset 0, rebuilt a chunk at a time
  if (recompute) rebuild_chunks();
  // round 5
  m.add(2 * nL);
  if (compact || recompute) rebuild_chunks();  // DEEP on the cosets not kept
  u64 log_m = s.log_n + s.log_l;
  u32 kmax = 0;
  for (u32 i = 0; i < s.sched_len; i++) {
    const u32 k = s.sched[i];
    kmax = std::max(kmax, k);
    const u64 lv_leaves = (1ull << (log_m - k)) / w;
    m.add(4 * lv_leaves);
    m.add(4 * (lv_leaves - capl));
    m.add((1ull << (log_m - k)) / w);
    m.add((1ull << (log_m - k)) / w);
    log_m -= k;
  }
  const u64 fft = 1ull << log_m;
  m.add(fft);
  m.add(fft);
  if (w > 1) {
    m.add(2 * fft / w);
    m.add(2 * fft);
    m.sub(2 * fft);
    m.sub(2 * fft / w);
  }
  m.sub(fft);
  m.sub(fft);
  // queries: one gather buffer at a time (leaf rows, Merkle paths, FRI leaves; the recompute plan gathers no row of the
  // setup, witness and stage-2 oracles here); the compact and recompute plans then recompute the rows of the cosets they
  // do not keep chunk by chunk, gathering all the queries' rows of a chunk at a time
  u32 depth = 0;
  while ((leaves >> depth) > capl) depth++;
  const u64 row_max = std::max<u64>({recompute ? 0 : std::max<u64>({S, s.W, s.n_s2}), 2 * (u64)s.Q, 4 * (u64)depth, 2ull << kmax});
  m.add((u64)s.n_queries * row_max);
  m.sub((u64)s.n_queries * row_max);
  if (compact || recompute) {
    m.add((u64)chunk * n);
    m.add((u64)chunk * (n >> s.split));
    m.add((u64)s.n_queries * chunk);
  }
  return m.peak;
}

// device bytes the library holds outside the pool during a proof (upper bounds): forward + inverse twiddles of the
// factor-D domain, the coset-power tables (capped by their 3 GiB budget in ntt.cu), the NTT / LDE / opening scratch, and a
// fixed 16 MiB for the parameter arena (8 MiB) and the long gate programs gates.cu uploads outside the context's pool
// The first two are the tables a context's lanes share (library_tables), the last two each lane holds itself (lane_reserve).
static u64 library_tables(const ProofShape& s) {
  const u64 n = s.n, D = 1ull << s.log_d;
  return sizeof(u64) * n * D + std::min<u64>(3ull << 30, sizeof(u64) * n * (D + s.Q + 2)) + 64 * 16 * (1ull << ((s.log_n + s.log_d + 2) / 2));
}
static u64 lane_reserve(const ProofShape& s) { return sizeof(u64) * std::max<u64>(1ull << 27, 4 * s.n) + (16ull << 20); }
static u64 library_reserve(const ProofShape& s) { return library_tables(s) + lane_reserve(s); }

static bool compact_applies(const ProofShape& s) { return s.world == 1 && s.Q < s.L; }
static bool recompute_applies(const ProofShape& s) { return s.world == 1; }
// one GPU, recompute plan: 1, 2, 4 or 8 row blocks per coset of at least 2 rows each
static constexpr u32 MAX_LOG_ROW_BLOCKS = 3;
static bool row_blocks_valid(const ProofShape& s, u32 rb) { return rb <= MAX_LOG_ROW_BLOCKS && s.log_n > rb; }
// the recompute plan on `world` ranks: the shapes a sharded context takes (at most 8 row blocks per coset, at least 2 rows each)
static bool sharded_shape_valid(const ProofShape& s) { return s.world <= 8 * s.L && s.log_n > s.split; }
// ... where every rank owns a unit of the quotient's cosets [0, Q) (with Q < L and more ranks than Q units some own none;
// the recompute plan is not taken there)
static bool recompute_sharded_applies(const ProofShape& s) { return sharded_shape_valid(s) && ((u64)s.Q << s.split) >= s.world; }
static bool streamed_applies(const ProofShape& s) { return s.Q > s.L; }  // on one GPU and on sharded contexts

static u64 plan_bytes(const ProofShape& s, MemoryPlan plan, u32 chunk = 2) { return pool_peak(s, plan, chunk) + library_reserve(s); }

// Lanes (bj_ctx_create_lane): one setup, proofs on n_lanes contexts at once.  The plan's bytes split in two: out[0] is the
// setup's part (the pool bytes the setup holds after bj_setup_create, and the shared twiddle / coset-power tables), out[1] a
// lane's part (the rest of the plan's pool peak, which is what a proof adds on top of the setup, and the lane's own scratch
// and parameter arena), out[2] = out[0] + n_lanes * out[1].  At one lane out[0] + out[1] is the plan.  The lane's pool part is
// its pool's high-water mark, or, where bj_setup_create itself peaks higher, that peak above what the setup keeps.
static void lane_plan(const ProofShape& s, MemoryPlan plan, u32 chunk, u32 n_lanes, uint64_t out[3]) {
  u64 held = 0;
  const u64 peak = pool_peak(s, plan, chunk, &held);
  out[0] = held + library_tables(s);
  out[1] = (peak - held) + lane_reserve(s);
  out[2] = out[0] + (u64)n_lanes * out[1];
}

}  // namespace bj

struct bj_setup {
  bj_ctx* ctx = nullptr;
  bj_circuit c{};
  std::vector<bj::GateCopy> gate_store;
  std::vector<bj_gate_desc> gates;
  std::vector<uint32_t> pi_cols, pi_rows;
  const uint64_t *sigmas = nullptr, *constants = nullptr, *tables = nullptr;  // borrowed, natural row order
  uint32_t n_tables = 0;
  // [V + C + T] sigmas | constants | tables and the setup tree.  The reference evaluates at D = max(fri_lde_factor, quotient
  // degree) and commits to the subset of the first fri_lde_factor cosets (prover.rs:178-196 `used_lde_degree`,
  // `subset_for_degree`): in the bit-reversed coset order the first L cosets of the factor-D domain ARE the factor-L domain,
  // so the trees, DEEP, FRI and the queries work on the prefix [0, n * L) of every column and only the quotient stage reads
  // the cosets beyond it.
  bj::ColumnSet cols;
  bj::MemoryPlan plan = bj::PLAN_RESIDENT;  // chosen by bj_setup_create, followed by bj_prove
  bj::ProofShape shape{};                   // the proof's shape on this context, with the chosen row blocks
  uint32_t log_blocks = 0;  // recompute plan on one GPU: log2 of the row blocks per coset (bj_setup_row_blocks), 0 elsewhere
  uint64_t limit = 0;    // the device-memory limit the plan was chosen under
  uint64_t plan_bytes[4] = {0, 0, 0, 0};  // resident, compact, streamed, recompute (0: the plan does not apply or was not allowed)
  uint32_t chunk = 2;         // compact and recompute plans: natural-order columns recomputed at a time
  uint64_t pool_bytes = 0, outside_pool_bytes = 0;  // the chosen plan (with its chunk): pool peak, library reserve
  uint64_t chosen_bytes() const { return pool_bytes + outside_pool_bytes; }
  // bj_setup_attach_variables_hint (witness_stream.cu): DenseVariablesCopyHint as u32 [V][hint_rows], 0xFFFFFFFF = placeholder
  bj::DevMem vars_hint;
  uint64_t hint_rows = 0;
  uint64_t hint_values = 0;  // 1 + the largest index the hint names: an all_values vector needs at least this many values
  bool has_hint = false;
  cudaEvent_t ready = nullptr;  // recorded on the context's stream when bj_setup_create returns: bj_prove on a lane waits for it
};

struct bj_proof {
  bj_circuit c{};
  std::vector<bj::u64> witness_cap, stage2_cap, quotient_cap;
  std::vector<std::vector<bj::u64>> fri_caps;
  std::vector<bj::u64> mono_c0, mono_c1;
  std::vector<gl::e2> values_at_z, values_at_z_omega, values_at_0;
  std::vector<bj::u64> public_inputs;
  uint64_t pow_challenge = 0;
  // queries[q][oracle]: witness, stage 2, quotient, setup, then one per FRI oracle
  std::vector<std::vector<bj::QueryAnswer>> queries;
  double stage_seconds[6] = {0, 0, 0, 0, 0, 0};
  std::string json;
};

using namespace bj;

namespace bj {
int32_t ctx_new_lane(bj_ctx* parent, bj_ctx** out);  // capi.cu
}

static bool is_pow2(uint32_t x) { return x && !(x & (x - 1)); }

// the limit a plan must fit under: the one set on the context, or what the device has free plus what the context's pool
// holds without using it
static int32_t memory_limit(bj_ctx* ctx, uint64_t* out) {
  if (ctx->memory_limit) {
    *out = ctx->memory_limit;
    return BJ_OK;
  }
  size_t free_b = 0, total_b = 0;
  BJ_CUDA(ctx, cudaMemGetInfo(&free_b, &total_b));
  uint64_t reserved = 0, used = 0;
  if (ctx->pool) {
    BJ_CUDA(ctx, cudaMemPoolGetAttribute(ctx->pool, cudaMemPoolAttrReservedMemCurrent, &reserved));
    BJ_CUDA(ctx, cudaMemPoolGetAttribute(ctx->pool, cudaMemPoolAttrUsedMemCurrent, &used));
  }
  *out = free_b + (reserved > used ? reserved - used : 0);
  return BJ_OK;
}

static std::string plan_message(const char* who, const uint64_t plan[4], uint64_t limit) {
  std::string m = std::string(who) + ": the proof needs " + std::to_string(plan[0]) + " bytes of device memory resident";
  m += plan[1] ? " and " + std::to_string(plan[1]) + " bytes on the compact plan" : std::string(" (no compact plan: sharded context or quotient degree >= LDE factor)");
  if (plan[2]) m += " and " + std::to_string(plan[2]) + " bytes on the streamed plan";
  if (plan[3]) m += " and " + std::to_string(plan[3]) + " bytes on the recompute plan";
  return m + ", above the limit of " + std::to_string(limit) + " bytes";
}


// The memory plan: resident if it fits under the limit, else compact (Q < L, one GPU), else streamed (Q > L), else recompute
// (one GPU when the context allows it, a context with a communicator when it allows the sharded recompute plan); refused
// before anything is launched.  On a sharded context every rank chooses under its own limit: every plan commits to the same
// units and runs the same collectives, so ranks on different plans still agree.  Sets s->plan, plan_bytes, limit, log_blocks,
// chunk, the chosen bytes and s->shape, the proof's shape with the chosen row blocks.
static int32_t choose_plan(bj_ctx* ctx, const bj_circuit* circuit, bj_setup* s) {
  ProofShape sh;
  BJ_TRY(proof_shape(*circuit, comm_world(ctx), &sh));
  s->plan_bytes[0] = plan_bytes(sh, PLAN_RESIDENT);
  s->plan_bytes[1] = compact_applies(sh) ? plan_bytes(sh, PLAN_COMPACT) : 0;
  s->plan_bytes[2] = streamed_applies(sh) ? plan_bytes(sh, PLAN_STREAMED) : 0;
  const bool recompute_allowed = (ctx->allow_recompute_plan && recompute_applies(sh)) ||
                                 (ctx->allow_sharded_recompute_plan && ctx->comm && recompute_sharded_applies(sh));
  BJ_TRY(memory_limit(ctx, &s->limit));
  // with lanes alive on the context, a plan must also hold their proofs: one lane part each beside the plan, and the
  // witness slot sets alive on the lanes
  const uint32_t lanes = ctx->lanes.load();
  uint64_t lane_sets = 0;
  {
    std::lock_guard<std::mutex> lock(ctx->tables_mu);
    lane_sets = ctx->lane_witness_set_bytes;
  }
  auto need_of = [&](const ProofShape& shape, MemoryPlan k) {
    uint64_t v = plan_bytes(shape, k);
    if (lanes) {
      uint64_t lp[3];
      lane_plan(shape, k, 2, 1, lp);
      v += (uint64_t)lanes * lp[1] + lane_sets;
    }
    return v;
  };
  uint64_t need[4];
  for (int k = 0; k < 3; k++) need[k] = s->plan_bytes[k] ? need_of(sh, (MemoryPlan)k) : 0;
  // the recompute plan on one GPU: the fewest row blocks per coset (up to the context's bj_ctx_set_max_row_blocks) whose
  // plan fits, or the most allowed when none does, so that a refusal names the smallest recompute plan on offer
  uint32_t rb = 0;
  need[3] = 0;
  if (recompute_allowed) {
    uint32_t max_rb = 0;
    while (!ctx->comm && (2u << max_rb) <= ctx->max_row_blocks && row_blocks_valid(sh, max_rb + 1)) max_rb++;
    ProofShape shb = sh;
    for (;; rb++) {
      shb.rb = rb;
      need[3] = need_of(shb, PLAN_RECOMPUTE);
      if (need[3] <= s->limit || rb == max_rb) break;
    }
    s->plan_bytes[3] = plan_bytes(shb, PLAN_RECOMPUTE);
  }
  auto fits = [&](int k) { return need[k] && need[k] <= s->limit; };
  if (need[0] > s->limit) {
    if (fits(2)) s->plan = PLAN_STREAMED;
    else if (fits(1)) s->plan = PLAN_COMPACT;
    else if (fits(3)) s->plan = PLAN_RECOMPUTE;
    else
      BJ_FAIL(ctx, BJ_ERR_OOM, plan_message("bj_setup_create", need, s->limit) +
                                   (lanes ? " (each plan counted with the " + std::to_string(lanes) + " lane(s) of the context" +
                                                (lane_sets ? " and their witness slot sets of " + std::to_string(lane_sets) + " bytes)" : std::string(")"))
                                          : std::string()));
  }
  if (ctx->comm && ctx->allow_sharded_recompute_plan && comm_world(ctx) > 1) {
    // The resident and streamed plans share their LDEs' monomials (lde_columns: every rank interpolates a block of the
    // columns, one all-gather per column group); the recompute plan evaluates its units from the natural-order columns and
    // takes part in no such exchange.  So the ranks agree before their first collective: once one rank needs the recompute
    // plan every rank takes it (a proof runs at its slowest rank's pace, so this costs the others no time), or, where a
    // rank's limit does not hold it, every rank refuses.
    const uint32_t world = comm_world(ctx);
    const u64 mine[2] = {s->plan == PLAN_RECOMPUTE ? 1u : 0u, fits(3) ? 1u : 0u};
    std::vector<u64> all(2 * (size_t)world);
    BJ_TRY(comm_all_gather_host(ctx->comm, mine, all.data(), 2));
    bool any = false, every = true;
    for (uint32_t r = 0; r < world; r++) {
      any = any || all[2 * r];
      every = every && all[2 * r + 1];
    }
    if (any && !every)
      BJ_FAIL(ctx, BJ_ERR_OOM, "bj_setup_create: a rank needs the recompute plan and another rank's limit does not hold it; " +
                                   plan_message("this rank", need, s->limit));
    if (any) s->plan = PLAN_RECOMPUTE;
  }
  if (s->plan == PLAN_RECOMPUTE) s->log_blocks = rb;
  sh.rb = s->log_blocks;
  if (s->plan == PLAN_COMPACT || s->plan == PLAN_RECOMPUTE) {
    // wider recompute chunks only save kernel launches: the chunk grows into at most half of the headroom the limit leaves
    // over the plan (the rest is slack for the pool's fragmentation) and stops at 16 columns
    const uint64_t planned = s->plan_bytes[s->plan];
    const uint64_t budget = planned + (s->limit - planned) / 2;
    uint32_t lo = 2, hi = std::max<uint32_t>(2, std::min<uint32_t>(16, sh.nat_cols()));
    while (lo < hi) {
      const uint32_t mid = lo + (hi - lo + 1) / 2;
      if (plan_bytes(sh, s->plan, mid) <= budget) lo = mid;
      else hi = mid - 1;
    }
    s->chunk = lo;
  }
  s->pool_bytes = pool_peak(sh, s->plan, s->chunk);
  s->outside_pool_bytes = library_reserve(sh);
  s->shape = sh;
  return BJ_OK;
}

// the proof's oracles, in the order of a query's answer
enum OracleId : u32 { WITNESS, STAGE2, QUOTIENT, SETUP };

// a polynomial opened and added to DEEP: column `col` of an oracle, or an Fp2 one (ext): columns col (c0) and col + 1 (c1)
struct Src {
  u32 oracle, col;
  bool ext;
};

// One proof (bj_prove): the transcript, the proof, the column sets and the quotient oracle, the challenges, round by round
struct Prover {
  bj_ctx* ctx;
  const bj_setup& setup;
  const bj_circuit& c;
  const uint64_t *d_variables, *d_multiplicities;
  bj_proof& pf;
  bj_transcript* tr;
  bj_fri_oracles* fri = nullptr;
  uint32_t V, C, T, Q, L, cap, log_n, log_l, log_d, log_q, world, rank, split, wdt, nsub, voff, n_partial, n_s2, a_off;
  bool lk;
  u64 n, nQ, nL, nD, nQl, nb;
  // domain shard (multi-GPU): this context holds (L << split) / world units of every LDE column and its units of the first
  // Q cosets; nL, nD = its length of the committed part of an LDE column and of a whole one (D = max(L, Q)), nQl its quotient
  // points, nb = n >> split the rows of a unit
  ColumnSet witness, stage2;  // variables | multiplicities, and z | partials | A_i | B (c0, c1 each)
  DevMem st2;                 // the natural-order stage-2 columns
  DevMem z_next;              // split shard, resident plan: z(omega x) on this rank's cosets
  DevMem qt_lde;
  Oracle qt;
  // DEEP and the queries rebuild the local committed units [first_rebuilt, units_l) of the setup, witness and stage-2
  // columns from their natural-order columns, a chunk of the flat order setup | witness | stage 2 (oracle o's columns from
  // base[o]) at a time
  u64 units_l, first_rebuilt;
  bool rebuild;
  uint32_t base[4] = {0, 0, 0, 0}, n_rebuilt = 0;
  gl::e2 beta, gamma, lookup_beta{0, 0}, lookup_gamma{0, 0}, z, z_omega;
  std::vector<Src> sources, z_omega_sources, zero_sources;
  DevMem deep;
  uint32_t num_queries = 0, sched[32], sched_len = 0;

  Prover(bj_ctx* x, const bj_setup& s, const uint64_t* vars, const uint64_t* mults, bj_proof& p)
      : ctx(x), setup(s), c(s.c), d_variables(vars), d_multiplicities(mults), pf(p) {
    tr = c.transcript == 1 ? bj_transcript_new_blake2s() : c.transcript == 2 ? bj_transcript_new_keccak256() : c.transcript == 3 ? bj_transcript_new_poseidon() : bj_transcript_new();
    V = c.num_variables, C = c.num_constants, T = setup.n_tables, Q = c.quotient_degree, L = c.fri_lde_factor, cap = c.merkle_tree_cap_size;
    log_n = c.log_n, log_l = setup.shape.log_l, log_d = setup.shape.log_d, log_q = setup.shape.log_q;
    n = 1ull << log_n, nQ = n << log_q;
    world = comm_world(ctx), rank = comm_rank(ctx);
    nL = (n << log_l) / world, nD = (n << log_d) / world, nQl = ctx->shard.local_points(Q, (int)log_n);
    split = ctx->shard.log_split, nb = n >> split;
    lk = c.lookup_width != 0, wdt = c.lookup_width, nsub = c.lookup_num_repetitions, voff = c.lookup_variables_offset;
    n_partial = (V + Q - 1) / Q - 1;
    n_s2 = 2 + 2 * n_partial + (lk ? 2 * (nsub + 1) : 0);
    a_off = 2 + 2 * n_partial;
    units_l = ctx->shard.local_units(L);
    first_rebuilt = setup.cols.first_rebuilt(units_l);
    rebuild = first_rebuilt < units_l;
    witness.init(setup.plan, setup.shape, {{d_variables, V}, {d_multiplicities, lk ? 1u : 0u}}, false);
    base[WITNESS] = setup.cols.size();
    base[STAGE2] = base[WITNESS] + witness.size();
    n_rebuilt = base[STAGE2] + n_s2;
  }
  ~Prover() {
    bj_fri_oracles_free(fri);
    bj_transcript_free(tr);
  }
  Prover(const Prover&) = delete;
  Prover& operator=(const Prover&) = delete;

  gl::e2 challenge2() {
    gl::e2 r;
    r.c0 = bj_transcript_get_challenge(tr);
    r.c1 = bj_transcript_get_challenge(tr);
    return r;
  }
  const ColumnSet& set(uint32_t o) const { return o == SETUP ? setup.cols : o == WITNESS ? witness : stage2; }
  const Oracle& oracle(uint32_t o) const { return o == QUOTIENT ? qt : set(o).tree; }
  const uint64_t* col(uint32_t o, uint32_t j) const { return oracle(o).cols[j]; }
  // every rebuilt column among [lo, hi) of the flat order: f(oracle, its column, flat index), in flat order
  template <class F>
  void for_flat(uint32_t lo, uint32_t hi, F&& f) const {
    for (uint32_t o : {SETUP, WITNESS, STAGE2})
      for (uint32_t i = std::max(lo, base[o]); i < std::min(hi, base[o] + set(o).size()); i++) f(o, i - base[o], i);
  }
  // flat column i and i + 1 are the c0, c1 of one Fp2 polynomial: stage 2 holds those pairs alone
  bool pair_start(uint32_t i) const { return i >= base[STAGE2] && (i - base[STAGE2]) % 2 == 0; }

  int32_t public_inputs() {
    bj_transcript_witness_merkle_tree_cap(tr, (const uint64_t*)setup.cols.tree.cap.data(), cap);  // prover.rs:211
    // public inputs: read from the witness, committed to before anything else (prover.rs:264-266)
    const uint32_t n_pi = c.n_public_inputs;
    pf.public_inputs.resize(n_pi);
    for (uint32_t i = 0; i < n_pi; i++)
      BJ_CUDA(ctx, cudaMemcpyAsync(&pf.public_inputs[i], d_variables + ((size_t)setup.pi_cols[i] << c.log_n) + setup.pi_rows[i], sizeof(u64),
                                   cudaMemcpyDeviceToHost, ctx->stream));
    if (n_pi) BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (uint32_t i = 0; i < n_pi; i++) {
      pf.public_inputs[i] = gl::canon(pf.public_inputs[i]);
      const uint64_t v = pf.public_inputs[i];
      bj_transcript_witness_field_elements(tr, &v, 1);
    }
    return BJ_OK;
  }

  // ---- round 1: witness commitment (variables | witness (none) | multiplicities) ----
  int32_t round1() {
    BJ_TRY(witness.evaluate(ctx));
    BJ_TRY(witness.build_tree(ctx, cap, c.tree_hasher));
    pf.witness_cap = witness.tree.cap;
    bj_transcript_witness_merkle_tree_cap(tr, (const uint64_t*)witness.tree.cap.data(), cap);
    return witness.keep_first_cosets(ctx);
  }

  // ---- round 2: copy-permutation grand product, partial products, lookup polynomials ----
  int32_t round2() {
    beta = challenge2();
    gamma = challenge2();
    if (lk) {
      lookup_beta = challenge2();  // prover.rs:402-406
      lookup_gamma = challenge2();
    }
    BJ_TRY(st2.alloc(ctx, (size_t)n_s2 * n));
    std::vector<const uint64_t*> vp(V), sp(V);
    for (uint32_t j = 0; j < V; j++) {
      vp[j] = d_variables + (size_t)j * n;
      sp[j] = setup.sigmas + (size_t)j * n;
    }
    std::vector<uint64_t> nr(V);
    BJ_TRY(bj_non_residues_for_copy_permutation(n, V, nr.data()));
    const uint64_t b[2] = {beta.c0, beta.c1}, g[2] = {gamma.c0, gamma.c1};
    if (world > 1 && n >= (u64)world * 16)  // rows split over the ranks, one all-gather (stage2.cu)
      BJ_TRY(copy_permutation_stage2_sharded(ctx, vp.data(), sp.data(), V, nr.data(), beta, gamma, log_n, Q, st2.p));
    else
      BJ_TRY(bj_copy_permutation_stage2(ctx, vp.data(), sp.data(), V, nr.data(), b, g, log_n, Q, (uint64_t*)st2.p, (uint64_t*)st2.p + n,
                                        (uint64_t*)st2.p + 2 * n));
    if (lk) {
      std::vector<const uint64_t*> lc(wdt * nsub), tc(T);
      for (uint32_t i = 0; i < wdt * nsub; i++) lc[i] = d_variables + (size_t)(voff + i) * n;
      for (uint32_t j = 0; j < T; j++) tc[j] = setup.tables + (size_t)j * n;
      const uint64_t lb[2] = {lookup_beta.c0, lookup_beta.c1}, lg[2] = {lookup_gamma.c0, lookup_gamma.c1};
      BJ_TRY(bj_lookup_polys_specialized(ctx, lc.data(), nsub, wdt, setup.constants + (size_t)c.lookup_table_id_column * n, tc.data(), T,
                                         d_multiplicities, lb, lg, log_n, (uint64_t*)st2.p + (size_t)a_off * n));
    }
    stage2.init(setup.plan, setup.shape, {{(const uint64_t*)st2.p, n_s2}}, false);
    BJ_TRY(stage2.evaluate(ctx));
    // a row block of a split shard does not hold z(omega x) (another block of the coset does).  On a unit with shift sigma,
    // z(omega x) is the LDE of z on the shift sigma * omega in the same row order: two more columns (c0, c1 of z).  The
    // streamed and recompute plans evaluate them one unit at a time with the quotient's other columns.
    if (split && stage2.keeps_quotient_cosets() && ctx->shard.local_units(Q)) {
      BJ_TRY(z_next.alloc(ctx, 2 * nD));
      BJ_TRY(bj_lde_next_row(ctx, (const uint64_t*)st2.p, n, (uint64_t*)z_next.p, log_n, log_d, 2, 0));
    }
    if (!stage2.reads_natural()) st2.release();
    BJ_TRY(stage2.build_tree(ctx, cap, c.tree_hasher));
    pf.stage2_cap = stage2.tree.cap;
    bj_transcript_witness_merkle_tree_cap(tr, (const uint64_t*)stage2.tree.cap.data(), cap);
    BJ_TRY(stage2.keep_first_cosets(ctx));
    return BJ_OK;
  }

  // ---- round 3: quotient ----
  // the columns the quotient reads, on the points it evaluates: the setup's (sigmas | constants | tables), the witness's
  // (variables | multiplicities) and stage 2's, and on a row block z(omega x)
  struct QuotientCols {
    const uint64_t* const* setup;
    const uint64_t* const* w;
    const uint64_t* const* s2;
    const uint64_t *z_next0, *z_next1;
  };
  int32_t quotient_terms(const QuotientCols& k, const std::vector<uint64_t>& powers, uint32_t n_lk_terms, uint32_t n_gate_terms, u64 n_points,
                         uint64_t* o0, uint64_t* o1) {
    const uint64_t* const* consts = k.setup + V;
    const uint64_t* const* tables = k.setup + V + C;
    if (lk) {
      std::vector<const uint64_t*> ll(wdt * nsub), al(2 * nsub);
      for (uint32_t i = 0; i < wdt * nsub; i++) ll[i] = k.w[voff + i];
      for (uint32_t i = 0; i < 2 * nsub; i++) al[i] = k.s2[a_off + i];
      const uint64_t lb[2] = {lookup_beta.c0, lookup_beta.c1}, lg[2] = {lookup_gamma.c0, lookup_gamma.c1};
      BJ_TRY(bj_quotient_lookup_specialized(ctx, ll.data(), nsub, wdt, consts[c.lookup_table_id_column], tables, T, k.w[V], al.data(),
                                            k.s2[a_off + 2 * nsub], k.s2[a_off + 2 * nsub + 1], lb, lg, powers.data(), n_points, o0, o1));
    }
    if (n_gate_terms)
      BJ_TRY(bj_quotient_gates_general_purpose(ctx, setup.gates.data(), (uint32_t)setup.gates.size(), k.w, V, nullptr, 0, consts, C,
                                               powers.data() + 2 * (size_t)n_lk_terms, n_gate_terms, n_points, o0, o1));
    std::vector<uint64_t> nr(V);
    BJ_TRY(bj_non_residues_for_copy_permutation(n, V, nr.data()));
    const uint64_t b[2] = {beta.c0, beta.c1}, g[2] = {gamma.c0, gamma.c1};
    const uint64_t* copy_powers = powers.data() + 2 * (size_t)(n_lk_terms + n_gate_terms);
    if (ctx->shard.log_split)  // a row block (split shard, or a recompute unit under its window) does not hold z(omega x)
      BJ_TRY(bj_quotient_copy_permutation_with_z_next(ctx, k.w, k.setup, V, nr.data(), k.s2[0], k.s2[1], k.z_next0, k.z_next1,
                                                      n_partial ? k.s2 + 2 : nullptr, b, g, copy_powers, log_n, log_d, log_q, Q, o0, o1));
    else
      BJ_TRY(bj_quotient_copy_permutation(ctx, k.w, k.setup, V, nr.data(), k.s2[0], k.s2[1], n_partial ? k.s2 + 2 : nullptr, b, g, copy_powers,
                                          log_n, log_d, log_q, Q, o0, o1));
    return bj_quotient_divide_by_vanishing(ctx, o0, o1, log_n, log_q);
  }
  int32_t quotient() {
    const gl::e2 alpha = challenge2();
    uint32_t n_gate_terms = 0;
    for (const auto& g : setup.gates) n_gate_terms += g.n_writes * g.num_repetitions;
    const uint32_t n_lk_terms = lk ? nsub + 1 : 0;  // lookup terms come first (prover.rs:608-625)
    const uint32_t total_terms = n_lk_terms + n_gate_terms + 1 + 1 + n_partial;
    std::vector<uint64_t> powers(2 * (size_t)total_terms);
    gl::e2 cur{1, 0};
    for (uint32_t i = 0; i < total_terms; i++) {
      powers[2 * i] = cur.c0;
      powers[2 * i + 1] = cur.c1;
      cur = gl::e2_mul(cur, alpha);
    }
    DevMem qq, qloc;  // qq: [2][nQ] global (c0 then c1); qloc: this rank's cosets among the first Q
    BJ_TRY(qq.alloc(ctx, 2 * nQ));
    uint64_t* q0 = (uint64_t*)qq.p;
    uint64_t* q1 = q0 + nQ;
    uint64_t* const gq0 = q0;
    uint64_t* const gq1 = q1;
    if (world > 1) {
      BJ_TRY(qloc.alloc(ctx, 2 * std::max<u64>(nQl, 1)));
      q0 = (uint64_t*)qloc.p;
      q1 = q0 + nQl;
      BJ_CUDA(ctx, cudaMemsetAsync(qloc.p, 0, sizeof(u64) * 2 * std::max<u64>(nQl, 1), ctx->stream));
    } else {
      BJ_CUDA(ctx, cudaMemsetAsync(qq.p, 0, sizeof(u64) * 2 * nQ, ctx->stream));
    }
    if (setup.cols.keeps_quotient_cosets()) {
      const uint64_t* zn = (const uint64_t*)z_next.p;
      if (nQl)
        BJ_TRY(quotient_terms({setup.cols.tree.cols.data(), witness.tree.cols.data(), stage2.tree.cols.data(), zn, zn ? zn + nD : nullptr}, powers,
                              n_lk_terms, n_gate_terms, nQl, q0, q1));
    } else {
      // one local quotient unit k at a time (global unit u: coset u on one GPU or a coset shard, a row block of ub rows of
      // coset u / B on a split shard or on one GPU with 2^rb row blocks per coset), under the window of unit u among the units
      // of the factor-D domain; each column set gives its columns on the unit (ColumnSet::quotient_unit), and on a row block
      // the unit's z(omega x) columns go to the scratch too.  The unit's quotient values land in its slot [k ub, (k + 1) ub)
      // of the local quotient cosets.
      CosetShard shard = ctx->shard;
      shard.log_split += setup.log_blocks;  // one GPU: every one of the Q * 2^rb units is local, global unit k = k
      const uint32_t usplit = shard.log_split;
      const u64 ub = n >> usplit;
      DevMem ev;
      BJ_TRY(ev.alloc(ctx, (size_t)(setup.cols.size() + witness.size() + n_s2 + (usplit ? 2 : 0)) * ub));
      std::vector<const uint64_t*> sc, wc, s2c;
      for (u64 k = 0; k < shard.local_units(Q); k++) {
        ShardWindow window(ctx, log_d + usplit, (u32)shard.global_unit(k), usplit);
        uint64_t* e = (uint64_t*)ev.p;
        BJ_TRY(setup.cols.quotient_unit(ctx, shard, k, e, sc));
        BJ_TRY(witness.quotient_unit(ctx, shard, k, e, wc));
        BJ_TRY(stage2.quotient_unit(ctx, shard, k, e, s2c));
        const uint64_t *z0 = nullptr, *z1 = nullptr;
        if (usplit) {
          BJ_TRY(bj_lde_next_row(ctx, (const uint64_t*)st2.p, n, e, log_n, log_d, 2, 0));
          z0 = e;
          z1 = e + ub;
        }
        BJ_TRY(quotient_terms({sc.data(), wc.data(), s2c.data(), z0, z1}, powers, n_lk_terms, n_gate_terms, ub, q0 + (size_t)k * ub, q1 + (size_t)k * ub));
      }
    }
    z_next.release();
    if (world > 1) {
      // the one bulk exchange: the quotient cosets recombine (they are interpolated together at size n * Q).  Every rank sends
      // `per` = ceil(Q * B / world) unit slots of nb = n / B rows (c0 | c1 per slot; ranks beyond the Q * B units send
      // padding), one all-gather, then the slots are scattered to their global unit positions.
      const u64 q_units = (u64)Q << split;
      const u64 per = std::max<u64>(1, q_units / world);
      DevMem snd, rcv;
      BJ_TRY(snd.alloc(ctx, per * 2 * nb));
      BJ_TRY(rcv.alloc(ctx, (u64)world * per * 2 * nb));
      BJ_CUDA(ctx, cudaMemsetAsync(snd.p, 0, sizeof(u64) * per * 2 * nb, ctx->stream));
      const u64 q_loc = ctx->shard.local_units(Q);
      for (u64 k = 0; k < q_loc; k++) {
        BJ_CUDA(ctx, cudaMemcpyAsync(snd.p + (2 * k) * nb, q0 + k * nb, sizeof(u64) * nb, cudaMemcpyDeviceToDevice, ctx->stream));
        BJ_CUDA(ctx, cudaMemcpyAsync(snd.p + (2 * k + 1) * nb, q1 + k * nb, sizeof(u64) * nb, cudaMemcpyDeviceToDevice, ctx->stream));
      }
      BJ_TRY(comm_all_gather(ctx->comm, snd.p, rcv.p, per * 2 * nb));
      for (uint32_t r = 0; r < world; r++)
        for (u64 k = 0; k < per; k++) {
          const u64 u = ctx->shard.unit_of(r, k);
          if (u >= q_units) continue;
          const u64* part = rcv.p + ((u64)r * per + k) * 2 * nb;
          BJ_CUDA(ctx, cudaMemcpyAsync(gq0 + u * nb, part, sizeof(u64) * nb, cudaMemcpyDeviceToDevice, ctx->stream));
          BJ_CUDA(ctx, cudaMemcpyAsync(gq1 + u * nb, part + nb, sizeof(u64) * nb, cudaMemcpyDeviceToDevice, ctx->stream));
        }
      q0 = gq0;
      q1 = gq1;
      qloc.release();
    }
    // cosets -> natural order, one interpolation of size n*Q on the coset 7, Q chunks of n coefficients (prover.rs:1399-1467)
    BJ_TRY(bj_bitreverse(ctx, q0, log_n + log_q, 2, nQ));
    BJ_TRY(bj_intt_natural_to_natural(ctx, q0, log_n + log_q, 2, nQ, gl::MULT_GEN));
    {
      // the reference's satisfiability guard: the top coefficient must vanish (prover.rs:1425-1438)
      uint64_t top[2];
      BJ_CUDA(ctx, cudaMemcpyAsync(&top[0], q0 + nQ - 1, sizeof(u64), cudaMemcpyDeviceToHost, ctx->stream));
      BJ_CUDA(ctx, cudaMemcpyAsync(&top[1], q1 + nQ - 1, sizeof(u64), cudaMemcpyDeviceToHost, ctx->stream));
      BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
      if (top[0] || top[1]) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_prove: unsatisfied circuit (quotient is not a polynomial of degree < n * quotient_degree)");
    }
    DevMem chunks;  // chunk j: c0 then c1
    BJ_TRY(chunks.alloc(ctx, 2 * nQ));
    for (uint32_t j = 0; j < Q; j++) {
      BJ_CUDA(ctx, cudaMemcpyAsync(chunks.p + (size_t)(2 * j) * n, q0 + (size_t)j * n, sizeof(u64) * n, cudaMemcpyDeviceToDevice, ctx->stream));
      BJ_CUDA(ctx, cudaMemcpyAsync(chunks.p + (size_t)(2 * j + 1) * n, q1 + (size_t)j * n, sizeof(u64) * n, cudaMemcpyDeviceToDevice, ctx->stream));
    }
    qq.release();
    BJ_TRY(qt_lde.alloc(ctx, (size_t)(2 * Q) * nL));
    BJ_TRY(bj_lde(ctx, (const uint64_t*)chunks.p, n, (uint64_t*)qt_lde.p, log_n, log_l, 2 * Q, 1));
    chunks.release();
    for (uint32_t j = 0; j < 2 * Q; j++) qt.cols.push_back((const uint64_t*)qt_lde.p + (size_t)j * nL);
    BJ_TRY(oracle_build(ctx, qt, n << log_l, cap, c.tree_hasher, L));
    pf.quotient_cap = qt.cap;
    bj_transcript_witness_merkle_tree_cap(tr, (const uint64_t*)qt.cap.data(), cap);
    return BJ_OK;
  }

  // chunks of `chunk` rebuilt columns among flat [lo, hi) (an Fp2 pair never split; a chunk may span two oracles): monomials
  // by one iNTT, then body(c0, cnt, monomials, scratch for one unit of the chunk: a coset, or nb rows of one on a split shard,
  // stride nb)
  int32_t for_chunks(uint32_t lo, uint32_t hi, const std::function<int32_t(uint32_t, uint32_t, const uint64_t*, uint64_t*)>& body) {
    DevMem mono, ev;
    BJ_TRY(mono.alloc(ctx, (size_t)setup.chunk * n));
    BJ_TRY(ev.alloc(ctx, (size_t)setup.chunk * nb));
    for (uint32_t c0 = lo; c0 < hi;) {
      uint32_t cnt = std::min<uint32_t>(setup.chunk, hi - c0);
      if (c0 + cnt < hi && pair_start(c0 + cnt - 1)) cnt--;
      std::vector<const uint64_t*> nat;
      for_flat(c0, c0 + cnt, [&](uint32_t o, uint32_t j, uint32_t) { nat.push_back(set(o).nat_col(j)); });
      for (uint32_t i = 0; i < cnt; i++)
        BJ_CUDA(ctx, cudaMemcpyAsync(mono.p + (size_t)i * n, nat[i], sizeof(u64) * n, cudaMemcpyDeviceToDevice, ctx->stream));
      BJ_TRY(bj_intt_natural_to_natural(ctx, (uint64_t*)mono.p, log_n, cnt, n, 1));
      BJ_TRY(body(c0, cnt, (const uint64_t*)mono.p, (uint64_t*)ev.p));
      c0 += cnt;
    }
    return BJ_OK;
  }

  // ---- round 4: openings.  Order (prover.rs:1549-1683): variables, witness, constants, sigmas, z, partial products,
  //      multiplicities, lookup A, lookup B, lookup tables, quotient chunks.
  // The barycentric sums of `cols` (oracle, column) at a into ev.  On the recompute plan the setup, witness and stage-2
  // columns come from local slot 0 (coset 0 on one GPU, this rank's coset or row block on a sharded context), rebuilt a chunk
  // at a time (only the chunks that hold one of them); the quotient oracle's columns are read directly.
  int32_t barycentric(const std::vector<std::pair<uint32_t, uint32_t>>& cols, const uint64_t a[2], uint64_t* ev) {
    auto evaluate = [&](const std::vector<const uint64_t*>& ptrs, const std::vector<size_t>& at) -> int32_t {
      if (ptrs.empty()) return BJ_OK;
      std::vector<uint64_t> got(2 * ptrs.size());
      BJ_TRY(bj_barycentric_evaluate(ctx, ptrs.data(), (uint32_t)ptrs.size(), log_n, a, got.data()));
      for (size_t k = 0; k < at.size(); k++) {
        ev[2 * at[k]] = got[2 * k];
        ev[2 * at[k] + 1] = got[2 * k + 1];
      }
      return BJ_OK;
    };
    std::vector<const uint64_t*> direct;
    std::vector<size_t> direct_at;
    uint32_t lo = n_rebuilt, hi = 0;
    const bool rebuilt = setup.plan == PLAN_RECOMPUTE;  // on coset 0 of the rebuilt columns
    for (size_t i = 0; i < cols.size(); i++) {
      const auto [o, j] = cols[i];
      if (!rebuilt || o == QUOTIENT) {
        direct.push_back(col(o, j));
        direct_at.push_back(i);
      } else {
        lo = std::min(lo, base[o] + j);
        hi = std::max(hi, base[o] + j + 1);
      }
    }
    BJ_TRY(evaluate(direct, direct_at));
    if (!rebuilt) return BJ_OK;
    return for_chunks(lo, hi, [&](uint32_t c0, uint32_t cnt, const uint64_t* mono, uint64_t* on_coset) -> int32_t {
      BJ_TRY(lde_unit(ctx, mono, on_coset, log_n, log_l, cnt, 0, 1));
      std::vector<const uint64_t*> ptrs;
      std::vector<size_t> at;
      for (size_t i = 0; i < cols.size(); i++) {
        const auto [o, j] = cols[i];
        if (o == QUOTIENT || base[o] + j < c0 || base[o] + j >= c0 + cnt) continue;
        ptrs.push_back(on_coset + (size_t)(base[o] + j - c0) * nb);
        at.push_back(i);
      }
      return evaluate(ptrs, at);
    });
  }
  int32_t open_at(const std::vector<Src>& srcs, gl::e2 at, std::vector<gl::e2>& vals) {
    std::vector<std::pair<uint32_t, uint32_t>> flat;
    for (const auto& s : srcs) {
      flat.push_back({s.oracle, s.col});
      if (s.ext) flat.push_back({s.oracle, s.col + 1});
    }
    vals.clear();
    if (flat.empty()) return BJ_OK;
    std::vector<uint64_t> ev(2 * flat.size());
    const uint64_t a[2] = {at.c0, at.c1};
    if (world == 1) {
      BJ_TRY(barycentric(flat, a, ev.data()));
    } else {
      // the columns are split over the coset groups: ranks [g B, (g + 1) B) hold the B row blocks of coset g (B = 1: one rank,
      // its whole coset) and open column block g from it, each rank its block's contribution (on the recompute plan from its
      // rebuilt local slot 0).  The contributions are gathered and the B of a group summed.
      const uint32_t groups = world >> split, g = rank >> split;
      const size_t per = (flat.size() + groups - 1) / groups, first = std::min(flat.size(), (size_t)g * per);
      const size_t cnt = std::min(per, flat.size() - first);
      std::vector<uint64_t> mine(2 * per, 0), all(2 * per * world);
      if (cnt) BJ_TRY(barycentric(std::vector<std::pair<uint32_t, uint32_t>>(flat.begin() + first, flat.begin() + first + cnt), a, mine.data()));
      BJ_TRY(comm_all_gather_host(ctx->comm, (const u64*)mine.data(), (u64*)all.data(), 2 * per));
      for (uint32_t gg = 0; gg < groups; gg++)
        for (size_t e = 0; e < 2 * per && gg * 2 * per + e < ev.size(); e++) {
          u64 v = 0;
          for (uint32_t p = 0; p < (1u << split); p++) v = gl::canon(gl::add(v, all[(((size_t)gg << split) + p) * 2 * per + e]));
          ev[gg * 2 * per + e] = v;  // group blocks are contiguous: [g][per] == flat order
        }
    }
    size_t k = 0;
    for (const auto& s : srcs) {
      if (s.ext) {  // f0 + u f1 at an Fp2 point (u^2 = 7)
        const gl::e2 a0{ev[2 * k], ev[2 * k + 1]}, b0{ev[2 * k + 2], ev[2 * k + 3]};
        vals.push_back({gl::canon(gl::add(a0.c0, gl::mul7(b0.c1))), gl::canon(gl::add(a0.c1, b0.c0))});
        k += 2;
      } else {
        vals.push_back({ev[2 * k], ev[2 * k + 1]});
        k += 1;
      }
    }
    return BJ_OK;
  }
  int32_t openings() {
    z = challenge2();
    z_omega = gl::e2_mul_base(z, gl::omega(log_n));
    for (uint32_t j = 0; j < V; j++) sources.push_back({WITNESS, j, false});
    for (uint32_t j = 0; j < C; j++) sources.push_back({SETUP, V + j, false});
    for (uint32_t j = 0; j < V; j++) sources.push_back({SETUP, j, false});
    for (uint32_t i = 0; i < 1 + n_partial; i++) sources.push_back({STAGE2, 2 * i, true});
    if (lk) {
      sources.push_back({WITNESS, V, false});
      for (uint32_t i = 0; i < nsub + 1; i++) {
        sources.push_back({STAGE2, a_off + 2 * i, true});
        zero_sources.push_back({STAGE2, a_off + 2 * i, true});
      }
      for (uint32_t j = 0; j < T; j++) sources.push_back({SETUP, V + C + j, false});
    }
    for (uint32_t i = 0; i < Q; i++) sources.push_back({QUOTIENT, 2 * i, true});
    z_omega_sources = {{STAGE2, 0, true}};
    BJ_TRY(open_at(sources, z, pf.values_at_z));
    BJ_TRY(open_at(z_omega_sources, z_omega, pf.values_at_z_omega));
    BJ_TRY(open_at(zero_sources, gl::e2{0, 0}, pf.values_at_0));
    for (const auto* vs : {&pf.values_at_z, &pf.values_at_z_omega, &pf.values_at_0})
      for (const auto& v : *vs) {
        const uint64_t e[2] = {v.c0, v.c1};
        bj_transcript_witness_field_elements(tr, e, 2);
      }
    return BJ_OK;
  }

  // ---- round 5: DEEP combination + FRI ----
  struct DeepGroup {
    const std::vector<Src>* srcs;
    const std::vector<gl::e2>* vals;
    gl::e2 at;
    const uint64_t* chs;
  };
  // sources i of a group with keep(i) on the local points [first, first + count), column j of oracle o read at at_col(o, j).
  // One GPU: any run of points.  Sharded (recompute plan): the whole local domain, or local unit k (first = k nb, count = nb)
  // under its window, whose points the kernel then places at their global indices.
  int32_t deep_range(const DeepGroup& g, const std::function<bool(size_t)>& keep, const std::function<const uint64_t*(uint32_t, uint32_t)>& at_col,
                     u64 first, u64 count) {
    std::vector<const uint64_t*> p0, p1;
    std::vector<uint64_t> v, ch;
    for (size_t i = 0; i < g.srcs->size(); i++) {
      if (!keep(i)) continue;
      const Src& sr = (*g.srcs)[i];
      p0.push_back(at_col(sr.oracle, sr.col));
      p1.push_back(sr.ext ? at_col(sr.oracle, sr.col + 1) : nullptr);
      v.push_back((*g.vals)[i].c0);
      v.push_back((*g.vals)[i].c1);
      ch.push_back(g.chs[2 * i]);
      ch.push_back(g.chs[2 * i + 1]);
    }
    if (p0.empty()) return BJ_OK;
    const uint64_t a[2] = {g.at.c0, g.at.c1};
    uint64_t *acc0 = (uint64_t*)deep.p + first, *acc1 = (uint64_t*)deep.p + nL + first;
    if (world == 1)
      return bj_deep_quotient_range(ctx, p0.data(), p1.data(), (uint32_t)p0.size(), v.data(), ch.data(), a, log_n + log_l, first, count, acc0, acc1);
    if (count == nL)
      return bj_deep_quotient_group(ctx, p0.data(), p1.data(), (uint32_t)p0.size(), v.data(), ch.data(), a, log_n + log_l, acc0, acc1);
    ShardWindow window(ctx, log_l + split, (u32)ctx->shard.global_unit(first / nb), split);
    return bj_deep_quotient_group(ctx, p0.data(), p1.data(), (uint32_t)p0.size(), v.data(), ch.data(), a, log_n + log_l, acc0, acc1);
  }
  int32_t deep_fri_pow() {
    // public inputs grouped by opening point w^row in order of first appearance (prover.rs:1805-1821)
    struct PiGroup {
      u64 at;
      std::vector<Src> srcs;
      std::vector<gl::e2> vals;
    };
    std::vector<PiGroup> pi_groups;
    for (uint32_t i = 0; i < c.n_public_inputs; i++) {
      const u64 at = gl::pow(gl::omega(log_n), setup.pi_rows[i]);
      PiGroup* g = nullptr;
      for (auto& e : pi_groups)
        if (e.at == at) g = &e;
      if (!g) {
        pi_groups.push_back({at, {}, {}});
        g = &pi_groups.back();
      }
      g->srcs.push_back({WITNESS, setup.pi_cols[i], false});
      g->vals.push_back({pf.public_inputs[i], 0});
    }
    const gl::e2 ch0 = challenge2();
    const size_t n_ch = pf.values_at_z.size() + 1 + pf.values_at_0.size() + c.n_public_inputs;
    std::vector<uint64_t> ch(2 * n_ch);
    gl::e2 cur{1, 0};
    for (size_t i = 0; i < n_ch; i++) {
      ch[2 * i] = cur.c0;
      ch[2 * i + 1] = cur.c1;
      cur = gl::e2_mul(cur, ch0);
    }
    BJ_TRY(deep.alloc(ctx, 2 * nL));
    BJ_CUDA(ctx, cudaMemsetAsync(deep.p, 0, sizeof(u64) * 2 * nL, ctx->stream));
    // with units rebuilt: units [0, first_rebuilt) from the kept columns, the quotient oracle's columns on all local units,
    // the rest added below
    const u64 Fn = rebuild ? first_rebuilt * n : 0;
    std::vector<DeepGroup> deep_groups;
    auto deep_group = [&](const std::vector<Src>& srcs, const std::vector<gl::e2>& vals, gl::e2 at, const uint64_t* chs) -> int32_t {
      if (srcs.empty()) return BJ_OK;
      const DeepGroup g{&srcs, &vals, at, chs};
      if (rebuild) {
        deep_groups.push_back(g);
        if (Fn) BJ_TRY(deep_range(g, [](size_t) { return true; }, [&](uint32_t o, uint32_t j) { return col(o, j); }, 0, Fn));
        return deep_range(g, [&](size_t i) { return srcs[i].oracle == QUOTIENT; }, [&](uint32_t o, uint32_t j) { return col(o, j) + Fn; }, Fn, nL - Fn);
      }
      std::vector<const uint64_t*> p0(srcs.size()), p1(srcs.size());
      std::vector<uint64_t> v(2 * srcs.size());
      for (size_t i = 0; i < srcs.size(); i++) {
        p0[i] = col(srcs[i].oracle, srcs[i].col);
        p1[i] = srcs[i].ext ? col(srcs[i].oracle, srcs[i].col + 1) : nullptr;
        v[2 * i] = vals[i].c0;
        v[2 * i + 1] = vals[i].c1;
      }
      const uint64_t a[2] = {at.c0, at.c1};
      return bj_deep_quotient_group(ctx, p0.data(), p1.data(), (uint32_t)srcs.size(), v.data(), chs, a, log_n + log_l /* global */,
                                    (uint64_t*)deep.p, (uint64_t*)deep.p + nL);
    };
    BJ_TRY(deep_group(sources, pf.values_at_z, z, ch.data()));
    BJ_TRY(deep_group(z_omega_sources, pf.values_at_z_omega, z_omega, ch.data() + 2 * sources.size()));
    BJ_TRY(deep_group(zero_sources, pf.values_at_0, gl::e2{0, 0}, ch.data() + 2 * (sources.size() + 1)));
    size_t off = sources.size() + 1 + zero_sources.size();
    for (const auto& g : pi_groups) {  // prover.rs:2010-2041
      BJ_TRY(deep_group(g.srcs, g.vals, gl::e2{g.at, 0}, ch.data() + 2 * off));
      off += g.srcs.size();
    }
    if (rebuild)  // units [first_rebuilt, units_l): every chunk of natural columns evaluated on one unit at a time, its DEEP terms added
      BJ_TRY(for_chunks(0, n_rebuilt, [&](uint32_t c0, uint32_t cnt, const uint64_t* mono, uint64_t* ev) -> int32_t {
        auto in_chunk = [&](const Src& s) { return s.oracle != QUOTIENT && base[s.oracle] + s.col >= c0 && base[s.oracle] + s.col < c0 + cnt; };
        auto on_unit = [&](uint32_t o, uint32_t j) -> const uint64_t* { return ev + (size_t)(base[o] + j - c0) * nb; };
        for (u64 k = first_rebuilt; k < units_l; k++) {
          BJ_TRY(lde_unit(ctx, mono, ev, log_n, log_l, cnt, k, 1));
          for (const DeepGroup& g : deep_groups) BJ_TRY(deep_range(g, [&](size_t i) { return in_chunk((*g.srcs)[i]); }, on_unit, k * nb, nb));
        }
        return BJ_OK;
      }));
    uint32_t new_pow = 0, final_degree = 0;
    BJ_TRY(bj_compute_fri_schedule(c.security_level, cap, c.pow_bits, log_l, log_n, &new_pow, &num_queries, sched, &sched_len, &final_degree));
    BJ_TRY(bj_do_fri_with_hasher(ctx, tr, (const uint64_t*)deep.p, (const uint64_t*)deep.p + nL, log_n + log_l, sched, sched_len, log_l, cap,
                                 c.tree_hasher, &fri));
    const uint32_t n_fri = bj_fri_oracles_num_oracles(fri);
    pf.fri_caps.resize(n_fri);
    for (uint32_t i = 0; i < n_fri; i++) {
      pf.fri_caps[i].resize(4 * (size_t)cap);
      BJ_TRY(bj_fri_oracles_get_cap(fri, i, (uint64_t*)pf.fri_caps[i].data()));
    }
    const uint32_t n_mono = bj_fri_oracles_num_monomials(fri);
    pf.mono_c0.resize(n_mono);
    pf.mono_c1.resize(n_mono);
    BJ_TRY(bj_fri_oracles_get_monomials(fri, (uint64_t*)pf.mono_c0.data(), (uint64_t*)pf.mono_c1.data()));
    if (new_pow) {  // prover.rs:2109-2132 with POW = Blake2s256: 5 challenges seed the search, the nonce re-enters the transcript
      uint8_t seed[40];
      for (int i = 0; i < 5; i++) {
        const uint64_t e = bj_transcript_get_challenge(tr);
        for (int k = 0; k < 8; k++) seed[8 * i + k] = (uint8_t)(e >> (8 * k));
      }
      uint64_t nonce = 0;
      BJ_TRY(bj_pow_blake2s(ctx, seed, 40, new_pow, &nonce));
      pf.pow_challenge = nonce;
      const uint64_t lh[2] = {nonce & 0xffffffffull, nonce >> 32};
      bj_transcript_witness_field_elements(tr, lh, 2);
    }
    return BJ_OK;
  }

  // ---- queries ----
  int32_t queries() {
    const uint32_t max_bits = log_n + log_l;
    std::vector<uint64_t> idxs(num_queries);
    for (auto& i : idxs) i = bj_transcript_get_index_bits(tr, max_bits, max_bits);
    pf.queries.assign(num_queries, {});
    // a query is answered by the rank that owns the unit of its index (leaf t = coset * n + row lies in that rank's subtree);
    // the other ranks look up a dummy leaf, the answers are exchanged and every rank keeps the owner's
    std::vector<uint64_t> loc_idx(num_queries);
    std::vector<uint32_t> owner(num_queries);
    for (uint32_t q = 0; q < num_queries; q++) {
      owner[q] = ctx->shard.owner(idxs[q], (int)log_n);
      loc_idx[q] = owner[q] == rank ? ctx->shard.owner_index(idxs[q], (int)log_n) : 0;
    }
    // every answer part (leaf elements / path of one oracle) is gathered locally first; ONE exchange then carries all of them
    struct Part {
      std::vector<uint64_t> data;  // [num_queries][rec_len]
      size_t rec_len;
    };
    std::vector<Part> parts;  // order: (rows, path) of the 4 base oracles (OracleId order), then (leaf elements, path) of every FRI level
    const u64 Fn = rebuild ? first_rebuilt * n : 0;
    for (uint32_t oi : {WITNESS, STAGE2, QUOTIENT, SETUP}) {
      const Oracle* o = &oracle(oi);
      const size_t row_len = o->cols.size();
      uint32_t depth = 0;
      while ((o->n_leaves >> depth) > o->cap_size) depth++;
      Part rows{std::vector<uint64_t>((size_t)num_queries * row_len), row_len};
      Part path{std::vector<uint64_t>((size_t)num_queries * depth * 4), (size_t)depth * 4};
      if (!rebuild || oi == QUOTIENT) {
        BJ_TRY(bj_query_leaf_elements(ctx, o->cols.data(), (uint32_t)row_len, 1, o->n_leaves, loc_idx.data(), num_queries, rows.data.data()));
      } else if (Fn) {  // kept columns hold the first units; the rows of the others are recomputed below
        std::vector<uint64_t> kept_idx(loc_idx);
        for (auto& i : kept_idx)
          if (i >= Fn) i = 0;
        BJ_TRY(bj_query_leaf_elements(ctx, o->cols.data(), (uint32_t)row_len, 1, Fn, kept_idx.data(), num_queries, rows.data.data()));
      }
      if (depth)
        BJ_TRY(bj_merkle_paths(ctx, (const uint64_t*)o->leaf_hashes.p, (const uint64_t*)o->nodes.p, o->n_leaves, o->cap_size, loc_idx.data(),
                               num_queries, path.data.data()));
      parts.push_back(std::move(rows));
      parts.push_back(std::move(path));
    }
    if (rebuild) {
      // queries this context answers whose leaf lies in a local unit k >= first_rebuilt (a coset on one GPU): one recompute of
      // each such unit per chunk, the queried rows gathered from it (the rows of every query, so that the gather buffer is the
      // one the plan counts) into the rows part of each column's oracle.  On a sharded context every rank runs the pass, also
      // one that answers none of these queries: its peers are rebuilding meanwhile and the exchange waits for them, so it
      // gathers from the chunk's monomials instead, and every rank's pool reaches the peak its plan counts.
      const u32 log_nb = log_n - split;
      std::vector<std::vector<uint32_t>> by_unit(units_l);
      for (uint32_t q = 0; q < num_queries; q++)
        if (owner[q] == rank && (loc_idx[q] >> log_nb) >= first_rebuilt) by_unit[loc_idx[q] >> log_nb].push_back(q);
      bool any = false;
      for (const auto& qs : by_unit) any = any || !qs.empty();
      if (any || world > 1)
        BJ_TRY(for_chunks(0, n_rebuilt, [&](uint32_t c0, uint32_t cnt, const uint64_t* mono, uint64_t* ev) -> int32_t {
          std::vector<const uint64_t*> cols(cnt);
          std::vector<uint64_t> rows_in(num_queries, 0), got((size_t)num_queries * cnt);
          if (!any) {
            for (uint32_t i = 0; i < cnt; i++) cols[i] = mono + (size_t)i * n;
            return bj_query_leaf_elements(ctx, cols.data(), cnt, 1, n, rows_in.data(), num_queries, got.data());
          }
          for (uint32_t i = 0; i < cnt; i++) cols[i] = ev + (size_t)i * nb;
          for (u64 k = first_rebuilt; k < units_l; k++) {
            const auto& qs = by_unit[k];
            if (qs.empty()) continue;
            BJ_TRY(lde_unit(ctx, mono, ev, log_n, log_l, cnt, k, 1));
            for (uint32_t q : qs) rows_in[q] = loc_idx[q] & (nb - 1);
            BJ_TRY(bj_query_leaf_elements(ctx, cols.data(), cnt, 1, nb, rows_in.data(), num_queries, got.data()));
            for_flat(c0, c0 + cnt, [&](uint32_t o, uint32_t j, uint32_t i) {
              Part& pt = parts[2 * o];
              for (uint32_t q : qs) pt.data[(size_t)q * pt.rec_len + j] = got[(size_t)q * cnt + (i - c0)];
            });
          }
          return BJ_OK;
        }));
    }
    uint32_t log_len = log_n;  // coset length of the level's codeword
    std::vector<uint64_t> sub(idxs);
    for (uint32_t lvl = 0; lvl < sched_len; lvl++) {
      const uint32_t k = sched[lvl];
      const size_t le_len = (size_t)2 << k;
      std::vector<uint64_t> locals(num_queries);
      for (uint32_t q = 0; q < num_queries; q++) {
        locals[q] = owner[q] == rank ? (ctx->shard.owner_index(sub[q], (int)log_len) >> k) : 0;
        sub[q] >>= k;
      }
      uint32_t plen = 0;
      Part les{std::vector<uint64_t>((size_t)num_queries * le_len, 0), le_len};
      Part path{std::vector<uint64_t>((size_t)num_queries * 40 * 4, 0), 0};  // [num_queries][plen][4] after the call
      BJ_TRY(bj_fri_oracles_query_batch(fri, lvl, locals.data(), num_queries, les.data.data(), path.data.data(), &plen));
      path.rec_len = (size_t)plen * 4;
      path.data.resize((size_t)num_queries * path.rec_len);
      parts.push_back(std::move(les));
      parts.push_back(std::move(path));
      log_len -= k;
    }
    if (world > 1) {
      size_t total = 0;
      for (const auto& pt : parts) total += pt.data.size();
      std::vector<uint64_t> mine(total), all((size_t)world * total);
      size_t off = 0;
      for (const auto& pt : parts) {
        if (!pt.data.empty()) memcpy(mine.data() + off, pt.data.data(), sizeof(uint64_t) * pt.data.size());
        off += pt.data.size();
      }
      BJ_TRY(comm_all_gather_host(ctx->comm, (const u64*)mine.data(), (u64*)all.data(), total));
      off = 0;
      for (auto& pt : parts) {
        for (uint32_t q = 0; q < num_queries && pt.rec_len; q++)
          memcpy(pt.data.data() + (size_t)q * pt.rec_len, all.data() + (size_t)owner[q] * total + off + (size_t)q * pt.rec_len,
                 sizeof(uint64_t) * pt.rec_len);
        off += pt.data.size();
      }
    }
    for (size_t o = 0; o + 1 < parts.size(); o += 2) {
      const Part &le = parts[o], &pa = parts[o + 1];
      for (uint32_t q = 0; q < num_queries; q++) {
        QueryAnswer a;
        a.leaf_elements.assign(le.data.begin() + (size_t)q * le.rec_len, le.data.begin() + (size_t)(q + 1) * le.rec_len);
        a.path.assign(pa.data.begin() + (size_t)q * pa.rec_len, pa.data.begin() + (size_t)(q + 1) * pa.rec_len);
        pf.queries[q].push_back(std::move(a));
      }
    }
    return BJ_OK;
  }
};

// ---- serde_json shape of Proof (proof.rs:57-143) ----
static std::string proof_json(const bj_proof& pf, uint32_t sched_len) {
  const bj_circuit& c = pf.c;
  const uint32_t cap = c.merkle_tree_cap_size;
  std::string s;
  s.reserve(1 << 20);
  const bool digest_bytes = c.tree_hasher != BJ_HASHER_POSEIDON2;
  s += "{\"proof_config\":{\"fri_lde_factor\":" + std::to_string(c.fri_lde_factor) + ",\"merkle_tree_cap_size\":" + std::to_string(cap) +
       ",\"fri_folding_schedule\":null,\"security_level\":" + std::to_string(c.security_level) + ",\"pow_bits\":" + std::to_string(c.pow_bits) +
       "},\"public_inputs\":";
  json_u64_list(s, pf.public_inputs.data(), pf.public_inputs.size());
  s += ",\"witness_oracle_cap\":";
  json_digests(s, pf.witness_cap.data(), cap, digest_bytes);
  s += ",\"stage_2_oracle_cap\":";
  json_digests(s, pf.stage2_cap.data(), cap, digest_bytes);
  s += ",\"quotient_oracle_cap\":";
  json_digests(s, pf.quotient_cap.data(), cap, digest_bytes);
  s += ",\"final_fri_monomials\":[";
  json_u64_list(s, pf.mono_c0.data(), pf.mono_c0.size());
  s += ',';
  json_u64_list(s, pf.mono_c1.data(), pf.mono_c1.size());
  s += "],\"values_at_z\":";
  json_ext_list(s, pf.values_at_z);
  s += ",\"values_at_z_omega\":";
  json_ext_list(s, pf.values_at_z_omega);
  s += ",\"values_at_0\":";
  json_ext_list(s, pf.values_at_0);
  s += ",\"fri_base_oracle_cap\":";
  json_digests(s, pf.fri_caps[0].data(), cap, digest_bytes);
  s += ",\"fri_intermediate_oracles_caps\":[";
  for (size_t i = 1; i < pf.fri_caps.size(); i++) {
    if (i > 1) s += ',';
    json_digests(s, pf.fri_caps[i].data(), cap, digest_bytes);
  }
  s += "],\"queries_per_fri_repetition\":[";
  static const char* names[4] = {"witness_query", "stage_2_query", "quotient_query", "setup_query"};
  auto json_answer = [&](const QueryAnswer& a) {
    s += "{\"leaf_elements\":";
    json_u64_list(s, a.leaf_elements.data(), a.leaf_elements.size());
    s += ",\"proof\":";
    json_digests(s, a.path.data(), a.path.size() / 4, digest_bytes);
    s += '}';
  };
  for (size_t q = 0; q < pf.queries.size(); q++) {
    if (q) s += ',';
    s += '{';
    for (int o = 0; o < 4; o++) {
      s += std::string("\"") + names[o] + "\":";
      json_answer(pf.queries[q][o]);
      s += ',';
    }
    s += "\"fri_queries\":[";
    for (uint32_t lvl = 0; lvl < sched_len; lvl++) {
      if (lvl) s += ',';
      json_answer(pf.queries[q][4 + lvl]);
    }
    s += "]}";
  }
  s += "],\"pow_challenge\":" + std::to_string(pf.pow_challenge) + ",\"_marker\":null}";
  return s;
}

extern "C" {

int32_t bj_setup_create(bj_ctx* ctx, const bj_circuit* circuit, const uint64_t* d_sigmas, const uint64_t* d_constants,
                        const uint64_t* d_lookup_tables, bj_setup** out) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || !circuit || !d_sigmas || !out || circuit->num_variables == 0 || circuit->log_n == 0 || circuit->log_n > 28 ||
      !is_pow2(circuit->fri_lde_factor) || !is_pow2(circuit->merkle_tree_cap_size) || !is_pow2(circuit->quotient_degree) ||
      (circuit->num_constants && !d_constants) ||
      (circuit->n_gates && !circuit->gates) || circuit->tree_hasher > BJ_HASHER_KECCAK256 || circuit->transcript > 3)
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_setup_create: bad argument");
  if (circuit->lookup_width && (!d_lookup_tables || circuit->lookup_table_id_column >= circuit->num_constants ||
                                circuit->lookup_variables_offset + circuit->lookup_width * circuit->lookup_num_repetitions >
                                    circuit->num_variables))
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_setup_create: inconsistent lookup description");
  if (ctx->parent)
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_setup_create: a lane proves against its parent's setups: create the setup on the parent");
  if (ctx->shard.log_stride && !ctx->comm)
    BJ_FAIL(ctx, BJ_ERR_UNSUPPORTED, "bj_setup_create: a coset-sharded context needs a communicator (bj_comm_create_*) for the native driver");
  const uint32_t split = ctx->shard.log_split;  // row blocks per coset = 2^split when there are more ranks than cosets
  if (ctx->comm && (circuit->merkle_tree_cap_size < std::max(circuit->fri_lde_factor, comm_world(ctx)) ||
                    (1u << ctx->shard_log_lde) != circuit->fri_lde_factor))
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_setup_create: sharded proving needs cap_size >= max(LDE factor, world) and the LDE factor the communicator was created for");
  if (ctx->comm && split && circuit->log_n <= split)
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_setup_create: a row block of the domain shard needs at least 2 rows (2^log_n >= 2 * world / LDE factor)");
  *out = nullptr;
  {
    // a proof needs at least one FRI folding step (the JSON has a fri_base_oracle_cap): reject circuits so small that
    // compute_fri_schedule (prover.rs:2281-2372) returns an empty schedule for this cap size, instead of failing inside bj_prove
    uint32_t log_l = 0, new_pow = 0, nq = 0, sched[32], sched_len = 0, fd = 0;
    while ((1u << log_l) < circuit->fri_lde_factor) log_l++;
    if (log_l == 0) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_setup_create: fri_lde_factor must be at least 2");
    BJ_TRY(bj_compute_fri_schedule(circuit->security_level, circuit->merkle_tree_cap_size, circuit->pow_bits, log_l, circuit->log_n, &new_pow, &nq,
                                   sched, &sched_len, &fd));
    if (sched_len == 0)
      BJ_FAIL(ctx, BJ_ERR_INVALID_ARG,
              "bj_setup_create: degenerate instance - 2^log_n * fri_lde_factor is too small for merkle_tree_cap_size (empty FRI schedule)");
    // a FRI fold stays inside one unit of the shard: every level's units must hold the 2^k elements it folds together
    uint32_t log_unit = circuit->log_n - (ctx->comm ? split : 0);
    for (uint32_t i = 0; i < sched_len; i++) {
      if (log_unit < sched[i])
        BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_setup_create: a FRI level has fewer elements per unit of the domain shard than it folds together");
      log_unit -= sched[i];
    }
  }
  std::unique_ptr<bj_setup> s(new bj_setup());
  // the setup is handed out with an event recorded behind its last kernel (lanes wait for it) and is listed on the context
  auto publish = [&]() -> int32_t {
    BJ_CUDA(ctx, cudaEventCreateWithFlags(&s->ready, cudaEventDisableTiming));
    BJ_CUDA(ctx, cudaEventRecord(s->ready, ctx->stream));
    {
      std::lock_guard<std::mutex> lock(ctx->tables_mu);
      ctx->setups.push_back(s.get());
    }
    *out = s.release();
    return BJ_OK;
  };
  BJ_TRY(choose_plan(ctx, circuit, s.get()));
  s->ctx = ctx;
  s->c = *circuit;
  // deep copy of the gate programs (the caller's arrays need not outlive this call)
  s->gate_store.resize(circuit->n_gates);
  s->gates.resize(circuit->n_gates);
  for (uint32_t g = 0; g < circuit->n_gates; g++) {
    const bj_gate_desc& d = circuit->gates[g];
    GateCopy& gc = s->gate_store[g];
    gc.relations.assign(d.relations, d.relations + d.n_relations);
    gc.writes.assign(d.writes, d.writes + d.n_writes);
    if (d.selector_path_len) gc.path.assign(d.selector_path, d.selector_path + d.selector_path_len);
    s->gates[g] = d;
    s->gates[g].relations = gc.relations.data();
    s->gates[g].writes = gc.writes.data();
    s->gates[g].selector_path = gc.path.data();
  }
  s->c.gates = s->gates.data();
  if (circuit->n_public_inputs) {
    if (!circuit->public_input_columns || !circuit->public_input_rows) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_setup_create: public input places missing");
    s->pi_cols.assign(circuit->public_input_columns, circuit->public_input_columns + circuit->n_public_inputs);
    s->pi_rows.assign(circuit->public_input_rows, circuit->public_input_rows + circuit->n_public_inputs);
    for (uint32_t i = 0; i < circuit->n_public_inputs; i++)
      if (s->pi_cols[i] >= circuit->num_variables || s->pi_rows[i] >= (1ull << circuit->log_n))
        BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_setup_create: public input place out of range");
  }
  s->c.public_input_columns = s->pi_cols.data();
  s->c.public_input_rows = s->pi_rows.data();
  s->sigmas = d_sigmas;
  s->constants = d_constants;
  s->tables = d_lookup_tables;
  s->n_tables = circuit->lookup_width ? circuit->lookup_width + 1 : 0;
  const uint32_t V = circuit->num_variables, C = circuit->num_constants, T = s->n_tables;
  // the streamed plan evaluates the committed cosets [0, L) only (this rank's units of them): the LDE at factor L, whose
  // cosets are the first L of the factor-D domain with the same shifts, so the values and trees do not change.  The
  // quotient recomputes the other cosets from the borrowed natural-order columns.  The recompute plan keeps no coset: the
  // tree is built one coset at a time, and s->cols.tree.cols are the natural-order columns every reader rebuilds its cosets from.
  s->cols.init(s->plan, s->shape, {{d_sigmas, V}, {d_constants, C}, {d_lookup_tables, T}}, true);
  BJ_TRY(s->cols.evaluate(ctx));
  BJ_TRY(s->cols.build_tree(ctx, circuit->merkle_tree_cap_size, circuit->tree_hasher));
  BJ_TRY(s->cols.keep_first_cosets(ctx));
  return publish();
}

void bj_setup_free(bj_setup* s) {
  if (!s) return;
  bj::DeviceGuard device_guard(s->ctx);
  if (s->ctx) {
    cudaStreamSynchronize(s->ctx->stream);
    std::lock_guard<std::mutex> lock(s->ctx->tables_mu);
    auto& v = s->ctx->setups;
    v.erase(std::remove(v.begin(), v.end(), s), v.end());
  }
  if (s->ready) cudaEventDestroy(s->ready);
  delete s;
}

int32_t bj_setup_get_cap(const bj_setup* s, uint64_t* h_cap) {
  if (!s || !h_cap) return BJ_ERR_INVALID_ARG;
  memcpy(h_cap, s->cols.tree.cap.data(), sizeof(uint64_t) * s->cols.tree.cap.size());
  return BJ_OK;
}

int32_t bj_prove(bj_ctx* ctx, const bj_setup* setup, const uint64_t* d_variables, const uint64_t* d_multiplicities, bj_proof** out) {
  bj::DeviceGuard device_guard(ctx);
  // a lane proves against its parent's setups
  if (!ctx || !setup || !d_variables || !out || (setup->ctx != ctx && (!ctx->parent || setup->ctx != ctx->parent)))
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_prove: bad argument");
  if (setup->ctx != ctx) BJ_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, setup->ready, 0));
  const bj_circuit& c = setup->c;
  if (c.lookup_width && !d_multiplicities) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_prove: the lookup argument needs the multiplicities column");
  *out = nullptr;
  std::unique_ptr<bj_proof> pf(new bj_proof());
  pf->c = c;
  pf->c.gates = nullptr;
  if (!setup->cols.built_for(comm_world(ctx))) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_prove: the setup was built with a different shard");
  {
    const uint64_t limit = ctx->memory_limit ? ctx->memory_limit : setup->limit;
    if (setup->chosen_bytes() > limit) BJ_FAIL(ctx, BJ_ERR_OOM, plan_message("bj_prove", setup->plan_bytes, limit));
  }
  auto t_prev = std::chrono::steady_clock::now();
  auto mark = [&](int stage) -> int32_t {
    BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    const auto now = std::chrono::steady_clock::now();
    pf->stage_seconds[stage] += std::chrono::duration<double>(now - t_prev).count();
    t_prev = now;
    return BJ_OK;
  };
  Prover p(ctx, *setup, d_variables, d_multiplicities, *pf);
  BJ_TRY(p.public_inputs());
  BJ_TRY(p.round1());
  BJ_TRY(mark(0));
  BJ_TRY(p.round2());
  BJ_TRY(mark(1));
  BJ_TRY(p.quotient());
  BJ_TRY(mark(2));
  BJ_TRY(p.openings());
  BJ_TRY(mark(3));
  BJ_TRY(p.deep_fri_pow());
  BJ_TRY(mark(4));
  BJ_TRY(p.queries());
  BJ_TRY(mark(5));
  pf->json = proof_json(*pf, p.sched_len);
  *out = pf.release();
  return BJ_OK;
}

static int32_t memory_plan_shape(const bj_circuit* circuit, uint32_t world, ProofShape* sh) {
  if (!circuit || world == 0 || (world & (world - 1)) || circuit->log_n == 0 || circuit->log_n > 28 || !is_pow2(circuit->fri_lde_factor) ||
      circuit->fri_lde_factor < 2 || !is_pow2(circuit->quotient_degree) || !is_pow2(circuit->merkle_tree_cap_size) ||
      circuit->merkle_tree_cap_size < world || circuit->num_variables == 0)
    return BJ_ERR_INVALID_ARG;
  BJ_TRY(proof_shape(*circuit, world, sh));
  return sh->sched_len == 0 ? BJ_ERR_INVALID_ARG : BJ_OK;
}

int32_t bj_proof_memory_plan(const bj_circuit* circuit, uint32_t world, uint64_t out[2]) {
  ProofShape sh;
  if (!out) return BJ_ERR_INVALID_ARG;
  BJ_TRY(memory_plan_shape(circuit, world, &sh));
  out[0] = plan_bytes(sh, PLAN_RESIDENT);
  out[1] = compact_applies(sh) ? plan_bytes(sh, PLAN_COMPACT) : 0;
  return BJ_OK;
}

int32_t bj_proof_memory_plan_streamed(const bj_circuit* circuit, uint32_t world, uint64_t* out) {
  ProofShape sh;
  if (!out) return BJ_ERR_INVALID_ARG;
  BJ_TRY(memory_plan_shape(circuit, world, &sh));
  *out = world == 1 && streamed_applies(sh) ? plan_bytes(sh, PLAN_STREAMED) : 0;
  return BJ_OK;
}

int32_t bj_proof_memory_plan_streamed_sharded(const bj_circuit* circuit, uint32_t world, uint64_t* out) {
  ProofShape sh;
  if (!out) return BJ_ERR_INVALID_ARG;
  BJ_TRY(memory_plan_shape(circuit, world, &sh));
  *out = streamed_applies(sh) ? plan_bytes(sh, PLAN_STREAMED) : 0;
  return BJ_OK;
}

int32_t bj_proof_memory_plan_recompute(const bj_circuit* circuit, uint32_t world, uint64_t* out) {
  ProofShape sh;
  if (!out) return BJ_ERR_INVALID_ARG;
  BJ_TRY(memory_plan_shape(circuit, world, &sh));
  *out = recompute_applies(sh) ? plan_bytes(sh, PLAN_RECOMPUTE) : 0;
  return BJ_OK;
}

int32_t bj_proof_memory_plan_recompute_sharded(const bj_circuit* circuit, uint32_t world, uint64_t* out) {
  ProofShape sh;
  if (!out) return BJ_ERR_INVALID_ARG;
  *out = 0;
  BJ_TRY(memory_plan_shape(circuit, world, &sh));
  if (!sharded_shape_valid(sh)) return BJ_ERR_INVALID_ARG;
  *out = recompute_sharded_applies(sh) ? plan_bytes(sh, PLAN_RECOMPUTE) : 0;
  return BJ_OK;
}

// log2 of a row-block count of the one-GPU recompute plan: 1, 2, 4 or 8 row blocks of at least 2 rows each
static int32_t log_row_blocks(const ProofShape& sh, uint32_t blocks, uint32_t* rb) {
  if (!is_pow2(blocks)) return BJ_ERR_INVALID_ARG;
  *rb = 0;
  while ((1u << *rb) < blocks) (*rb)++;
  return row_blocks_valid(sh, *rb) ? BJ_OK : BJ_ERR_INVALID_ARG;
}

int32_t bj_proof_memory_plan_recompute_blocks(const bj_circuit* circuit, uint32_t blocks, uint64_t* out) {
  ProofShape sh;
  if (!out) return BJ_ERR_INVALID_ARG;
  *out = 0;
  BJ_TRY(memory_plan_shape(circuit, 1, &sh));
  BJ_TRY(log_row_blocks(sh, blocks, &sh.rb));
  *out = plan_bytes(sh, PLAN_RECOMPUTE);
  return BJ_OK;
}

int32_t bj_proof_memory_plan_lanes_host_blocks(const bj_circuit* circuit, uint32_t plan, uint32_t blocks, uint32_t n_lanes, uint64_t out[3]) {
  ProofShape sh;
  if (!out || n_lanes == 0 || plan > BJ_PLAN_RECOMPUTE || (plan != BJ_PLAN_RECOMPUTE && blocks != 1)) return BJ_ERR_INVALID_ARG;
  BJ_TRY(memory_plan_shape(circuit, 1, &sh));
  BJ_TRY(log_row_blocks(sh, blocks, &sh.rb));
  const bool applies = plan == PLAN_RESIDENT || (plan == PLAN_COMPACT && compact_applies(sh)) || (plan == PLAN_STREAMED && streamed_applies(sh)) ||
                       (plan == PLAN_RECOMPUTE && recompute_applies(sh));
  if (!applies) {
    out[0] = out[1] = out[2] = 0;
    return BJ_OK;
  }
  lane_plan(sh, (MemoryPlan)plan, 2, n_lanes, out);
  return BJ_OK;
}

int32_t bj_proof_memory_plan_lanes_host(const bj_circuit* circuit, uint32_t plan, uint32_t n_lanes, uint64_t out[3]) {
  return bj_proof_memory_plan_lanes_host_blocks(circuit, plan, 1, n_lanes, out);
}

// the one-GPU shape of a setup's chosen plan, row blocks included
static int32_t setup_shape(const bj_setup* s, ProofShape* sh) {
  BJ_TRY(proof_shape(s->c, 1, sh));
  sh->rb = s->log_blocks;
  return BJ_OK;
}

int32_t bj_proof_memory_plan_lanes(const bj_setup* setup, uint32_t n_lanes, uint64_t out[3]) {
  ProofShape sh;
  if (!setup || !out || n_lanes == 0 || comm_world(setup->ctx) != 1) return BJ_ERR_INVALID_ARG;
  BJ_TRY(setup_shape(setup, &sh));
  lane_plan(sh, setup->plan, setup->chunk, n_lanes, out);
  return BJ_OK;
}

int32_t bj_proof_memory_plan_lane_pool(const bj_setup* setup, uint64_t* pool_bytes) {
  ProofShape sh;
  if (!setup || !pool_bytes || comm_world(setup->ctx) != 1) return BJ_ERR_INVALID_ARG;
  BJ_TRY(setup_shape(setup, &sh));
  uint64_t out[3];
  lane_plan(sh, setup->plan, setup->chunk, 1, out);
  *pool_bytes = out[1] - lane_reserve(sh);
  return BJ_OK;
}

int32_t bj_ctx_create_lane(bj_ctx* parent, bj_ctx** out) {
  if (!out) BJ_FAIL(parent, BJ_ERR_INVALID_ARG, "bj_ctx_create_lane: out is NULL");
  *out = nullptr;
  if (!parent) return BJ_ERR_INVALID_ARG;
  bj::DeviceGuard device_guard(parent);
  if (parent->parent) BJ_FAIL(parent, BJ_ERR_INVALID_ARG, "bj_ctx_create_lane: a lane has no lanes of its own: create them on its parent");
  if (parent->comm || parent->shard.log_stride)
    BJ_FAIL(parent, BJ_ERR_INVALID_ARG, "bj_ctx_create_lane: a sharded context (communicator or domain shard) has no lanes");
  {
    // every setup of the parent, with the lanes alive, this one, and the parent itself (its pool keeps what its setup and its
    // own proofs reached, so it counts as one proving context) must fit under the limit its plan was chosen under
    // (and the witness slot sets alive on the lanes)
    std::lock_guard<std::mutex> lock(parent->tables_mu);
    const uint32_t lanes_after = parent->lanes.load() + 1;
    const uint64_t lane_sets = parent->lane_witness_set_bytes;
    for (const bj_setup* s : parent->setups) {
      ProofShape sh;
      BJ_TRY(setup_shape(s, &sh));
      uint64_t p[3];
      lane_plan(sh, s->plan, s->chunk, lanes_after + 1, p);
      const uint64_t limit = parent->memory_limit ? parent->memory_limit : s->limit;
      if (p[2] + lane_sets > limit)
        BJ_FAIL(parent, BJ_ERR_OOM, "bj_ctx_create_lane: the setup's plan needs " + std::to_string(s->chosen_bytes()) + " bytes and every lane " +
                                        std::to_string(p[1]) + " bytes more; with " + std::to_string(lanes_after) + " lane(s) that is " +
                                        std::to_string(p[2]) + " bytes" +
                                        (lane_sets ? ", and the lanes' witness slot sets " + std::to_string(lane_sets) + " bytes" : std::string()) +
                                        ", above the limit of " + std::to_string(limit) + " bytes");
    }
  }
  return ctx_new_lane(parent, out);
}

int32_t bj_setup_is_compact(const bj_setup* s) { return s ? (s->plan == PLAN_COMPACT ? 1 : 0) : BJ_ERR_INVALID_ARG; }

int32_t bj_setup_plan(const bj_setup* s) {
  if (!s) return BJ_ERR_INVALID_ARG;
  return s->plan;
}

int32_t bj_setup_row_blocks(const bj_setup* s) { return s ? (int32_t)(1u << s->log_blocks) : BJ_ERR_INVALID_ARG; }

int32_t bj_setup_memory_plan(const bj_setup* s, uint64_t out[3]) {
  if (!s || !out) return BJ_ERR_INVALID_ARG;
  out[0] = s->pool_bytes;
  out[1] = s->outside_pool_bytes;
  out[2] = s->plan == PLAN_COMPACT || s->plan == PLAN_RECOMPUTE ? s->chunk : 0;
  return BJ_OK;
}

void bj_proof_free(bj_proof* p) { delete p; }

int32_t bj_proof_to_json(const bj_proof* p, char* buf, size_t capacity, size_t* needed) {
  if (!p || !needed) return BJ_ERR_INVALID_ARG;
  *needed = p->json.size() + 1;
  if (!buf || capacity < *needed) return buf ? BJ_ERR_INVALID_ARG : BJ_OK;
  memcpy(buf, p->json.c_str(), *needed);
  return BJ_OK;
}

int32_t bj_proof_stage_seconds(const bj_proof* p, double out[6]) {
  if (!p || !out) return BJ_ERR_INVALID_ARG;
  for (int i = 0; i < 6; i++) out[i] = p->stage_seconds[i];
  return BJ_OK;
}

}  // extern "C"
