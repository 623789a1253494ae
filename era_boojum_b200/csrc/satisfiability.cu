// Satisfiability check of a witness against its circuit on the trace domain, and the lookup multiplicity column.
//   CSReferenceAssembly::check_if_satisfied            src/cs/implementations/satisfiability_test.rs:15-353
//   materialize_multiplicities_polynomials             src/cs/implementations/witness.rs:225-272
// Exact, no random challenge: the three conditions bj_prove needs.
//   * gates: the quotient's interpreter (gates.cu) in check mode over the n rows of the trace: every pushed term of a selected
//     gate must be 0;
//   * copy constraints from sigma alone: an entry s = k_c' w^r' names the cell (c', r').  s^n = k_c'^n identifies c' (the k^n
//     of make_non_residues are pairwise distinct, k_0 = 1), r' is the discrete log of s / k_c' in <w_n>, read from a device
//     hash table of the n powers of w.  Every cell must hold the value of the cell it names; every cell must be named exactly
//     once (two bitmaps: "named once" and "named again", set with atomicOr);
//   * lookups: a device hash table over the table rows maps every distinct content to its first row; the n * R tuples are
//     counted against it, and the count of each content must equal the sum of the multiplicities over its rows.
// Counts are atomic sums and every "first" is an atomicMin over a key in the report's order, so the report is the same for the
// same inputs whatever the scheduling; one single-thread kernel then fills the report from the keys.
#include <cstring>
#include <vector>
#include "ctx.hpp"

namespace bj {

constexpr u32 SAT_EMPTY = 0xffffffffu;
constexpr unsigned long long SAT_NO_KEY = ~0ull;

// device accumulators: a count and the smallest key of each failure kind
struct SatAcc {
  unsigned long long gate_failures, gate_key;      // key: row << 32 | global term index
  unsigned long long copy_failures, copy_key;      // key: row * V + column
  unsigned long long sigma_failures, sigma_key;    // key: (row * V + column) << 2 | kind
  unsigned long long lookup_unmatched, lookup_key; // key: row * R + sub-argument
  unsigned long long mult_failures, mult_key;      // key: first table row of the content
};

__device__ __forceinline__ u64 sat_hash(u64 x) {
  x ^= x >> 33;
  x *= 0xff51afd7ed558ccdull;
  x ^= x >> 33;
  x *= 0xc4ceb9fe1a85ec53ull;
  return x ^ (x >> 33);
}

// every lane of the warp calls this: one atomic per warp for the count and one for the smallest key
__device__ __forceinline__ void sat_warp_report(bool fail, u64 key, unsigned long long* count, unsigned long long* min_key) {
  const unsigned mask = __ballot_sync(0xffffffffu, fail);
  if (!mask) return;
  u64 k = fail ? key : SAT_NO_KEY;
#pragma unroll
  for (int o = 16; o; o >>= 1) k = min(k, (u64)__shfl_xor_sync(0xffffffffu, k, o));
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(count, (unsigned long long)__popc(mask));
    atomicMin(min_key, (unsigned long long)k);
  }
}

// ---- sigma decode ----
struct SigmaDecode {
  const u64* kn;     // [V] k_c^n, ascending
  const u32* kn_col; // [V] its column
  const u64* k_inv;  // [V] k_c^-1 by column
  const u64* w_key;  // hash table of the powers of w_n: key w^r (0 = empty slot) ...
  const u32* w_row;  // ... and r
  u64 w_mask;
  u32 V, log_n;
};

__device__ bool sigma_decode(const SigmaDecode& d, u64 s, u32* col, u64* row) {
  s = gl::canon(s);
  if (s == 0) return false;
  u64 t = s;
  for (u32 i = 0; i < d.log_n; i++) t = gl::mul(t, t);
  u32 lo = 0, hi = d.V;  // t among the k_c^n
  while (lo < hi) {
    const u32 mid = (lo + hi) / 2;
    if (__ldg(d.kn + mid) < t) lo = mid + 1;
    else hi = mid;
  }
  if (lo == d.V || __ldg(d.kn + lo) != t) return false;
  const u32 c = __ldg(d.kn_col + lo);
  const u64 x = gl::canon(gl::mul(s, __ldg(d.k_inv + c)));  // an n-th root of unity, as x^n = s^n / k_c^n = 1
  for (u64 h = sat_hash(x) & d.w_mask;; h = (h + 1) & d.w_mask) {
    const u64 k = __ldg(d.w_key + h);
    if (k == 0) return false;
    if (k == x) {
      *col = c;
      *row = __ldg(d.w_row + h);
      return true;
    }
  }
}

__global__ void sat_omega_table_kernel(u64 w, u64 n, u64* keys, u32* rows, u64 mask) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const u64 x = gl::canon(gl::pow(w, i));
  for (u64 h = sat_hash(x) & mask;; h = (h + 1) & mask) {
    if (atomicCAS((unsigned long long*)keys + h, 0ull, (unsigned long long)x) == 0ull) {
      rows[h] = (u32)i;
      return;
    }
  }
}

struct CopyParams {
  const u64* vars;    // [V][n]
  const u64* sigmas;  // [V][n]
  SigmaDecode dec;
  u32* named_once;    // bitmaps over cells c * n + r
  u32* named_again;
  SatAcc* acc;
};

// every cell: decode its sigma entry, mark the named cell, compare the two values
__global__ void __launch_bounds__(256) sat_copy_kernel(const CopyParams p) {
  const u64 total = (u64)p.dec.V << p.dec.log_n;
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  const u64 n_mask = (1ull << p.dec.log_n) - 1;
  bool bad_copy = false, bad_sigma = false;
  u64 cell_key = 0;
  if (i < total) {
    const u64 r = i & n_mask, c = i >> p.dec.log_n;
    cell_key = r * p.dec.V + c;
    u32 c2;
    u64 r2;
    if (sigma_decode(p.dec, __ldg(p.sigmas + i), &c2, &r2)) {
      const u64 j = ((u64)c2 << p.dec.log_n) | r2;
      const u32 bit = 1u << (j & 31);
      if (atomicOr(p.named_once + (j >> 5), bit) & bit) atomicOr(p.named_again + (j >> 5), bit);
      bad_copy = gl::canon(__ldg(p.vars + i)) != gl::canon(__ldg(p.vars + j));
    } else {
      bad_sigma = true;
    }
  }
  sat_warp_report(bad_copy, cell_key, &p.acc->copy_failures, &p.acc->copy_key);
  sat_warp_report(bad_sigma, cell_key << 2 | 1, &p.acc->sigma_failures, &p.acc->sigma_key);
}

// every cell: named by no entry (kind 2) or by two or more (kind 3)
__global__ void __launch_bounds__(256) sat_named_kernel(const CopyParams p) {
  const u64 total = (u64)p.dec.V << p.dec.log_n;
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  bool bad = false;
  u64 key = 0;
  if (i < total) {
    const u32 bit = 1u << (i & 31);
    const bool once = p.named_once[i >> 5] & bit, again = p.named_again[i >> 5] & bit;
    bad = !once || again;
    key = (((i & ((1ull << p.dec.log_n) - 1)) * p.dec.V + (i >> p.dec.log_n)) << 2) | (once ? 3 : 2);
  }
  sat_warp_report(bad, key, &p.acc->sigma_failures, &p.acc->sigma_key);
}

// ---- lookups ----
struct LookupCheckParams {
  const u64* tables;  // [W + 1][n]: t_0 .. t_{W-1}, table id
  const u64* vars;    // [V][n]; tuple (row, sub i) = columns voff + i * W + j
  const u64* id_col;  // the constant column with the table id
  const u64* mult;    // [n] or nullptr
  u32 W, R, voff, log_n;
  u32* slots;  // hash table: first table row of each distinct content (SAT_EMPTY = free)
  u64 slot_mask;
  unsigned long long* count;    // [n] tuples per content, at its first row
  unsigned long long* msum_lo;  // [n] sum of the low / high 32 bits of the canonical multiplicities of its rows
  unsigned long long* msum_hi;
  SatAcc* acc;
};

__device__ __forceinline__ void lk_table_row(const LookupCheckParams& p, u64 r, u64 (&v)[LK_MAX_WIDTH]) {
  const u64 n = 1ull << p.log_n;
  for (u32 j = 0; j <= p.W; j++) v[j] = gl::canon(__ldg(p.tables + j * n + r));
}
__device__ __forceinline__ u64 lk_hash(const u64 (&v)[LK_MAX_WIDTH], u32 len) {
  u64 h = 0x9e3779b97f4a7c15ull;
  for (u32 j = 0; j < len; j++) h = sat_hash(h ^ v[j]) + j;
  return h;
}
__device__ __forceinline__ bool lk_row_equals(const LookupCheckParams& p, u64 r, const u64 (&v)[LK_MAX_WIDTH]) {
  const u64 n = 1ull << p.log_n;
  for (u32 j = 0; j <= p.W; j++)
    if (gl::canon(__ldg(p.tables + j * n + r)) != v[j]) return false;
  return true;
}
// first table row with content v, or SAT_EMPTY
__device__ u32 lk_find(const LookupCheckParams& p, const u64 (&v)[LK_MAX_WIDTH]) {
  for (u64 h = lk_hash(v, p.W + 1) & p.slot_mask;; h = (h + 1) & p.slot_mask) {
    const u32 r = p.slots[h];
    if (r == SAT_EMPTY || lk_row_equals(p, r, v)) return r;
  }
}

// a distinct content takes one slot, which ends up holding its smallest row: every row of the content probes the same chain,
// claims the first free slot or meets the content's slot (atomicMin).  A row equal to the row above it is not its first.
__global__ void lk_insert_kernel(const LookupCheckParams p) {
  const u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >> p.log_n) return;
  u64 v[LK_MAX_WIDTH];
  lk_table_row(p, r, v);
  if (r && lk_row_equals(p, r - 1, v)) return;
  for (u64 h = lk_hash(v, p.W + 1) & p.slot_mask;; h = (h + 1) & p.slot_mask) {
    u32 cur = p.slots[h];
    if (cur == SAT_EMPTY) {
      cur = atomicCAS(p.slots + h, SAT_EMPTY, (u32)r);
      if (cur == SAT_EMPTY) return;
    }
    if (lk_row_equals(p, cur, v)) {
      atomicMin(p.slots + h, (u32)r);
      return;
    }
  }
}

// tuple (row, sub i), i = blockIdx.y: count it at the first row of its content, or report it
__global__ void __launch_bounds__(256) lk_count_kernel(const LookupCheckParams p) {
  const u64 n = 1ull << p.log_n;
  const u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  const u32 i = blockIdx.y;
  bool miss = false;
  if (r < n) {
    u64 v[LK_MAX_WIDTH];
    for (u32 j = 0; j < p.W; j++) v[j] = gl::canon(__ldg(p.vars + (u64)(p.voff + i * p.W + j) * n + r));
    v[p.W] = gl::canon(__ldg(p.id_col + r));
    const u32 f = lk_find(p, v);
    if (f == SAT_EMPTY) miss = true;
    else atomicAdd(p.count + f, 1ull);
  }
  sat_warp_report(miss, r * p.R + i, &p.acc->lookup_unmatched, &p.acc->lookup_key);
}

// table row r adds its multiplicity to the sum of its content (split in 32-bit halves: n * 2^32 < 2^64 for n <= 2^28)
__global__ void lk_multiplicity_sum_kernel(const LookupCheckParams p) {
  const u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >> p.log_n) return;
  const u64 m = gl::canon(__ldg(p.mult + r));
  if (m == 0) return;
  u64 v[LK_MAX_WIDTH];
  lk_table_row(p, r, v);
  const u32 f = lk_find(p, v);
  atomicAdd(p.msum_lo + f, m & 0xffffffffull);
  atomicAdd(p.msum_hi + f, m >> 32);
}

__device__ __forceinline__ u64 lk_multiplicity_sum(const LookupCheckParams& p, u32 f) {
  return gl::canon(gl::add(gl::mul(gl::canon(p.msum_hi[f]), 1ull << 32), gl::canon(p.msum_lo[f])));
}

// every distinct content (one slot each): tuple count == multiplicity sum mod p
__global__ void __launch_bounds__(256) lk_compare_kernel(const LookupCheckParams p) {
  const u64 h = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  bool bad = false;
  u64 f = 0;
  if (h <= p.slot_mask) {
    f = p.slots[h];
    if (f != SAT_EMPTY) bad = (u64)p.count[f] != lk_multiplicity_sum(p, (u32)f);
  }
  sat_warp_report(bad, f, &p.acc->mult_failures, &p.acc->mult_key);
}

// bj_lookup_multiplicities: the count of each content on its first row (the other rows stay 0)
__global__ void lk_write_multiplicities_kernel(const LookupCheckParams p, u64* out) {
  const u64 h = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (h > p.slot_mask) return;
  const u32 f = p.slots[h];
  if (f != SAT_EMPTY) out[f] = p.count[f];
}

// ---- the report ----
struct FinishParams {
  const SatAcc* acc;
  const u64* gate_value;     // [n] (nullptr without gates)
  const u64* gate_selector;
  CopyParams copy;
  LookupCheckParams lk;
  bool lookup;
  bj_satisfiability_report* out;
};

__global__ void sat_finish_kernel(const FinishParams p) {
  const SatAcc& a = *p.acc;
  bj_satisfiability_report rep;
  memset(&rep, 0, sizeof(rep));
  const u64 V = p.copy.dec.V, n = 1ull << p.copy.dec.log_n;
  rep.gate_failures = a.gate_failures;
  if (a.gate_failures) {
    rep.gate_row = a.gate_key >> 32;
    rep.gate_term = (u32)a.gate_key;  // global term index: the host splits it into (gate, repetition, term)
    rep.gate_value = p.gate_value[rep.gate_row];
    rep.gate_selector = p.gate_selector[rep.gate_row];
  }
  rep.copy_failures = a.copy_failures;
  if (a.copy_failures) {
    rep.copy_row = a.copy_key / V;
    rep.copy_column = (u32)(a.copy_key % V);
    const u64 i = (u64)rep.copy_column * n + rep.copy_row;
    u32 c2 = 0;
    u64 r2 = 0;
    sigma_decode(p.copy.dec, p.copy.sigmas[i], &c2, &r2);
    rep.copy_other_column = c2;
    rep.copy_other_row = r2;
    rep.copy_value = gl::canon(p.copy.vars[i]);
    rep.copy_other_value = gl::canon(p.copy.vars[(u64)c2 * n + r2]);
  }
  rep.sigma_failures = a.sigma_failures;
  if (a.sigma_failures) {
    rep.sigma_row = (a.sigma_key >> 2) / V;
    rep.sigma_column = (u32)((a.sigma_key >> 2) % V);
    rep.sigma_kind = (u32)(a.sigma_key & 3);
  }
  if (p.lookup) {
    rep.lookup_unmatched = a.lookup_unmatched;
    if (a.lookup_unmatched) {
      rep.lookup_row = a.lookup_key / p.lk.R;
      rep.lookup_subargument = (u32)(a.lookup_key % p.lk.R);
    }
    rep.multiplicity_failures = a.mult_failures;
    if (a.mult_failures) {
      rep.multiplicity_row = a.mult_key;
      rep.multiplicity_count = p.lk.count[a.mult_key];
      rep.multiplicity_sum = lk_multiplicity_sum(p.lk, (u32)a.mult_key);
    }
  }
  rep.satisfied = !(rep.gate_failures || rep.copy_failures || rep.sigma_failures || rep.lookup_unmatched || rep.multiplicity_failures);
  *p.out = rep;
}

static unsigned sat_blocks(u64 n, unsigned threads) { return (unsigned)((n + threads - 1) / threads); }

// shared argument rules of the two entry points (no kernel is launched before they pass)
static int32_t sat_validate(bj_ctx* ctx, const char* who, const bj_circuit* c, const uint64_t* d_constants, const uint64_t* d_lookup_tables,
                            const uint64_t* d_variables, bool need_lookup) {
  const std::string w(who);
  if (!c || !d_variables || c->num_variables == 0 || c->log_n == 0 || c->log_n > 28 || (c->num_constants && !d_constants) ||
      (c->n_gates && !c->gates))
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, w + ": bad argument (NULL column, empty or oversized circuit)");
  if (need_lookup && !c->lookup_width) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, w + ": the circuit has no lookup argument");
  if (c->lookup_width) {
    if (!d_lookup_tables) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, w + ": the lookup argument needs the table columns");
    if (c->lookup_table_id_column >= c->num_constants) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, w + ": lookup table-id column out of range");
    if (c->lookup_num_repetitions == 0 || c->lookup_num_repetitions > (uint32_t)LK_MAX_SUB || c->lookup_width + 1 > (uint32_t)LK_MAX_WIDTH ||
        (uint64_t)c->lookup_variables_offset + (uint64_t)c->lookup_width * c->lookup_num_repetitions > c->num_variables)
      BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, w + ": inconsistent lookup description");
  }
  return BJ_OK;
}

// the lookup hash table and the tuple counts (shared by the check and bj_lookup_multiplicities)
struct LookupScratch {
  DevMem slots, count, msum;
  LookupCheckParams p{};
};
static int32_t lookup_build_and_count(bj_ctx* ctx, const bj_circuit* c, const uint64_t* d_constants, const uint64_t* d_lookup_tables,
                                      const uint64_t* d_variables, const uint64_t* d_multiplicities, SatAcc* d_acc, LookupScratch& s) {
  const u64 n = 1ull << c->log_n, n_slots = 2 * n;
  BJ_TRY(s.slots.alloc(ctx, n_slots / 2));  // u32 slots
  BJ_TRY(s.count.alloc(ctx, n));
  BJ_CUDA(ctx, cudaMemsetAsync(s.slots.p, 0xff, sizeof(u32) * n_slots, ctx->stream));
  BJ_CUDA(ctx, cudaMemsetAsync(s.count.p, 0, sizeof(u64) * n, ctx->stream));
  LookupCheckParams& p = s.p;
  p.tables = (const u64*)d_lookup_tables;
  p.vars = (const u64*)d_variables;
  p.id_col = (const u64*)d_constants + (size_t)c->lookup_table_id_column * n;
  p.mult = (const u64*)d_multiplicities;
  p.W = c->lookup_width;
  p.R = c->lookup_num_repetitions;
  p.voff = c->lookup_variables_offset;
  p.log_n = c->log_n;
  p.slots = (u32*)s.slots.p;
  p.slot_mask = n_slots - 1;
  p.count = (unsigned long long*)s.count.p;
  p.acc = d_acc;
  if (d_multiplicities) {
    BJ_TRY(s.msum.alloc(ctx, 2 * n));
    BJ_CUDA(ctx, cudaMemsetAsync(s.msum.p, 0, sizeof(u64) * 2 * n, ctx->stream));
    p.msum_lo = (unsigned long long*)s.msum.p;
    p.msum_hi = p.msum_lo + n;
  }
  lk_insert_kernel<<<sat_blocks(n, 256), 256, 0, ctx->stream>>>(p);
  BJ_LAUNCH_CHECK(ctx);
  lk_count_kernel<<<dim3(sat_blocks(n, 256), p.R), 256, 0, ctx->stream>>>(p);
  BJ_LAUNCH_CHECK(ctx);
  return BJ_OK;
}

static int32_t sat_acc_init(bj_ctx* ctx, DevMem& acc) {
  BJ_TRY(acc.alloc(ctx, sizeof(SatAcc) / sizeof(u64)));
  SatAcc h;
  h.gate_failures = h.copy_failures = h.sigma_failures = h.lookup_unmatched = h.mult_failures = 0;
  h.gate_key = h.copy_key = h.sigma_key = h.lookup_key = h.mult_key = SAT_NO_KEY;
  BJ_CUDA(ctx, cudaMemcpyAsync(acc.p, &h, sizeof(h), cudaMemcpyHostToDevice, ctx->stream));
  return BJ_OK;
}

}  // namespace bj

using namespace bj;

extern "C" int32_t bj_check_satisfied(bj_ctx* ctx, const bj_circuit* circuit, const uint64_t* d_sigmas, const uint64_t* d_constants,
                                      const uint64_t* d_lookup_tables, const uint64_t* d_variables, const uint64_t* d_multiplicities,
                                      bj_satisfiability_report* out) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx) return BJ_ERR_INVALID_ARG;
  if (!out || !d_sigmas) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_check_satisfied: bad argument (NULL column or report)");
  BJ_TRY(sat_validate(ctx, "bj_check_satisfied", circuit, d_constants, d_lookup_tables, d_variables, false));
  const bj_circuit& c = *circuit;
  if (c.lookup_width && !d_multiplicities) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_check_satisfied: the lookup argument needs the multiplicities column");
  CompiledGates compiled;
  if (c.n_gates) {
    GateCompileError err;
    if (compile_gates(&err, ctx->gate_peephole, c.gates, c.n_gates, c.num_variables, 0, c.num_constants, compiled) != BJ_OK)
      BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_check_satisfied: " + err.last_error);
    if (compiled.total_terms >> 32) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_check_satisfied: more than 2^32 gate terms per row");
  }
  const u32 V = c.num_variables, log_n = c.log_n;
  const u64 n = 1ull << log_n, cells = (u64)V << log_n;
  // sigma decode tables (host): k_c^n ascending with their columns, k_c^-1 by column
  std::vector<u64> k(V), kn(V), kinv(V);
  std::vector<u32> kn_col(V);
  BJ_TRY(bj_non_residues_for_copy_permutation(n, V, (uint64_t*)k.data()));
  {
    std::vector<std::pair<u64, u32>> sorted(V);
    for (u32 j = 0; j < V; j++) {
      sorted[j] = {gl::pow(k[j], n), j};
      kinv[j] = gl::inv(k[j]);
    }
    std::sort(sorted.begin(), sorted.end());
    for (u32 j = 0; j < V; j++) kn[j] = sorted[j].first, kn_col[j] = sorted[j].second;
  }
  DevMem acc, gate_first, omega_tab, bitmaps, small;
  BJ_TRY(sat_acc_init(ctx, acc));
  SatAcc* d_acc = (SatAcc*)acc.p;
  FinishParams fp{};
  fp.acc = d_acc;
  // ---- gates: the interpreter in check mode over the n rows ----
  if (c.n_gates) {
    BJ_TRY(gate_first.alloc(ctx, 2 * n));
    GateEvalParams p{};
    std::vector<const u64*> table;
    for (u32 j = 0; j < V; j++) table.push_back((const u64*)d_variables + (size_t)j * n);
    for (u32 j = 0; j < c.num_constants; j++) table.push_back((const u64*)d_constants + (size_t)j * n);
    BJ_TRY(gate_program_upload(ctx, compiled, table, V, &p));
    p.n_rows = n;
    GateCheckOut chk{gate_first.p, gate_first.p + n, &d_acc->gate_failures, &d_acc->gate_key};
    const int k_pts = gate_points_per_thread(ctx, n);
    const bool small_slots = compiled.max_slots <= 32;
    if (k_pts == 4) small_slots ? gate_check_launch<4, 32>(p, chk, ctx->stream) : gate_check_launch<4, GATE_MAX_TMP>(p, chk, ctx->stream);
    else if (k_pts == 2) small_slots ? gate_check_launch<2, 32>(p, chk, ctx->stream) : gate_check_launch<2, GATE_MAX_TMP>(p, chk, ctx->stream);
    else small_slots ? gate_check_launch<1, 32>(p, chk, ctx->stream) : gate_check_launch<1, GATE_MAX_TMP>(p, chk, ctx->stream);
    BJ_LAUNCH_CHECK(ctx);
    fp.gate_value = gate_first.p;
    fp.gate_selector = gate_first.p + n;
  }
  // ---- copy constraints ----
  const u64 w_slots = 2 * n;
  BJ_TRY(omega_tab.alloc(ctx, w_slots + w_slots / 2));  // u64 keys, then u32 rows
  BJ_TRY(bitmaps.alloc(ctx, 2 * ((cells + 63) / 64)));
  BJ_TRY(small.alloc(ctx, 3 * (size_t)V));
  const u64 bitmap_words = 2 * ((cells + 63) / 64);  // u32 words of one bitmap
  BJ_CUDA(ctx, cudaMemsetAsync(omega_tab.p, 0, sizeof(u64) * w_slots, ctx->stream));
  BJ_CUDA(ctx, cudaMemsetAsync(bitmaps.p, 0, sizeof(u32) * 2 * bitmap_words, ctx->stream));
  BJ_CUDA(ctx, cudaMemcpyAsync(small.p, kn.data(), sizeof(u64) * V, cudaMemcpyHostToDevice, ctx->stream));
  BJ_CUDA(ctx, cudaMemcpyAsync(small.p + V, kinv.data(), sizeof(u64) * V, cudaMemcpyHostToDevice, ctx->stream));
  BJ_CUDA(ctx, cudaMemcpyAsync(small.p + 2 * (size_t)V, kn_col.data(), sizeof(u32) * V, cudaMemcpyHostToDevice, ctx->stream));
  // the host vectors must outlive the asynchronous copies from pageable memory: cudaMemcpyAsync stages them before returning
  CopyParams cp{};
  cp.vars = (const u64*)d_variables;
  cp.sigmas = (const u64*)d_sigmas;
  cp.dec.kn = small.p;
  cp.dec.k_inv = small.p + V;
  cp.dec.kn_col = (const u32*)(small.p + 2 * (size_t)V);
  cp.dec.w_key = omega_tab.p;
  cp.dec.w_row = (const u32*)(omega_tab.p + w_slots);
  cp.dec.w_mask = w_slots - 1;
  cp.dec.V = V;
  cp.dec.log_n = log_n;
  cp.named_once = (u32*)bitmaps.p;
  cp.named_again = (u32*)bitmaps.p + bitmap_words;
  cp.acc = d_acc;
  sat_omega_table_kernel<<<sat_blocks(n, 256), 256, 0, ctx->stream>>>(gl::omega(log_n), n, omega_tab.p, (u32*)(omega_tab.p + w_slots), w_slots - 1);
  BJ_LAUNCH_CHECK(ctx);
  sat_copy_kernel<<<sat_blocks(cells, 256), 256, 0, ctx->stream>>>(cp);
  BJ_LAUNCH_CHECK(ctx);
  sat_named_kernel<<<sat_blocks(cells, 256), 256, 0, ctx->stream>>>(cp);
  BJ_LAUNCH_CHECK(ctx);
  fp.copy = cp;
  // ---- lookups ----
  LookupScratch lks;
  if (c.lookup_width) {
    BJ_TRY(lookup_build_and_count(ctx, circuit, d_constants, d_lookup_tables, d_variables, d_multiplicities, d_acc, lks));
    lk_multiplicity_sum_kernel<<<sat_blocks(n, 256), 256, 0, ctx->stream>>>(lks.p);
    BJ_LAUNCH_CHECK(ctx);
    lk_compare_kernel<<<sat_blocks(lks.p.slot_mask + 1, 256), 256, 0, ctx->stream>>>(lks.p);
    BJ_LAUNCH_CHECK(ctx);
    fp.lk = lks.p;
    fp.lookup = true;
  }
  // ---- the report ----
  DevMem d_rep;
  BJ_TRY(d_rep.alloc(ctx, (sizeof(bj_satisfiability_report) + 7) / 8));
  fp.out = (bj_satisfiability_report*)d_rep.p;
  sat_finish_kernel<<<1, 1, 0, ctx->stream>>>(fp);
  BJ_LAUNCH_CHECK(ctx);
  bj_satisfiability_report rep;
  BJ_CUDA(ctx, cudaMemcpyAsync(&rep, d_rep.p, sizeof(rep), cudaMemcpyDeviceToHost, ctx->stream));
  BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (rep.gate_failures) {  // global term index -> (gate, repetition, term)
    const u32 t = rep.gate_term;
    u32 g = 0;
    while (g + 1 < compiled.gates.size() && compiled.gates[g + 1].term_base <= t) g++;
    const DevGate& dg = compiled.gates[g];
    rep.gate_index = g;
    rep.gate_repetition = (t - dg.term_base) / dg.n_writes;
    rep.gate_term = (t - dg.term_base) % dg.n_writes;
  }
  *out = rep;
  return BJ_OK;
}

extern "C" int32_t bj_lookup_multiplicities(bj_ctx* ctx, const bj_circuit* circuit, const uint64_t* d_constants, const uint64_t* d_lookup_tables,
                                            const uint64_t* d_variables, uint64_t* d_multiplicities) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx) return BJ_ERR_INVALID_ARG;
  if (!d_multiplicities) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_lookup_multiplicities: bad argument (NULL output column)");
  BJ_TRY(sat_validate(ctx, "bj_lookup_multiplicities", circuit, d_constants, d_lookup_tables, d_variables, true));
  const u64 n = 1ull << circuit->log_n;
  DevMem acc;
  BJ_TRY(sat_acc_init(ctx, acc));
  LookupScratch lks;
  BJ_TRY(lookup_build_and_count(ctx, circuit, d_constants, d_lookup_tables, d_variables, nullptr, (SatAcc*)acc.p, lks));
  SatAcc h;
  BJ_CUDA(ctx, cudaMemcpyAsync(&h, acc.p, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
  BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (h.lookup_unmatched) {
    const u64 row = h.lookup_key / circuit->lookup_num_repetitions, sub = h.lookup_key % circuit->lookup_num_repetitions;
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_lookup_multiplicities: " + std::to_string(h.lookup_unmatched) +
                                         " lookup tuple(s) match no table row; the first is sub-argument " + std::to_string(sub) + " of row " +
                                         std::to_string(row));
  }
  BJ_CUDA(ctx, cudaMemsetAsync(d_multiplicities, 0, sizeof(u64) * n, ctx->stream));
  lk_write_multiplicities_kernel<<<sat_blocks(lks.p.slot_mask + 1, 256), 256, 0, ctx->stream>>>(lks.p, (u64*)d_multiplicities);
  BJ_LAUNCH_CHECK(ctx);
  BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return BJ_OK;
}
