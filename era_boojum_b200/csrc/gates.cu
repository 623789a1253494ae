// Per-row gate / quotient evaluator over general-purpose columns and over specialised columns.
//
// Reference semantics (what is computed, bit-exact):
//   * a gate's constraint terms come from GateConstraintEvaluator::evaluate_once (src/cs/traits/evaluator.rs:145-152),
//     repeated `num_repetitions` times per row with PerChunkOffset (RowwiseEvaluator, evaluator.rs:376-397); row-shared
//     constants are read once at repetition 0 (load_row_shared_constants);
//   * every pushed term is folded with the next alpha power, the power index running on across the gates of the row
//     (push_evaluation_result, src/cs/implementations/buffering_source.rs:304-362), the per-gate sum is multiplied by the
//     gate's selector and added to the quotient (proceed_to_next_gate, :158-221);
//   * the selector of a gate is the product along its path in the selector tree of const_i or (1 - const_i)
//     (compute_selector_subpath, src/cs/implementations/prover.rs:2775-2916); the gate's own constants start at column
//     `path length` (constant_placement_offset, prover.rs:1000-1013);
//   * driver: the row loop of prove_cpu_basic (prover.rs:1031-1080) over the first Q cosets of the LDE.
//   * gates placed on SPECIALISED columns (GatePlacementStrategy::UseSpecializedColumns, prover.rs:653-801) own a fixed range
//     of columns: no selector, the first repetition starts at the gate's initial offset, constants start behind those of
//     the general-purpose gates (shared by the repetitions when share_constants); their terms precede the general-purpose ones.
// The gate itself is data: the SSA program the reference's own GPU hook records (gpu_synthesizer::GPUDataCapture,
// src/gpu_synthesizer/mod.rs:115-133, 354-443) - Index::{VariablePoly, WitnessPoly, ConstantPoly, TemporaryValue,
// ConstantValue} and Relation::{Add, Double, Sub, Negate, Mul, Square, Inverse} - so any evaluator the reference can
// capture runs here unchanged.  One thread owns up to four (coset, row) points and interprets the programs for all of them at
// once (one decode per step); column loads are coalesced across threads, temporaries live in thread-local memory.
#include <algorithm>
#include <cstring>
#include <functional>
#include <vector>
#include "ctx.hpp"

namespace bj {

constexpr int GATE_MAX_TMP = 128;            // live temporaries per thread after host-side slot allocation
constexpr u32 GATE_MAX_PROGRAM_TMP = 1u << 20;  // temporaries a recorded program may name (SSA: one per relation)
// internal steps next to the seven recorded relation kinds (BJ_REL_* = 0..6)
constexpr u32 GATE_OP_PUSH = 7;               // fold operand a into the accumulator with alpha power `dst` of the repetition
constexpr u32 GATE_OP_MADD = 8;               // dst = a * b + c, a product whose only use is the sum that follows (host peephole)
constexpr u32 GATE_OP_LINCOMB = 9;            // dst = bias + sum_j k_j * x_j, 2..16 terms, k_j < 2^28 (host peephole: sum trees)
constexpr u32 GATE_CODE_LINCOMB = 48;         // its opcode (gate_code() numbers the others 0..47)
constexpr u32 GATE_LINCOMB_MAX_TERMS = 16, GATE_LINCOMB_MAX_COEFF = 1u << 28;  // 16 * 2^64 * 2^28 + 2^64 <= 2^96: one 96-bit sum

struct DevOperand {
  u32 kind;  // bj_gate_index kinds
  u32 pad;
  u64 value;
};
struct DevOp {  // host-side form of one step (the device reads PackedOp)
  u32 op;
  u32 dst;
  DevOperand a, b;
  DevOperand c;     // GATE_OP_MADD only
  int32_t lc = -1;  // GATE_OP_LINCOMB: index of its term list; a.value = the constant term
  bool push = false;  // the step's value is a quotient term read by nothing else: it is pushed (dst = term index), not stored
};
struct LcTerm {      // k * x, x a temporary or a variable column
  DevOperand x;
  u32 k;
};
struct DevGate {  // placement (PerChunkOffset, specialised-column bases, first constant column) is folded into the steps' operands
  u32 ops_begin, n_ops;                       // records of the gate's program in GateEvalParams::ops
  u32 n_writes;                               // quotient terms per repetition
  u32 num_repetitions;
  u32 path_len;
  u32 path_bits;  // bit i = path[i]
  u32 term_base;  // index of the gate's first alpha power
};

// Device form of one program step (32 bytes, read with two 128-bit uniform loads).  The host lowers the recorded program to
// it: operand kinds collapse to three classes - T: temporary slot, L: column of the unified table [variables | witnesses |
// constants] (index of repetition 0 plus a per-repetition stride), I: immediate field element - and the opcode carries the
// classes, so the interpreter decodes ONE dense switch per step and the step bodies contain no operand dispatch.
struct PackedOp {
  u32 code_dst;  // code (7 bits) | push flag (bit 7) | destination slot, or the term index when the value is pushed (24 bits)
  u32 strides;   // per-repetition column stride of operand a (low 16 bits) and b (high 16 bits)
  u64 a, b;      // slot / column index / immediate
  u64 c;         // GATE_OP_MADD: slot of the addend
};
// GATE_OP_LINCOMB: the header {code | dst, variables stride, a = number of terms, b = constant term} is followed by
// ceil(n / 4) records of four (ref, k) pairs; ref = slot, or 0x80000000 | variable column of repetition 0
struct PackedTerm {
  u32 ref, k;
};
static_assert(sizeof(PackedOp) == 32, "PackedOp is read as two uint4");
constexpr int KIND_T = 0, KIND_L = 1, KIND_I = 2;
// dense numbering: ADD 0-8, SUB 9-17, MUL 18-26 by (class a, class b); DOUBLE, NEGATE, SQUARE, INVERSE, PUSH 27-41 by class a;
// MADD 42-47 by (class a in {T, L}, class b), its addend is always a temporary
__host__ __device__ constexpr u32 gate_code(u32 op, int ka, int kb) {
  return op == GATE_OP_MADD ? 42u + (u32)(ka * 3 + kb)
       : op == BJ_REL_ADD ? (u32)(ka * 3 + kb)
       : op == BJ_REL_SUB ? 9u + (u32)(ka * 3 + kb)
       : op == BJ_REL_MUL ? 18u + (u32)(ka * 3 + kb)
       : op == BJ_REL_DOUBLE ? 27u + (u32)ka
       : op == BJ_REL_NEGATE ? 30u + (u32)ka
       : op == BJ_REL_SQUARE ? 33u + (u32)ka
       : op == BJ_REL_INVERSE ? 36u + (u32)ka
       : 39u + (u32)ka;
}

struct GateEvalParams {
  const DevGate* gates;
  u32 n_gates;
  const PackedOp* ops;
  const u64* const* cols;  // [variables | witnesses | constants]
  u32 consts_base;         // index of constant column 0 in `cols` (the selector path reads constants 0 .. path_len - 1)
  const u64* alphas;       // (c0, c1) per term
  u64 n_rows;
  u64* q_c0;
  u64* q_c1;
};

// Temporaries of the K points of a thread live in thread-local memory, [slot][point] (32 bytes per slot for K = 4: two 128-bit
// accesses).  A shared-memory slab was tried instead: the slab limits the block residency and
// the interpreter then waits on latencies it cannot hide - slower than the L1-cached local array.
template <int K>
struct GateSlots {
  u64 (*v)[K];
  __device__ __forceinline__ void load(u32 slot, u64 (&out)[K]) const {
#pragma unroll
    for (int k = 0; k < K; k++) out[k] = v[slot][k];
  }
  __device__ __forceinline__ void store(u32 slot, const u64 (&r)[K]) const {
#pragma unroll
    for (int k = 0; k < K; k++) v[slot][k] = r[k];
  }
};

template <int KIND, int K>
__device__ __forceinline__ void gate_operand(u64 (&out)[K], u64 raw, u32 stride, u32 rep, const GateSlots<K>& tmp, const u64* const* cols,
                                             const u64 (&pt)[K]) {
  if (KIND == KIND_T) {
    tmp.load((u32)raw, out);
  } else if (KIND == KIND_L) {
    const u64* col = cols[(u32)raw + rep * stride];
#pragma unroll
    for (int k = 0; k < K; k++) out[k] = __ldg(col + pt[k]);
  } else {
#pragma unroll
    for (int k = 0; k < K; k++) out[k] = raw;
  }
}

// One step for the K points of the thread: the value it computes is returned in r; the caller stores it in the destination slot
// or, for a step that carries the push flag, folds it into the gate's accumulator.  Values in the slots are LAZY (any u64
// congruent to the value): products skip the final canonicalisation, sums canonicalise their second operand only.
template <int OP, int KA, int KB, int K>
__device__ __forceinline__ void gate_step(u64 (&r)[K], const uint4* op, u32 strides, u64 a_raw, u32 rep, const GateSlots<K>& tmp,
                                          const u64* const* cols, const u64 (&pt)[K]) {
  u64 a[K], b[K];
  gate_operand<KA, K>(a, a_raw, strides & 0xffffu, rep, tmp, cols, pt);
  u64 b_raw = 0;
  if (OP == BJ_REL_ADD || OP == BJ_REL_SUB || OP == BJ_REL_MUL || OP == (int)GATE_OP_MADD) {
    const uint4 wb = __ldg(op + 1);
    b_raw = ((u64)wb.y << 32) | wb.x;
    gate_operand<KB, K>(b, b_raw, strides >> 16, rep, tmp, cols, pt);
    if (OP == (int)GATE_OP_MADD) {
      u64 c[K];
      tmp.load(wb.z, c);
      if (KB == KIND_I && (b_raw >> 32) == 0) {  // 32-bit immediate (uniform test): a * k + c exactly in 96 bits, one reduction
#pragma unroll
        for (int k = 0; k < K; k++) r[k] = gl::w96_reduce(gl::w96_add64(gl::mul_u32_wide(a[k], (u32)b_raw), c[k]));
      } else {
#pragma unroll
        for (int k = 0; k < K; k++) r[k] = gl::fma_lazy(a[k], b[k], c[k]);
      }
    }
  }
  if (OP != (int)GATE_OP_MADD) {
#pragma unroll
  for (int k = 0; k < K; k++) {
    if (OP == BJ_REL_ADD) r[k] = gl::add_lazy(a[k], b[k]);
    else if (OP == BJ_REL_DOUBLE) r[k] = gl::add_lazy(a[k], a[k]);
    else if (OP == BJ_REL_SUB) r[k] = gl::sub_lazy(a[k], b[k]);
    else if (OP == BJ_REL_NEGATE) r[k] = gl::neg(a[k]);
    else if (OP == BJ_REL_MUL) r[k] = (KB == KIND_I && (b_raw >> 32) == 0) ? gl::w96_reduce(gl::mul_u32_wide(a[k], (u32)b_raw)) : gl::mul_lazy(a[k], b[k]);
    else if (OP == BJ_REL_SQUARE) r[k] = gl::mul_lazy(a[k], a[k]);
    else if (OP == BJ_REL_INVERSE) r[k] = gl_inv_chain(gl::canon(a[k]));
    else r[k] = a[k];  // GATE_OP_PUSH of a bare operand (column / constant / a temporary that is also read elsewhere)
  }
  }
}

#define GATE_CASE(OP, KA, KB) \
  case gate_code(OP, KA, KB): gate_step<(int)(OP), KA, KB, K>(r, op, w.y, a_raw, rep, tmp, p.cols, pt); break;
#define GATE_CASES_UNARY(OP) GATE_CASE(OP, KIND_T, 0) GATE_CASE(OP, KIND_L, 0) GATE_CASE(OP, KIND_I, 0)
#define GATE_CASES_BINARY(OP)                                                                     \
  GATE_CASE(OP, KIND_T, KIND_T) GATE_CASE(OP, KIND_T, KIND_L) GATE_CASE(OP, KIND_T, KIND_I)      \
  GATE_CASE(OP, KIND_L, KIND_T) GATE_CASE(OP, KIND_L, KIND_L) GATE_CASE(OP, KIND_L, KIND_I)      \
  GATE_CASE(OP, KIND_I, KIND_T) GATE_CASE(OP, KIND_I, KIND_L) GATE_CASE(OP, KIND_I, KIND_I)

// Check mode (bj_check_satisfied): the same interpreter on the trace domain, where every pushed term of a selected gate must be
// 0.  A gate runs only where its selector is nonzero; per point the thread counts the (gate, repetition) instances with a
// nonzero term and keeps the first one in (gate, repetition, term) order.  Each row belongs to one thread, so its first
// failure is written to the row's slot without a race; the smallest (row, term index) key is found with atomicMin.
struct GateCheckOut {
  u64* first_value;              // [n_rows] the row's first nonzero term (written on failing rows only)
  u64* first_selector;           // [n_rows] the selector of its gate
  unsigned long long* failures;  // (row, gate, repetition) instances with a nonzero term
  unsigned long long* first_key; // min of row << 32 | global term index (gate.term_base + rep * n_writes + term)
};
constexpr u32 GATE_NO_TERM = 0xffffffffu;

// One thread owns K points (block b: points b * 128 * K + k * 128 + thread, so every column load is coalesced).  Decoding a
// step costs the same for K points as for one (the one-point interpreter is bound by the instruction issue rate).  Tried and
// dropped: fetching the next step's words ahead, a register budget of 128 with half the resident blocks, temporaries in
// shared memory.
template <int K, int S, bool CHECK>
__device__ __forceinline__ void gate_eval_body(const GateEvalParams& p, const GateCheckOut& chk) {
  u64 slots[S][K];
  const GateSlots<K> tmp{slots};
  const u64 first = (u64)blockIdx.x * (128 * K) + threadIdx.x;
  u64 pt[K];
#pragma unroll
  for (int k = 0; k < K; k++) pt[k] = min(first + (u64)k * 128, p.n_rows - 1);  // out-of-range points repeat the last one, not stored
  gl::e2 q[K];
#pragma unroll
  for (int k = 0; k < K; k++) q[k] = {0, 0};
  u32 fails[K], first_term[K];  // check mode: failing instances of the point, its first failing term (global index)
  u64 first_val[K], first_sel[K];
  if constexpr (CHECK) {
#pragma unroll
    for (int k = 0; k < K; k++) fails[k] = 0, first_term[k] = GATE_NO_TERM, first_val[k] = first_sel[k] = 0;
  }
  for (u32 g = 0; g < p.n_gates; g++) {
    const DevGate gate = p.gates[g];
    gl::e2 acc[K];
#pragma unroll
    for (int k = 0; k < K; k++) acc[k] = {0, 0};
    u64 csel[K];  // check mode: the selector, known before the program runs
    bool selected = true;
    if constexpr (CHECK) {
      selected = false;
#pragma unroll
      for (int k = 0; k < K; k++) {
        u64 sel = 1;
        for (u32 i = 0; i < gate.path_len; i++) {
          const u64 c = gl::canon(__ldg(p.cols[p.consts_base + i] + pt[k]));
          sel = gl::mul(sel, ((gate.path_bits >> i) & 1) ? c : gl::canon(gl::sub(1, c)));
        }
        csel[k] = gl::canon(sel);
        selected |= csel[k] != 0;
      }
    }
    if (gate.n_ops && selected) {
      for (u32 rep = 0; rep < gate.num_repetitions; rep++) {
        u32 rep_term[K];  // check mode: smallest failing term index of this repetition (pushes come in program order)
        u64 rep_val[K];
        if constexpr (CHECK) {
#pragma unroll
          for (int k = 0; k < K; k++) rep_term[k] = GATE_NO_TERM, rep_val[k] = 0;
        }
        const u64* alpha_rep = p.alphas + 2 * (size_t)(gate.term_base + rep * gate.n_writes);
        const uint4* op = reinterpret_cast<const uint4*>(p.ops + gate.ops_begin);
        for (u32 i = 0; i < gate.n_ops; i++, op += 2) {
          const uint4 w = __ldg(op);  // code | dst, strides, operand a; operand b is fetched by the binary steps only
          const u32 dst = w.x >> 8;   // destination slot, or the term index when the step pushes its value (bit 7 of the code)
          const u64 a_raw = ((u64)w.w << 32) | w.z;
          u64 r[K];
          switch (w.x & 0x7fu) {
            case GATE_CODE_LINCOMB: {
              const uint4 wb = __ldg(op + 1);
              const u32 n = w.z;
              const PackedTerm* terms = reinterpret_cast<const PackedTerm*>(op + 2);
              gl::w96 sum[K];
#pragma unroll
              for (int k = 0; k < K; k++) sum[k] = gl::w96_from(((u64)wb.y << 32) | wb.x);
              for (u32 t = 0; t < n; t++) {
                const uint2 tm = __ldg(reinterpret_cast<const uint2*>(terms + t));
                u64 x[K];
                if (tm.x >> 31) gate_operand<KIND_L, K>(x, tm.x & 0x7fffffffu, w.y, rep, tmp, p.cols, pt);
                else tmp.load(tm.x, x);
#pragma unroll
                for (int k = 0; k < K; k++) sum[k] = gl::w96_add(sum[k], gl::mul_u32_wide(x[k], tm.y));
              }
#pragma unroll
              for (int k = 0; k < K; k++) r[k] = gl::w96_reduce(sum[k]);
              const u32 extra = (n + 3) / 4;  // the term records are part of the step
              op += 2 * (size_t)extra;
              i += extra;
              break;
            }
            GATE_CASES_BINARY(BJ_REL_ADD)
            GATE_CASES_BINARY(BJ_REL_SUB)
            GATE_CASES_BINARY(BJ_REL_MUL)
            GATE_CASES_UNARY(BJ_REL_DOUBLE)
            GATE_CASES_UNARY(BJ_REL_NEGATE)
            GATE_CASES_UNARY(BJ_REL_SQUARE)
            GATE_CASES_UNARY(BJ_REL_INVERSE)
            GATE_CASES_UNARY(GATE_OP_PUSH)
            GATE_CASE(GATE_OP_MADD, KIND_T, KIND_T) GATE_CASE(GATE_OP_MADD, KIND_T, KIND_L) GATE_CASE(GATE_OP_MADD, KIND_T, KIND_I)
            GATE_CASE(GATE_OP_MADD, KIND_L, KIND_T) GATE_CASE(GATE_OP_MADD, KIND_L, KIND_L) GATE_CASE(GATE_OP_MADD, KIND_L, KIND_I)
            default:
#pragma unroll
              for (int k = 0; k < K; k++) r[k] = 0;
              break;
          }
          if (w.x & 0x80u) {
            if constexpr (CHECK) {  // the term must be 0 where the gate is selected
#pragma unroll
              for (int k = 0; k < K; k++) {
                const u64 v = gl::canon(r[k]);
                if (csel[k] != 0 && v != 0 && dst < rep_term[k]) rep_term[k] = dst, rep_val[k] = v;
              }
            } else {  // push_evaluation_result: the term times its alpha power goes into the gate's accumulator
              const u64 a0 = __ldg(alpha_rep + 2 * dst), a1 = __ldg(alpha_rep + 2 * dst + 1);
#pragma unroll
              for (int k = 0; k < K; k++) {
                acc[k].c0 = gl::fma_lazy(r[k], a0, acc[k].c0);  // the running sum enters the 128-bit product before its one reduction
                acc[k].c1 = gl::fma_lazy(r[k], a1, acc[k].c1);
              }
            }
          } else {
            tmp.store(dst, r);
          }
        }
        if constexpr (CHECK) {
#pragma unroll
          for (int k = 0; k < K; k++) {
            if (rep_term[k] == GATE_NO_TERM) continue;
            fails[k]++;
            if (first_term[k] == GATE_NO_TERM)
              first_term[k] = gate.term_base + rep * gate.n_writes + rep_term[k], first_val[k] = rep_val[k], first_sel[k] = csel[k];
          }
        }
      }
    }
    if constexpr (!CHECK) {
#pragma unroll
      for (int k = 0; k < K; k++) {
        u64 sel = 1;
        for (u32 i = 0; i < gate.path_len; i++) {
          const u64 c = gl::canon(__ldg(p.cols[p.consts_base + i] + pt[k]));
          sel = gl::mul(sel, ((gate.path_bits >> i) & 1) ? c : gl::canon(gl::sub(1, c)));
        }
        q[k].c0 = gl::add(q[k].c0, gl::mul(acc[k].c0, sel));
        q[k].c1 = gl::add(q[k].c1, gl::mul(acc[k].c1, sel));
      }
    }
  }
#pragma unroll
  for (int k = 0; k < K; k++) {
    const u64 t = first + (u64)k * 128;
    if (t < p.n_rows) {
      if constexpr (CHECK) {
        if (fails[k]) {
          atomicAdd(chk.failures, (unsigned long long)fails[k]);
          chk.first_value[t] = first_val[k];
          chk.first_selector[t] = first_sel[k];
          atomicMin(chk.first_key, (unsigned long long)((t << 32) | first_term[k]));
        }
      } else {
        p.q_c0[t] = gl::canon(gl::add(p.q_c0[t], gl::canon(q[k].c0)));
        p.q_c1[t] = gl::canon(gl::add(p.q_c1[t], gl::canon(q[k].c1)));
      }
    }
  }
}

template <int K, int S>
__global__ void __launch_bounds__(128) gate_eval_kernel(const GateEvalParams p) {
  gate_eval_body<K, S, false>(p, GateCheckOut{});
}

template <int K, int S>
__global__ void __launch_bounds__(128) gate_check_kernel(const GateEvalParams p, const GateCheckOut chk) {
  gate_eval_body<K, S, true>(p, chk);
}

template <int K, int S>
static void gate_eval_launch(const GateEvalParams& p, cudaStream_t stream) {
  gate_eval_kernel<K, S><<<(unsigned)((p.n_rows + 128 * K - 1) / (128 * K)), 128, 0, stream>>>(p);
}

template <int K, int S>
static void gate_check_launch(const GateEvalParams& p, const GateCheckOut& chk, cudaStream_t stream) {
  gate_check_kernel<K, S><<<(unsigned)((p.n_rows + 128 * K - 1) / (128 * K)), 128, 0, stream>>>(p, chk);
}

}  // namespace bj

using namespace bj;

// Host compiler of the recorded programs: validation, push placement, peephole, slot allocation, lowering.  Pure host code (no
// device, no context): bj_gate_programs_compile exposes its output, and the CPU test suite runs an emulator of the step format
// over it for every gate of the library under every peephole setting (tests/test_gate_compiler_cpu.py).
namespace {
struct GateCompileError {  // what BJ_FAIL writes to
  std::string last_error;
};
struct CompiledGates {
  std::vector<DevGate> gates;
  std::vector<PackedOp> ops;
  uint32_t max_slots = 0;
  uint64_t total_terms = 0;
};
struct GatePeephole {
  int gate_peephole;
};

int32_t compile_gates(GateCompileError* err, int peephole, const bj_gate_desc* h_gates, uint32_t n_gates, uint32_t n_variables,
                      uint32_t n_witnesses, uint32_t n_constants, CompiledGates& compiled) {
  GateCompileError* const ctx_err = err;
  const GatePeephole settings{peephole};
  const GatePeephole* const ctx = &settings;  // the passes below read ctx->gate_peephole
#define GATE_FAIL(code, msg)               \
  do {                                     \
    if (ctx_err) ctx_err->last_error = (msg); \
    return (code);                         \
  } while (0)
  std::vector<DevGate>& gates = compiled.gates;
  std::vector<PackedOp>& ops = compiled.ops;
  uint32_t& max_slots = compiled.max_slots;
  uint64_t& total_terms = compiled.total_terms;
  // operand range checks against the columns the caller passed (all repetitions)
  auto check_index = [&](const bj_gate_index& ix, const bj_gate_desc& g, DevOperand* out) -> bool {
    const uint32_t reps = g.num_repetitions ? g.num_repetitions - 1 : 0;
    switch (ix.kind) {
      case BJ_IDX_VARIABLE:
        if (g.variables_initial_offset + ix.value + (uint64_t)reps * g.variables_offset >= n_variables) return false;
        break;
      case BJ_IDX_WITNESS:
        if (g.witnesses_initial_offset + ix.value + (uint64_t)reps * g.witnesses_offset >= n_witnesses) return false;
        break;
      case BJ_IDX_CONSTANT_POLY:
        if (g.constants_placement_offset + ix.value + (uint64_t)reps * g.constants_offset >= n_constants) return false;
        break;
      case BJ_IDX_CONSTANT_POLY_SHARED:
        if (g.constants_placement_offset + ix.value >= n_constants) return false;
        break;
      case BJ_IDX_TEMPORARY:
        if (ix.value >= GATE_MAX_PROGRAM_TMP) return false;
        break;
      case BJ_IDX_CONSTANT_VALUE: break;
      default: return false;
    }
    out->kind = ix.kind;
    out->pad = 0;
    out->value = ix.kind == BJ_IDX_CONSTANT_VALUE ? gl::canon(ix.value) : ix.value;
    return true;
  };
  for (uint32_t gi = 0; gi < n_gates; gi++) {
    const bj_gate_desc& g = h_gates[gi];
    if (g.selector_path_len > 32 || g.selector_path_len > n_constants || (g.n_relations && !g.relations) ||
        (g.n_writes && !g.writes))
      GATE_FAIL(BJ_ERR_INVALID_ARG, "gate descriptor: bad selector path or NULL program");
    DevGate d{};
    d.ops_begin = (u32)ops.size();
    d.n_writes = g.n_writes;
    d.num_repetitions = g.num_repetitions;
    d.path_len = g.selector_path_len;
    d.path_bits = 0;
    d.term_base = (u32)total_terms;
    for (uint32_t i = 0; i < g.selector_path_len; i++)
      if (g.selector_path[i]) d.path_bits |= 1u << i;
    // 1. the recorded program (SSA as GPUVariablesContext records it: every relation defines a fresh TemporaryValue, used
    //    only afterwards), with the pushes of the quotient terms placed right behind the relation that defines them
    //    (push_evaluation_result is called inline by evaluate_once; the alpha power of a term is fixed by its write index)
    std::vector<DevOp> prog;
    std::vector<std::vector<LcTerm>> lincombs;  // term lists of the GATE_OP_LINCOMB steps (DevOp::lc)
    // every temporary a step reads (operands a / b, the addend of a multiply-add, the terms of a linear combination)
    const auto each_temp = [&](DevOp& o, const std::function<void(DevOperand&)>& fn) {
      if (o.a.kind == BJ_IDX_TEMPORARY) fn(o.a);
      if ((o.op == BJ_REL_ADD || o.op == BJ_REL_SUB || o.op == BJ_REL_MUL || o.op == GATE_OP_MADD) && o.b.kind == BJ_IDX_TEMPORARY) fn(o.b);
      if (o.op == GATE_OP_MADD) fn(o.c);
      if (o.op == GATE_OP_LINCOMB)
        for (LcTerm& t : lincombs[o.lc])
          if (t.x.kind == BJ_IDX_TEMPORARY) fn(t.x);
    };
    prog.reserve(g.n_relations + g.n_writes);
    std::vector<int32_t> def_at;  // program temporary -> index in `prog` of its defining op (-1: undefined)
    auto defined = [&](const bj_gate_index& ix) { return ix.kind != BJ_IDX_TEMPORARY || (ix.value < def_at.size() && def_at[ix.value] >= 0); };
    std::vector<std::vector<uint32_t>> pushes_of(g.n_relations);  // relation index -> write indices it feeds
    std::vector<uint32_t> late_pushes;                              // writes of bare columns / constants
    for (uint32_t i = 0; i < g.n_relations; i++) {
      const bj_gate_relation& r = g.relations[i];
      if (r.op > BJ_REL_INVERSE || r.dst_temporary >= GATE_MAX_PROGRAM_TMP)
        GATE_FAIL(BJ_ERR_UNSUPPORTED, "gate program: unknown relation or temporary index beyond 2^20");
      if (r.dst_temporary >= def_at.size()) def_at.resize(r.dst_temporary + 1, -1);
    }
    {
      std::vector<int32_t> def_rel(def_at.size(), -1);
      for (uint32_t i = 0; i < g.n_relations; i++) {
        if (def_rel[g.relations[i].dst_temporary] >= 0)
          GATE_FAIL(BJ_ERR_INVALID_ARG, "gate program: temporary defined twice (programs are SSA)");
        def_rel[g.relations[i].dst_temporary] = (int32_t)i;
      }
      for (uint32_t k = 0; k < g.n_writes; k++) {
        const bj_gate_index& w = g.writes[k];
        if (w.kind == BJ_IDX_TEMPORARY) {
          if (w.value >= def_rel.size() || def_rel[w.value] < 0) GATE_FAIL(BJ_ERR_INVALID_ARG, "gate program: write of an undefined temporary");
          pushes_of[def_rel[w.value]].push_back(k);
        } else {
          late_pushes.push_back(k);
        }
      }
    }
    auto emit_push = [&](uint32_t k) -> bool {
      DevOp o{};
      o.op = GATE_OP_PUSH;
      o.dst = k;
      return check_index(g.writes[k], g, &o.a) && (prog.push_back(o), true);
    };
    for (uint32_t i = 0; i < g.n_relations; i++) {
      const bj_gate_relation& r = g.relations[i];
      DevOp o{};
      o.op = r.op;
      o.dst = r.dst_temporary;
      const bool binary = r.op == BJ_REL_ADD || r.op == BJ_REL_SUB || r.op == BJ_REL_MUL;
      const bj_gate_index bdummy{BJ_IDX_CONSTANT_VALUE, 0, 0};
      if (!defined(r.a) || (binary && !defined(r.b)) || !check_index(r.a, g, &o.a) || !check_index(binary ? r.b : bdummy, g, &o.b))
        GATE_FAIL(BJ_ERR_INVALID_ARG, "gate program: operand out of range or temporary used before definition");
      def_at[r.dst_temporary] = (int32_t)prog.size();
      prog.push_back(o);
      for (uint32_t k : pushes_of[i])
        if (!emit_push(k)) GATE_FAIL(BJ_ERR_INVALID_ARG, "gate program: write operand out of range");
    }
    for (uint32_t k : late_pushes)
      if (!emit_push(k)) GATE_FAIL(BJ_ERR_INVALID_ARG, "gate program: write operand out of range");
    // 1b. peephole over the recorded program.  Evaluators written against a generic field interface record what they execute:
    //     the Poseidon2 flattened gate multiplies by the matrix entry 1 3228 times and starts 372 sums at the constant 0
    //     (9636 relations, 6036 after this pass).  x * 1, x + 0, x - 0 become aliases of x, x * 0 the constant 0; a product
    //     whose only use is a sum with a temporary becomes one multiply-add step (its 128-bit product takes the addend before
    //     the single reduction).  Values mod p are unchanged, so the quotient is bit-identical.
    {
      const auto is_const = [](const DevOperand& o, u64 v) { return o.kind == BJ_IDX_CONSTANT_VALUE && o.value == v; };
      std::vector<DevOperand> alias(def_at.size(), DevOperand{0xffffffffu, 0, 0});
      const auto resolve = [&](DevOperand& o) {
        while (o.kind == BJ_IDX_TEMPORARY && alias[o.value].kind != 0xffffffffu) o = alias[o.value];
      };
      std::vector<DevOp> kept;
      kept.reserve(prog.size());
      for (DevOp o : prog) {
        resolve(o.a);
        const bool binary = o.op == BJ_REL_ADD || o.op == BJ_REL_SUB || o.op == BJ_REL_MUL;
        if (binary) resolve(o.b);
        const DevOperand zero{BJ_IDX_CONSTANT_VALUE, 0, 0};
        if (!(ctx->gate_peephole & 1)) { kept.push_back(o); continue; }
        if (o.op == BJ_REL_MUL && (is_const(o.a, 0) || is_const(o.b, 0))) { alias[o.dst] = zero; continue; }
        if (o.op == BJ_REL_MUL && is_const(o.b, 1)) { alias[o.dst] = o.a; continue; }
        if (o.op == BJ_REL_MUL && is_const(o.a, 1)) { alias[o.dst] = o.b; continue; }
        if ((o.op == BJ_REL_ADD || o.op == BJ_REL_SUB) && is_const(o.b, 0)) { alias[o.dst] = o.a; continue; }
        if (o.op == BJ_REL_ADD && is_const(o.a, 0)) { alias[o.dst] = o.b; continue; }
        kept.push_back(o);
      }
      // sums of products with small immediates -> ONE step.  A matrix row of the Poseidon2 gate is 12 products by constants and
      // 11 sums; with the single-use sums merged bottom-up (an inner sum hands its term list to the sum that consumes it) the
      // row becomes one GATE_OP_LINCOMB: bias + sum_j k_j * x_j, accumulated in 96 bits and reduced once.
      if (ctx->gate_peephole & 4) {
        const size_t NT = def_at.size();
        std::vector<uint32_t> uses(NT, 0);
        std::vector<int32_t> def_idx(NT, -1), consumer(NT, -1);
        for (size_t i = 0; i < kept.size(); i++) {
          each_temp(kept[i], [&](DevOperand& t) {
            uses[t.value]++;
            consumer[t.value] = (int32_t)i;
          });
          if (kept[i].op != GATE_OP_PUSH) def_idx[kept[i].dst] = (int32_t)i;
        }
        struct Pending {
          std::vector<LcTerm> terms;
          u64 bias = 0;
          bool fused = false;  // something was merged into it (a plain a + b of two leaves stays an ADD)
        };
        std::vector<int32_t> pending(kept.size(), -1);
        std::vector<Pending> pend;
        std::vector<char> dead(kept.size(), 0);
        const auto leaf = [&](const DevOperand& o, Pending& acc, std::vector<int32_t>& kill) -> bool {
          if (o.kind == BJ_IDX_CONSTANT_VALUE) {
            acc.bias = gl::canon(gl::add(acc.bias, o.value));
            acc.fused = true;
            return true;
          }
          if (o.kind == BJ_IDX_VARIABLE) {
            acc.terms.push_back({o, 1u});
            return true;
          }
          if (o.kind != BJ_IDX_TEMPORARY) return false;  // witness / constant columns stay with the plain steps
          const int32_t di = def_idx[o.value];
          if (uses[o.value] == 1 && di >= 0 && !dead[di]) {
            const DevOp& d = kept[di];
            if (d.op == BJ_REL_ADD && pending[di] >= 0 && acc.terms.size() + pend[pending[di]].terms.size() <= GATE_LINCOMB_MAX_TERMS) {
              const Pending& c = pend[pending[di]];
              acc.terms.insert(acc.terms.end(), c.terms.begin(), c.terms.end());
              acc.bias = gl::canon(gl::add(acc.bias, c.bias));
              acc.fused = true;
              kill.push_back(di);
              return true;
            }
            if (d.op == BJ_REL_MUL) {
              const DevOperand *x = &d.a, *k = &d.b;
              if (x->kind == BJ_IDX_CONSTANT_VALUE) std::swap(x, k);
              if (k->kind == BJ_IDX_CONSTANT_VALUE && k->value < GATE_LINCOMB_MAX_COEFF &&
                  (x->kind == BJ_IDX_TEMPORARY || x->kind == BJ_IDX_VARIABLE)) {
                acc.terms.push_back({*x, (u32)k->value});
                acc.fused = true;
                kill.push_back(di);
                return true;
              }
            }
          }
          acc.terms.push_back({o, 1u});
          return true;
        };
        const auto finalize = [&](size_t j, const Pending& pd) {
          if (!pd.fused) return;  // a + b of two plain leaves: unchanged
          DevOp& o = kept[j];
          o.op = GATE_OP_LINCOMB;
          o.a = DevOperand{BJ_IDX_CONSTANT_VALUE, 0, pd.bias};
          o.b = DevOperand{BJ_IDX_CONSTANT_VALUE, 0, 0};
          o.lc = (int32_t)lincombs.size();
          lincombs.push_back(pd.terms);
        };
        for (size_t j = 0; j < kept.size(); j++) {
          if (kept[j].op != BJ_REL_ADD) continue;
          Pending acc;
          std::vector<int32_t> kill;
          if (!leaf(kept[j].a, acc, kill) || !leaf(kept[j].b, acc, kill) || acc.terms.size() > GATE_LINCOMB_MAX_TERMS || acc.terms.empty()) continue;
          for (int32_t d : kill) dead[d] = 1;
          const uint32_t t = kept[j].dst;
          const bool inner = uses[t] == 1 && consumer[t] >= 0 && kept[consumer[t]].op == BJ_REL_ADD;
          if (inner) {
            pending[j] = (int32_t)pend.size();
            pend.push_back(std::move(acc));
          } else {
            finalize(j, acc);
          }
        }
        for (size_t j = 0; j < kept.size(); j++)  // inner sums their consumer did not take (size limit, unsupported sibling)
          if (pending[j] >= 0 && !dead[j]) finalize(j, pend[pending[j]]);
        std::vector<DevOp> compact;
        compact.reserve(kept.size());
        for (size_t i = 0; i < kept.size(); i++)
          if (!dead[i]) compact.push_back(kept[i]);
        kept.swap(compact);
      }
      // multiply-add fusion (products that are not by a small immediate, or whose sum was not merged above)
      std::vector<uint32_t> uses(def_at.size(), 0);
      std::vector<int32_t> def_idx(def_at.size(), -1);
      for (size_t i = 0; i < kept.size(); i++) {
        each_temp(kept[i], [&](DevOperand& t) { uses[t.value]++; });
        if (kept[i].op != GATE_OP_PUSH) def_idx[kept[i].dst] = (int32_t)i;
      }
      std::vector<char> dead(kept.size(), 0);
      for (size_t j = 0; j < kept.size(); j++) {
        DevOp& o = kept[j];
        if (o.op != BJ_REL_ADD || !(ctx->gate_peephole & 2)) continue;
        for (int side = 0; side < 2; side++) {
          const DevOperand& prod = side ? o.b : o.a;
          const DevOperand& other = side ? o.a : o.b;
          if (prod.kind != BJ_IDX_TEMPORARY || other.kind != BJ_IDX_TEMPORARY || uses[prod.value] != 1) continue;
          const int32_t i = def_idx[prod.value];
          if (i < 0 || dead[i] || kept[i].op != BJ_REL_MUL) continue;
          DevOperand ma = kept[i].a, mb = kept[i].b;
          if (ma.kind == BJ_IDX_CONSTANT_VALUE) std::swap(ma, mb);  // the immediate goes second
          if (ma.kind == BJ_IDX_CONSTANT_VALUE) continue;            // constant * constant: left alone
          const DevOperand addend = other;
          o.op = GATE_OP_MADD;
          o.a = ma;
          o.b = mb;
          o.c = addend;
          dead[i] = 1;
          break;
        }
      }
      prog.clear();
      for (size_t i = 0; i < kept.size(); i++)
        if (!dead[i]) prog.push_back(kept[i]);
    }
    // 1c. a step whose value is read by nothing but the push_evaluation_result that follows it pushes the value itself
    if (ctx->gate_peephole & 8) {
      std::vector<uint32_t> uses(def_at.size(), 0);
      for (DevOp& o : prog) each_temp(o, [&](DevOperand& t) { uses[t.value]++; });
      std::vector<DevOp> out;
      out.reserve(prog.size());
      for (const DevOp& o : prog) {
        if (o.op == GATE_OP_PUSH && o.a.kind == BJ_IDX_TEMPORARY && !out.empty() && out.back().op != GATE_OP_PUSH && !out.back().push &&
            out.back().dst == o.a.value && uses[o.a.value] == 1) {
          out.back().push = true;
          out.back().dst = o.dst;  // the term index
          continue;
        }
        out.push_back(o);
      }
      prog.swap(out);
    }
    // 2. slot allocation: a temporary lives from its definition to its last use; its slot is then reused (the kernel reads both
    //    operands before it writes the destination, so a destination may take over the slot of an operand that dies there)
    {
      std::vector<int32_t> last_use(def_at.size(), -1), slot(def_at.size(), -1);
      for (size_t i = 0; i < prog.size(); i++) each_temp(prog[i], [&](DevOperand& t) { last_use[t.value] = (int32_t)i; });
      std::vector<uint32_t> free_slots;
      std::vector<uint64_t> read;  // program temporaries this step reads (distinct)
      uint32_t next_slot = 0;
      for (size_t i = 0; i < prog.size(); i++) {
        DevOp& o = prog[i];
        const bool is_push = o.op == GATE_OP_PUSH || o.push;
        read.clear();
        each_temp(o, [&](DevOperand& t) {
          if (std::find(read.begin(), read.end(), t.value) == read.end()) read.push_back(t.value);
          t.value = (uint64_t)slot[t.value];
        });
        for (uint64_t t : read)
          if (last_use[t] == (int32_t)i) free_slots.push_back((uint32_t)slot[t]);
        if (is_push) continue;
        const uint32_t t_dst = o.dst;
        uint32_t sl;
        if (!free_slots.empty()) {
          sl = free_slots.back();
          free_slots.pop_back();
        } else {
          sl = next_slot++;
        }
        if (sl >= (uint32_t)GATE_MAX_TMP)
          GATE_FAIL(BJ_ERR_UNSUPPORTED, "gate program: more than 128 temporaries live at once");
        slot[t_dst] = (int32_t)sl;
        o.dst = sl;
        if (last_use[t_dst] < 0) free_slots.push_back(sl);  // defined but never read
      }
      max_slots = std::max(max_slots, next_slot);
    }
    // 3. lowering to the device form: operand classes T / L / I, column operands as indices into the unified table
    //    [variables | witnesses | constants] of repetition 0 plus the per-repetition stride (PerChunkOffset)
    {
      auto lower = [&](const DevOperand& o, u64* raw, u32* stride) -> int {
        *stride = 0;
        switch (o.kind) {
          case BJ_IDX_TEMPORARY: *raw = o.value; return KIND_T;
          case BJ_IDX_CONSTANT_VALUE: *raw = o.value; return KIND_I;
          case BJ_IDX_VARIABLE: *raw = (u64)g.variables_initial_offset + o.value; *stride = g.variables_offset; return KIND_L;
          case BJ_IDX_WITNESS: *raw = (u64)n_variables + g.witnesses_initial_offset + o.value; *stride = g.witnesses_offset; return KIND_L;
          case BJ_IDX_CONSTANT_POLY:
            *raw = (u64)n_variables + n_witnesses + g.constants_placement_offset + o.value;
            *stride = g.constants_offset;
            return KIND_L;
          default: *raw = (u64)n_variables + n_witnesses + g.constants_placement_offset + o.value; return KIND_L;  // row-shared constant
        }
      };
      if (g.variables_offset > 0xffffu || g.witnesses_offset > 0xffffu || g.constants_offset > 0xffffu || g.n_writes >= (1u << 24))
        GATE_FAIL(BJ_ERR_UNSUPPORTED, "gate descriptor: per-repetition offset beyond 65535 or more than 2^24 terms");
      for (const DevOp& o : prog) {
        if (o.op == GATE_OP_LINCOMB) {
          const std::vector<LcTerm>& terms = lincombs[o.lc];
          PackedOp head{};
          head.code_dst = GATE_CODE_LINCOMB | (o.push ? 0x80u : 0u) | (o.dst << 8);
          head.strides = g.variables_offset;
          head.a = terms.size();
          head.b = o.a.value;
          ops.push_back(head);
          for (size_t t0 = 0; t0 < terms.size(); t0 += 4) {
            PackedTerm rec[4] = {};
            for (size_t t = t0; t < std::min(terms.size(), t0 + 4); t++) {
              const LcTerm& lt = terms[t];
              rec[t - t0].ref = lt.x.kind == BJ_IDX_TEMPORARY ? (u32)lt.x.value : (0x80000000u | (u32)(g.variables_initial_offset + lt.x.value));
              rec[t - t0].k = lt.k;
            }
            PackedOp raw;
            static_assert(sizeof(rec) == sizeof(PackedOp), "four terms per record");
            memcpy(&raw, rec, sizeof(raw));
            ops.push_back(raw);
          }
          continue;
        }
        PackedOp po{};
        u32 sa = 0, sb = 0;
        const int ka = lower(o.a, &po.a, &sa);
        const bool binary = o.op == BJ_REL_ADD || o.op == BJ_REL_SUB || o.op == BJ_REL_MUL || o.op == GATE_OP_MADD;
        const int kb = binary ? lower(o.b, &po.b, &sb) : 0;
        if (o.op == GATE_OP_MADD) po.c = o.c.value;
        po.code_dst = gate_code(o.op, ka, kb) | ((o.op == GATE_OP_PUSH || o.push) ? 0x80u : 0u) | (o.dst << 8);
        po.strides = sa | (sb << 16);
        ops.push_back(po);
      }
    }
    d.n_ops = (u32)ops.size() - d.ops_begin;  // records, incl. the term records of linear combinations
    total_terms += (uint64_t)g.n_writes * g.num_repetitions;
    gates.push_back(d);
  }
  return BJ_OK;
#undef GATE_FAIL
}
}  // namespace

namespace bj {
// K = 4 points per thread once there is enough work to fill the machine with such blocks
static int gate_points_per_thread(const bj_ctx* ctx, u64 n_points) {
  const int k = ctx->gate_points_per_thread;
  if (k == 1 || k == 2 || k == 4) return k;
  return n_points >= (u64)ctx->sm_count * 4 * 512 ? 4 : n_points >= (u64)ctx->sm_count * 4 * 256 ? 2 : 1;
}

// gates, steps and the column table [variables | witnesses | constants] of a compiled program set -> p.gates, p.ops, p.cols,
// p.consts_base.  Small programs ride in the parameter arena; a long one (the Poseidon2 flattened gate is ~9k relations) goes
// to the context's program buffer, which only grows: repeated proofs allocate nothing here (a cudaMalloc / cudaFree would
// synchronise the device and serialise the lanes of a context).  The copy is ordered on the stream after the last kernel
// that read the previous program.
static int32_t gate_program_upload(bj_ctx* ctx, const CompiledGates& compiled, std::vector<const u64*> table, uint32_t consts_base,
                                   GateEvalParams* p) {
  const std::vector<PackedOp>& ops = compiled.ops;
  void* d;
  BJ_TRY(param_upload(ctx, compiled.gates.data(), sizeof(DevGate) * compiled.gates.size(), &d));
  p->gates = (const DevGate*)d;
  p->n_gates = (u32)compiled.gates.size();
  static const PackedOp dummy_op{};
  const size_t ops_bytes = sizeof(PackedOp) * std::max<size_t>(ops.size(), 1);
  if (ops_bytes > (128u << 10)) {
    if (ctx->gate_program_bytes < ops_bytes) {
      if (ctx->gate_program) {
        BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        BJ_CUDA(ctx, cudaFree(ctx->gate_program));
        ctx->gate_program = nullptr;
        ctx->gate_program_bytes = 0;
      }
      BJ_CUDA(ctx, cudaMalloc(&ctx->gate_program, ops_bytes));
      ctx->gate_program_bytes = ops_bytes;
    }
    const cudaError_t e = cudaMemcpyAsync(ctx->gate_program, ops.data(), ops_bytes, cudaMemcpyHostToDevice, ctx->stream);
    if (e != cudaSuccess)
      BJ_FAIL(ctx, BJ_ERR_CUDA, std::string("gate program upload: ") + cudaGetErrorString(e));
    d = ctx->gate_program;
  } else {
    BJ_TRY(param_upload(ctx, ops.empty() ? &dummy_op : ops.data(), ops_bytes, &d));
  }
  p->ops = (const PackedOp*)d;
  if (table.empty()) table.push_back(nullptr);
  BJ_TRY(param_upload(ctx, table.data(), sizeof(u64*) * table.size(), &d));
  p->cols = (const u64* const*)d;
  p->consts_base = consts_base;
  return BJ_OK;
}
}  // namespace bj

extern "C" int32_t bj_gate_programs_compile(const bj_gate_desc* h_gates, uint32_t n_gates, uint32_t n_variables, uint32_t n_witnesses,
                                            uint32_t n_constants, uint32_t peephole, uint64_t* h_records, uint64_t capacity_records,
                                            uint64_t* n_records, uint32_t* h_gate_first_record, uint32_t* max_live_temporaries) {
  if (!h_gates || n_gates == 0 || !n_records) return BJ_ERR_INVALID_ARG;
  CompiledGates c;
  const int32_t st = compile_gates(nullptr, (int)peephole, h_gates, n_gates, n_variables, n_witnesses, n_constants, c);
  if (st != BJ_OK) return st;
  *n_records = c.ops.size();
  if (max_live_temporaries) *max_live_temporaries = c.max_slots;
  if (h_gate_first_record) {
    for (uint32_t g = 0; g < n_gates; g++) h_gate_first_record[g] = c.gates[g].ops_begin;
    h_gate_first_record[n_gates] = (uint32_t)c.ops.size();
  }
  if (h_records) {
    if (capacity_records < c.ops.size()) return BJ_ERR_INVALID_ARG;
    memcpy(h_records, c.ops.data(), sizeof(PackedOp) * c.ops.size());
  }
  return BJ_OK;
}

extern "C" int32_t bj_quotient_gates_general_purpose(bj_ctx* ctx, const bj_gate_desc* h_gates, uint32_t n_gates,
                                                     const uint64_t* const* h_variable_cols, uint32_t n_variables,
                                                     const uint64_t* const* h_witness_cols, uint32_t n_witnesses,
                                                     const uint64_t* const* h_constant_cols, uint32_t n_constants,
                                                     const uint64_t* h_alpha_powers, uint32_t n_alpha_powers,
                                                     uint64_t n_points, uint64_t* d_q_c0, uint64_t* d_q_c1) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || !h_gates || n_gates == 0 || !d_q_c0 || !d_q_c1 || n_points == 0 || (!h_alpha_powers && n_alpha_powers))
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_quotient_gates_general_purpose: bad argument");
  CompiledGates compiled;
  {
    GateCompileError err;
    const int32_t st = compile_gates(&err, ctx->gate_peephole, h_gates, n_gates, n_variables, n_witnesses, n_constants, compiled);
    if (st != BJ_OK) BJ_FAIL(ctx, st, err.last_error);
  }
  const uint32_t max_slots = compiled.max_slots;
  const uint64_t total_terms = compiled.total_terms;
  if (total_terms > n_alpha_powers) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "not enough alpha powers for the gate terms");
  std::vector<u64> alphas(2 * (size_t)total_terms);
  for (size_t i = 0; i < alphas.size(); i++) alphas[i] = gl::canon(h_alpha_powers[i]);
  GateEvalParams p{};
  {
    std::vector<const u64*> table;
    table.reserve((size_t)n_variables + n_witnesses + n_constants + 1);
    for (uint32_t i = 0; i < n_variables; i++) table.push_back((const u64*)h_variable_cols[i]);
    for (uint32_t i = 0; i < n_witnesses; i++) table.push_back((const u64*)h_witness_cols[i]);
    for (uint32_t i = 0; i < n_constants; i++) table.push_back((const u64*)h_constant_cols[i]);
    for (const u64* c : table)
      if (!c) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_quotient_gates_general_purpose: NULL column");
    BJ_TRY(gate_program_upload(ctx, compiled, table, n_variables + n_witnesses, &p));
  }
  void* d;
  static const u64 zero2[2] = {0, 0};
  BJ_TRY(param_upload(ctx, alphas.empty() ? (const void*)zero2 : (const void*)alphas.data(), sizeof(u64) * std::max<size_t>(alphas.size(), 2), &d));
  p.alphas = (const u64*)d;
  p.n_rows = n_points;
  p.q_c0 = (u64*)d_q_c0;
  p.q_c1 = (u64*)d_q_c1;
  // slots sized to the live maximum
  const int k = gate_points_per_thread(ctx, n_points);
  const bool small = max_slots <= 32;
  if (k == 4) small ? gate_eval_launch<4, 32>(p, ctx->stream) : gate_eval_launch<4, GATE_MAX_TMP>(p, ctx->stream);
  else if (k == 2) small ? gate_eval_launch<2, 32>(p, ctx->stream) : gate_eval_launch<2, GATE_MAX_TMP>(p, ctx->stream);
  else small ? gate_eval_launch<1, 32>(p, ctx->stream) : gate_eval_launch<1, GATE_MAX_TMP>(p, ctx->stream);
  BJ_LAUNCH_CHECK(ctx);
  return BJ_OK;
}
