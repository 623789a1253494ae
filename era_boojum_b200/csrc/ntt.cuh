// Goldilocks radix-2 NTT family for sm_90a: device-side pass descriptor + host planner interface.
//
// What is computed is fixed by the reference (bit-exact after canonicalisation):
//   forward  fft_natural_to_bitreversed  src/fft/mod.rs:398-411 (+ distribute_powers :308-317)
//            out[bitrev_n(k)] = sum_i a_i (c w_n^k)^i ; butterfly network :659-734 with the bit-reversed
//            twiddle table of src/cs/implementations/utils.rs:88-125
//   inverse  ifft_natural_to_natural      src/fft/mod.rs:464-491 (network with w^-1, bit-reverse, c^-i n^-1)
//   LDE      transform_raw_storages_to_lde src/cs/implementations/utils.rs:270-403
// How it is computed: the log n rounds are split into 1-3 "passes"; one pass keeps a tile of
// 2^t rows x 2^w columns in shared memory, runs t rounds as radix-16 register stages, and touches HBM once.
#pragma once
#include "gl64.cuh"

namespace bj {

using gl::u64;

enum NttScaleMode : int { SCALE_NONE = 0, SCALE_CONST = 1, SCALE_POW = 2, SCALE_FULL = 3 };
enum NttPassKind : int { PASS_TILE = 0, PASS_TRANSPOSE_LAST = 1 };

struct NttPass {
  const u64* src;
  u64* dst;
  u64 src_col_stride;  // elements between consecutive batch columns
  u64 dst_col_stride;
  const u64* tab;      // bit-reversed twiddle table (prefix property: valid for every size <= table size)
  int log_n;           // m
  int r0;              // rounds done by earlier passes (= number of index prefix bits)
  int t;               // rounds in this pass, tile rows = 2^t
  int w;               // log2 tile columns
  int kind;            // NttPassKind
  int scale_mode;      // NttScaleMode
  int scale_on_load;   // 1: factor indexed by the load position (forward coset), 0: by the store position (inverse)
  u64 scale_const;     // SCALE_CONST factor (canonical)
  const u64* pw_lo;    // SCALE_POW: c^x, x < 2^pw_split
  const u64* pw_hi;    // SCALE_POW: s * c^(y 2^pw_split)
  int pw_split;
  const u64* pw_full;  // SCALE_FULL: s * c^i for every i < 2^log_n (one load, one multiplication per element)
  int canon_out;       // canonicalise values at the store (last pass)
  // PASS_TILE with a coset's twisted table as tab (forward coset transform, run_transform): 2^r0, else 0.  The twiddles of
  // round rho start at tab + 2^rho, so the kernels put this 1 above the r0 prefix bits of the tile's twiddle index
  unsigned tw_prefix;
  // specialised PASS_TILE kernels on a one-dimensional grid (n_cols > 0): block w is the tile w / n_cols of column
  // w % n_cols (column-fastest: the same tile of every column back to back); n_cols == 0: grid (tile, column)
  unsigned n_cols;
};

}  // namespace bj
