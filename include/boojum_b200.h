/*
 * libboojum_b200 -- C-ABI of the H100-native (sm_90a) backend for Boojum's polynomial-commitment hot path.
 *
 * The reference (matter-labs/era-boojum, Rust) has no FFI for this path: the work sits behind generic
 * traits.  Each entry point below is what a Rust `extern "C"` shim (INTEGRATION.md) binds in place of the
 * cited reference function.  Conventions:
 *   - every call returns an int32 status (BJ_OK == 0, < 0 error); nothing aborts or throws across the ABI;
 *     bj_last_error(ctx) holds a message for the last failure on that context;
 *   - a bj_ctx is bound to one CUDA device and one stream; calls on one context are issued in order on that
 *     stream and are asynchronous unless stated (use bj_ctx_synchronize); one host thread per context;
 *   - field elements are little-endian u64; inputs may be non-canonical (any u64 congruent mod
 *     p = 2^64 - 2^32 + 1, as the reference tolerates, src/field/goldilocks/mod.rs:147-171); outputs are always
 *     CANONICAL (< p), i.e. exactly the values the reference serialises (mod.rs:99-107);
 *   - Fp2 elements are (c0, c1) pairs; Fp2 vectors are two separate u64 columns (SoA), as in the reference;
 *   - Poseidon2 digests are 4 x u64;
 *   - pointers named d_* are DEVICE pointers (cudaMalloc / bj_alloc / torch tensor data_ptr); h_* are host.
 *   - there is no CPU fallback: without a CUDA device bj_ctx_create fails with BJ_ERR_NO_DEVICE;
 *   - objects created through a context (bj_fri_oracles, bj_setup) hold device memory from that context's private
 *     stream-ordered pool: free them before bj_ctx_destroy.  A bj_proof is host memory only.
 */
#ifndef BOOJUM_B200_H
#define BOOJUM_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define BJ_API __attribute__((visibility("default")))
#else
#define BJ_API
#endif

#define BJ_OK 0
#define BJ_ERR_INVALID_ARG (-1)
#define BJ_ERR_CUDA (-2)
#define BJ_ERR_NO_DEVICE (-3)
#define BJ_ERR_OOM (-4)
#define BJ_ERR_UNSUPPORTED (-5)

#define BJ_GOLDILOCKS_P 0xFFFFFFFF00000001ull

typedef struct bj_ctx bj_ctx;

/* ---- context (replaces Worker, src/worker/mod.rs:5-87, as the executor handle) ---- */
BJ_API const char* bj_version(void);
BJ_API const char* bj_status_string(int32_t status);
/* stream: a cudaStream_t owned by the caller (e.g. torch.cuda.current_stream().cuda_stream); NULL is the CUDA
 * legacy default stream.  Kernels only ever run on this stream; the host-buffer entry points additionally use two
 * private copy streams so that upload, transform and download of successive column chunks overlap. */
BJ_API int32_t bj_ctx_create(int32_t device, void* stream, bj_ctx** out_ctx);
BJ_API int32_t bj_ctx_destroy(bj_ctx* ctx);
BJ_API int32_t bj_ctx_set_stream(bj_ctx* ctx, void* stream);
BJ_API int32_t bj_ctx_synchronize(bj_ctx* ctx);
/* Multi-GPU proving (one process and one context per GPU): declare that this context is rank `rank` of `world` (a power
 * of two, <= the LDE factor 2^log_lde of the proof).  Every buffer on the LDE domain then holds only the cosets j = rank (mod world), stored
 * [local coset][row]: bj_lde produces just those cosets, and bj_quotient_copy_permutation,
 * bj_quotient_divide_by_vanishing, bj_deep_quotient_group and bj_fri_fold take local buffers (sizes in their signatures
 * stay the GLOBAL domain sizes) and use the domain points of the owned cosets.  Merkle trees are built per rank over the
 * local leaves (a coset is a contiguous subtree: leaf index = coset * n + row, src/cs/implementations/proof.rs:89-91),
 * so caps and query paths are gathered by the caller.  bj_barycentric_evaluate reads local slot 0 (the global coset `rank`) and
 * uses that coset's shift, so any rank can open any column - the same value comes out.
 * The reference has no counterpart (its Worker is one machine's thread pool).  Default: rank 0 of 1. */
BJ_API int32_t bj_ctx_set_coset_shard(bj_ctx* ctx, uint32_t rank, uint32_t world, uint32_t log_lde);
/* Domain shard: bj_ctx_set_coset_shard for world <= 2^log_lde.  Above it (world a power of two <= 8 * 2^log_lde) every coset
 * is cut into B = world / 2^log_lde row blocks: the domain is made of UNITS u = j * B + p, unit u being rows
 * [p n / B, (p + 1) n / B) of coset j in its bit-reversed row order (flat index t = u * (n / B) + i'), and this context holds
 * the units u = rank (mod world), stored [local unit][n / B rows].  Row block p of coset j is the coset
 * sigma * <w_{n/B}> with sigma = 7 w_{nL}^{bitrev_L(j)} w_n^{bitrev_s(p)} (B = 2^s), rows bit-reversed.  Every entry point
 * that works on a coset shard works on units the same way, with two exceptions: bj_barycentric_evaluate returns the
 * CONTRIBUTION of the local row block (the B contributions of the ranks that hold coset j add up to the value), and
 * bj_quotient_copy_permutation, which would read z(omega x) from another row block, returns BJ_ERR_UNSUPPORTED -
 * bj_quotient_copy_permutation_with_z_next takes z(omega x) as columns (bj_lde_next_row) instead. */
BJ_API int32_t bj_ctx_set_domain_shard(bj_ctx* ctx, uint32_t rank, uint32_t world, uint32_t log_lde);
BJ_API const char* bj_last_error(const bj_ctx* ctx);
/* number of kernels this library launched through ctx so far (for launch accounting) */
BJ_API uint64_t bj_launch_count(const bj_ctx* ctx);
/* Device-memory limit of the prover driver on this context (bytes; 0, the default: what the device has free when
 * bj_setup_create runs, plus what the context's pool holds without using it).  bj_setup_create compares the memory plans of
 * bj_proof_memory_plan and bj_proof_memory_plan_streamed(_sharded) with it: RESIDENT if that fits, else COMPACT (one GPU,
 * quotient degree < LDE factor), else STREAMED (quotient degree > LDE factor, one GPU or sharded), else RECOMPUTE (one GPU only
 * after bj_ctx_allow_recompute_plan(ctx, 1); a context with a communicator only after bj_ctx_allow_sharded_recompute_plan(ctx,
 * 1), counted by bj_proof_memory_plan_recompute_sharded), else BJ_ERR_OOM with every applicable byte count in the message and
 * no kernel launched.  With quotient degree = LDE factor only RESIDENT (and the opt-in RECOMPUTE) applies.  On a sharded
 * context every rank chooses under its own limit; ranks on different plans (resident, streamed, recompute) still return the
 * same proof.  bj_prove follows the setup's plan and refuses the same way if the limit was lowered below it since. */
BJ_API int32_t bj_ctx_set_memory_limit(bj_ctx* ctx, uint64_t bytes);
/* allow != 0 lets bj_setup_create fall back to the RECOMPUTE plan (bj_proof_memory_plan_recompute) when none of RESIDENT,
 * COMPACT and STREAMED fits under the limit; the refusal below every plan then names the recompute bytes too.  Off by default:
 * the recompute plan rebuilds every coset of the setup, witness and stage-2 columns wherever it is read, so it is slower, and
 * a caller that relies on BJ_ERR_OOM below the smaller plans keeps it.  A sharded context ignores the switch. */
BJ_API int32_t bj_ctx_allow_recompute_plan(bj_ctx* ctx, int32_t allow);
/* Row blocks per coset the one-GPU RECOMPUTE plan may use: max_blocks = 1 (the default), 2, 4 or 8, anything else
 * BJ_ERR_INVALID_ARG.  When bj_setup_create takes the recompute plan (still only after bj_ctx_allow_recompute_plan) it takes
 * the fewest row blocks B <= max_blocks whose plan (bj_proof_memory_plan_recompute_blocks) fits under the limit; the refusal
 * below every plan names the recompute bytes at the largest allowed B.  With B > 1 the trees and the quotient work on the
 * L * B and Q * B row blocks of n / B rows (B >= 2 rows each) instead of whole cosets, so their scratch falls by B while the
 * quotient repeats the inverse NTT of its columns B times as often; every other choice, refusal and proof is unchanged.
 * bj_setup_row_blocks reports the B chosen.  A context with a communicator ignores the switch; lanes inherit it. */
BJ_API int32_t bj_ctx_set_max_row_blocks(bj_ctx* ctx, uint32_t max_blocks);
/* allow != 0 lets bj_setup_create on a context with a communicator fall back to the RECOMPUTE plan on this rank
 * (bj_proof_memory_plan_recompute_sharded) when neither RESIDENT nor STREAMED fits under the rank's limit; the refusal below
 * every plan then names the recompute bytes too.  Off by default, for the reasons of bj_ctx_allow_recompute_plan, which a
 * sharded context still ignores.  Set it alike on every rank: with it on, the ranks exchange their choice before their first
 * collective, and once one rank needs the recompute plan every rank takes it (the resident and streamed plans share LDE
 * monomials the recompute plan does not compute), or every rank refuses with BJ_ERR_OOM where a rank's limit does not hold
 * it.  A context without a communicator ignores this switch. */
BJ_API int32_t bj_ctx_allow_sharded_recompute_plan(bj_ctx* ctx, int32_t allow);
/* highest device memory the context's pool has had in use (cudaMemPoolAttrUsedMemHigh); reset != 0 restarts the mark.
 * Synchronises.  Memory the library keeps outside the pool (twiddles, coset-power tables, scratch) is not included. */
BJ_API int32_t bj_ctx_memory_high_water(bj_ctx* ctx, uint64_t* bytes, int32_t reset);
/* Lanes: several proofs of one setup in flight on one GPU.  A lane is a context on the parent's device with its own stream
 * (non-blocking), stream-ordered pool, scratch, parameter arena, launch counter and last error; it inherits the parent's memory
 * limit and recompute-plan switch.  bj_prove(lane, setup, ...) takes a setup created on the parent and returns the bytes
 * bj_prove(parent, setup, ...) returns, on every single-GPU plan.  Distinct lanes of one parent may run bj_prove at the same
 * time from different host threads (one thread per lane); they read the setup and the parent's twiddle and coset-power tables,
 * which nothing frees while a lane is alive.  After its first proof a lane allocates every proof buffer from its pool (no
 * cudaMalloc / cudaFree).  A lane creates no setup, has no lanes and keeps its stream (bj_ctx_set_stream is refused).
 * Refused with BJ_ERR_INVALID_ARG on a sharded parent (communicator or domain shard) and with BJ_ERR_OOM, naming the bytes and
 * the limit and launching nothing, when for some setup alive on the parent bj_proof_memory_plan_lanes(setup, lanes + 1)[2]
 * exceeds the parent's limit (bj_ctx_set_memory_limit, else the one the setup was planned under): `lanes` counts the lanes
 * alive after this one, and the parent counts as one more because its pool keeps what its setup and its own proofs reached.
 * A bj_setup_create on a parent with lanes alive counts them too: each plan must fit with one lane part per live lane.
 * Witness slot sets (bj_witness_slots_create) may live on a lane too, one copy stream per lane; the lane's thread alone
 * touches them.  bj_ctx_create_lane and bj_setup_create also count the bytes of the slot sets alive on the lanes.
 * Create the lanes of one parent from one thread.  Teardown: bj_ctx_destroy(parent) refuses with BJ_ERR_INVALID_ARG while a
 * lane is alive (destroy the lanes first), and bj_ctx_destroy(lane) while a slot set of the lane is alive (free it first); a
 * setup may be freed once every bj_prove that reads it has returned. */
BJ_API int32_t bj_ctx_create_lane(bj_ctx* parent, bj_ctx** out_lane);

/* ---- multi-GPU: communicator of the sharded prover (one process - or one thread - per GPU) ----
 * Creating a communicator on a context declares its domain shard (bj_ctx_set_domain_shard(ctx, rank, world, log_lde)) and makes
 * bj_setup_create / bj_prove / bj_do_fri on that context run SHARDED: every rank passes the same full witness, keeps the LDE
 * units u = rank (mod world) of every committed polynomial (whole cosets for world <= the LDE factor, row blocks of cosets
 * above it), builds the Merkle subtrees of its units, and all ranks return the same proof (identical to the single-GPU
 * proof).  What crosses GPUs: cap digests of every oracle, the quotient units (one all-gather of 2 * Q * n u64 - they are
 * interpolated together, prover.rs:1399-1467), the openings (each column block opened by one coset group, row-block
 * contributions summed on the host), the last FRI codeword and the query answers.  Requirements: world a power of two
 * <= 8 * the LDE factor, merkle_tree_cap_size >= max(LDE factor, world); with row blocks, 2^log_n >= 2 * world / LDE factor
 * and every FRI level must keep at least the 2^k elements it folds together in each unit.
 *   NCCL transport: rank 0 calls bj_comm_unique_id and hands the 128 bytes to the other ranks by any side channel (MPI, TCP,
 *   torch.distributed ...); every rank then calls bj_comm_create_nccl.  libnccl.so.2 is loaded at run time (the copy already
 *   in the process is reused); BJ_ERR_UNSUPPORTED if it is absent.
 *   Local transport: bj_comm_group_create(world) once, bj_comm_create_local per rank (ranks = host threads whose contexts sit
 *   on one device): lets one GPU run the sharded driver end to end.
 * Destroy the communicator before its context.  The raw collectives are exported for host code that shards other stages. */
typedef struct bj_comm bj_comm;
typedef struct bj_comm_group bj_comm_group;
#define BJ_COMM_UNIQUE_ID_BYTES 128
BJ_API int32_t bj_comm_unique_id(uint8_t out[BJ_COMM_UNIQUE_ID_BYTES]);
BJ_API int32_t bj_comm_create_nccl(bj_ctx* ctx, const uint8_t unique_id[BJ_COMM_UNIQUE_ID_BYTES], uint32_t rank, uint32_t world,
                            uint32_t log_lde, bj_comm** out);
BJ_API int32_t bj_comm_group_create(uint32_t world, bj_comm_group** out);
BJ_API void bj_comm_group_destroy(bj_comm_group* group);
BJ_API int32_t bj_comm_create_local(bj_ctx* ctx, bj_comm_group* group, uint32_t rank, uint32_t log_lde, bj_comm** out);
BJ_API int32_t bj_comm_destroy(bj_comm* comm);
BJ_API uint32_t bj_comm_rank(const bj_comm* comm);
BJ_API uint32_t bj_comm_world(const bj_comm* comm);
/* d_recv[r * n .. (r + 1) * n) = rank r's d_send[0 .. n): ncclAllGather on the context's stream (asynchronous); the local
 * transport completes before returning.  d_send may be its own slot of d_recv. */
BJ_API int32_t bj_comm_all_gather(bj_comm* comm, const uint64_t* d_send, uint64_t* d_recv, uint64_t n_u64_per_rank);
/* the same for small host buffers (staged through the device); synchronises */
BJ_API int32_t bj_comm_all_gather_host(bj_comm* comm, const uint64_t* h_send, uint64_t* h_recv, uint64_t n_u64_per_rank);
BJ_API int32_t bj_comm_broadcast_host(bj_comm* comm, uint64_t* h_buf, uint64_t n_u64, uint32_t root);

/* ---- device memory (GoodAllocator hook, src/cs/traits/mod.rs:13-15) ---- */
BJ_API int32_t bj_alloc(bj_ctx* ctx, size_t bytes, void** d_ptr);
BJ_API int32_t bj_free(bj_ctx* ctx, void* d_ptr);
BJ_API int32_t bj_upload(bj_ctx* ctx, void* d_dst, const void* h_src, size_t bytes);   /* async on ctx stream */
BJ_API int32_t bj_download(bj_ctx* ctx, void* h_dst, const void* d_src, size_t bytes); /* async on ctx stream */
BJ_API int32_t bj_alloc_host_pinned(size_t bytes, void** h_ptr);
BJ_API int32_t bj_free_host_pinned(void* h_ptr);

/* ---- twiddles: precompute_twiddles_for_fft::<_,_,_,INVERSED> (src/cs/implementations/utils.rs:88-125) ----
 * Copies tab[i] = w^bitrev_{n/2}(i), i < n/2 (w = omega_n or omega_n^-1) into d_out (n/2 u64).  The library
 * caches its own tables; this export exists for parity tests and for callers that want the reference table. */
BJ_API int32_t bj_twiddles(bj_ctx* ctx, uint32_t log_n, int32_t inverse, uint64_t* d_out);

/* ---- NTT: PrimeFieldLikeVectorized::fft_natural_to_bitreversed / ifft_natural_to_natural
 *      (src/field/traits/field_like.rs:139-161 -> src/fft/mod.rs:398-411, 464-491) ----
 * In place on n_cols columns of 2^log_n elements; column c starts at d_data + c*col_stride (elements).
 * forward: out[bitrev(k)] = sum_i a_i (coset w^k)^i.  inverse: natural-order values on coset<w> -> natural-order
 * monomial coefficients (network with w^-1, bit reversal, scaling by coset^-i n^-1).  coset == 1 means none. */
BJ_API int32_t bj_ntt_natural_to_bitreversed(bj_ctx* ctx, uint64_t* d_data, uint32_t log_n, uint32_t n_cols,
                                      uint64_t col_stride, uint64_t coset);
BJ_API int32_t bj_intt_natural_to_natural(bj_ctx* ctx, uint64_t* d_data, uint32_t log_n, uint32_t n_cols,
                                   uint64_t col_stride, uint64_t coset);
/* bitreverse_enumeration_inplace (src/fft/mod.rs:41-155), batched */
BJ_API int32_t bj_bitreverse(bj_ctx* ctx, uint64_t* d_data, uint32_t log_n, uint32_t n_cols, uint64_t col_stride);

/* ---- LDE: transform_raw_storages_to_lde / transform_monomials_to_lde (src/cs/implementations/utils.rs:270-403)
 * d_in : n_cols columns (column c at d_in + c*in_col_stride) of 2^log_n Lagrange values in natural row order
 *        (or monomial coefficients if from_monomials != 0).  Not modified.
 * d_out: [col][coset j][row], 2^log_lde cosets of 2^log_n values each; coset j is evaluated on
 *        7 * w_{nL}^{bitrev_L(j)} * <w_n>, values bit-reversed within the coset (ArcGenericLdeStorage layout,
 *        src/cs/implementations/polynomial/lde.rs:161-170).  Column c starts at d_out + c * (n << log_lde). */
BJ_API int32_t bj_lde(bj_ctx* ctx, const uint64_t* d_in, uint64_t in_col_stride, uint64_t* d_out, uint32_t log_n,
               uint32_t log_lde, uint32_t n_cols, int32_t from_monomials);
/* bj_lde of g(x) = f(w_n x), same layout: the value at a point is f at the next row's point.  A row block of a split domain
 * shard reads z(omega x) of the copy-permutation quotient from here (the row itself lives in another block). */
BJ_API int32_t bj_lde_next_row(bj_ctx* ctx, const uint64_t* d_in, uint64_t in_col_stride, uint64_t* d_out, uint32_t log_n,
                               uint32_t log_lde, uint32_t n_cols, int32_t from_monomials);
/* bj_lde onto the cosets [coset_begin, coset_end) of the factor-2^log_lde domain only: d_out [col][coset_end - coset_begin][row],
 * each coset bit-identical to its slot of the full bj_lde.  Unsharded contexts (BJ_ERR_UNSUPPORTED otherwise). */
BJ_API int32_t bj_lde_cosets(bj_ctx* ctx, const uint64_t* d_in, uint64_t in_col_stride, uint64_t* d_out, uint32_t log_n, uint32_t log_lde,
                             uint32_t coset_begin, uint32_t coset_end, uint32_t n_cols, int32_t from_monomials);

/* ---- Poseidon2 Merkle tree: MerkleTreeWithCap::construct / construct_by_chunking /
 *      construct_by_chunking_from_flat_sources / continue_from_leaf_hashes (src/cs/oracle/merkle_tree.rs:78-449)
 *      with H = GoldilocksPoseidon2Sponge<AbsorptionModeOverwrite> (src/cs/oracle/mod.rs:114-175) ----
 * h_sources: HOST array of n_sources DEVICE pointers; source s is a flat array of n_leaves*elems_per_leaf u64
 *            (a column's cosets flattened coset-major).  Leaf m absorbs, for s = 0..n_sources-1 in order,
 *            source_s[m*elems_per_leaf .. (m+1)*elems_per_leaf).
 * d_leaf_hashes: n_leaves digests.  d_nodes: concatenated levels n_leaves/2, n_leaves/4, ..., cap_size digests
 *            (node_hashes_enumerated_from_leafs); total n_leaves - cap_size digests.  The cap is the last level
 *            (or the leaf hashes when n_leaves == cap_size). */
BJ_API int32_t bj_merkle_build_poseidon2(bj_ctx* ctx, const uint64_t* const* h_sources, uint32_t n_sources,
                                  uint64_t n_leaves, uint32_t elems_per_leaf, uint32_t cap_size,
                                  uint64_t* d_leaf_hashes, uint64_t* d_nodes);
/* Same tree with H = blake2::Blake2s256 (src/cs/oracle/mod.rs:179-245): leaf = Blake2s-256 over the LE bytes of the reduced
 * elements, node = Blake2s-256(left || right); 32-byte digests stored as 4 LE u64 (same [n][4] layout). */
BJ_API int32_t bj_merkle_build_blake2s(bj_ctx* ctx, const uint64_t* const* h_sources, uint32_t n_sources, uint64_t n_leaves,
                                uint32_t elems_per_leaf, uint32_t cap_size, uint64_t* d_leaf_hashes, uint64_t* d_nodes);
/* impl TreeHasher for sha3::Keccak256 (src/cs/oracle/mod.rs:247-313): same layout and arguments, Keccak-256 digests */
BJ_API int32_t bj_merkle_build_keccak256(bj_ctx* ctx, const uint64_t* const* h_sources, uint32_t n_sources, uint64_t n_leaves,
                                uint32_t elems_per_leaf, uint32_t cap_size, uint64_t* d_leaf_hashes, uint64_t* d_nodes);
/* TreeHasher::hash_into_leaf on rows given contiguously: n_rows rows of row_len u64 (row-major) -> digests */
BJ_API int32_t bj_poseidon2_hash_rows(bj_ctx* ctx, const uint64_t* d_rows, uint64_t n_rows, uint32_t row_len,
                               uint64_t* d_digests);
/* raw permutation on n_states states of 12 u64 (src/implementations/poseidon2/state_generic_impl.rs:219-233) */
BJ_API int32_t bj_poseidon2_permute(bj_ctx* ctx, uint64_t* d_states, uint64_t n_states);

/* ---- FRI fold: fold_multiple / interpolate_flattened_cosets (src/cs/implementations/fri/mod.rs:362-474, 587-678)
 * One oracle step = `log_fold` (1..3) successive fold-by-2 of a flat Fp2 vector of 2^log_m values:
 *   out[i] = (f[2i] + f[2i+1]) + alpha * (f[2i] - f[2i+1]) * R[i] * kappa,
 *   R = inverse twiddle table of the full LDE domain (prefix), kappa = *coset_inv, squared after every fold;
 *   fold j uses challenge alpha^(2^j).  h_alpha = (c0, c1) of the first challenge.  On return *h_coset_inv_io holds
 *   the updated kappa (as the reference's `coset_inverse.square()` leaves it).  Output length 2^(log_m-log_fold). */
BJ_API int32_t bj_fri_fold(bj_ctx* ctx, const uint64_t* d_c0, const uint64_t* d_c1, uint32_t log_m, uint32_t log_fold,
                    const uint64_t h_alpha[2], uint64_t* h_coset_inv_io, uint64_t* d_out_c0, uint64_t* d_out_c1);

/* ---- batch inverse: batch_inverse_inplace / batch_inverse_inplace_in_extension (src/cs/implementations/utils.rs:405-600)
 * In place.  The reference panics on a zero element ("must be called on sets without zeroes", utils.rs:425-427); here a
 * zero is mapped to zero and does not disturb the other elements. */
BJ_API int32_t bj_batch_inverse(bj_ctx* ctx, uint64_t* d_data, uint64_t n);
BJ_API int32_t bj_batch_inverse_ext(bj_ctx* ctx, uint64_t* d_c0, uint64_t* d_c1, uint64_t n);

/* ---- DEEP: quotening_operation_in_extension (src/cs/implementations/prover.rs:2523-2706), one call per opening point
 * For every point t of the LDE domain (2^log_rows = n*L points, coset-major, bit-reversed inside a coset; x(t) =
 * 7 * w_{nL}^{bitrev(t)}):   acc[t] += ( sum_i ch_i * (f_i(t) - v_i) ) / (x(t) - at)      in Fp2.
 * h_src_c0 / h_src_c1: HOST arrays of n_src DEVICE pointers to the c0 / c1 columns (each n*L u64, LDE layout);
 *   h_src_c1[i] == NULL marks a base-field polynomial (prover.rs:2655-2677).
 * h_values_at / h_challenges: n_src (c0, c1) pairs: f_i(at) and the challenge coefficient of term i.
 * d_acc_c0 / d_acc_c1: the Fp2 codeword accumulated across calls (zero-initialised by the caller). */
BJ_API int32_t bj_deep_quotient_group(bj_ctx* ctx, const uint64_t* const* h_src_c0, const uint64_t* const* h_src_c1,
                               uint32_t n_src, const uint64_t* h_values_at, const uint64_t* h_challenges,
                               const uint64_t h_at[2], uint32_t log_rows, uint64_t* d_acc_c0, uint64_t* d_acc_c1);
/* the same on the points [first_point, first_point + n_points) of the domain only: source columns and accumulators hold
 * those n_points values (e.g. one coset recomputed by bj_lde_cosets, t = j * n + row).  Unsharded contexts. */
BJ_API int32_t bj_deep_quotient_range(bj_ctx* ctx, const uint64_t* const* h_src_c0, const uint64_t* const* h_src_c1, uint32_t n_src,
                                      const uint64_t* h_values_at, const uint64_t* h_challenges, const uint64_t h_at[2], uint32_t log_rows,
                                      uint64_t first_point, uint64_t n_points, uint64_t* d_acc_c0, uint64_t* d_acc_c1);

/* ---- stage 2, copy-permutation argument: compute_partial_products_in_extension
 *      (src/cs/implementations/copy_permutation.rs:649-766; rational :114-248, grand product :425-510) ----
 * Inputs are Lagrange columns on the trace domain in natural row order (n = 2^log_n values each): the copy-permutation
 * (variable) columns and their sigma columns; non-residues k_j from bj_non_residues_for_copy_permutation.
 * chunk_size = quotient degree (columns multiplied per partial product).
 * Outputs: z (c0, c1) = exclusive prefix product of prod_j (w_j + beta k_j x + gamma)/(w_j + beta sigma_j + gamma), and the
 * ceil(n_cols/chunk_size) - 1 partial products, laid out [partial][c0|c1][n] in d_partials.
 * Returns BJ_ERR_INVALID_ARG if the grand product over the domain is not 1 (the reference asserts, :479). Synchronises. */
BJ_API int32_t bj_non_residues_for_copy_permutation(uint64_t domain_size, uint32_t num_columns, uint64_t* h_out);
BJ_API int32_t bj_copy_permutation_stage2(bj_ctx* ctx, const uint64_t* const* h_variable_cols, const uint64_t* const* h_sigma_cols,
                                   uint32_t n_cols, const uint64_t* h_non_residues, const uint64_t h_beta[2],
                                   const uint64_t h_gamma[2], uint32_t log_n, uint32_t chunk_size, uint64_t* d_z_c0,
                                   uint64_t* d_z_c1, uint64_t* d_partials);

/* ---- lookup argument over specialised columns, table id in a constant column
 *      (LookupParameters::UseSpecializedColumnsWithTableIdAsConstant; src/cs/implementations/lookup_argument_in_ext.rs) ----
 * stage 2 (compute_lookup_poly_pairs_specialized, :320-947), trace domain, natural order:
 *   A_i[r] = 1/(beta + sum_j gamma^j col_{i,j}[r] + gamma^w table_id[r]),  B[r] = m[r]/(beta + sum_j gamma^j t_j[r]).
 * h_lookup_cols: n_subarguments*width device pointers (the sub-arguments' variable columns, in order); d_table_id_col: the
 * constant column with the table id (NULL if none); h_table_cols: the n_table_cols = width (+1) lookup-table setup columns.
 * d_out: [n_subarguments + 1][c0|c1][n]  (A_0, ..., A_{k-1}, B). */
BJ_API int32_t bj_lookup_polys_specialized(bj_ctx* ctx, const uint64_t* const* h_lookup_cols, uint32_t n_subarguments, uint32_t width,
                                    const uint64_t* d_table_id_col, const uint64_t* const* h_table_cols, uint32_t n_table_cols,
                                    const uint64_t* d_multiplicity, const uint64_t h_beta[2], const uint64_t h_gamma[2],
                                    uint32_t log_n, uint64_t* d_out);
/* quotient terms (compute_quotient_terms_for_lookup_specialized, :949-1319) on the first n_points = Q*n points of the LDE:
 *   q += alpha_i (A_i (beta + sum gamma^j col_ij + gamma^w id) - 1)  for every sub-argument,  + alpha_k (B (beta + sum gamma^j t_j) - m).
 * All column arguments are LDE columns; h_a_ldes: 2*n_subarguments pointers (c0, c1); h_alphas: n_subarguments + 1 Fp2. */
BJ_API int32_t bj_quotient_lookup_specialized(bj_ctx* ctx, const uint64_t* const* h_lookup_ldes, uint32_t n_subarguments, uint32_t width,
                                       const uint64_t* d_table_id_lde, const uint64_t* const* h_table_ldes, uint32_t n_table_cols,
                                       const uint64_t* d_multiplicity_lde, const uint64_t* const* h_a_ldes, const uint64_t* d_b_c0,
                                       const uint64_t* d_b_c1, const uint64_t h_beta[2], const uint64_t h_gamma[2],
                                       const uint64_t* h_alphas, uint64_t n_points, uint64_t* d_q_c0, uint64_t* d_q_c1);

/* ---- gate / quotient evaluator over general-purpose columns: the row loop of prove_cpu_basic
 *      (src/cs/implementations/prover.rs:1031-1080; gates over specialised columns, :653-801, use the same call) with GateConstraintEvaluator::evaluate_once (src/cs/traits/evaluator.rs:145-152)
 *      supplied as DATA: the SSA program recorded by the reference's own GPU hook, gpu_synthesizer::GPUDataCapture
 *      (src/gpu_synthesizer/mod.rs:115-133 Index / Relation, :354-443 capture). */
enum { /* Index<F> (gpu_synthesizer/mod.rs:115-121); SHARED = a ConstantPoly listed in row_shared_constants_set */
  BJ_IDX_VARIABLE = 0, BJ_IDX_WITNESS = 1, BJ_IDX_CONSTANT_POLY = 2, BJ_IDX_TEMPORARY = 3, BJ_IDX_CONSTANT_VALUE = 4,
  BJ_IDX_CONSTANT_POLY_SHARED = 5
};
enum { /* Relation<F> (gpu_synthesizer/mod.rs:125-133) */
  BJ_REL_ADD = 0, BJ_REL_DOUBLE = 1, BJ_REL_SUB = 2, BJ_REL_NEGATE = 3, BJ_REL_MUL = 4, BJ_REL_SQUARE = 5, BJ_REL_INVERSE = 6
};
typedef struct bj_gate_index {
  uint32_t kind;   /* BJ_IDX_* */
  uint32_t reserved;
  uint64_t value;  /* column / temporary index, or the field element for BJ_IDX_CONSTANT_VALUE */
} bj_gate_index;
typedef struct bj_gate_relation {
  uint32_t op;            /* BJ_REL_* */
  uint32_t dst_temporary; /* TemporaryValue index this relation defines: programs are SSA (one fresh index per relation, < 2^20);
                           * the library assigns slots by liveness - at most 128 temporaries may be live at once */
  bj_gate_index a, b;     /* b ignored by the unary relations */
} bj_gate_relation;
typedef struct bj_gate_desc {
  const bj_gate_relation* relations; /* GPUDataCapture::relations, in recording order */
  uint32_t n_relations;
  uint32_t n_writes;
  const bj_gate_index* writes;       /* GPUDataCapture::writes_per_repetition (one quotient term each) */
  uint32_t num_repetitions;          /* num_repetitions_on_row */
  uint32_t variables_offset;         /* PerChunkOffset (GatePlacementType::MultipleOnRow) */
  uint32_t witnesses_offset;
  uint32_t constants_offset;
  uint32_t constants_placement_offset; /* first constant column of the gate = selector path length (prover.rs:1000-1013) */
  uint32_t selector_path_len;          /* TreeNode path of the gate; 0 = no selector */
  const uint8_t* selector_path;        /* path[i] != 0: factor const_i, else (1 - const_i) (prover.rs:2775-2916) */
  /* gates on SPECIALISED columns (GatePlacementStrategy::UseSpecializedColumns, prover.rs:653-801): first column of
   * repetition 0 among the variable / witness columns (initial_offset of offsets_for_specialized_evaluators); 0 for
   * general-purpose gates.  Such a gate has selector_path_len = 0, constants_placement_offset = (constants of the
   * general-purpose gates) + initial constants offset, and constants_offset = 0 when share_constants. */
  uint32_t variables_initial_offset;
  uint32_t witnesses_initial_offset;
} bj_gate_desc;
/* For every point t < n_points (= Q * n, the first Q cosets of the LDE, flat coset-major):
 *   q[t] += sum_g selector_g(t) * sum_k alpha_pow[k] * term_k(t),  k running over the terms of all gates in order
 * (gates with zero terms, e.g. NOP, are simply not passed).  Column pointer arrays are HOST arrays of DEVICE pointers,
 * each column flat [coset][row] as produced by bj_lde.  h_alpha_powers: (c0, c1) pairs, one per term. */
BJ_API int32_t bj_quotient_gates_general_purpose(bj_ctx* ctx, const bj_gate_desc* h_gates, uint32_t n_gates,
                                          const uint64_t* const* h_variable_cols, uint32_t n_variables,
                                          const uint64_t* const* h_witness_cols, uint32_t n_witnesses,
                                          const uint64_t* const* h_constant_cols, uint32_t n_constants,
                                          const uint64_t* h_alpha_powers, uint32_t n_alpha_powers,
                                          uint64_t n_points, uint64_t* d_q_c0, uint64_t* d_q_c1);
/* What the evaluator will execute for these gates - pure host code, no device needed.  The recorded programs are validated
 * (SSA, operand ranges against n_variables / n_witnesses / n_constants), rewritten (peephole bits: 1 = x*1, x+0, x*0 become
 * aliases; 2 = a product whose only use is a sum becomes a multiply-add; 4 = trees of single-use sums over products with
 * immediates < 2^28 become one linear combination; 8 = a value read only by push_evaluation_result is pushed by the step that
 * computes it; 15 = what bj_quotient_gates_general_purpose uses) and lowered to 32-byte records = 4 little-endian u64:
 *   word 0: code (bits 0-6) | pushes-its-value flag (bit 7) | destination slot or term index (bits 8-31) |
 *           per-repetition column stride of operand a (bits 32-47) and b (bits 48-63);  word 1: operand a;  word 2: operand b;
 *   word 3: addend slot of a multiply-add.  Operand classes T (slot), L (index into [variables | witnesses | constants] at
 *   repetition 0), I (immediate).  Codes: ADD 0-8, SUB 9-17, MUL 18-26 = base + 3 * class(a) + class(b) with T, L, I = 0, 1, 2;
 *   DOUBLE 27-29, NEGATE 30-32, SQUARE 33-35, INVERSE 36-38, MOVE 39-41 = base + class(a); multiply-add a * b + slot 42-47 =
 *   42 + 3 * class(a) + class(b), class(a) in {T, L}; 48 = linear combination: word 0 stride = variables stride, word 1 = number
 *   of terms n, word 2 = constant term, followed by ceil(n / 4) records of four (u32 ref, u32 k) pairs, ref = slot or
 *   0x80000000 | variable column.
 * h_records may be NULL (sizes only); h_gate_first_record has n_gates + 1 entries.  Used by the CPU test suite, which runs an
 * emulator of this format against the gate evaluators (tests/test_gate_compiler_cpu.py). */
BJ_API int32_t bj_gate_programs_compile(const bj_gate_desc* h_gates, uint32_t n_gates, uint32_t n_variables, uint32_t n_witnesses,
                                 uint32_t n_constants, uint32_t peephole, uint64_t* h_records, uint64_t capacity_records,
                                 uint64_t* n_records, uint32_t* h_gate_first_record, uint32_t* max_live_temporaries);

/* ---- quotient: copy-permutation relations + the z(1) = 1 term (src/cs/implementations/copy_permutation.rs:1000-1249,
 *      src/cs/implementations/prover.rs:1189-1227) over the first 2^log_quotient_degree cosets of the LDE ----
 * All polynomial arguments are LDE columns (flat [L][n], 2^log_lde cosets).  h_partial_ldes: 2*(n_chunks-1) device
 * pointers (c0, c1 per partial product).  h_alphas: (n_chunks + 1) Fp2 challenge powers: the z(1)=1 term first, then one
 * per copy-permutation relation (order of prover.rs:1176-1250).  Accumulates into q. */
BJ_API int32_t bj_quotient_copy_permutation(bj_ctx* ctx, const uint64_t* const* h_variable_ldes, const uint64_t* const* h_sigma_ldes,
                                     uint32_t n_cols, const uint64_t* h_non_residues, const uint64_t* d_z_c0,
                                     const uint64_t* d_z_c1, const uint64_t* const* h_partial_ldes, const uint64_t h_beta[2],
                                     const uint64_t h_gamma[2], const uint64_t* h_alphas, uint32_t log_n, uint32_t log_lde,
                                     uint32_t log_quotient_degree, uint32_t chunk_size, uint64_t* d_q_c0, uint64_t* d_q_c1);
/* the same with z(omega x) given as LDE columns (bj_lde_next_row of z) instead of read from z's next row: what a split domain
 * shard uses, where bj_quotient_copy_permutation returns BJ_ERR_UNSUPPORTED */
BJ_API int32_t bj_quotient_copy_permutation_with_z_next(bj_ctx* ctx, const uint64_t* const* h_variable_ldes, const uint64_t* const* h_sigma_ldes,
                                                        uint32_t n_cols, const uint64_t* h_non_residues, const uint64_t* d_z_c0,
                                                        const uint64_t* d_z_c1, const uint64_t* d_z_next_c0, const uint64_t* d_z_next_c1,
                                                        const uint64_t* const* h_partial_ldes, const uint64_t h_beta[2], const uint64_t h_gamma[2],
                                                        const uint64_t* h_alphas, uint32_t log_n, uint32_t log_lde, uint32_t log_quotient_degree,
                                                        uint32_t chunk_size, uint64_t* d_q_c0, uint64_t* d_q_c1);
/* divide_by_vanishing_for_bitreversed_coset_enumeration (src/cs/implementations/utils.rs:770-817): q[coset j] *= 1/((7 w^bitrev(j))^n - 1) */
BJ_API int32_t bj_quotient_divide_by_vanishing(bj_ctx* ctx, uint64_t* d_q_c0, uint64_t* d_q_c1, uint32_t log_n,
                                        uint32_t log_quotient_degree);

/* ---- openings: values of n_cols base-field polynomials at the Fp2 point `at`, from their first LDE coset
 *      (barycentric evaluation, src/cs/implementations/utils.rs:907-1243; prover.rs:1519-1802).
 * h_cols: host array of device pointers to LDE columns (only the first 2^log_n values, coset 0, are read).
 * h_out: n_cols (c0, c1) pairs.  `at` must not lie on the coset 7<w_n> (on a sharded context: on the coset of local slot 0).
 * On a split domain shard (bj_ctx_set_domain_shard with world > the LDE factor) local slot 0 is one row block of a coset and
 * h_out is that block's CONTRIBUTION: summing the outputs of the ranks that hold the coset's blocks gives the values.
 * Synchronises. */
BJ_API int32_t bj_barycentric_evaluate(bj_ctx* ctx, const uint64_t* const* h_cols, uint32_t n_cols, uint32_t log_n,
                                const uint64_t h_at[2], uint64_t* h_out);

/* ---- host-buffer convenience entry points (what the Rust shim calls when columns live in host Vecs).
 * They upload, run, download and synchronise; used for the end-to-end measurement. */
BJ_API int32_t bj_ntt_natural_to_bitreversed_host(bj_ctx* ctx, uint64_t* h_data, uint32_t log_n, uint32_t n_cols,
                                           uint64_t coset);
BJ_API int32_t bj_intt_natural_to_natural_host(bj_ctx* ctx, uint64_t* h_data, uint32_t log_n, uint32_t n_cols,
                                        uint64_t coset);

/* ---- host-side Fiat-Shamir (never on the GPU; must be replayed bit-exactly):
 * GoldilocksPoisedon2Transcript = AlgebraicSpongeBasedTranscript<_, 8, 12, 4, Poseidon2, Overwrite>
 * (src/cs/implementations/transcript.rs:62-129), BoolsBuffer::get_bits (:369-417), compute_fri_schedule
 * (src/cs/implementations/prover.rs:2281-2372). */
typedef struct bj_transcript bj_transcript;
BJ_API bj_transcript* bj_transcript_new(void);          /* GoldilocksPoisedon2Transcript */
/* Blake2sTranscript (transcript.rs:155-260; the transcript of sha256_bench_non_recursive): field elements enter as the
 * 8 LE bytes of their reduced value, caps as raw 32-byte digests; a challenge is 8 output bytes reduced mod p; query bits
 * take all 64 bits of 8 challenge bytes (BoolsBuffer, non-algebraic branch). */
BJ_API bj_transcript* bj_transcript_new_blake2s(void);
BJ_API bj_transcript* bj_transcript_new_keccak256(void); /* Keccak256Transcript (transcript.rs:262-367): same scheme, Keccak-256 */
/* GoldilocksPoisedonTranscript (transcript.rs:131-138): the algebraic sponge transcript over the Poseidon (v1) permutation
 * (src/implementations/poseidon_goldilocks_naive.rs) - the TR of run_sha256_prover_recursive_mode and
 * run_sha256_prover_recursive_mode_poseidon2 (src/gadgets/sha256/mod.rs:275-293) */
BJ_API bj_transcript* bj_transcript_new_poseidon(void);
BJ_API void bj_transcript_free(bj_transcript* t);
BJ_API void bj_transcript_witness_field_elements(bj_transcript* t, const uint64_t* els, size_t n);
BJ_API void bj_transcript_witness_merkle_tree_cap(bj_transcript* t, const uint64_t* cap_digests, size_t n_digests);
BJ_API uint64_t bj_transcript_get_challenge(bj_transcript* t);
/* num_bits query-index bits, LSB first, as one integer; each refill keeps the (64 - max_needed) low bits of a challenge */
BJ_API uint64_t bj_transcript_get_index_bits(bj_transcript* t, uint32_t num_bits, uint32_t max_needed);
/* schedule: caller array of >= 32 entries */
BJ_API int32_t bj_compute_fri_schedule(uint32_t security_bits, uint32_t cap_size, uint32_t pow_bits, uint32_t rate_log_two,
                                uint32_t initial_degree_log_two, uint32_t* new_pow_bits, uint32_t* num_queries,
                                uint32_t* schedule, uint32_t* schedule_len, uint32_t* final_degree);

/* ---- FRI commit phase: do_fri (src/cs/implementations/fri/mod.rs:49-357) ----
 * d_c0 / d_c1: the DEEP codeword on the full LDE domain (2^log_full_size values each, LDE layout; borrowed - must stay
 * alive as long as the returned oracles are queried).  schedule: interpolation_log2s_schedule (compute_fri_schedule).
 * Builds the base oracle and every intermediate oracle (Poseidon2 trees with 2^k c0 values then 2^k c1 values per
 * leaf), absorbs each cap into the transcript, draws the two challenge elements, folds, and finally bit-reverses +
 * iNTTs the last vector into the monomial forms which are absorbed as well.  Returns BJ_ERR_INVALID_ARG if the folded
 * codeword is not of low degree (the reference's self-check panics, fri/mod.rs:326-334). */
typedef struct bj_fri_oracles bj_fri_oracles;
BJ_API int32_t bj_do_fri(bj_ctx* ctx, bj_transcript* transcript, const uint64_t* d_c0, const uint64_t* d_c1,
                  uint32_t log_full_size, const uint32_t* schedule, uint32_t n_schedule, uint32_t log_lde,
                  uint32_t cap_size, bj_fri_oracles** out);
#define BJ_HASHER_POSEIDON2 0u
#define BJ_HASHER_BLAKE2S 1u
#define BJ_HASHER_KECCAK256 2u
/* same with the tree hasher chosen (BJ_HASHER_*: GoldilocksPoseidon2Sponge, Blake2s256 or Keccak256, src/cs/oracle/mod.rs:114-313) */
BJ_API int32_t bj_do_fri_with_hasher(bj_ctx* ctx, bj_transcript* transcript, const uint64_t* d_c0, const uint64_t* d_c1,
                              uint32_t log_full_size, const uint32_t* schedule, uint32_t n_schedule, uint32_t log_lde,
                              uint32_t cap_size, uint32_t hasher, bj_fri_oracles** out);
BJ_API void bj_fri_oracles_free(bj_fri_oracles* o);
BJ_API uint32_t bj_fri_oracles_num_oracles(const bj_fri_oracles* o);
BJ_API uint32_t bj_fri_oracles_num_monomials(const bj_fri_oracles* o);
BJ_API int32_t bj_fri_oracles_get_cap(const bj_fri_oracles* o, uint32_t oracle_idx, uint64_t* h_out /* 4*cap u64 */);
BJ_API int32_t bj_fri_oracles_get_monomials(const bj_fri_oracles* o, uint64_t* h_c0, uint64_t* h_c1);
BJ_API int32_t bj_fri_oracles_get_challenges(const bj_fri_oracles* o, uint64_t* h_out /* 2 u64 per oracle */);
/* OracleQuery::construct for one FRI oracle (src/cs/implementations/proof.rs:65-97): leaf elements (2 * 2^k u64:
 * c0 values then c1 values) and the sibling path (path_len digests, bottom-up, cap level excluded). */
BJ_API int32_t bj_fri_oracles_query(bj_fri_oracles* o, uint32_t oracle_idx, uint64_t leaf_index, uint64_t* h_leaf_elements,
                             uint64_t* h_path, uint32_t* path_len);
/* n leaves of one oracle at once (two device round trips): h_leaf_elements [n][2 * 2^k], h_paths [n][*path_len][4] */
BJ_API int32_t bj_fri_oracles_query_batch(bj_fri_oracles* o, uint32_t oracle_idx, const uint64_t* h_leaf_indices, uint32_t n_indices,
                                   uint64_t* h_leaf_elements, uint64_t* h_paths, uint32_t* path_len);
/* Query helpers for the base oracles (witness / stage 2 / quotient / setup): gather the leaf preimages of n_indices
 * leaves (h_out[q][s * elems_per_leaf + e]) and their Merkle paths (h_out[q][depth][4]); both synchronise.  Every source
 * column holds n_leaves * elems_per_leaf elements; an index >= n_leaves is rejected with BJ_ERR_INVALID_ARG (no launch). */
BJ_API int32_t bj_query_leaf_elements(bj_ctx* ctx, const uint64_t* const* h_sources, uint32_t n_sources, uint32_t elems_per_leaf,
                               uint64_t n_leaves, const uint64_t* h_indices, uint32_t n_indices, uint64_t* h_out);
BJ_API int32_t bj_merkle_paths(bj_ctx* ctx, const uint64_t* d_leaf_hashes, const uint64_t* d_nodes, uint64_t n_leaves,
                        uint32_t cap_size, const uint64_t* h_indices, uint32_t n_indices, uint64_t* h_out);

/* ---- proof of work: impl PoWRunner for Blake2s256 (src/cs/implementations/pow.rs:52-147).  Returns the smallest u64
 * `challenge` of the first successful 2^24-candidate batch for which the first 8 bytes (little endian) of
 * Blake2s-256(seed || challenge.to_le_bytes()) have at least pow_bits (<= 32) trailing zero bits.  The seed is the byte
 * string of run_from_field_elements (the LE bytes of the reduced field elements; 5 challenges = 40 bytes in
 * prove_cpu_basic, prover.rs:2109-2126).  Synchronises. */
BJ_API int32_t bj_pow_blake2s(bj_ctx* ctx, const uint8_t* h_seed, uint32_t seed_len, uint32_t pow_bits, uint64_t* h_challenge);
/* impl PoWRunner for Keccak256 (pow.rs:140-230): the same search with Keccak-256 (seed <= 120 bytes) */
BJ_API int32_t bj_pow_keccak256(bj_ctx* ctx, const uint8_t* h_seed, uint32_t seed_len, uint32_t pow_bits, uint64_t* h_challenge);

/* ---- setup / witness materialisation on the device (what feeds bj_setup_create and bj_prove) ----
 * Variable encoding as in the reference (src/cs/mod.rs:44-47, :155-180): a u64 whose bit 63 marks a placeholder and whose
 * low 48 bits are the variable index.
 * bj_materialize_columns: materialize_variables_polynomials_from_dense_hint (src/cs/implementations/witness.rs:325-385):
 *   d_out[c][row] = d_all_values[hint[c][row]] for row < hint_rows (hint laid out [n_cols][hint_rows]); placeholders and
 *   the rows beyond the hint are zero.  Fails if a hint points past n_values.  Synchronises.
 * bj_create_permutation_polys: create_permutation_polys (src/cs/implementations/setup.rs:419-502): d_placement is
 *   copy_permutation_data, [n_cols][2^log_n] variables; d_sigmas [n_cols][2^log_n] receives the sigma columns (identity
 *   k_c * w^row on cells that are never copied, one cycle per variable over its occurrences in column-major order). */
BJ_API int32_t bj_materialize_columns(bj_ctx* ctx, const uint64_t* d_all_values, uint64_t n_values, const uint64_t* d_hint,
                               uint32_t n_cols, uint64_t hint_rows, uint32_t log_n, uint64_t* d_out);
BJ_API int32_t bj_create_permutation_polys(bj_ctx* ctx, const uint64_t* d_placement, uint32_t n_cols, uint32_t log_n,
                                    uint64_t* d_sigmas);

/* ---- the prover entry point: CSReferenceAssembly::prove_cpu_basic (src/cs/implementations/prover.rs:153-2269) and the part of
 *      the setup materialisation it depends on (setup.rs:1093-1255: sigma / constant / lookup-table columns -> LDE -> setup tree).
 * Scope: gates on general-purpose columns (bj_gate_desc programs), copy permutation over all variable columns, optional
 * log-derivative lookup over specialised columns with the table id in a constant column (lookup_width = 0: none), Poseidon2
 * or Blake2s tree hasher and transcript, public inputs, Blake2s proof of work (pow_bits > 0).  Host C++ inside the library: transcript, schedule, query
 * indices and proof assembly never leave the host; every heavy step is one of the entry points above.
 * Column arguments are DEVICE arrays [column][2^log_n] in natural row order.  bj_setup BORROWS d_sigmas / d_constants /
 * d_lookup_tables (stage 2 reads them again): they must outlive the setup.  The gate programs are copied.
 * bj_prove returns BJ_ERR_INVALID_ARG for an unsatisfied circuit (the reference panics, prover.rs:1425-1438). */
typedef struct bj_circuit {
  uint32_t log_n;            /* trace length 2^log_n */
  uint32_t num_variables;    /* columns under the copy permutation (general purpose + specialised lookup columns) */
  uint32_t num_constants;
  uint32_t quotient_degree;  /* power of two; may exceed fri_lde_factor (production: factor 2, degree 8) - columns are then evaluated
                              * at max(fri_lde_factor, quotient_degree) cosets and the oracles commit to the first fri_lde_factor
                              * of them (prover.rs:178-196 used_lde_degree / subset_for_degree) */
  uint32_t fri_lde_factor, merkle_tree_cap_size, security_level, pow_bits; /* ProofConfig (prover.rs:55-73) */
  const bj_gate_desc* gates;
  uint32_t n_gates;
  uint32_t lookup_width;            /* columns per lookup tuple without the table id; 0 = no lookup argument */
  uint32_t lookup_num_repetitions;  /* sub-arguments */
  uint32_t lookup_variables_offset; /* first lookup column among the variables */
  uint32_t lookup_table_id_column;  /* constant column holding the table id */
  /* public inputs: places (variable column, row) whose witness values are published (CSReferenceAssembly::public_inputs;
   * prover.rs:264-266, 1805-1821, 2010-2041) */
  const uint32_t* public_input_columns;
  const uint32_t* public_input_rows;
  uint32_t n_public_inputs;
  uint32_t tree_hasher; /* BJ_HASHER_POSEIDON2 (recursive-mode bench), BJ_HASHER_BLAKE2S (sha256_bench_non_recursive), BJ_HASHER_KECCAK256 */
  uint32_t transcript;  /* 0: Poseidon2 sponge transcript, 1: Blake2sTranscript, 2: Keccak256Transcript, 3: Poseidon (v1) sponge transcript */
} bj_circuit;
typedef struct bj_setup bj_setup;
typedef struct bj_proof bj_proof;
BJ_API int32_t bj_setup_create(bj_ctx* ctx, const bj_circuit* circuit, const uint64_t* d_sigmas, const uint64_t* d_constants,
                        const uint64_t* d_lookup_tables /* [lookup_width + 1][n] or NULL */, bj_setup** out);
BJ_API void bj_setup_free(bj_setup* setup);
/* Device bytes of bj_setup_create + bj_prove at their peak on each of `world` GPUs, counted from the circuit's shapes (host
 * only, no device needed): out[0] the RESIDENT plan (every LDE column on all max(L, Q) cosets), out[1] the COMPACT plan (0
 * when it does not apply: world > 1 or quotient degree >= LDE factor), which keeps cosets [0, Q) of the setup, witness and
 * stage-2 columns after their trees are built and recomputes cosets [Q, L) from the natural-order columns for DEEP and the
 * query answers.  Both are the context pool's allocations replayed in the driver's order plus an upper bound of what the
 * library keeps outside the pool (twiddles, coset-power tables, NTT scratch). */
BJ_API int32_t bj_proof_memory_plan(const bj_circuit* circuit, uint32_t world, uint64_t out[2]);
/* The STREAMED plan's bytes, counted the same way (0 when it does not apply: world > 1 or quotient degree <= LDE factor).  With
 * Q > L the resident plan evaluates every setup, witness and stage-2 column on all Q cosets, and cosets [L, Q) are read by the
 * quotient only.  The streamed plan evaluates those columns on the committed cosets [0, L) only (stride n * L) and keeps the
 * natural-order stage-2 columns.  The quotient then runs one coset j at a time: coset j < L from the kept columns, coset
 * j >= L evaluated from the natural-order columns into one coset-sized scratch of every column the quotient reads.  Proofs
 * are bit-identical to the resident plan's. */
BJ_API int32_t bj_proof_memory_plan_streamed(const bj_circuit* circuit, uint32_t world, uint64_t* out);
/* The STREAMED plan's bytes on each of `world` GPUs (0 when quotient degree <= LDE factor; at world 1 the value of
 * bj_proof_memory_plan_streamed).  Each rank evaluates the setup, witness and stage-2 columns on its units of the committed
 * cosets [0, L) only (stride n * L / world) and keeps the natural-order stage-2 columns.  The quotient then runs one of the
 * rank's units of cosets [0, Q) at a time - the units the resident sharded plan gives the rank: whole cosets on a coset
 * shard (world <= L), row blocks of n * L / world rows on a split shard - a unit of a committed coset from the kept columns,
 * any other unit evaluated from the natural-order columns into one unit-sized scratch (with its z(omega x) columns on a
 * split shard).  The gathered quotient and everything after it are unchanged: every rank returns the single-GPU proof. */
BJ_API int32_t bj_proof_memory_plan_streamed_sharded(const bj_circuit* circuit, uint32_t world, uint64_t* out);
/* The RECOMPUTE plan's bytes, counted the same way with 2 columns recomputed at a time (0 when world > 1).  It applies on one
 * GPU to any quotient degree Q and LDE factor L, and keeps no coset of the setup, witness or stage-2 columns: only the trees,
 * the natural-order stage-2 columns, the quotient oracle and the quotient buffers.  Each tree is built one committed coset at
 * a time (the coset's columns evaluated from natural order into an n-row scratch per column, its n leaves hashed into their
 * slice of the leaf array, the node levels after the last coset).  The quotient evaluates every column it reads onto one
 * coset of [0, Q) at a time, the openings rebuild coset 0 a chunk of columns at a time, and DEEP and the query answers
 * rebuild cosets [0, L) the same way.  Proofs are bit-identical to the resident plan's; opt in with
 * bj_ctx_allow_recompute_plan. */
BJ_API int32_t bj_proof_memory_plan_recompute(const bj_circuit* circuit, uint32_t world, uint64_t* out);
/* The RECOMPUTE plan's bytes on each of `world` GPUs, counted like bj_proof_memory_plan_streamed_sharded (at world 1 the value
 * of bj_proof_memory_plan_recompute), for any quotient degree.  Each rank keeps no coset of the setup, witness or stage-2
 * columns and works on its own units u = rank (mod world) - whole cosets on a coset shard (world <= L), row blocks of
 * n * L / world rows on a split shard: it builds each tree one of its committed units at a time (the unit's columns
 * evaluated from natural order into a unit-sized scratch, its leaves hashed into their slice), evaluates every column the
 * quotient reads onto one of its quotient units at a time (with the unit's z(omega x) columns on a split shard), rebuilds its
 * local slot 0 a chunk of columns at a time for the openings, and its committed units for DEEP and for the queries it
 * answers.  The gathered quotient, the collectives and the proof are unchanged.  *out = 0 where some rank would own no
 * quotient unit (Q < L and world > Q: the plan does not apply there).  *out = 0 and BJ_ERR_INVALID_ARG for the
 * shapes sharding rejects: cap_size < world, world > 8 * LDE factor, a row block of fewer than 2 rows.  Chosen only after
 * bj_ctx_allow_sharded_recompute_plan. */
BJ_API int32_t bj_proof_memory_plan_recompute_sharded(const bj_circuit* circuit, uint32_t world, uint64_t* out);
/* The one-GPU RECOMPUTE plan's bytes with every coset cut into `blocks` row blocks (host only, no device needed): each tree is
 * built one row block of n / blocks rows at a time (its columns evaluated from natural order into a row-block scratch per
 * column, its leaves hashed into their slice) and the quotient evaluates every column it reads, and z(omega x), onto one of
 * the Q * blocks row blocks of cosets [0, Q) at a time.  The openings, DEEP and the query answers rebuild whole cosets as on
 * the recompute plan.  At blocks = 1 the value of bj_proof_memory_plan_recompute(circuit, 1, out).  *out = 0 and
 * BJ_ERR_INVALID_ARG for blocks other than 1, 2, 4 or 8, or row blocks of fewer than 2 rows.  Proofs are bit-identical to
 * the resident plan's; chosen only after bj_ctx_allow_recompute_plan and bj_ctx_set_max_row_blocks. */
BJ_API int32_t bj_proof_memory_plan_recompute_blocks(const bj_circuit* circuit, uint32_t blocks, uint64_t* out);
/* 1 if bj_setup_create chose the compact plan, 0 otherwise (resident, streamed or recompute) */
BJ_API int32_t bj_setup_is_compact(const bj_setup* setup);
/* the plan bj_setup_create chose: BJ_PLAN_RESIDENT, BJ_PLAN_COMPACT, BJ_PLAN_STREAMED or BJ_PLAN_RECOMPUTE */
#define BJ_PLAN_RESIDENT 0
#define BJ_PLAN_COMPACT 1
#define BJ_PLAN_STREAMED 2
#define BJ_PLAN_RECOMPUTE 3
BJ_API int32_t bj_setup_plan(const bj_setup* setup);
/* the row blocks per coset bj_setup_create chose for the recompute plan on one GPU (bj_ctx_set_max_row_blocks); 1 on every
 * other plan and on a sharded context */
BJ_API int32_t bj_setup_row_blocks(const bj_setup* setup);
/* the plan bj_setup_create chose: out[0] the peak bytes of the context's pool over bj_setup_create + bj_prove (what
 * bj_ctx_memory_high_water reads on a fresh context), out[1] the bound on what the library holds outside the pool, out[2] the
 * columns the compact or recompute plan recomputes at a time (0 on the resident and streamed plans) */
BJ_API int32_t bj_setup_memory_plan(const bj_setup* setup, uint64_t out[3]);
/* device bytes of one setup proved on n_lanes >= 1 lanes at once (bj_ctx_create_lane), the setup's chosen plan split in two:
 * out[0] the setup's part (the pool bytes it holds after bj_setup_create, and the twiddle and coset-power tables the lanes
 * share), out[1] one lane's part (what a proof's pool adds on top of the setup - a fresh lane's bj_ctx_memory_high_water - and
 * the lane's own scratch and parameter arena), out[2] = out[0] + n_lanes * out[1].  With n_lanes = 1, out[2] is the plan
 * (bj_setup_memory_plan out[0] + out[1]).  BJ_ERR_INVALID_ARG for a setup of a sharded context. */
BJ_API int32_t bj_proof_memory_plan_lanes(const bj_setup* setup, uint32_t n_lanes, uint64_t out[3]);
/* the pool part of bj_proof_memory_plan_lanes out[1]: what a fresh lane's bj_ctx_memory_high_water reaches proving the setup
 * (the rest of out[1] is the lane's scratch and parameter arena) */
BJ_API int32_t bj_proof_memory_plan_lane_pool(const bj_setup* setup, uint64_t* pool_bytes);
/* the same from the circuit's shapes alone (no device), for plan = BJ_PLAN_RESIDENT / COMPACT / STREAMED / RECOMPUTE on one GPU
 * with the smallest recompute chunk: out[0] + out[1] equals bj_proof_memory_plan(_streamed / _recompute) for that plan; all
 * three are 0 where the plan does not apply to the circuit */
BJ_API int32_t bj_proof_memory_plan_lanes_host(const bj_circuit* circuit, uint32_t plan, uint32_t n_lanes, uint64_t out[3]);
/* bj_proof_memory_plan_lanes_host with the recompute plan cut into `blocks` row blocks per coset (1, 2, 4 or 8; only 1 on the
 * other plans, else BJ_ERR_INVALID_ARG): out[0] + out[1] equals bj_proof_memory_plan_recompute_blocks.  bj_proof_memory_plan_lanes
 * and bj_witness_slots_create count the row blocks a setup chose by themselves. */
BJ_API int32_t bj_proof_memory_plan_lanes_host_blocks(const bj_circuit* circuit, uint32_t plan, uint32_t blocks, uint32_t n_lanes,
                                                      uint64_t out[3]);
BJ_API int32_t bj_setup_get_cap(const bj_setup* setup, uint64_t* h_cap /* 4 * cap_size u64: VerificationKey::setup_merkle_tree_cap */);
BJ_API int32_t bj_prove(bj_ctx* ctx, const bj_setup* setup, const uint64_t* d_variables, const uint64_t* d_multiplicities /* or NULL */,
                 bj_proof** out);
BJ_API void bj_proof_free(bj_proof* proof);
/* the proof in the reference's serde_json shape (Proof<F, H, EXT>, src/cs/implementations/proof.rs:57-143).
 * Call with buf == NULL to learn the size (incl. the terminating 0), then with a buffer of at least that size. */
BJ_API int32_t bj_proof_to_json(const bj_proof* proof, char* buf, size_t capacity, size_t* needed);
/* wall-clock seconds of the six stages (witness, stage 2, quotient, openings, DEEP+FRI, queries), device work included */
BJ_API int32_t bj_proof_stage_seconds(const bj_proof* proof, double out[6]);

/* ---- repeated proving: a stream of witnesses against one setup (prove_from_witness_vec_and_precomputations,
 *      src/cs/implementations/convenience.rs:159-195) ----
 * A witness slot set holds n_slots (1 to 4) witnesses on the device, each in the layout bj_prove reads: [V][n] variables, then
 * n multiplicities when the circuit has a lookup.  Uploads run on a copy stream of the context (created by the first slot set),
 * so the upload of the next witness overlaps the running proof; bj_prove_slot makes the context's stream wait for the slot's
 * upload and runs bj_prove on it (same proof bytes).  An upload into a slot whose proof has been issued is ordered after that
 * proof.  Host memory: pinned memory (bj_alloc_host_pinned, cudaHostRegister) is copied directly - the call returns at once and
 * the buffer must stay unchanged until bj_prove_slot on that slot has returned; pageable memory is copied through a ring of
 * four 16 MiB pinned staging chunks on the calling thread - the call returns when the last chunk is staged (it blocks only to
 * refill a chunk whose copy has not finished) and the buffer may be reused at once.
 * The slot set allocates once, from the context's pool: n_slots * (V + lookup) * n u64, and with max_values > 0 an all_values
 * buffer of max_values u64 shared by the slots plus, with a lookup, n u32 multiplicities.  bj_witness_slots_bytes counts those
 * the way bj_proof_memory_plan counts the proof (host only), and with max_values > 0 the u32 variables hint at its largest
 * (V * n u32); it is the same on each of `world` GPUs: every rank of a sharded context holds the whole witness.
 * bj_witness_slots_create refuses with BJ_ERR_OOM, naming both numbers and launching nothing, if the setup's chosen plan plus
 * those bytes exceed the context's limit (bj_ctx_set_memory_limit, else the limit the setup was planned under).  Free the slot
 * set before its setup and context (both drain its copy stream).  Argument errors return BJ_ERR_INVALID_ARG with a message
 * before any launch: another context's setup, a slot out of range, a slot never uploaded, a witness vector without hint or
 * buffer, a lookup without multiplicities.
 * On a lane (bj_ctx_create_lane): `ctx` may be a lane of the setup's context.  The set's buffers then come from the lane's pool
 * and its uploads run on a copy stream the lane owns (created by the lane's first set, destroyed with the lane); it has its
 * own staging ring, all_values and u32 multiplicities, and a WitnessVec gather reads the setup's hint from the lane's copy
 * stream.  Uploads, bj_witness_slot_columns and bj_prove_slot(lane, setup, set, slot) behave as on the parent, and the proofs
 * are the bytes bj_prove(parent, setup, ...) returns, on every single-GPU plan.  Only the lane's thread touches its sets.  The
 * memory check on a lane sums bj_proof_memory_plan_lanes(setup, m + 1)[2] (m = the parent's live lanes), the hint once
 * (out[1] of bj_witness_slots_bytes_split, when max_values > 0 or the setup has a hint), the full bytes of the parent's live
 * sets, out[0] of the live sets of its lanes and out[0] of the new set, and refuses with BJ_ERR_OOM, naming every term and
 * allocating nothing, above the parent's limit (else the one the setup was planned under).  bj_prove_slot refuses with
 * BJ_ERR_INVALID_ARG a set of another context: another lane's, a lane's on the parent, the parent's on a lane.
 * bj_setup_attach_variables_hint refuses with BJ_ERR_INVALID_ARG while a lane of the setup's context has a set alive (attach
 * the hint before creating lane sets); bj_ctx_destroy(lane) refuses while a set of the lane is alive. */
typedef struct bj_witness_slots bj_witness_slots;
BJ_API int32_t bj_witness_slots_bytes(const bj_circuit* circuit, uint32_t world, uint32_t n_slots, uint64_t max_values, uint64_t* out);
/* bj_witness_slots_bytes at world 1 split in two (host only): out[0] the bytes the set itself allocates in its context's pool,
 * out[1] the u32 variables hint at its largest, which lives once on the setup (0 when max_values == 0).  out[0] + out[1] equals
 * bj_witness_slots_bytes(circuit, 1, ...).  A set on a lane counts out[0] only. */
BJ_API int32_t bj_witness_slots_bytes_split(const bj_circuit* circuit, uint32_t n_slots, uint64_t max_values, uint64_t out[2]);
BJ_API int32_t bj_witness_slots_create(bj_ctx* ctx, const bj_setup* setup, uint32_t n_slots, uint64_t max_values, bj_witness_slots** out);
BJ_API void bj_witness_slots_free(bj_witness_slots* slots);
/* columns from host memory into a slot: h_variables [V][n], h_multiplicities n values (NULL without a lookup) */
BJ_API int32_t bj_witness_upload(bj_witness_slots* slots, uint32_t slot, const uint64_t* h_variables, const uint64_t* h_multiplicities);
/* DenseVariablesCopyHint (witness.rs:325-385) in the Variable encoding, [V][hint_rows], hint_rows <= n: kept on the device as u32
 * with placeholders as 0xFFFFFFFF (half the bytes).  BJ_ERR_INVALID_ARG if an index is >= 2^32 - 1.  Synchronises. */
BJ_API int32_t bj_setup_attach_variables_hint(bj_setup* setup, const uint64_t* h_hint, uint64_t hint_rows);
/* the host conversion it uses: n Variables -> u32 (placeholder 0xFFFFFFFF); *h_values_needed (may be NULL) = 1 + the largest
 * index, 0 if none.  BJ_ERR_INVALID_ARG on an index >= 2^32 - 1. */
BJ_API int32_t bj_variables_hint_to_u32(const uint64_t* h_hint, uint64_t n, uint32_t* h_out, uint64_t* h_values_needed);
/* WitnessVec (witness.rs:32-40): all_values (n_values <= max_values, at least what the hint names) and the u32 multiplicities
 * (1 to n of them, widened and zero-padded to n as witness.rs:493-520 does), gathered into the slot on the copy stream:
 * variables[c][row] = all_values[hint[c][row]] for row < hint_rows, zero for placeholders and later rows (bj_materialize_columns'
 * result).  The next upload refills all_values after that gather. */
BJ_API int32_t bj_witness_upload_vec(bj_witness_slots* slots, uint32_t slot, const uint64_t* h_all_values, uint64_t n_values,
                                     const uint32_t* h_multiplicities, uint64_t n_multiplicities);
/* bj_prove on the slot's witness, ordered after its upload; a sharded context runs the sharded driver (every rank uploads the
 * same witness into its own slot set) */
BJ_API int32_t bj_prove_slot(bj_ctx* ctx, const bj_setup* setup, bj_witness_slots* slots, uint32_t slot, bj_proof** out);
/* the slot's device columns (variables [V][n], then the multiplicities), e.g. for bj_check_satisfied: the context's stream is
 * made to wait for the slot's upload, so work queued on it afterwards reads the whole witness.  Valid until the next upload into
 * the slot is issued. */
BJ_API int32_t bj_witness_slot_columns(bj_witness_slots* slots, uint32_t slot, uint64_t** d_columns);

/* ---- satisfiability check: CSReferenceAssembly::check_if_satisfied (src/cs/implementations/satisfiability_test.rs:15-353) ----
 * Checks a witness against its circuit exactly (no random challenge) on the trace domain, from the natural-order device columns
 * bj_setup_create and bj_prove take, with no setup (no LDE, no tree).  It reads log_n, num_variables, num_constants,
 * gates / n_gates and the lookup_* fields of the circuit and ignores the rest.  Three conditions, the ones bj_prove needs:
 *   - gates: every pushed term of every repetition of every gate is 0 on every row where the gate's selector (the product along
 *     its path over constant columns 0 .. path_len - 1) is nonzero; gates on specialised columns have no selector and run on
 *     every row;
 *   - copy constraints, from sigma alone: the entry s = k_c' w^r' of cell (c, r) names cell (c', r') (c' from s^n = k_c'^n, r'
 *     the discrete log of s / k_c' in <w_n>); each cell holds the value of the cell it names, and sigma is well formed: every
 *     entry names a cell (BJ_SIGMA_NO_CELL) and every cell is named by exactly one entry (BJ_SIGMA_UNNAMED, BJ_SIGMA_NAMED_TWICE);
 *   - lookups (lookup_width > 0): every tuple (the row's lookup_width columns of a sub-argument, then the table id from constant
 *     column lookup_table_id_column) equals a row of the table columns [lookup_width + 1][n] (id last), and for every distinct
 *     table content the number of tuples equal to it is the sum mod p of d_multiplicities over the table rows with that content.
 * Values are compared canonically (x + p equals x).  Returns BJ_OK whether or not the witness is satisfied (the report says
 * which); BJ_ERR_INVALID_ARG, with a message and no kernel launched, for malformed arguments: NULL columns, lookup_width > 0
 * without tables or multiplicities, a table-id column out of range, a lookup shape bj_prove refuses (more than 32
 * sub-arguments or 7 columns per tuple), gate programs the gate compiler rejects.  Synchronises.  Never communicates: it runs
 * the same on a sharded context.
 * Scratch from the context's pool, released before it returns: 16 n (gates) + 24 n (powers of w) + V n / 4 (two bitmaps) +
 * 24 V + 32 n (lookups) bytes, n = 2^log_n, V = num_variables - e.g. 72 n + V n / 4 bytes, about 400 MB at n = 2^22, V = 92.
 * Every count and "first" field is deterministic.  A "first" field is 0 when its count is 0. */
#define BJ_SIGMA_NO_CELL 1u      /* the cell's sigma entry is not k_c w^r for any column c < num_variables and row r */
#define BJ_SIGMA_UNNAMED 2u      /* no sigma entry names the cell */
#define BJ_SIGMA_NAMED_TWICE 3u  /* two or more sigma entries name the cell */
typedef struct bj_satisfiability_report {
  uint32_t satisfied; /* 1 if every count below is 0 */
  uint32_t reserved0;
  /* gates: (row, gate, repetition) instances with a nonzero term; the first in (row, gate, repetition, term) order */
  uint64_t gate_failures;
  uint64_t gate_row;
  uint32_t gate_index;      /* into circuit->gates */
  uint32_t gate_repetition;
  uint32_t gate_term;       /* index into the gate's writes */
  uint32_t reserved1;
  uint64_t gate_value;      /* the term's value (canonical) */
  uint64_t gate_selector;   /* the gate's selector on that row */
  /* copy constraints: cells whose value differs from the cell their sigma entry names; the first in (row, column) order */
  uint64_t copy_failures;
  uint64_t copy_row, copy_other_row;
  uint32_t copy_column, copy_other_column;
  uint64_t copy_value, copy_other_value;
  /* malformed sigma: entries naming no cell + cells named by no entry + cells named more than once; the first in
   * (row, column, kind) order */
  uint64_t sigma_failures;
  uint64_t sigma_row;
  uint32_t sigma_column;
  uint32_t sigma_kind;      /* BJ_SIGMA_* */
  /* lookups: tuples that match no table row, the first in (row, sub-argument) order */
  uint64_t lookup_unmatched;
  uint64_t lookup_row;
  uint32_t lookup_subargument;
  uint32_t reserved2;
  /* distinct table contents whose tuple count is not their multiplicity sum, the first by its first table row */
  uint64_t multiplicity_failures;
  uint64_t multiplicity_row;
  uint64_t multiplicity_count; /* tuples equal to the content */
  uint64_t multiplicity_sum;   /* sum mod p of d_multiplicities over the rows with that content */
} bj_satisfiability_report;
BJ_API int32_t bj_check_satisfied(bj_ctx* ctx, const bj_circuit* circuit, const uint64_t* d_sigmas, const uint64_t* d_constants,
                                  const uint64_t* d_lookup_tables /* or NULL */, const uint64_t* d_variables,
                                  const uint64_t* d_multiplicities /* or NULL */, bj_satisfiability_report* out);
/* materialize_multiplicities_polynomials (src/cs/implementations/witness.rs:225-272) on the device: d_multiplicities (n values)
 * receives, on the first table row of every distinct content, the number of lookup tuples equal to it, and 0 on every other
 * row.  The circuit fields read and the argument rules are those of bj_check_satisfied; the circuit must have a lookup
 * argument.  BJ_ERR_INVALID_ARG, naming the first such tuple, if a tuple matches no table row (no valid column exists then).
 * Scratch: 16 n bytes.  Synchronises. */
BJ_API int32_t bj_lookup_multiplicities(bj_ctx* ctx, const bj_circuit* circuit, const uint64_t* d_constants, const uint64_t* d_lookup_tables,
                                        const uint64_t* d_variables, uint64_t* d_multiplicities /* out: n values */);

/* device self-test: PTX field arithmetic vs the portable C versions on n pseudo-random + edge inputs */
BJ_API int32_t bj_selftest_field(bj_ctx* ctx, uint64_t n, uint64_t seed, uint64_t* h_mismatches);

/* ---- host self-test hooks: the same gl64 source compiled for the host (CPU tests, no device needed) ---- */
BJ_API uint64_t bj_host_gl_mul(uint64_t a, uint64_t b);
BJ_API uint64_t bj_host_gl_add(uint64_t a, uint64_t b);
BJ_API uint64_t bj_host_gl_sub(uint64_t a, uint64_t b);
BJ_API uint64_t bj_host_gl_inv(uint64_t a);
BJ_API uint64_t bj_host_gl_mul_pow2(uint64_t a, uint32_t s);
BJ_API void bj_host_e2_mul(const uint64_t a[2], const uint64_t b[2], uint64_t out[2]);
BJ_API void bj_host_e2_inv(const uint64_t a[2], uint64_t out[2]);
BJ_API void bj_host_poseidon2_permutation(uint64_t state[12]);
BJ_API void bj_host_poseidon_permutation(uint64_t state[12]); /* Poseidon (v1), poseidon_goldilocks_naive.rs:154-165 */
BJ_API void bj_host_keccak256(const uint8_t* data, size_t n, uint8_t out[32]);

#ifdef __cplusplus
}
#endif
#endif /* BOOJUM_B200_H */
