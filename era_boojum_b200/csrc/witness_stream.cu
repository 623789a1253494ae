// Repeated proving against one setup (prove_from_witness_vec_and_precomputations, src/cs/implementations/convenience.rs:159-195):
// witness slot sets.  A slot holds one witness in the layout bj_prove reads ([V][n] variables, then n multiplicities when the
// circuit has a lookup).  Uploads run on the context's witness copy stream, so the copy engine fills slot k+1 while the
// compute stream proves slot k; events order the two streams:
//   ready[s]  recorded on the copy stream when slot s holds its witness; bj_prove_slot makes the compute stream wait on it;
//   free[s]   recorded on the compute stream when the proof of slot s has returned; the next upload into s waits on it.
// The WitnessVec form (all_values + u32 multiplicities, witness.rs:32-40) lands in one all_values buffer shared by the slots
// and is gathered into the slot on the copy stream through the setup's u32 copy hint (materialize_variables_polynomials_from_
// dense_hint, witness.rs:325-385); the next upload overwrites all_values only after that gather, by the copy stream's order.
// Pageable host memory is copied through a ring of pinned staging chunks on the calling thread (no helper thread).
// A slot set may also live on a lane of the setup's context (bj_ctx_create_lane): its buffers come from the lane's pool, its
// uploads run on the lane's own copy stream and its proofs on the lane's stream, so each lane streams its own witnesses.

namespace bj {

constexpr uint32_t WITNESS_MAX_SLOTS = 4;
constexpr uint32_t HINT32_PLACEHOLDER = 0xFFFFFFFFu;
constexpr uint32_t STAGING_CHUNKS = 4;
constexpr size_t STAGING_CHUNK_BYTES = 16ull << 20;

// column[c][row] = all_values[hint[c][row]] for row < hint_rows; placeholders and rows past the hint are zero.  Thread i
// handles element i of the [n_cols][n] output, so consecutive threads read consecutive hint entries of a column.
__global__ void __launch_bounds__(256) gather_columns_u32_kernel(const u64* __restrict__ values, const u32* __restrict__ hint, u64 hint_rows,
                                                                  u64 n, u32 n_cols, u64* __restrict__ out) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * n_cols) return;
  const u64 c = i / n, row = i % n;
  u64 v = 0;
  if (row < hint_rows) {
    const u32 h = hint[c * hint_rows + row];
    if (h != HINT32_PLACEHOLDER) v = gl::canon(values[h]);
  }
  out[i] = v;
}

// the multiplicity column from the reference's Vec<u32> (witness.rs:493-520): widened, zero past n_mult
__global__ void __launch_bounds__(256) widen_multiplicities_kernel(const u32* __restrict__ m, u64 n_mult, u64 n, u64* __restrict__ out) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[i] = i < n_mult ? (u64)m[i] : 0;
}

// pool bytes the set itself allocates in its context's pool: the slots; with max_values > 0 the all_values buffer and the u32
// multiplicities (lookup); each counted as one pool allocation the way pool_peak counts them
static u64 witness_slots_own_bytes(const bj_circuit& c, uint32_t n_slots, uint64_t max_values) {
  const u64 n = 1ull << c.log_n, lk = c.lookup_width ? 1 : 0;
  u64 b = pool_bytes((u64)n_slots * (c.num_variables + lk) * n);
  if (max_values) {
    b += pool_bytes(max_values);
    if (lk) b += pool_bytes((n + 1) / 2);
  }
  return b;
}

// the u32 hint at its largest (n rows), which bj_setup_attach_variables_hint allocates once, on the setup
static u64 witness_hint_bytes(const bj_circuit& c) { return pool_bytes(((u64)c.num_variables * (1ull << c.log_n) + 1) / 2); }

// pool bytes of a slot set on a parent: its own buffers, and with max_values > 0 the hint
static u64 witness_slots_pool_bytes(const bj_circuit& c, uint32_t n_slots, uint64_t max_values) {
  return witness_slots_own_bytes(c, n_slots, max_values) + (max_values ? witness_hint_bytes(c) : 0);
}

static bool witness_shape_valid(const bj_circuit* c, uint32_t n_slots) {
  return c && n_slots && n_slots <= WITNESS_MAX_SLOTS && c->num_variables && c->log_n && c->log_n <= 28;
}

}  // namespace bj

struct bj_witness_slots {
  bj_ctx* ctx = nullptr;
  const bj_setup* setup = nullptr;
  uint32_t n_slots = 0;
  uint64_t max_values = 0;
  uint64_t slot_len = 0;  // u64 of one slot: (V + lookup) * n
  uint64_t counted = 0;   // pool bytes the set counts on its context (bj_ctx::witness_set_bytes)
  bj::DevMem slots, values, mult32;
  cudaEvent_t ready[bj::WITNESS_MAX_SLOTS] = {}, freed[bj::WITNESS_MAX_SLOTS] = {};
  bool filled[bj::WITNESS_MAX_SLOTS] = {};
  bool proved[bj::WITNESS_MAX_SLOTS] = {};
  // pinned staging ring for pageable host memory (allocated by the first pageable upload)
  void* staging = nullptr;
  cudaEvent_t staged[bj::STAGING_CHUNKS] = {};
  bool staged_used[bj::STAGING_CHUNKS] = {};
  uint32_t next_chunk = 0;
  uint64_t* slot_ptr(uint32_t s) const { return (uint64_t*)slots.p + (size_t)s * slot_len; }
};

using namespace bj;

// one host-to-device copy on the witness stream: pinned memory directly, pageable memory chunk by chunk through the staging
// ring (the host waits only for a chunk's previous copy to finish before refilling it)
static int32_t witness_copy(bj_witness_slots* s, void* d_dst, const void* h_src, size_t bytes) {
  bj_ctx* ctx = s->ctx;
  if (!bytes) return BJ_OK;
  cudaPointerAttributes attr;
  if (cudaPointerGetAttributes(&attr, h_src) != cudaSuccess) {
    cudaGetLastError();
    attr.type = cudaMemoryTypeUnregistered;
  }
  if (attr.type == cudaMemoryTypeHost) {
    BJ_CUDA(ctx, cudaMemcpyAsync(d_dst, h_src, bytes, cudaMemcpyHostToDevice, ctx->witness_stream));
    return BJ_OK;
  }
  if (attr.type != cudaMemoryTypeUnregistered) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_witness_upload: the source is not host memory");
  if (!s->staging) {
    if (cudaMallocHost(&s->staging, STAGING_CHUNKS * STAGING_CHUNK_BYTES) != cudaSuccess) {
      cudaGetLastError();
      s->staging = nullptr;
      BJ_FAIL(ctx, BJ_ERR_OOM, "bj_witness_upload: pinned staging allocation failed");
    }
    for (uint32_t i = 0; i < STAGING_CHUNKS; i++) BJ_CUDA(ctx, cudaEventCreateWithFlags(&s->staged[i], cudaEventDisableTiming));
  }
  for (size_t off = 0; off < bytes; off += STAGING_CHUNK_BYTES) {
    const size_t cnt = std::min(STAGING_CHUNK_BYTES, bytes - off);
    const uint32_t k = s->next_chunk;
    s->next_chunk = (k + 1) % STAGING_CHUNKS;
    if (s->staged_used[k]) BJ_CUDA(ctx, cudaEventSynchronize(s->staged[k]));
    char* chunk = (char*)s->staging + (size_t)k * STAGING_CHUNK_BYTES;
    memcpy(chunk, (const char*)h_src + off, cnt);
    BJ_CUDA(ctx, cudaMemcpyAsync((char*)d_dst + off, chunk, cnt, cudaMemcpyHostToDevice, ctx->witness_stream));
    BJ_CUDA(ctx, cudaEventRecord(s->staged[k], ctx->witness_stream));
    s->staged_used[k] = true;
  }
  return BJ_OK;
}

// checks shared by both upload forms; on success the copy stream is ordered after the last proof that read the slot
static int32_t witness_upload_begin(bj_witness_slots* s, uint32_t slot, const char* who) {
  if (!s) return BJ_ERR_INVALID_ARG;
  if (slot >= s->n_slots)
    BJ_FAIL(s->ctx, BJ_ERR_INVALID_ARG, std::string(who) + ": slot " + std::to_string(slot) + " out of range (the set has " + std::to_string(s->n_slots) + ")");
  if (s->proved[slot]) BJ_CUDA(s->ctx, cudaStreamWaitEvent(s->ctx->witness_stream, s->freed[slot], 0));
  s->filled[slot] = false;  // until the whole witness is queued
  return BJ_OK;
}

static int32_t witness_upload_end(bj_witness_slots* s, uint32_t slot) {
  BJ_CUDA(s->ctx, cudaEventRecord(s->ready[slot], s->ctx->witness_stream));
  s->filled[slot] = true;
  return BJ_OK;
}

extern "C" {

int32_t bj_variables_hint_to_u32(const uint64_t* h_hint, uint64_t n, uint32_t* h_out, uint64_t* h_values_needed) {
  if ((!h_hint || !h_out) && n) return BJ_ERR_INVALID_ARG;
  uint64_t need = 0;
  for (uint64_t i = 0; i < n; i++) {
    const uint64_t h = h_hint[i];
    if (h & VAR_PLACEHOLDER_BIT) {
      h_out[i] = HINT32_PLACEHOLDER;
      continue;
    }
    const uint64_t idx = h & VAR_INDEX_MASK;
    if (idx >= HINT32_PLACEHOLDER) return BJ_ERR_INVALID_ARG;
    h_out[i] = (uint32_t)idx;
    need = std::max(need, idx + 1);
  }
  if (h_values_needed) *h_values_needed = need;
  return BJ_OK;
}

int32_t bj_setup_attach_variables_hint(bj_setup* setup, const uint64_t* h_hint, uint64_t hint_rows) {
  if (!setup || !setup->ctx) return BJ_ERR_INVALID_ARG;
  bj_ctx* ctx = setup->ctx;
  bj::DeviceGuard device_guard(ctx);
  const uint32_t V = setup->c.num_variables;
  if (!h_hint || hint_rows == 0 || hint_rows > (1ull << setup->c.log_n))
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_setup_attach_variables_hint: need a hint of 1 to 2^log_n rows");
  const u64 cells = (u64)V * hint_rows;
  std::vector<uint32_t> h32(cells);
  uint64_t need = 0;
  if (bj_variables_hint_to_u32(h_hint, cells, h32.data(), &need) != BJ_OK)
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_setup_attach_variables_hint: a variable index does not fit the u32 hint (>= 2^32 - 1)");
  {
    // a gather on a lane's copy stream may read the current hint; only the parent's streams are drained below
    std::lock_guard<std::mutex> lock(ctx->tables_mu);
    if (ctx->lane_witness_sets)
      BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_setup_attach_variables_hint: " + std::to_string(ctx->lane_witness_sets) +
                                           " witness slot set(s) of the context's lanes are alive: attach the hint before creating them");
  }
  BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // a previous hint may still be read by a gather
  if (ctx->witness_stream) BJ_CUDA(ctx, cudaStreamSynchronize(ctx->witness_stream));
  BJ_TRY(setup->vars_hint.alloc(ctx, (cells + 1) / 2));
  BJ_CUDA(ctx, cudaMemcpyAsync(setup->vars_hint.p, h32.data(), sizeof(uint32_t) * cells, cudaMemcpyHostToDevice, ctx->stream));
  BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  setup->hint_rows = hint_rows;
  setup->hint_values = need;
  setup->has_hint = true;
  return BJ_OK;
}

int32_t bj_witness_slots_bytes(const bj_circuit* c, uint32_t world, uint32_t n_slots, uint64_t max_values, uint64_t* out) {
  if (!out || world == 0 || (world & (world - 1)) || !witness_shape_valid(c, n_slots)) return BJ_ERR_INVALID_ARG;
  *out = witness_slots_pool_bytes(*c, n_slots, max_values);  // every rank holds the whole witness: the same on each of `world` GPUs
  return BJ_OK;
}

int32_t bj_witness_slots_bytes_split(const bj_circuit* c, uint32_t n_slots, uint64_t max_values, uint64_t out[2]) {
  if (!out || !witness_shape_valid(c, n_slots)) return BJ_ERR_INVALID_ARG;
  out[0] = witness_slots_own_bytes(*c, n_slots, max_values);
  out[1] = max_values ? witness_hint_bytes(*c) : 0;
  return BJ_OK;
}

// the memory check of a slot set on a lane, and its bytes counted on the lane and the parent (under the parent's tables_mu, so
// that sets created at once on several lanes are checked against one another).  Everything that shares the limit is summed:
// the setup with the live lanes and the parent proving at once, the hint once, the parent's sets, the lanes' sets, this set.
static int32_t lane_witness_slots_reserve(bj_ctx* lane, const bj_setup* setup, uint32_t n_slots, uint64_t max_values, uint64_t* counted) {
  bj_ctx* parent = lane->parent;
  const bj_circuit& c = setup->c;
  const uint64_t own = witness_slots_own_bytes(c, n_slots, max_values);
  ProofShape sh;
  BJ_TRY(setup_shape(setup, &sh));
  std::lock_guard<std::mutex> lock(parent->tables_mu);
  const uint32_t m = parent->lanes.load();
  uint64_t p[3];
  lane_plan(sh, setup->plan, setup->chunk, m + 1, p);
  const uint64_t hint = max_values || setup->has_hint ? witness_hint_bytes(c) : 0;
  const uint64_t total = p[2] + hint + parent->witness_set_bytes + parent->lane_witness_set_bytes + own;
  const uint64_t limit = parent->memory_limit ? parent->memory_limit : setup->limit;
  if (total > limit)
    BJ_FAIL(lane, BJ_ERR_OOM, "bj_witness_slots_create: on a lane, the setup with " + std::to_string(m) + " lane(s) and the parent proving needs " +
                                  std::to_string(p[2]) + " bytes, the variables hint " + std::to_string(hint) + " bytes, the parent's slot sets " +
                                  std::to_string(parent->witness_set_bytes) + " bytes, the lanes' slot sets " +
                                  std::to_string(parent->lane_witness_set_bytes) + " bytes and " + std::to_string(n_slots) + " witness slots " +
                                  std::to_string(own) + " bytes: " + std::to_string(total) + " bytes, above the limit of " + std::to_string(limit) +
                                  " bytes");
  lane->witness_sets++;
  lane->witness_set_bytes += own;
  parent->lane_witness_sets++;
  parent->lane_witness_set_bytes += own;
  *counted = own;
  return BJ_OK;
}

// takes back what a set counted on its context (and, for a lane, on the parent)
static void witness_slots_unreserve(bj_ctx* ctx, uint64_t counted) {
  bj_ctx* owner = ctx->parent ? ctx->parent : ctx;
  std::lock_guard<std::mutex> lock(owner->tables_mu);
  ctx->witness_sets--;
  ctx->witness_set_bytes -= counted;
  if (ctx->parent) {
    ctx->parent->lane_witness_sets--;
    ctx->parent->lane_witness_set_bytes -= counted;
  }
}

int32_t bj_witness_slots_create(bj_ctx* ctx, const bj_setup* setup, uint32_t n_slots, uint64_t max_values, bj_witness_slots** out) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || !setup || !out) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_witness_slots_create: bad argument");
  *out = nullptr;
  const bool lane = ctx->parent != nullptr;
  if (setup->ctx != (lane ? ctx->parent : ctx)) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_witness_slots_create: the setup belongs to another context");
  if (n_slots == 0 || n_slots > WITNESS_MAX_SLOTS) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_witness_slots_create: 1 to 4 slots");
  const bj_circuit& c = setup->c;
  uint64_t counted = 0;
  if (lane) {
    BJ_TRY(lane_witness_slots_reserve(ctx, setup, n_slots, max_values, &counted));
  } else {
    const uint64_t bytes = witness_slots_pool_bytes(c, n_slots, max_values);
    const uint64_t limit = ctx->memory_limit ? ctx->memory_limit : setup->limit;
    if (setup->chosen_bytes() + bytes > limit)
      BJ_FAIL(ctx, BJ_ERR_OOM, "bj_witness_slots_create: the setup's plan needs " + std::to_string(setup->chosen_bytes()) + " bytes and " +
                                   std::to_string(n_slots) + " witness slots " + std::to_string(bytes) + " bytes, above the limit of " +
                                   std::to_string(limit) + " bytes");
    std::lock_guard<std::mutex> lock(ctx->tables_mu);
    ctx->witness_sets++;
    ctx->witness_set_bytes += bytes;
    counted = bytes;
  }
  // from here on the set is counted: a failure below frees it with bj_witness_slots_free, which takes the count back
  std::unique_ptr<bj_witness_slots, void (*)(bj_witness_slots*)> s(new bj_witness_slots(), bj_witness_slots_free);
  s->ctx = ctx;
  s->counted = counted;
  s->setup = setup;
  s->n_slots = n_slots;
  if (!ctx->witness_stream) BJ_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->witness_stream, cudaStreamNonBlocking));
  s->max_values = max_values;
  const u64 n = 1ull << c.log_n;
  s->slot_len = (u64)(c.num_variables + (c.lookup_width ? 1 : 0)) * n;
  for (uint32_t i = 0; i < n_slots; i++) {
    BJ_CUDA(ctx, cudaEventCreateWithFlags(&s->ready[i], cudaEventDisableTiming));
    BJ_CUDA(ctx, cudaEventCreateWithFlags(&s->freed[i], cudaEventDisableTiming));
  }
  BJ_TRY(s->slots.alloc(ctx, (size_t)n_slots * s->slot_len));
  if (max_values) {
    BJ_TRY(s->values.alloc(ctx, max_values));
    if (c.lookup_width) BJ_TRY(s->mult32.alloc(ctx, (n + 1) / 2));
  }
  BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // the copy stream writes these buffers next
  *out = s.release();
  return BJ_OK;
}

void bj_witness_slots_free(bj_witness_slots* s) {
  if (!s) return;
  bj_ctx* ctx = s->ctx;
  bj::DeviceGuard device_guard(ctx);
  if (ctx->witness_stream) cudaStreamSynchronize(ctx->witness_stream);
  cudaStreamSynchronize(ctx->stream);
  for (uint32_t i = 0; i < s->n_slots; i++) {
    if (s->ready[i]) cudaEventDestroy(s->ready[i]);
    if (s->freed[i]) cudaEventDestroy(s->freed[i]);
  }
  if (s->staging) {
    for (uint32_t i = 0; i < STAGING_CHUNKS; i++)
      if (s->staged[i]) cudaEventDestroy(s->staged[i]);
    cudaFreeHost(s->staging);
  }
  witness_slots_unreserve(ctx, s->counted);
  delete s;  // the device buffers go back to the context's pool, ordered on its stream
}

int32_t bj_witness_upload(bj_witness_slots* s, uint32_t slot, const uint64_t* h_variables, const uint64_t* h_multiplicities) {
  if (!s) return BJ_ERR_INVALID_ARG;
  bj_ctx* ctx = s->ctx;
  bj::DeviceGuard device_guard(ctx);
  const bj_circuit& c = s->setup->c;
  const u64 n = 1ull << c.log_n;
  if (!h_variables) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_witness_upload: no variables");
  if (c.lookup_width && !h_multiplicities) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_witness_upload: the lookup argument needs the multiplicities column");
  BJ_TRY(witness_upload_begin(s, slot, "bj_witness_upload"));
  uint64_t* d = s->slot_ptr(slot);
  BJ_TRY(witness_copy(s, d, h_variables, sizeof(u64) * c.num_variables * n));
  if (c.lookup_width) BJ_TRY(witness_copy(s, d + (size_t)c.num_variables * n, h_multiplicities, sizeof(u64) * n));
  return witness_upload_end(s, slot);
}

int32_t bj_witness_upload_vec(bj_witness_slots* s, uint32_t slot, const uint64_t* h_all_values, uint64_t n_values, const uint32_t* h_multiplicities,
                              uint64_t n_multiplicities) {
  if (!s) return BJ_ERR_INVALID_ARG;
  bj_ctx* ctx = s->ctx;
  bj::DeviceGuard device_guard(ctx);
  const bj_setup* setup = s->setup;
  const bj_circuit& c = setup->c;
  const u64 n = 1ull << c.log_n;
  if (!setup->has_hint) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_witness_upload_vec: the setup has no variables hint (bj_setup_attach_variables_hint)");
  if (!s->max_values) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_witness_upload_vec: the slot set was created without a witness-vector buffer (max_values = 0)");
  if (!h_all_values || n_values > s->max_values || n_values < setup->hint_values)
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_witness_upload_vec: " + std::to_string(n_values) + " values, the hint needs " + std::to_string(setup->hint_values) +
                                         " and the buffer holds " + std::to_string(s->max_values));
  if (c.lookup_width && (!h_multiplicities || n_multiplicities == 0 || n_multiplicities > n))
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_witness_upload_vec: the lookup argument needs 1 to 2^log_n multiplicities");
  BJ_TRY(witness_upload_begin(s, slot, "bj_witness_upload_vec"));
  uint64_t* d = s->slot_ptr(slot);
  BJ_TRY(witness_copy(s, s->values.p, h_all_values, sizeof(u64) * n_values));
  const u64 total = (u64)c.num_variables * n;
  gather_columns_u32_kernel<<<(unsigned)((total + 255) / 256), 256, 0, ctx->witness_stream>>>(s->values.p, (const u32*)setup->vars_hint.p, setup->hint_rows,
                                                                                              n, c.num_variables, (u64*)d);
  BJ_LAUNCH_CHECK(ctx);
  if (c.lookup_width) {
    BJ_TRY(witness_copy(s, s->mult32.p, h_multiplicities, sizeof(uint32_t) * n_multiplicities));
    widen_multiplicities_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->witness_stream>>>((const u32*)s->mult32.p, n_multiplicities, n, (u64*)d + total);
    BJ_LAUNCH_CHECK(ctx);
  }
  return witness_upload_end(s, slot);
}

int32_t bj_witness_slot_columns(bj_witness_slots* s, uint32_t slot, uint64_t** d_columns) {
  if (!s || !d_columns) return BJ_ERR_INVALID_ARG;
  bj_ctx* ctx = s->ctx;
  bj::DeviceGuard device_guard(ctx);
  if (slot >= s->n_slots || !s->filled[slot]) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_witness_slot_columns: slot out of range or never uploaded");
  BJ_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, s->ready[slot], 0));
  *d_columns = s->slot_ptr(slot);
  return BJ_OK;
}

int32_t bj_prove_slot(bj_ctx* ctx, const bj_setup* setup, bj_witness_slots* s, uint32_t slot, bj_proof** out) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || !setup || !s || !out) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_prove_slot: bad argument");
  if (s->ctx != ctx || s->setup != setup) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_prove_slot: the slot set belongs to another setup or context");
  if (slot >= s->n_slots) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_prove_slot: slot out of range");
  if (!s->filled[slot]) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_prove_slot: nothing was uploaded into the slot");
  BJ_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, s->ready[slot], 0));
  const uint64_t* d = s->slot_ptr(slot);
  const int32_t st = bj_prove(ctx, setup, d, setup->c.lookup_width ? d + ((size_t)setup->c.num_variables << setup->c.log_n) : nullptr, out);
  // the next upload into this slot waits for everything the proof queued on the compute stream
  BJ_CUDA(ctx, cudaEventRecord(s->freed[slot], ctx->stream));
  s->proved[slot] = true;
  return st;
}

}  // extern "C"
