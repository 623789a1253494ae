// Context management, device memory and host self-test hooks of the C-ABI (include/boojum_b200.h).
#include <cstdlib>
#include <cstring>
#include <memory>
#include "ctx.hpp"

namespace bj {
int32_t poseidon2_init_constants(bj_ctx* ctx);
}

namespace bj {
// device self-test of the PTX field arithmetic against the portable C versions (same inputs, same thread)
__global__ void field_selftest_kernel(u64 n, u64 seed, unsigned long long* mismatches) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  // splitmix64 stream + edge values
  auto next = [](u64& s) {
    s += 0x9E3779B97F4A7C15ull;
    u64 z = s;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
  };
  u64 st = seed + i * 0x632BE59BD9B4E019ull;
  const u64 edges[12] = {0, 1, gl::P - 1, gl::P, gl::P + 1, ~0ull, gl::EPS, gl::EPS + 1, 1ull << 63, gl::P - gl::EPS, 2, gl::P - 2};
  u64 a = next(st), b = next(st);
  if ((i & 7) == 0) a = edges[(i >> 3) % 12];
  if ((i & 15) < 2) b = edges[(i >> 4) % 12];
  if ((i & 7) == 3) {
    // structured operands that drive the rare wrap paths of the reduction: a = 2^s (+-1), b with all-zero / all-one
    // 32-bit halves (e.g. 2^63 * (r << 33) leaves x = -r3: the borrow path; 2^32 * ~0 takes the carry path)
    const u64 r = next(st);
    a = (1ull << ((i >> 3) & 63)) + (((i >> 9) & 3) == 1 ? 1 : 0) - (((i >> 9) & 3) == 2 ? 1 : 0);
    const unsigned sel = (unsigned)(i >> 11) & 7;
    u64 lo = r & 0xffffffffull, hi = r >> 32;
    if (sel & 1) lo = (sel & 4) ? 0xffffffffull : 0;
    if (sel & 2) hi = (sel & 4) ? 0xffffffffull : 0;
    b = (hi << 32) | lo;
  }
  if ((i & 63) == 5) {  // every pair of edge values
    a = edges[(i >> 6) % 12];
    b = edges[(i >> 6) / 12 % 12];
  }
  unsigned bad = 0;
  if (gl::mul(a, b) != gl::mul_c(a, b)) bad++;
  if (gl::canon(gl::mul_lazy(a, b)) != gl::mul_c(a, b)) bad++;
  const u64 bc = gl::canon(b);
  if (gl::canon(gl::add(a, bc)) != gl::canon(gl::add_c(a, bc))) bad++;
  if (gl::canon(gl::sub(a, bc)) != gl::canon(gl::sub_c(a, bc))) bad++;
  // b == p is allowed by the contract
  if (gl::canon(gl::add(a, gl::P)) != gl::canon(a)) bad++;
  if (gl::canon(gl::sub(a, gl::P)) != gl::canon(a)) bad++;
  if (gl::mul(a, b) >= gl::P) bad++;
  if (bad) atomicAdd(mismatches, (unsigned long long)bad);
}
}  // namespace bj

namespace bj {
// the prover driver allocates tens of GB per proof: a private pool that never trims keeps the second and later proofs free
// of cudaMalloc / page-mapping cost (the default pool returns memory to the OS at every synchronisation); nullptr if the
// device has none
static cudaMemPool_t private_pool(int device) {
  cudaMemPoolProps props = {};
  props.allocType = cudaMemAllocationTypePinned;
  props.handleTypes = cudaMemHandleTypeNone;
  props.location.type = cudaMemLocationTypeDevice;
  props.location.id = device;
  cudaMemPool_t pool = nullptr;
  if (cudaMemPoolCreate(&pool, &props) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  uint64_t keep = ~0ull;
  cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
  return pool;
}

// a lane of `parent` (bj_ctx_create_lane checks the arguments and the memory first): the parent's device, settings and tunables,
// its own non-blocking stream (no implicit ordering with the legacy default stream or with the other lanes) and pool, and
// tw_* viewing the parent's twiddles.  Every table the parent queued before this call is complete when it returns.
int32_t ctx_new_lane(bj_ctx* parent, bj_ctx** out) {
  std::unique_ptr<bj_ctx> lane(new bj_ctx());
  lane->device = parent->device;
  lane->sm_count = parent->sm_count;
  lane->l2_persist_bytes = parent->l2_persist_bytes;
  lane->l2_window_max = parent->l2_window_max;
  lane->ntt_use_v2 = parent->ntt_use_v2;
  lane->ntt_col_fastest = parent->ntt_col_fastest;
  lane->ntt_max_tile_log = parent->ntt_max_tile_log;
  lane->ntt_pass1_w = parent->ntt_pass1_w;
  lane->ntt_chunk_mb = parent->ntt_chunk_mb;
  lane->ntt_full_pow = parent->ntt_full_pow;
  lane->ntt_twist = parent->ntt_twist;
  lane->gate_peephole = parent->gate_peephole;
  lane->gate_points_per_thread = parent->gate_points_per_thread;
  lane->ntt_l2_persist = 0;  // the carve-out is sized for one stream's table (ctx.hpp)
  lane->ntt_bulk = parent->ntt_bulk;
  lane->memory_limit = parent->memory_limit;
  lane->allow_recompute_plan = parent->allow_recompute_plan;
  lane->max_row_blocks = parent->max_row_blocks;
  lane->own_twiddles = false;
  BJ_CUDA(parent, cudaStreamCreateWithFlags(&lane->stream, cudaStreamNonBlocking));
  lane->own_stream = true;
  lane->pool = private_pool(parent->device);
  {
    std::lock_guard<std::mutex> lock(parent->tables_mu);
    const cudaError_t e = cudaStreamSynchronize(parent->stream);
    if (e != cudaSuccess) {
      cudaStreamDestroy(lane->stream);
      if (lane->pool) cudaMemPoolDestroy(lane->pool);
      BJ_FAIL(parent, BJ_ERR_CUDA, std::string("bj_ctx_create_lane: cudaStreamSynchronize: ") + cudaGetErrorString(e));
    }
    lane->parent = parent;
    parent->lanes++;
  }
  *out = lane.release();
  return BJ_OK;
}
}  // namespace bj

using namespace bj;

extern "C" {

int32_t bj_selftest_field(bj_ctx* ctx, uint64_t n, uint64_t seed, uint64_t* h_mismatches) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || !h_mismatches) return BJ_ERR_INVALID_ARG;
  *h_mismatches = 0;
  if (n == 0) return BJ_OK;
  struct Counter {  // freed on every exit path
    unsigned long long* d = nullptr;
    ~Counter() {
      if (d) cudaFree(d);
    }
  } c;
  BJ_CUDA(ctx, cudaMalloc(&c.d, sizeof(unsigned long long)));
  BJ_CUDA(ctx, cudaMemsetAsync(c.d, 0, sizeof(unsigned long long), ctx->stream));
  field_selftest_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(n, seed, c.d);
  BJ_LAUNCH_CHECK(ctx);
  unsigned long long h = 0;
  BJ_CUDA(ctx, cudaMemcpyAsync(&h, c.d, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
  BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  *h_mismatches = h;
  return BJ_OK;
}

const char* bj_version(void) { return "boojum_b200 0.1.0 (sm_90a)"; }

const char* bj_status_string(int32_t s) {
  switch (s) {
    case BJ_OK: return "ok";
    case BJ_ERR_INVALID_ARG: return "invalid argument";
    case BJ_ERR_CUDA: return "CUDA error";
    case BJ_ERR_NO_DEVICE: return "no CUDA device (this library has no CPU fallback)";
    case BJ_ERR_OOM: return "out of device memory";
    case BJ_ERR_UNSUPPORTED: return "unsupported";
    default: return "unknown status";
  }
}

static int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return v && *v ? atoi(v) : dflt;
}

int32_t bj_ctx_create(int32_t device, void* stream, bj_ctx** out_ctx) {
  if (!out_ctx) return BJ_ERR_INVALID_ARG;
  *out_ctx = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) {
    cudaGetLastError();
    return BJ_ERR_NO_DEVICE;
  }
  if (device < 0 || device >= count) return BJ_ERR_INVALID_ARG;
  bj_ctx* ctx = new bj_ctx();
  ctx->device = device;
  bj::DeviceGuard device_guard(ctx);  // the caller's current device is restored on return
  {
    int cur = -1;
    if (cudaGetDevice(&cur) != cudaSuccess || cur != device) {
      cudaGetLastError();
      delete ctx;
      return BJ_ERR_CUDA;
    }
  }
  ctx->stream = (cudaStream_t)stream;  // NULL == the CUDA legacy default stream (what torch uses by default)
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) {
    ctx->sm_count = prop.multiProcessorCount;
    ctx->l2_persist_bytes = std::min<size_t>((size_t)prop.l2CacheSize * 3 / 8, (size_t)prop.persistingL2CacheMaxSize);
    ctx->l2_window_max = (size_t)prop.accessPolicyMaxWindowSize;
  }
  ctx->ntt_max_tile_log = env_int("BJ_NTT_MAX_TILE_LOG", 13);
  ctx->gate_points_per_thread = env_int("BJ_GATE_POINTS_PER_THREAD", 0);
  ctx->gate_peephole = env_int("BJ_GATE_PEEPHOLE", 15);
  if (ctx->ntt_max_tile_log < 8) ctx->ntt_max_tile_log = 8;
  if (ctx->ntt_max_tile_log > 14) ctx->ntt_max_tile_log = 14;
  ctx->ntt_pass1_w = env_int("BJ_NTT_PASS1_W", -1);
  ctx->ntt_use_v2 = env_int("BJ_NTT_V2", 1);
  ctx->ntt_col_fastest = env_int("BJ_NTT_COL_FASTEST", -1);
  ctx->ntt_full_pow = env_int("BJ_NTT_FULL_POW", 1);
  ctx->ntt_twist = env_int("BJ_NTT_TWIST", 1);
  ctx->ntt_bulk = env_int("BJ_NTT_BULK", 0);
  ctx->ntt_l2_persist = env_int("BJ_NTT_L2_PERSIST", 1);
  ctx->ntt_chunk_mb = env_int("BJ_NTT_CHUNK_MB", 0);
  ctx->pool = private_pool(device);
  int32_t st = poseidon2_init_constants(ctx);
  if (st != BJ_OK) {
    if (ctx->pool) cudaMemPoolDestroy(ctx->pool);
    delete ctx;
    return st;
  }
  *out_ctx = ctx;
  return BJ_OK;
}

int32_t bj_ctx_destroy(bj_ctx* ctx) {
  if (!ctx) return BJ_OK;
  bj::DeviceGuard device_guard(ctx);
  if (const uint32_t alive = ctx->lanes.load())
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_ctx_destroy: " + std::to_string(alive) + " lane(s) of this context are alive: destroy them first");
  if (ctx->parent) {
    std::lock_guard<std::mutex> lock(ctx->parent->tables_mu);
    if (ctx->witness_sets)
      BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_ctx_destroy: " + std::to_string(ctx->witness_sets) + " witness slot set(s) of this lane are alive: free them first");
  }
  cudaStreamSynchronize(ctx->stream);
  if (ctx->witness_stream) {  // uploads of witness slot sets still in flight finish before the memory goes
    cudaStreamSynchronize(ctx->witness_stream);
    cudaStreamDestroy(ctx->witness_stream);
  }
  if (ctx->own_twiddles) {  // a lane's view of its parent's pair is not its own
    if (ctx->tw_fwd) cudaFree(ctx->tw_fwd);
    if (ctx->tw_inv) cudaFree(ctx->tw_inv);
  }
  for (auto& e : ctx->pow_cache) {
    cudaFree(e.lo);
    cudaFree(e.hi);
    if (e.full) cudaFree(e.full);
  }
  for (auto& e : ctx->twist_cache) cudaFree(e.tab);
  for (void* p : ctx->tables_retired) cudaFree(p);
  if (ctx->pow_best) cudaFree(ctx->pow_best);
  if (ctx->gate_program) cudaFree(ctx->gate_program);
  if (ctx->pool) cudaMemPoolDestroy(ctx->pool);
  if (ctx->scratch) cudaFree(ctx->scratch);
  if (ctx->ptr_table) cudaFree(ctx->ptr_table);
  if (ctx->param_arena) cudaFree(ctx->param_arena);
  if (ctx->host_ring) cudaFree(ctx->host_ring);
  if (ctx->copy_streams_ready) {
    cudaStreamDestroy(ctx->h2d_stream);
    cudaStreamDestroy(ctx->d2h_stream);
    for (int i = 0; i < 3; i++) {
      cudaEventDestroy(ctx->ev_up[i]);
      cudaEventDestroy(ctx->ev_done[i]);
      cudaEventDestroy(ctx->ev_down[i]);
    }
  }
  if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
  if (ctx->parent) {
    std::lock_guard<std::mutex> lock(ctx->parent->tables_mu);
    ctx->parent->lanes--;
  }
  delete ctx;
  return BJ_OK;
}

int32_t bj_ctx_set_stream(bj_ctx* ctx, void* stream) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx) return BJ_ERR_INVALID_ARG;
  if (ctx->parent) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_ctx_set_stream: a lane keeps the stream it was created with");
  BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  ctx->stream = (cudaStream_t)stream;
  return BJ_OK;
}

int32_t bj_ctx_set_coset_shard(bj_ctx* ctx, uint32_t rank, uint32_t world, uint32_t log_lde) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx) return BJ_ERR_INVALID_ARG;
  if (world == 0 || (world & (world - 1)) || rank >= world || log_lde > 16 || world > (1u << log_lde))
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_ctx_set_coset_shard: world must be a power of two <= the LDE factor and rank < world");
  uint32_t ls = 0;
  while ((1u << ls) < world) ls++;
  ctx->shard_log_lde = log_lde;
  ctx->shard.first = rank;
  ctx->shard.log_stride = ls;
  ctx->shard.log_split = 0;
  return BJ_OK;
}

int32_t bj_ctx_set_domain_shard(bj_ctx* ctx, uint32_t rank, uint32_t world, uint32_t log_lde) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx) return BJ_ERR_INVALID_ARG;
  if (world == 0 || (world & (world - 1)) || rank >= world || log_lde > 16 || world > (8u << log_lde))
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_ctx_set_domain_shard: world must be a power of two <= 8 * the LDE factor and rank < world");
  uint32_t ls = 0;
  while ((1u << ls) < world) ls++;
  ctx->shard_log_lde = log_lde;
  ctx->shard.first = rank;
  ctx->shard.log_stride = ls;
  ctx->shard.log_split = ls > log_lde ? ls - log_lde : 0;  // row blocks per coset when there are more ranks than cosets
  return BJ_OK;
}

int32_t bj_ctx_synchronize(bj_ctx* ctx) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx) return BJ_ERR_INVALID_ARG;
  BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return BJ_OK;
}

int32_t bj_ctx_set_memory_limit(bj_ctx* ctx, uint64_t bytes) {
  if (!ctx) return BJ_ERR_INVALID_ARG;
  ctx->memory_limit = bytes;
  return BJ_OK;
}

int32_t bj_ctx_allow_recompute_plan(bj_ctx* ctx, int32_t allow) {
  if (!ctx) return BJ_ERR_INVALID_ARG;
  ctx->allow_recompute_plan = allow != 0;
  return BJ_OK;
}

int32_t bj_ctx_set_max_row_blocks(bj_ctx* ctx, uint32_t max_blocks) {
  if (!ctx) return BJ_ERR_INVALID_ARG;
  if (max_blocks == 0 || max_blocks > 8 || (max_blocks & (max_blocks - 1)))
    BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_ctx_set_max_row_blocks: 1, 2, 4 or 8 row blocks per coset");
  ctx->max_row_blocks = max_blocks;
  return BJ_OK;
}

int32_t bj_ctx_allow_sharded_recompute_plan(bj_ctx* ctx, int32_t allow) {
  if (!ctx) return BJ_ERR_INVALID_ARG;
  ctx->allow_sharded_recompute_plan = allow != 0;
  return BJ_OK;
}

int32_t bj_ctx_memory_high_water(bj_ctx* ctx, uint64_t* bytes, int32_t reset) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || !bytes) return BJ_ERR_INVALID_ARG;
  if (!ctx->pool) BJ_FAIL(ctx, BJ_ERR_UNSUPPORTED, "bj_ctx_memory_high_water: the context has no memory pool");
  BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  uint64_t v = 0;
  BJ_CUDA(ctx, cudaMemPoolGetAttribute(ctx->pool, cudaMemPoolAttrUsedMemHigh, &v));
  *bytes = v;
  if (reset) {
    uint64_t zero = 0;  // the attribute can only be reset to 0: the high-water mark restarts from the current use
    BJ_CUDA(ctx, cudaMemPoolSetAttribute(ctx->pool, cudaMemPoolAttrUsedMemHigh, &zero));
  }
  return BJ_OK;
}

const char* bj_last_error(const bj_ctx* ctx) { return ctx ? ctx->last_error.c_str() : "no context"; }
uint64_t bj_launch_count(const bj_ctx* ctx) { return ctx ? ctx->launches : 0; }

int32_t bj_alloc(bj_ctx* ctx, size_t bytes, void** d_ptr) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || !d_ptr) return BJ_ERR_INVALID_ARG;
  cudaError_t e = cudaMalloc(d_ptr, bytes ? bytes : 1);
  if (e != cudaSuccess) {
    cudaGetLastError();
    *d_ptr = nullptr;
    BJ_FAIL(ctx, e == cudaErrorMemoryAllocation ? BJ_ERR_OOM : BJ_ERR_CUDA, std::string("cudaMalloc: ") + cudaGetErrorString(e));
  }
  return BJ_OK;
}
int32_t bj_free(bj_ctx* ctx, void* d_ptr) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx) return BJ_ERR_INVALID_ARG;
  if (!d_ptr) return BJ_OK;
  BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  BJ_CUDA(ctx, cudaFree(d_ptr));
  return BJ_OK;
}
int32_t bj_upload(bj_ctx* ctx, void* d_dst, const void* h_src, size_t bytes) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || (!d_dst && bytes) || (!h_src && bytes)) return BJ_ERR_INVALID_ARG;
  BJ_CUDA(ctx, cudaMemcpyAsync(d_dst, h_src, bytes, cudaMemcpyHostToDevice, ctx->stream));
  return BJ_OK;
}
int32_t bj_download(bj_ctx* ctx, void* h_dst, const void* d_src, size_t bytes) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || (!h_dst && bytes) || (!d_src && bytes)) return BJ_ERR_INVALID_ARG;
  BJ_CUDA(ctx, cudaMemcpyAsync(h_dst, d_src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  return BJ_OK;
}
int32_t bj_alloc_host_pinned(size_t bytes, void** h_ptr) {
  if (!h_ptr) return BJ_ERR_INVALID_ARG;
  if (cudaMallocHost(h_ptr, bytes ? bytes : 1) != cudaSuccess) {
    cudaGetLastError();
    *h_ptr = nullptr;
    return BJ_ERR_OOM;
  }
  return BJ_OK;
}
int32_t bj_free_host_pinned(void* h_ptr) {
  if (h_ptr && cudaFreeHost(h_ptr) != cudaSuccess) return BJ_ERR_CUDA;
  return BJ_OK;
}

// ---- host self-test hooks (same gl64 / poseidon2 source, host compilation) ----
uint64_t bj_host_gl_mul(uint64_t a, uint64_t b) { return gl::mul(a, b); }
uint64_t bj_host_gl_add(uint64_t a, uint64_t b) { return gl::canon(gl::add_lazy(a, b)); }
uint64_t bj_host_gl_sub(uint64_t a, uint64_t b) { return gl::canon(gl::sub_lazy(a, b)); }
uint64_t bj_host_gl_inv(uint64_t a) { return gl::inv(a); }
uint64_t bj_host_gl_mul_pow2(uint64_t a, uint32_t s) { return gl::mul_pow2(a, s); }
void bj_host_e2_mul(const uint64_t a[2], const uint64_t b[2], uint64_t out[2]) {
  gl::e2 r = gl::e2_mul({a[0], a[1]}, {b[0], b[1]});
  out[0] = r.c0;
  out[1] = r.c1;
}
void bj_host_e2_inv(const uint64_t a[2], uint64_t out[2]) {
  gl::e2 r = gl::e2_inv({gl::canon(a[0]), gl::canon(a[1])});
  out[0] = r.c0;
  out[1] = r.c1;
}

}  // extern "C"
