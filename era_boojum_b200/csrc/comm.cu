// Multi-GPU communicator of the coset-sharded prover: one bj_comm per (process, GPU), rank r of `world`.
//
// The reference has no counterpart (its Worker is one machine's thread pool, src/worker/mod.rs); what crosses GPUs is fixed
// by the data dependencies of prove_cpu_basic (SURVEY.md 8e): cap digests of every oracle, the quotient cosets that are
// interpolated together (src/cs/implementations/prover.rs:1399-1467), the openings, the last FRI codeword, query answers.
//
// Two transports behind one interface:
//   * NCCL over NVLink / NVSwitch (one process per GPU).  libnccl.so.2 is resolved at run time with dlopen - the copy a host
//     framework already loaded is reused (RTLD_NOLOAD first) - so the library itself has no link-time NCCL dependency and still
//     loads on a box without it; the few NCCL declarations needed are restated below (stable C ABI of NCCL 2.x).
//   * "local": the ranks are threads of one process whose contexts sit on the same device (or on peer-accessible devices):
//     collectives are device-to-device copies between the ranks' buffers, ordered by a host barrier.  It exists so that the
//     sharded driver can be exercised end to end on a single GPU (NCCL refuses two ranks on one device).
#include <dlfcn.h>
#include <condition_variable>
#include <cstring>
#include <mutex>
#include <vector>
#include "ctx.hpp"

namespace bj {

// ---- the slice of the NCCL C API used here ----
typedef void* nccl_comm_t;
struct nccl_unique_id {
  char internal[128];
};
enum { NCCL_UINT64 = 5 };  // ncclDataType_t: ncclInt8 0, ncclUint8 1, ncclInt32 2, ncclUint32 3, ncclInt64 4, ncclUint64 5
struct NcclApi {
  int (*GetUniqueId)(nccl_unique_id*) = nullptr;
  int (*CommInitRank)(nccl_comm_t*, int, nccl_unique_id, int) = nullptr;
  int (*CommDestroy)(nccl_comm_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, nccl_comm_t, cudaStream_t) = nullptr;
  int (*Broadcast)(const void*, void*, size_t, int, int, nccl_comm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  bool ok = false;
};
static NcclApi& nccl_api() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);  // the copy already in the process (e.g. torch's), if any
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return;
    api.GetUniqueId = (int (*)(nccl_unique_id*))dlsym(h, "ncclGetUniqueId");
    api.CommInitRank = (int (*)(nccl_comm_t*, int, nccl_unique_id, int))dlsym(h, "ncclCommInitRank");
    api.CommDestroy = (int (*)(nccl_comm_t))dlsym(h, "ncclCommDestroy");
    api.AllGather = (int (*)(const void*, void*, size_t, int, nccl_comm_t, cudaStream_t))dlsym(h, "ncclAllGather");
    api.Broadcast = (int (*)(const void*, void*, size_t, int, int, nccl_comm_t, cudaStream_t))dlsym(h, "ncclBroadcast");
    api.GetErrorString = (const char* (*)(int))dlsym(h, "ncclGetErrorString");
    api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllGather && api.Broadcast;
  });
  return api;
}

}  // namespace bj

// ranks-as-threads group (the "local" transport)
struct bj_comm_group {
  uint32_t world = 0;
  std::mutex m;
  std::condition_variable cv;
  uint32_t arrived = 0;
  uint64_t generation = 0;
  std::vector<const void*> slots;
  void barrier() {
    std::unique_lock<std::mutex> lk(m);
    const uint64_t gen = generation;
    if (++arrived == world) {
      arrived = 0;
      generation++;
      cv.notify_all();
    } else {
      cv.wait(lk, [&] { return generation != gen; });
    }
  }
};

struct bj_comm {
  bj_ctx* ctx = nullptr;
  uint32_t rank = 0, world = 1;
  bj::nccl_comm_t nccl = nullptr;
  bj_comm_group* group = nullptr;
  bj::u64* stage = nullptr;  // device staging for the host-buffer collectives
  size_t stage_u64 = 0;
  // second stream for collectives that overlap with compute on the context's stream (NCCL transport)
  cudaStream_t aux = nullptr;
  std::vector<cudaEvent_t> events;  // pool, grown on demand
  size_t next_event = 0;
  cudaEvent_t event() {
    if (next_event == events.size()) {
      cudaEvent_t e = nullptr;
      cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
      events.push_back(e);
    }
    return events[next_event++ % events.size()];
  }
};

namespace bj {

#define BJ_NCCL(comm, expr)                                                                                        \
  do {                                                                                                             \
    const int _r = (expr);                                                                                         \
    if (_r != 0) {                                                                                                 \
      const NcclApi& _a = nccl_api();                                                                              \
      (comm)->ctx->last_error = std::string(#expr) + ": " + (_a.GetErrorString ? _a.GetErrorString(_r) : "NCCL error"); \
      return BJ_ERR_CUDA;                                                                                          \
    }                                                                                                              \
  } while (0)

static int32_t comm_stage(bj_comm* c, size_t n_u64) {
  if (c->stage_u64 >= n_u64) return BJ_OK;
  bj_ctx* ctx = c->ctx;
  if (c->stage) {
    BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    cudaFree(c->stage);
    c->stage = nullptr;
    c->stage_u64 = 0;
  }
  const size_t want = std::max<size_t>(n_u64, 1 << 16);
  BJ_CUDA(ctx, cudaMalloc((void**)&c->stage, sizeof(u64) * want));
  c->stage_u64 = want;
  return BJ_OK;
}

// recv[r * n .. (r+1) * n) = rank r's send[0 .. n); device buffers, asynchronous on the context's stream (NCCL) or complete
// on return (local transport).  send may alias its own slot of recv.
int32_t comm_all_gather(bj_comm* c, const u64* d_send, u64* d_recv, u64 n) {
  bj_ctx* ctx = c->ctx;
  if (c->world == 1) {
    if (d_send != d_recv) BJ_CUDA(ctx, cudaMemcpyAsync(d_recv, d_send, sizeof(u64) * n, cudaMemcpyDeviceToDevice, ctx->stream));
    return BJ_OK;
  }
  if (c->nccl) {
    BJ_NCCL(c, nccl_api().AllGather(d_send, d_recv, (size_t)n, NCCL_UINT64, c->nccl, ctx->stream));
    return BJ_OK;
  }
  bj_comm_group* g = c->group;
  BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // my send buffer is complete
  g->slots[c->rank] = d_send;
  g->barrier();
  for (uint32_t r = 0; r < c->world; r++)
    if (d_recv + (size_t)r * n != (const u64*)g->slots[r])
      BJ_CUDA(ctx, cudaMemcpyAsync(d_recv + (size_t)r * n, g->slots[r], sizeof(u64) * n, cudaMemcpyDeviceToDevice, ctx->stream));
  BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  g->barrier();  // every rank has read every send buffer: they may be reused
  return BJ_OK;
}

// The same all-gather issued on the communicator's auxiliary stream: it starts when the work enqueued so far on the context's
// stream is done, and returns an event the caller makes the context's stream wait for (comm_wait) right before it consumes
// d_recv - compute enqueued in between overlaps with the transfer.  The local transport has no streams to overlap: it runs
// the blocking all-gather and returns a null event.
int32_t comm_all_gather_overlapped(bj_comm* c, const u64* d_send, u64* d_recv, u64 n, cudaEvent_t* done) {
  *done = nullptr;
  if (c->world == 1 || !c->nccl) return comm_all_gather(c, d_send, d_recv, n);
  bj_ctx* ctx = c->ctx;
  if (!c->aux) BJ_CUDA(ctx, cudaStreamCreateWithFlags(&c->aux, cudaStreamNonBlocking));
  if (c->events.size() < 64) {
    while (c->events.size() < 64) {
      cudaEvent_t e = nullptr;
      BJ_CUDA(ctx, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
      c->events.push_back(e);
    }
  }
  cudaEvent_t ready = c->event(), fin = c->event();
  BJ_CUDA(ctx, cudaEventRecord(ready, ctx->stream));
  BJ_CUDA(ctx, cudaStreamWaitEvent(c->aux, ready, 0));
  BJ_NCCL(c, nccl_api().AllGather(d_send, d_recv, (size_t)n, NCCL_UINT64, c->nccl, c->aux));
  BJ_CUDA(ctx, cudaEventRecord(fin, c->aux));
  *done = fin;
  return BJ_OK;
}
int32_t comm_wait(bj_comm* c, cudaEvent_t done) {
  if (!done) return BJ_OK;
  BJ_CUDA(c->ctx, cudaStreamWaitEvent(c->ctx->stream, done, 0));
  return BJ_OK;
}

// host buffers (small: caps, codeword tails, query answers): h_recv[r * n ..] = rank r's h_send; synchronises
int32_t comm_all_gather_host(bj_comm* c, const u64* h_send, u64* h_recv, u64 n) {
  bj_ctx* ctx = c->ctx;
  if (c->world == 1) {
    if (h_send != h_recv) memcpy(h_recv, h_send, sizeof(u64) * n);
    return BJ_OK;
  }
  if (c->nccl) {
    BJ_TRY(comm_stage(c, (size_t)n * (c->world + 1)));
    u64* snd = c->stage;
    u64* rcv = c->stage + n;
    BJ_CUDA(ctx, cudaMemcpyAsync(snd, h_send, sizeof(u64) * n, cudaMemcpyHostToDevice, ctx->stream));
    BJ_NCCL(c, nccl_api().AllGather(snd, rcv, (size_t)n, NCCL_UINT64, c->nccl, ctx->stream));
    BJ_CUDA(ctx, cudaMemcpyAsync(h_recv, rcv, sizeof(u64) * n * c->world, cudaMemcpyDeviceToHost, ctx->stream));
    BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return BJ_OK;
  }
  bj_comm_group* g = c->group;
  g->slots[c->rank] = h_send;
  g->barrier();
  for (uint32_t r = 0; r < c->world; r++) memcpy(h_recv + (size_t)r * n, g->slots[r], sizeof(u64) * n);
  g->barrier();
  return BJ_OK;
}

int32_t comm_broadcast_host(bj_comm* c, u64* h_buf, u64 n, uint32_t root) {
  bj_ctx* ctx = c->ctx;
  if (c->world == 1 || n == 0) return BJ_OK;
  if (c->nccl) {
    BJ_TRY(comm_stage(c, (size_t)n));
    if (c->rank == root) BJ_CUDA(ctx, cudaMemcpyAsync(c->stage, h_buf, sizeof(u64) * n, cudaMemcpyHostToDevice, ctx->stream));
    BJ_NCCL(c, nccl_api().Broadcast(c->stage, c->stage, (size_t)n, NCCL_UINT64, (int)root, c->nccl, ctx->stream));
    if (c->rank != root) BJ_CUDA(ctx, cudaMemcpyAsync(h_buf, c->stage, sizeof(u64) * n, cudaMemcpyDeviceToHost, ctx->stream));
    BJ_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return BJ_OK;
  }
  bj_comm_group* g = c->group;
  if (c->rank == root) g->slots[root] = h_buf;
  g->barrier();
  if (c->rank != root) memcpy(h_buf, g->slots[root], sizeof(u64) * n);
  g->barrier();
  return BJ_OK;
}

uint32_t comm_world(const bj_ctx* ctx) { return ctx && ctx->comm ? ctx->comm->world : 1; }
uint32_t comm_rank(const bj_ctx* ctx) { return ctx && ctx->comm ? ctx->comm->rank : 0; }

int32_t comm_assemble_cap(bj_ctx* ctx, const u64* h_local_cap, uint32_t cap_size, uint32_t lde_factor, u64* h_global_cap) {
  const uint32_t world = comm_world(ctx);
  if (world == 1) {
    if (h_local_cap != h_global_cap) memcpy(h_global_cap, h_local_cap, sizeof(u64) * 4 * cap_size);
    return BJ_OK;
  }
  // every unit (a coset, or a row block of one) is a whole subtree: `per` cap nodes
  const uint32_t units = lde_factor << ctx->shard.log_split;
  if (cap_size < units || units % world) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "sharded proving needs cap_size >= LDE factor * row blocks and world | units");
  const uint32_t per = cap_size / units, local = cap_size / world;
  std::vector<u64> all((size_t)4 * cap_size);
  BJ_TRY(comm_all_gather_host(ctx->comm, h_local_cap, all.data(), (u64)4 * local));
  for (uint32_t r = 0; r < world; r++)
    for (uint32_t k = 0; k < units / world; k++) {
      const u64 j = ctx->shard.unit_of(r, k);
      memcpy(h_global_cap + (size_t)4 * j * per, all.data() + (size_t)4 * (r * local + k * per), sizeof(u64) * 4 * per);
    }
  return BJ_OK;
}

}  // namespace bj

using namespace bj;

extern "C" {

int32_t bj_comm_unique_id(uint8_t out[BJ_COMM_UNIQUE_ID_BYTES]) {
  if (!out) return BJ_ERR_INVALID_ARG;
  const NcclApi& a = nccl_api();
  if (!a.ok) return BJ_ERR_UNSUPPORTED;
  nccl_unique_id id;
  if (a.GetUniqueId(&id) != 0) return BJ_ERR_CUDA;
  static_assert(sizeof(id) == BJ_COMM_UNIQUE_ID_BYTES, "ncclUniqueId is 128 bytes");
  memcpy(out, &id, sizeof(id));
  return BJ_OK;
}

static int32_t comm_attach(bj_ctx* ctx, bj_comm* c, uint32_t log_lde) {
  // the communicator defines the domain shard of its context: rank r keeps the units u = r (mod world) - the cosets
  // j = r (mod world) for world <= the LDE factor, row blocks of cosets above it
  BJ_TRY(bj_ctx_set_domain_shard(ctx, c->rank, c->world, log_lde));
  ctx->comm = c;
  return BJ_OK;
}

int32_t bj_comm_create_nccl(bj_ctx* ctx, const uint8_t unique_id[BJ_COMM_UNIQUE_ID_BYTES], uint32_t rank, uint32_t world, uint32_t log_lde,
                            bj_comm** out) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || !unique_id || !out || world == 0 || rank >= world) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_comm_create_nccl: bad argument");
  *out = nullptr;
  if (ctx->comm) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_comm_create_nccl: the context already has a communicator");
  const NcclApi& a = nccl_api();
  if (!a.ok) BJ_FAIL(ctx, BJ_ERR_UNSUPPORTED, "bj_comm_create_nccl: libnccl.so.2 not found");
  bj_comm* c = new bj_comm();
  c->ctx = ctx;
  c->rank = rank;
  c->world = world;
  nccl_unique_id id;
  memcpy(&id, unique_id, sizeof(id));
  const int r = a.CommInitRank(&c->nccl, (int)world, id, (int)rank);
  if (r != 0) {
    ctx->last_error = std::string("ncclCommInitRank: ") + (a.GetErrorString ? a.GetErrorString(r) : "error");
    delete c;
    return BJ_ERR_CUDA;
  }
  const int32_t st = comm_attach(ctx, c, log_lde);
  if (st != BJ_OK) {
    a.CommDestroy(c->nccl);
    delete c;
    return st;
  }
  *out = c;
  return BJ_OK;
}

int32_t bj_comm_group_create(uint32_t world, bj_comm_group** out) {
  if (!out || world == 0) return BJ_ERR_INVALID_ARG;
  bj_comm_group* g = new bj_comm_group();
  g->world = world;
  g->slots.assign(world, nullptr);
  *out = g;
  return BJ_OK;
}
void bj_comm_group_destroy(bj_comm_group* g) { delete g; }

int32_t bj_comm_create_local(bj_ctx* ctx, bj_comm_group* group, uint32_t rank, uint32_t log_lde, bj_comm** out) {
  bj::DeviceGuard device_guard(ctx);
  if (!ctx || !group || !out || rank >= group->world) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_comm_create_local: bad argument");
  *out = nullptr;
  if (ctx->comm) BJ_FAIL(ctx, BJ_ERR_INVALID_ARG, "bj_comm_create_local: the context already has a communicator");
  bj_comm* c = new bj_comm();
  c->ctx = ctx;
  c->rank = rank;
  c->world = group->world;
  c->group = group;
  const int32_t st = comm_attach(ctx, c, log_lde);
  if (st != BJ_OK) {
    delete c;
    return st;
  }
  *out = c;
  return BJ_OK;
}

int32_t bj_comm_destroy(bj_comm* c) {
  if (!c) return BJ_OK;
  bj_ctx* ctx = c->ctx;
  bj::DeviceGuard device_guard(ctx);
  cudaStreamSynchronize(ctx->stream);
  if (c->aux) cudaStreamSynchronize(c->aux);
  if (c->nccl) nccl_api().CommDestroy(c->nccl);
  if (c->stage) cudaFree(c->stage);
  for (cudaEvent_t e : c->events) cudaEventDestroy(e);
  if (c->aux) cudaStreamDestroy(c->aux);
  if (ctx->comm == c) {
    ctx->comm = nullptr;
    bj_ctx_set_coset_shard(ctx, 0, 1, ctx->shard_log_lde);
  }
  delete c;
  return BJ_OK;
}

uint32_t bj_comm_rank(const bj_comm* c) { return c ? c->rank : 0; }
uint32_t bj_comm_world(const bj_comm* c) { return c ? c->world : 1; }

int32_t bj_comm_all_gather(bj_comm* c, const uint64_t* d_send, uint64_t* d_recv, uint64_t n_u64_per_rank) {
  if (!c || !d_send || !d_recv) return BJ_ERR_INVALID_ARG;
  bj::DeviceGuard device_guard(c->ctx);
  return comm_all_gather(c, (const u64*)d_send, (u64*)d_recv, n_u64_per_rank);
}
int32_t bj_comm_all_gather_host(bj_comm* c, const uint64_t* h_send, uint64_t* h_recv, uint64_t n_u64_per_rank) {
  if (!c || !h_send || !h_recv) return BJ_ERR_INVALID_ARG;
  bj::DeviceGuard device_guard(c->ctx);
  return comm_all_gather_host(c, (const u64*)h_send, (u64*)h_recv, n_u64_per_rank);
}
int32_t bj_comm_broadcast_host(bj_comm* c, uint64_t* h_buf, uint64_t n_u64, uint32_t root) {
  if (!c || (!h_buf && n_u64) || root >= c->world) return BJ_ERR_INVALID_ARG;
  bj::DeviceGuard device_guard(c->ctx);
  return comm_broadcast_host(c, (u64*)h_buf, n_u64, root);
}

}  // extern "C"
