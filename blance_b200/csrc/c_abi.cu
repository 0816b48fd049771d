// blance_b200/csrc/c_abi.cu — the C ABI of libblance_b200.so (include/blance_b200.h):
// validation, pooling of a batch of plan instances into one set of device arrays,
// the host side of the convergence loop (plan.go:32-56) and the launches.
// No CPU fallback: every compute entry point needs a CUDA device.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <utility>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_radix_sort.cuh>

#include "assign_pass.cuh"
#include "assign_pass_seq.cuh"
#include "assign_pass_spec.cuh"
#include "audit.cuh"
#include "aux_kernels.cuh"
#include "blance_b200.h"
#include "count_bound.hpp"
#include "device_types.cuh"
#include "exposure.cuh"
#include "wave_schedule.cuh"

using namespace blance_dev;

static std::string g_create_error;

// Opted-in dynamic shared memory of k_assign_pass_seq<1|2|4|8>, per device.  The attribute belongs to the
// (function, device) pair, not to a blance_ctx, and must only ever be raised.
static std::mutex g_dyn_smem_mu;
static size_t g_seq_dyn[64][4][4];   // [device][NPT index][K - 1]
static size_t g_spec_dyn[64][4];     // [device][K - 1], k_assign_pass_spec

// A failure inside this file.  It is thrown, and entry() / fan_out() turn it into a status and a message.
struct Error {
  int status;
  std::string msg;
};

[[noreturn]] static void throw_err(int status, const std::string& msg) { throw Error{status, msg}; }

static void cuda_check(cudaError_t e, const char* call) {
  if (e != cudaSuccess) throw_err(BLANCE_ERR_CUDA, std::string(call) + " failed: " + cudaGetErrorString(e));
}
#define CUDA(call) cuda_check((call), #call)

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// One stream-ordered device allocation carved into slices, each aligned to 256 bytes.  The slice list alone
// gives the size, so a layout is priced without allocating it; carve() lays the same list over a host buffer.
class Arena {
 public:
  Arena() = default;
  Arena(const Arena&) = delete;
  Arena& operator=(const Arena&) = delete;
  ~Arena() {
    if (base_) cudaFreeAsync(base_, stream_);       // back to the pool (stream ordered)
  }
  template <class T> void add(T*& p, size_t count) { slices_.push_back(Slice{(void**)&p, sizeof(T) * count}); }
  void add(void*& p, size_t bytes) { slices_.push_back(Slice{&p, bytes}); }
  size_t bytes() const {
    size_t total = 0;
    for (const Slice& s : slices_) total += span(s);
    return total;
  }
  void carve(void* base) const {
    char* p = (char*)base;
    for (const Slice& s : slices_) { *s.ptr = p; p += span(s); }
  }
  // The context's memory pool keeps the arena of the previous call around.
  void alloc(cudaStream_t st, const char* what) {
    void* p = nullptr;
    const cudaError_t e = cudaMallocAsync(&p, bytes(), st);
    if (e != cudaSuccess) {
      cudaGetLastError();
      throw_err(BLANCE_ERR_NOMEM, std::string("cudaMalloc of ") + what + " failed: " + cudaGetErrorString(e));
    }
    base_ = p;
    stream_ = st;
    carve(p);
  }

 private:
  struct Slice { void** ptr; size_t bytes; };
  static size_t span(const Slice& s) { return align_up(std::max<size_t>(s.bytes, 1), 256); }   // no two slices alias
  std::vector<Slice> slices_;
  void* base_ = nullptr;
  cudaStream_t stream_ = nullptr;
};

struct blance_ctx {
  int device = 0;
  int sm_count = 132;
  cudaStream_t stream = nullptr;
  std::string err;
  std::mutex mu;
  void* cub_tmp = nullptr;
  size_t cub_tmp_bytes = 0;
  std::vector<cudaEvent_t> events;   // pool for pass timing
  cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};   // [4], [5]: around the audit kernels
  int* d_any_active = nullptr;
  int* h_any_active = nullptr;       // pinned
  long long launches = 0;            // kernels of this library launched so far
  void* h_stage = nullptr;           // pinned staging of a batch (kept between calls, grow-only)
  size_t h_stage_bytes = 0;
  std::vector<blance_ctx*> children; // blance_ctx_create_multi: one single-device context per GPU
};

static int fail(blance_ctx* ctx, int st, const std::string& msg) {
  if (ctx) ctx->err = msg; else g_create_error = msg;
  return st;
}

// The entry ritual on the context that does a call's work: its lock is taken, its device made current, and an
// earlier CUDA error still pending on this thread is reported instead of being blamed on this call's first launch.
static std::unique_lock<std::mutex> enter(blance_ctx* dev) {
  std::unique_lock<std::mutex> lock(dev->mu);
  CUDA(cudaSetDevice(dev->device));
  const cudaError_t stale = cudaGetLastError();
  if (stale != cudaSuccess)
    throw_err(BLANCE_ERR_CUDA, std::string("a previous CUDA call on this thread failed: ") + cudaGetErrorString(stale));
  return lock;
}

// device() takes the entry ritual on the context that does the work (the first device of a multi-device context)
// and returns it.  An entry point calls it after the argument checks that need no device.
struct Device {
  blance_ctx* ctx;
  std::unique_lock<std::mutex> lock;
  blance_ctx* operator()() {
    if (!ctx) throw_err(BLANCE_ERR_INVALID_ARG, "ctx is NULL");
    blance_ctx* dev = ctx->children.empty() ? ctx : ctx->children[0];
    lock = enter(dev);
    return dev;
  }
};

// The boundary of every entry point that reports into a context: runs body(device) and turns what it throws into
// the status and the message of the context the caller passed (of blance_last_error(NULL) when that is NULL).
template <class F>
static int entry(blance_ctx* ctx, F&& body) noexcept {
  Device device{ctx, {}};
  try {
    body(device);
    return BLANCE_OK;
  } catch (const Error& e) {
    return fail(ctx, e.status, e.msg);
  } catch (const std::exception& e) {                   // host memory or threads
    return fail(ctx, BLANCE_ERR_NOMEM, std::string("host resources exhausted: ") + e.what());
  }
}

// Runs work(d, dev) on devices d = 0 .. G-1 of ctx (ctx itself when it is a single-device context, with G = 1),
// one host thread per device, each after the entry ritual.  The first failing device's error is rethrown as
// "device N: ...".
template <class F>
static void fan_out(blance_ctx* ctx, int G, F&& work) {
  if (ctx->children.empty()) {
    auto lock = enter(ctx);
    work(0, ctx);
    return;
  }
  std::vector<Error> err((size_t)G, Error{BLANCE_OK, std::string()});
  auto one = [&](int d) {
    blance_ctx* dev = ctx->children[(size_t)d];
    try {
      auto lock = enter(dev);
      work(d, dev);
    } catch (const Error& e) {
      err[(size_t)d] = e;
    } catch (const std::exception& e) {
      err[(size_t)d] = Error{BLANCE_ERR_NOMEM, std::string("host resources exhausted: ") + e.what()};
    }
  };
  std::vector<std::thread> th;
  for (int d = 0; d < G; ++d) th.emplace_back(one, d);
  for (auto& t : th) t.join();
  for (int d = 0; d < G; ++d)
    if (err[(size_t)d].status != BLANCE_OK)
      throw_err(err[(size_t)d].status, "device " + std::to_string(ctx->children[(size_t)d]->device) + ": " + err[(size_t)d].msg);
}

// Launches a kernel of this library on the context's stream, counts it and checks the launch.
template <class... P, class... A>
static void launch(blance_ctx* ctx, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, A&&... args) {
  kernel<<<grid, block, smem, ctx->stream>>>(std::forward<A>(args)...);
  ++ctx->launches;
  CUDA(cudaGetLastError());
}

// Raises a kernel's dynamic shared memory opt-in on the current device to `bytes` (it is never lowered).
// `configured` is the (kernel, device) pair's current opt-in.
static void opt_in_smem(const void* kernel, size_t* configured, size_t bytes) {
  std::lock_guard<std::mutex> g(g_dyn_smem_mu);
  if (bytes <= *configured) return;
  CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  *configured = bytes;
}

extern "C" int blance_version(void) { return 100; }

extern "C" int64_t blance_ctx_kernel_launches(const blance_ctx* ctx) {
  if (!ctx) return 0;
  long long n = ctx->launches;
  for (const blance_ctx* c : ctx->children) n += c->launches;
  return n;
}

extern "C" int blance_ctx_device_count(const blance_ctx* ctx) { return !ctx ? 0 : ctx->children.empty() ? 1 : (int)ctx->children.size(); }

extern "C" const char* blance_last_error(const blance_ctx* ctx) {
  return ctx ? ctx->err.c_str() : g_create_error.c_str();
}

extern "C" int blance_ctx_create(blance_ctx** out, int device_id) {
  if (!out) return fail(nullptr, BLANCE_ERR_INVALID_ARG, "blance_ctx_create: out is NULL");
  *out = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count <= 0)
    return fail(nullptr, BLANCE_ERR_CUDA, std::string("no CUDA device available (") +
                                              (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0") +
                                              "); libblance_b200 has no CPU fallback");
  if (device_id < 0) {
    if (cudaGetDevice(&device_id) != cudaSuccess) device_id = 0;
  }
  if (device_id >= count) return fail(nullptr, BLANCE_ERR_INVALID_ARG, "blance_ctx_create: device id out of range");
  blance_ctx* ctx = new blance_ctx();
  ctx->device = device_id;
  auto bail = [&](const char* what, cudaError_t er) {
    std::string msg = std::string(what) + ": " + cudaGetErrorString(er);
    delete ctx;
    return fail(nullptr, BLANCE_ERR_CUDA, msg);
  };
  if ((e = cudaSetDevice(device_id)) != cudaSuccess) return bail("cudaSetDevice", e);
  cudaDeviceProp prop;
  if ((e = cudaGetDeviceProperties(&prop, device_id)) != cudaSuccess) return bail("cudaGetDeviceProperties", e);
  ctx->sm_count = prop.multiProcessorCount;
  if ((e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking)) != cudaSuccess) return bail("cudaStreamCreate", e);
  for (auto& ev : ctx->ev)
    if ((e = cudaEventCreate(&ev)) != cudaSuccess) return bail("cudaEventCreate", e);
  {
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, device_id) == cudaSuccess) {
      unsigned long long keep = ~0ull;              // keep freed arenas cached in the pool between calls
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    }
  }
  if ((e = cudaMalloc(&ctx->d_any_active, sizeof(int))) != cudaSuccess) return bail("cudaMalloc", e);
  if ((e = cudaMallocHost(&ctx->h_any_active, sizeof(int))) != cudaSuccess) return bail("cudaMallocHost", e);
  *out = ctx;
  return BLANCE_OK;
}

// One context over several GPUs of the node (SURVEY.md section 8b: blance_ctx_create(gpu_ids, n_gpus)).  A batch
// (blance_plan_next_map_batch) is sharded instance i -> device i mod n, one host thread per device, no collective:
// plan instances are independent; scenarios are sharded the same way (fan_out()).  Everything else runs on the
// first device (entry()).
extern "C" int blance_ctx_create_multi(blance_ctx** out, const int* device_ids, int n_devices) {
  if (!out) return fail(nullptr, BLANCE_ERR_INVALID_ARG, "blance_ctx_create_multi: out is NULL");
  *out = nullptr;
  if (!device_ids || n_devices <= 0) return fail(nullptr, BLANCE_ERR_INVALID_ARG, "blance_ctx_create_multi: no devices given");
  for (int a = 0; a < n_devices; ++a)
    for (int b = 0; b < a; ++b)
      if (device_ids[a] == device_ids[b]) return fail(nullptr, BLANCE_ERR_INVALID_ARG, "blance_ctx_create_multi: a device is listed twice");
  blance_ctx* parent = new blance_ctx();
  for (int a = 0; a < n_devices; ++a) {
    blance_ctx* c = nullptr;
    const int st = blance_ctx_create(&c, device_ids[a]);
    if (st != BLANCE_OK) {
      for (blance_ctx* k : parent->children) blance_ctx_destroy(k);
      delete parent;
      return st;                       // g_create_error already says why
    }
    parent->children.push_back(c);
  }
  parent->device = parent->children[0]->device;
  parent->sm_count = parent->children[0]->sm_count;
  *out = parent;
  return BLANCE_OK;
}

extern "C" void blance_ctx_destroy(blance_ctx* ctx) {
  if (!ctx) return;
  if (!ctx->children.empty()) {
    for (blance_ctx* c : ctx->children) blance_ctx_destroy(c);
    delete ctx;
    return;
  }
  cudaSetDevice(ctx->device);
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  for (auto ev : ctx->events) cudaEventDestroy(ev);
  for (auto ev : ctx->ev) if (ev) cudaEventDestroy(ev);
  if (ctx->cub_tmp) cudaFree(ctx->cub_tmp);
  if (ctx->d_any_active) cudaFree(ctx->d_any_active);
  if (ctx->h_any_active) cudaFreeHost(ctx->h_any_active);
  if (ctx->h_stage) cudaFreeHost(ctx->h_stage);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
}

// ---------------------------------------------------------------------------------------
// A batch of instances resident on the device.

struct blance_plan {
  int n_inst = 0;
  std::vector<DInst> h_insts;          // initial descriptors (dynamic fields at their start values)
  std::vector<long long> raw_rows_off, raw_shape_off;   // caller-layout offsets per instance
  long long PT = 0, RT = 0, NT = 0, NUT = 0, CT = 0, N2T = 0, MT = 0, RRT = 0, RST = 0, ST = 0;
  int max_N = 0, max_S = 0, max_NU = 0;
  int pair_inst_shift = 0, pair_end_bit = 64;   // key layout of the (top, node) pair sort (k_pair_keys)
  bool any_state_active[BL_S_MAX] = {};
  Arena arena;                         // one device allocation, carved by plan_slices()
  DPool pool{};
  // immutable copies of the mutable state, to replay the plan (blance_plan_run)
  int32_t *rows_init = nullptr, *prev_rows_init = nullptr;
  uint32_t *pmeta_init = nullptr, *prev_meta_init = nullptr;
  uint8_t* pflags_init = nullptr;
  // device staging in caller layout
  int32_t *raw_a = nullptr, *raw_b = nullptr;           // cur/prev rows in, next rows out (raw_a)
  uint8_t *rawsh_a = nullptr, *rawsh_b = nullptr;       // cur/prev shape in, next shape (a) / warn (b) out
  long long *d_raw_rows_off = nullptr, *d_raw_shape_off = nullptr;
  int* d_seg_off = nullptr;            // [n_inst+1] partition offsets for the segmented sort
  // where a staged batch's results land in the context's pinned buffer (upload() carves them; unused by a
  // single instance, whose results are copied straight to the caller)
  int32_t* h_rows = nullptr;
  uint8_t *h_shape = nullptr, *h_warn = nullptr;
  float last_kernel_ms = 0, last_pass_ms = 0;
  int pass_launches = 0;
};
using PlanPtr = std::unique_ptr<blance_plan>;

// A batch of one instance is copied between the caller's arrays and the device directly; a larger batch goes
// through the pinned staging buffer.
static bool direct(const blance_plan* pl) { return pl->n_inst == 1; }

// sizes, pointers and limits of one instance (no table contents: those are blance_plan_in_check's)
static int check_structure(const blance_plan_in* in, std::string& why) {
  auto bad = [&](const char* what, int st = BLANCE_ERR_INVALID_ARG) {
    why = what;
    return st;
  };
  if (!in) return bad("plan_in is NULL");
  if (in->n_nodes < 0 || in->n_node_ids < in->n_nodes || in->n_states < 0 || in->n_parts < 0 || in->n_slots < 0)
    return bad("negative size or n_node_ids < n_nodes");
  if (in->n_states > BL_S_MAX) return bad("more than 8 model states", BLANCE_ERR_UNSUPPORTED);
  if (in->n_slots > BL_SLP_MAX) return bad("more than 32 slots per row", BLANCE_ERR_UNSUPPORTED);
  if (in->n_nodes > 8192) return bad("more than 8192 nodes", BLANCE_ERR_UNSUPPORTED);   /* 512 compute threads x 16 nodes */
  if (in->n_states > 0 && (!in->state_priority || !in->state_constraints || !in->state_slot_off ||
                           !in->state_stickiness || !in->state_has_stickiness))
    return bad("state tables are NULL");
  if (in->n_states > 0 && (in->top_state < 0 || in->top_state >= in->n_states)) return bad("top_state out of range");
  if (in->n_states > 0 && in->state_slot_off[in->n_states] != in->n_slots) return bad("state_slot_off[S] != n_slots");
  for (int s = 0; s < in->n_states; ++s) {
    if (in->state_slot_off[s + 1] < in->state_slot_off[s]) return bad("state_slot_off not monotone");
    if (in->state_constraints[s] > BL_K_MAX) return bad("constraints > 16", BLANCE_ERR_UNSUPPORTED);
    if (in->state_constraints[s] > in->state_slot_off[s + 1] - in->state_slot_off[s])
      return bad("a state's slot range is smaller than its constraints");
  }
  if (in->n_parts > 0 && (!in->part_in_prev || !in->part_in_assign || !in->part_weight || !in->part_has_weight ||
                          !in->part_name_rank))
    return bad("partition tables are NULL");
  if (in->n_parts > 0 && in->n_states > 0 && (!in->prev_shape || !in->cur_shape)) return bad("shape tables are NULL");
  if (in->n_parts > 0 && in->n_slots > 0 && (!in->prev_rows || !in->cur_rows)) return bad("row tables are NULL");
  if (in->n_node_ids > 0 && (!in->node_removed || !in->node_added)) return bad("node flag tables are NULL");
  if (in->n_nodes > 0 && in->has_node_weights && (!in->node_weight || !in->node_has_weight)) return bad("node weight tables are NULL");
  if (in->n_parts >= (1 << 30)) return bad("2^30 or more partitions", BLANCE_ERR_UNSUPPORTED);
  if (in->has_hier_rules) {
    if (!in->rule_off) return bad("rule_off is NULL");
    if (in->n_rules > 0 && !in->ie_mask) return bad("ie_mask is NULL");
    if (in->n_hier_bits < in->n_nodes) return bad("n_hier_bits < n_nodes");
    if ((in->n_hier_bits + 31) / 32 > 128) return bad("hierarchy universe above 4096 bits", BLANCE_ERR_UNSUPPORTED);
    for (int s = 0; s < in->n_states; ++s)
      if ((in->rule_off[s + 1] - in->rule_off[s]) * std::max(0, in->state_constraints[s]) > BL_PICK_MAX)
        return bad("rules x constraints > 32 for one state", BLANCE_ERR_UNSUPPORTED);
  }
  if (in->engine != BLANCE_ENGINE_AUTO && in->engine != BLANCE_ENGINE_LOCKSTEP && in->engine != BLANCE_ENGINE_SEQUENCER) return bad("unknown engine", BLANCE_ERR_UNSUPPORTED);
  if (in->booster_kind != BLANCE_BOOSTER_NONE && in->booster_kind != BLANCE_BOOSTER_CBGT_MAX)
    return bad("unknown booster_kind", BLANCE_ERR_UNSUPPORTED);
  return BLANCE_OK;
}

static void validate(const blance_plan_in* in, int idx) {
  std::string why;
  const int st = check_structure(in, why);
  if (st != BLANCE_OK) throw_err(st, "instance " + std::to_string(idx) + ": " + why);
}

/* The contents of the tables, for bindings that do not trust their own marshalling (the planning entry points
 * check sizes, pointers and limits only: a scan of every row would sit in the timed path of every call). */
extern "C" int blance_plan_in_check(const blance_plan_in* in, char* msg, int32_t msg_cap) {
  std::string why;
  auto done = [&](int st) {
    if (msg && msg_cap > 0) std::snprintf(msg, (size_t)msg_cap, "%s", why.c_str());
    return st;
  };
  int st = check_structure(in, why);
  if (st != BLANCE_OK) return done(st);
  auto bad = [&](const std::string& what, int code = BLANCE_ERR_INVALID_ARG) { why = what; return done(code); };
  if (in->n_states > 0 && in->state_slot_off[0] != 0) return bad("state_slot_off[0] != 0");
  const long long P = in->n_parts, SL = in->n_slots, S = in->n_states;
  for (int which = 0; which < 2; ++which) {
    const int32_t* rows = which ? in->cur_rows : in->prev_rows;
    const uint8_t* shape = which ? in->cur_shape : in->prev_shape;
    const char* name = which ? "cur" : "prev";
    int32_t lo = 0, hi = -1;
    for (long long i = 0; i < P * SL; ++i) { lo = std::min(lo, rows[i]); hi = std::max(hi, rows[i]); }
    if (lo < BLANCE_NO_NODE || hi >= in->n_node_ids)
      return bad(std::string(name) + "_rows holds a node id outside [-1, n_node_ids)");
    uint8_t sh = 0;
    for (long long i = 0; i < P * S; ++i) sh = std::max(sh, shape[i]);
    if (sh > BLANCE_SHAPE_LIST) return bad(std::string(name) + "_shape holds a value above BLANCE_SHAPE_LIST");
    // a state's list is filled from the left: no node after an empty slot
    for (long long p = 0; p < P; ++p)
      for (int s = 0; s < in->n_states; ++s) {
        bool gap = false;
        for (int c = in->state_slot_off[s]; c < in->state_slot_off[s + 1]; ++c) {
          const int32_t x = rows[p * SL + c];
          if (x == BLANCE_NO_NODE) gap = true;
          else if (gap) return bad(std::string(name) + "_rows: partition " + std::to_string(p) + " has a node after an empty slot of state " + std::to_string(s));
        }
      }
  }
  {
    // part_name_rank: 0 <= rank < 2^30, unique (it is the last word of the partition sort key, plan.go:512-528)
    std::vector<uint64_t> seen;
    std::vector<int32_t> big;
    seen.assign((size_t)((P + 63) / 64), 0);
    for (long long p = 0; p < P; ++p) {
      const int32_t r = in->part_name_rank[p];
      if (r < 0 || r >= (1 << 30)) return bad("part_name_rank outside [0, 2^30) at partition " + std::to_string(p));
      if (r < P) {
        if (seen[(size_t)(r >> 6)] >> (r & 63) & 1ull) return bad("part_name_rank " + std::to_string(r) + " appears twice");
        seen[(size_t)(r >> 6)] |= 1ull << (r & 63);
      } else big.push_back(r);
    }
    std::sort(big.begin(), big.end());
    if (std::adjacent_find(big.begin(), big.end()) != big.end()) return bad("a part_name_rank appears twice");
    // the weight word of the key is 999999999 - w printed with %10d (plan.go:539): beyond 999999999 the reference's
    // STRING order and a numeric order part ways
    for (long long p = 0; p < P; ++p)
      if (in->has_part_weights && in->part_has_weight[p] && in->part_weight[p] > 999999999)
        return bad("partition weight above 999999999 at partition " + std::to_string(p), BLANCE_ERR_UNSUPPORTED);
  }
  if (!count_bound_fits(*in)) return bad(BLANCE_COUNT_BOUND_MSG, BLANCE_ERR_UNSUPPORTED);
  if (in->has_hier_rules)
    for (int s = 0; s <= in->n_states; ++s) {
      if (in->rule_off[s] < 0 || in->rule_off[s] > in->n_rules || (s > 0 && in->rule_off[s] < in->rule_off[s - 1]))
        return bad("rule_off is not a monotone offset table into the rules");
    }
  why.clear();
  return done(BLANCE_OK);
}

static int grid_for(const blance_ctx* ctx, long long n, int block) {
  long long want = (n + block - 1) / block;
  long long cap = (long long)ctx->sm_count * 8;      // multiples of the SM count; kernels are grid-stride
  if (want > cap) want = cap;
  if (want < 1) want = 1;
  return (int)want;
}

// The device code (NR_REMOVE | NR_OUTSIDE) of node id q of an instance.  A caller's node_removed says only "in
// nodesToRemove", any nonzero value meaning yes; `coded` tables (blance_plan_chains' stages) already hold the code.
static uint8_t rm_code(const blance_plan_in& in, int q, bool coded) {
  const uint8_t v = in.node_removed[q];
  return coded ? v : (uint8_t)(v ? NR_REMOVE : 0);
}

// The node fields of a descriptor that a scenario or a chain stage changes, and the loop state they start it in:
// nodesNext's size, whether nodesToRemove is non-empty (also with ids outside nodesAll), nodesToAdd == nil.  n_prev =
// len(prevMap).
static void node_state(DInst& D, const blance_plan_in& in, bool coded, int n_prev) {
  int n_valid = 0, rm_active = 0, masked = 0;
  for (int q = 0; q < in.n_nodes; ++q) { n_valid += rm_code(in, q, coded) == 0; masked |= (rm_code(in, q, coded) & NR_OUTSIDE) != 0; }
  for (int q = 0; q < in.n_node_ids; ++q) rm_active |= rm_code(in, q, coded) & NR_REMOVE;
  D.has_node_weights = in.has_node_weights;
  D.n_valid = n_valid; D.masked = masked;
  D.P = n_prev; D.rm_active = rm_active; D.add_active = 1; D.add_is_nil = in.add_is_nil; D.use_rest = 0;
  D.active = in.max_iters > 0 ? 1 : 0;
  D.iters_run = 0; D.converged = 0; D.mismatch = 0;
}

// Host side of a batch: the per-instance descriptors, their offsets into the pooled arrays and the totals.
static void layout(blance_plan* pl, int n, const blance_plan_in* ins, std::vector<int>& seg_off, bool coded = false) {
  pl->n_inst = n;
  pl->h_insts.resize(n);
  pl->raw_rows_off.resize(n + 1);
  pl->raw_shape_off.resize(n + 1);
  seg_off.assign(n + 1, 0);
  int n_prev = 0, n_assign = 0;
  for (int i = 0; i < n; ++i) {
    const blance_plan_in& in = ins[i];
    DInst& D = pl->h_insts[i];
    std::memset(&D, 0, sizeof D);
    D.N = in.n_nodes; D.NU = in.n_node_ids; D.S = in.n_states; D.PU = in.n_parts; D.SL = in.n_slots;
    D.SLP = std::max(4, (int)align_up((size_t)in.n_slots, 4));
    D.HW = in.has_hier_rules ? (in.n_hier_bits + 31) / 32 : 0;
    D.n_rules = in.has_hier_rules ? in.n_rules : 0;
    D.top_state = in.top_state; D.booster = in.booster_kind;
    D.has_part_weights = in.has_part_weights; D.has_node_weights = in.has_node_weights;
    D.has_hier_rules = in.has_hier_rules; D.max_iters = in.max_iters; D.engine = in.engine;
    D.debug = getenv("BLANCE_SPEC_STATS") ? 1 : 0;
    for (int s = 0; s < in.n_states; ++s) {
      D.state_priority[s] = in.state_priority[s];
      D.state_constraints[s] = in.state_constraints[s];
      D.state_slot_off[s] = in.state_slot_off[s];
      D.state_stickiness[s] = in.state_stickiness[s];
      D.state_has_stickiness[s] = in.state_has_stickiness[s];
      D.rule_off[s] = in.has_hier_rules ? in.rule_off[s] : 0;
      if (in.state_constraints[s] > 0) pl->any_state_active[s] = true;
    }
    D.state_slot_off[in.n_states] = in.n_slots;
    D.rule_off[in.n_states] = in.has_hier_rules ? in.rule_off[in.n_states] : 0;
    // (the instances of a scenario wave share their partition tables: counted once)
    const bool same_parts = i > 0 && in.n_parts == ins[i - 1].n_parts && in.part_in_prev == ins[i - 1].part_in_prev &&
                            in.part_in_assign == ins[i - 1].part_in_assign;
    if (!same_parts) {
      n_prev = 0; n_assign = 0;
      for (int p = 0; p < in.n_parts; ++p) { n_prev += in.part_in_prev[p] != 0; n_assign += in.part_in_assign[p] != 0; }
    }
    D.n_assign = n_assign;
    node_state(D, in, coded, n_prev);
    D.part_off = pl->PT; D.rows_off = pl->RT; D.node_off = pl->NT; D.nodeid_off = pl->NUT;
    D.counts_off = pl->CT; D.n2n_off = pl->N2T; D.mask_off = pl->MT; D.stream_off = pl->ST;
    pl->raw_rows_off[i] = pl->RRT; pl->raw_shape_off[i] = pl->RST;
    seg_off[i] = (int)pl->PT;
    pl->ST += (long long)D.PU * (D.SLP + 8);
    pl->PT += D.PU; pl->RT += (long long)D.PU * D.SLP; pl->NT += D.N; pl->NUT += D.NU;
    pl->CT += (long long)D.S * D.N; pl->N2T += (long long)(D.NU + 1) * D.N;
    pl->MT += (long long)D.n_rules * (D.NU + 1) * D.HW;
    pl->RRT += (long long)D.PU * D.SL; pl->RST += (long long)D.PU * D.S;
    pl->max_N = std::max(pl->max_N, D.N); pl->max_S = std::max(pl->max_S, D.S); pl->max_NU = std::max(pl->max_NU, D.NU);
  }
  seg_off[n] = (int)pl->PT;
  pl->raw_rows_off[n] = pl->RRT; pl->raw_shape_off[n] = pl->RST;
  {
    int top_bits = 1, inst_bits = 1;
    while ((1ll << top_bits) < (long long)pl->max_NU + 2) ++top_bits;
    while ((1ll << inst_bits) < (long long)n + 1) ++inst_bits;
    pl->pair_inst_shift = 13 + top_bits;
    pl->pair_end_bit = pl->pair_inst_shift + inst_bits;
  }
}

// Adds the device slices of a laid-out batch (sizes from layout()) to an arena.
static void plan_slices(Arena& a, blance_plan* pl, int n) {
  DPool& P = pl->pool;
  const size_t PT = (size_t)pl->PT + 1, RT = (size_t)pl->RT + 4, NT = (size_t)pl->NT + 1, NUT = (size_t)pl->NUT + 1;
  const size_t CT = (size_t)pl->CT + 1, N2T = (size_t)pl->N2T + 1, MT = (size_t)pl->MT + 1;
  const size_t RRT = (size_t)pl->RRT + 1, RST = (size_t)pl->RST + 1;
  a.add(P.rows, RT); a.add(P.prev_rows, RT); a.add(pl->rows_init, RT); a.add(pl->prev_rows_init, RT);
  a.add(P.pmeta, PT); a.add(P.prev_meta, PT); a.add(pl->pmeta_init, PT); a.add(pl->prev_meta_init, PT);
  a.add(P.pflags, PT); a.add(pl->pflags_init, PT);
  a.add(P.pweight, PT); a.add(P.name_rank, PT); a.add(P.part_inst, PT);
  a.add(P.stream, (size_t)pl->ST + 4); a.add(P.ostream, (size_t)pl->ST + 4);
  a.add(P.keys, PT); a.add(P.keys_alt, PT); a.add(P.order, PT); a.add(P.order_alt, PT);
  a.add(P.node_removed, NUT); a.add(P.node_added, NUT); a.add(P.node_weight, NT); a.add(P.node_has_weight, NT);
  a.add(P.extra_first, NT); a.add(P.extra_rest, NT);
  a.add(P.counts, CT); a.add(P.n2n, N2T); a.add(P.ie_mask, MT);
  a.add(P.n2n_dev, N2T); a.add(P.qstat, 4 * PT); a.add(P.srank, PT);
  a.add(P.pair_keys, 4 * PT); a.add(P.pair_keys_alt, 4 * PT);
  a.add(P.pair_vals, 4 * PT); a.add(P.pair_vals_alt, 4 * PT);
  a.add(P.insts, (size_t)n);
  a.add(pl->raw_a, RRT); a.add(pl->raw_b, RRT); a.add(pl->rawsh_a, RST); a.add(pl->rawsh_b, RST);
  a.add(pl->d_raw_rows_off, (size_t)n + 1); a.add(pl->d_raw_shape_off, (size_t)n + 1);
  a.add(pl->d_seg_off, (size_t)n + 1);
}

// Device bytes of the radix sorts' scratch for a batch of PT partitions in n segments (a size query only).
static size_t sort_scratch_bytes(long long PT, int n, cudaStream_t st) {
  size_t need = 0, need2 = 0, need3 = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, need, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int32_t*)nullptr,
                                  (int32_t*)nullptr, (int)PT, 0, 64, st);
  cub::DeviceSegmentedRadixSort::SortPairs(nullptr, need2, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int32_t*)nullptr,
                                           (int32_t*)nullptr, (int)PT, n, (int*)nullptr, (int*)nullptr, 0, 64, st);
  cub::DeviceRadixSort::SortPairs(nullptr, need3, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (uint32_t*)nullptr,
                                  (uint32_t*)nullptr, (int)(4 * PT), 0, 64, st);
  return std::max(need, std::max(need2, need3));
}

// Grows the context's sort scratch to what the batch needs, then waits for the uploads.
static void finish_upload(blance_ctx* ctx, const blance_plan* pl) {
  const size_t need = sort_scratch_bytes(pl->PT, pl->n_inst, ctx->stream);
  if (need > ctx->cub_tmp_bytes) {
    if (ctx->cub_tmp) cudaFree(ctx->cub_tmp);
    ctx->cub_tmp = nullptr; ctx->cub_tmp_bytes = 0;
    const cudaError_t e = cudaMalloc(&ctx->cub_tmp, need);
    if (e != cudaSuccess) { cudaGetLastError(); throw_err(BLANCE_ERR_NOMEM, "cudaMalloc of the sort scratch failed"); }
    ctx->cub_tmp_bytes = need;
  }
  CUDA(cudaStreamSynchronize(ctx->stream));
}

// Host arrays of a batch's node tables, extra counts and hierarchy masks, in the pooled layout of layout().
struct NodeTables {
  uint8_t *rm, *ad, *hw;
  int32_t *nw, *ef, *er;
  uint32_t* mask;
};

// Writes instance `in` (descriptor D) into its slices of t.
static void stage_nodes(const blance_plan_in& in, const DInst& D, const NodeTables& t, bool coded = false) {
  for (int q = 0; q < D.NU; ++q) t.rm[D.nodeid_off + q] = rm_code(in, q, coded);
  if (D.NU) std::memcpy(t.ad + D.nodeid_off, in.node_added, (size_t)D.NU);
  for (int q = 0; q < D.N; ++q) {
    t.nw[D.node_off + q] = in.has_node_weights ? in.node_weight[q] : 0;
    t.hw[D.node_off + q] = in.has_node_weights ? in.node_has_weight[q] : 0;
    t.ef[D.node_off + q] = in.extra_tot_first ? in.extra_tot_first[q] : 0;
    t.er[D.node_off + q] = in.extra_tot_rest ? in.extra_tot_rest[q] : 0;
  }
  const size_t mw = (size_t)D.n_rules * (D.NU + 1) * D.HW;
  if (mw) std::memcpy(t.mask + D.mask_off, in.ie_mask, sizeof(uint32_t) * mw);
}

static uint8_t part_flags(const blance_plan_in& in, int p) {
  return (uint8_t)((in.part_in_prev[p] ? PF_IN_PREV : 0) | ((in.part_in_prev[p] & 2) ? PF_PREV_EXTRA : 0) |
                   (in.part_in_assign[p] ? PF_IN_ASSIGN : 0) | (in.part_has_weight[p] ? PF_HAS_WEIGHT : 0));
}

static PlanPtr upload(blance_ctx* ctx, int n, const blance_plan_in* ins, bool coded = false) {
  if (n <= 0) throw_err(BLANCE_ERR_INVALID_ARG, "batch size must be positive");
  for (int i = 0; i < n; ++i) validate(&ins[i], i);
  PlanPtr pl(new blance_plan());
  std::vector<int> seg_off;
  layout(pl.get(), n, ins, seg_off, coded);
  if (pl->PT >= (1LL << 29)) throw_err(BLANCE_ERR_UNSUPPORTED, "2^29 or more partitions in one batch");
  plan_slices(pl->arena, pl.get(), n);
  pl->arena.alloc(ctx->stream, "the plan arena");
  DPool& P = pl->pool;

  // ---- host side of the copy: a single instance straight from the caller's arrays, a batch concatenated in
  // caller layout into the context's pinned staging buffer
  const int32_t *h_cur = nullptr, *h_prev = nullptr, *h_pw = nullptr, *h_rank = nullptr, *h_inst = nullptr;
  const int32_t *h_nw = nullptr, *h_ef = nullptr, *h_er = nullptr;
  const uint8_t *h_csh = nullptr, *h_psh = nullptr, *h_flags = nullptr, *h_rm = nullptr, *h_ad = nullptr, *h_hw = nullptr;
  const uint32_t* h_mask = nullptr;
  std::vector<uint8_t> v_flags, v_rm;
  if (direct(pl.get())) {
    const blance_plan_in& in = ins[0];
    v_flags.resize((size_t)in.n_parts + 1);
    for (int p = 0; p < in.n_parts; ++p) v_flags[(size_t)p] = part_flags(in, p);
    v_rm.resize((size_t)in.n_node_ids + 1);
    for (int q = 0; q < in.n_node_ids; ++q) v_rm[(size_t)q] = rm_code(in, q, coded);
    h_cur = in.cur_rows; h_prev = in.prev_rows; h_csh = in.cur_shape; h_psh = in.prev_shape;
    h_flags = v_flags.data(); h_pw = in.part_weight; h_rank = in.part_name_rank;     // h_inst stays NULL: all zero
    h_rm = v_rm.data(); h_ad = in.node_added;
    if (in.has_node_weights) { h_nw = in.node_weight; h_hw = in.node_has_weight; }
    h_ef = in.extra_tot_first; h_er = in.extra_tot_rest; h_mask = in.ie_mask;
  } else {
    const size_t PT = (size_t)pl->PT + 1, NT = (size_t)pl->NT + 1, NUT = (size_t)pl->NUT + 1;
    const size_t MT = (size_t)pl->MT + 1, RRT = (size_t)pl->RRT + 1, RST = (size_t)pl->RST + 1;
    int32_t *s_cur, *s_prev, *s_pw, *s_rank, *s_inst;
    uint8_t *s_csh, *s_psh, *s_flags;
    NodeTables s;
    Arena stage;                // carved over the pinned buffer; fetch() reads the results from s_cur / s_csh / s_psh
    stage.add(s_cur, RRT); stage.add(s_prev, RRT); stage.add(s_csh, RST); stage.add(s_psh, RST);
    stage.add(s_flags, PT); stage.add(s_pw, PT); stage.add(s_rank, PT); stage.add(s_inst, PT);
    stage.add(s.rm, NUT); stage.add(s.ad, NUT); stage.add(s.nw, NT); stage.add(s.ef, NT); stage.add(s.er, NT);
    stage.add(s.hw, NT); stage.add(s.mask, MT);
    const size_t stage_bytes = stage.bytes();
    if (stage_bytes > ctx->h_stage_bytes) {          // grow-only, kept by the context between calls
      if (ctx->h_stage) cudaFreeHost(ctx->h_stage);
      ctx->h_stage = nullptr; ctx->h_stage_bytes = 0;
      const cudaError_t e = cudaMallocHost(&ctx->h_stage, stage_bytes + stage_bytes / 4);
      if (e != cudaSuccess)
        throw_err(BLANCE_ERR_NOMEM, std::string("cudaMallocHost of the staging buffer failed: ") + cudaGetErrorString(e));
      ctx->h_stage_bytes = stage_bytes + stage_bytes / 4;
    }
    stage.carve(ctx->h_stage);
    pl->h_rows = s_cur; pl->h_shape = s_csh; pl->h_warn = s_psh;
    auto stage_one = [&](int i) {
      const blance_plan_in& in = ins[i];
      const DInst& D = pl->h_insts[i];
      const size_t rr = (size_t)D.PU * D.SL, rs = (size_t)D.PU * D.S;
      if (rr) { std::memcpy(s_cur + pl->raw_rows_off[i], in.cur_rows, sizeof(int32_t) * rr);
                std::memcpy(s_prev + pl->raw_rows_off[i], in.prev_rows, sizeof(int32_t) * rr); }
      if (rs) { std::memcpy(s_csh + pl->raw_shape_off[i], in.cur_shape, rs); std::memcpy(s_psh + pl->raw_shape_off[i], in.prev_shape, rs); }
      for (int p = 0; p < D.PU; ++p) {
        const size_t g = (size_t)D.part_off + p;
        s_flags[g] = part_flags(in, p);
        s_pw[g] = in.part_weight[p];
        s_rank[g] = in.part_name_rank[p];
        s_inst[g] = i;
      }
      stage_nodes(in, D, s, coded);
    };
    // instances are staged by a few host threads (a 1 024-instance fan-out is ~1 M partitions of flag packing)
    int T = (int)std::min<long long>(8, std::max<long long>(1, pl->PT / 65536));
    T = std::min(T, std::max(1, (int)std::thread::hardware_concurrency()));
    if (T <= 1) { for (int i = 0; i < n; ++i) stage_one(i); }
    else {
      std::vector<std::thread> th;
      for (int t = 0; t < T; ++t) th.emplace_back([&, t]() { for (int i = t; i < n; i += T) stage_one(i); });
      for (auto& x : th) x.join();
    }
    h_cur = s_cur; h_prev = s_prev; h_csh = s_csh; h_psh = s_psh; h_flags = s_flags; h_pw = s_pw; h_rank = s_rank;
    h_inst = s_inst; h_rm = s.rm; h_ad = s.ad; h_nw = s.nw; h_hw = s.hw; h_ef = s.ef; h_er = s.er; h_mask = s.mask;
  }
  cudaStream_t st = ctx->stream;
  auto h2d = [&](const void* dst, const void* src, size_t bytes) {      // a NULL source uploads zeros
    if (bytes > 0)
      cuda_check(src ? cudaMemcpyAsync((void*)dst, src, bytes, cudaMemcpyHostToDevice, st) : cudaMemsetAsync((void*)dst, 0, bytes, st), "H2D copy");
  };
  h2d(pl->raw_a, h_cur, sizeof(int32_t) * (size_t)pl->RRT); h2d(pl->raw_b, h_prev, sizeof(int32_t) * (size_t)pl->RRT);
  h2d(pl->rawsh_a, h_csh, (size_t)pl->RST); h2d(pl->rawsh_b, h_psh, (size_t)pl->RST);
  h2d(pl->pflags_init, h_flags, (size_t)pl->PT); h2d(P.pweight, h_pw, sizeof(int32_t) * (size_t)pl->PT);
  h2d(P.name_rank, h_rank, sizeof(int32_t) * (size_t)pl->PT); h2d(P.part_inst, h_inst, sizeof(int32_t) * (size_t)pl->PT);
  h2d(P.node_removed, h_rm, (size_t)pl->NUT); h2d(P.node_added, h_ad, (size_t)pl->NUT);
  h2d(P.node_weight, h_nw, sizeof(int32_t) * (size_t)pl->NT); h2d(P.node_has_weight, h_hw, (size_t)pl->NT);
  h2d(P.extra_first, h_ef, sizeof(int32_t) * (size_t)pl->NT); h2d(P.extra_rest, h_er, sizeof(int32_t) * (size_t)pl->NT);
  h2d(P.ie_mask, h_mask, sizeof(uint32_t) * (size_t)pl->MT);
  h2d(P.insts, pl->h_insts.data(), sizeof(DInst) * (size_t)n);
  h2d(pl->d_raw_rows_off, pl->raw_rows_off.data(), sizeof(long long) * (size_t)(n + 1));
  h2d(pl->d_raw_shape_off, pl->raw_shape_off.data(), sizeof(long long) * (size_t)(n + 1));
  h2d(pl->d_seg_off, seg_off.data(), sizeof(int) * (size_t)(n + 1));
  // device layout of the rows / shapes, into the *_init copies via the working arrays
  if (pl->PT > 0) {
    launch(ctx, k_unpack, grid_for(ctx, pl->PT, 256), 256, 0, P, pl->raw_a, pl->raw_b, pl->rawsh_a, pl->rawsh_b,
           pl->d_raw_rows_off, pl->d_raw_shape_off, pl->PT);
    CUDA(cudaMemcpyAsync(pl->rows_init, P.rows, sizeof(int32_t) * (size_t)pl->RT, cudaMemcpyDeviceToDevice, st));
    CUDA(cudaMemcpyAsync(pl->prev_rows_init, P.prev_rows, sizeof(int32_t) * (size_t)pl->RT, cudaMemcpyDeviceToDevice, st));
    CUDA(cudaMemcpyAsync(pl->pmeta_init, P.pmeta, sizeof(uint32_t) * (size_t)pl->PT, cudaMemcpyDeviceToDevice, st));
    CUDA(cudaMemcpyAsync(pl->prev_meta_init, P.prev_meta, sizeof(uint32_t) * (size_t)pl->PT, cudaMemcpyDeviceToDevice, st));
  }
  finish_upload(ctx, pl.get());
  return pl;
}

static cudaEvent_t get_event(blance_ctx* ctx, size_t idx) {
  while (ctx->events.size() <= idx) {
    cudaEvent_t ev;
    if (cudaEventCreate(&ev) != cudaSuccess) return nullptr;
    ctx->events.push_back(ev);
  }
  return ctx->events[idx];
}

// Calls f(std::integral_constant<int, NPT>()) for the pass kernel's nodes per thread npt (1, 2, 4, 8 or 16).
template <class F>
static void dispatch_npt(int npt, F&& f) {
  switch (npt) {
    case 1: f(std::integral_constant<int, 1>()); break;
    case 2: f(std::integral_constant<int, 2>()); break;
    case 4: f(std::integral_constant<int, 4>()); break;
    case 8: f(std::integral_constant<int, 8>()); break;
    default: f(std::integral_constant<int, 16>()); break;
  }
}

// Calls f(std::integral_constant<int, K>()) for K = 1 .. 4 in ascending order where bit K of kmask is set: the
// sequencer and speculative kernels have one instantiation per constraint count K.  CTAs whose instance picked
// another kernel (or has a different K for this state) exit at once.
template <class F>
static void for_each_k(unsigned kmask, F&& f) {
  if (kmask & 2u) f(std::integral_constant<int, 1>());
  if (kmask & 4u) f(std::integral_constant<int, 2>());
  if (kmask & 8u) f(std::integral_constant<int, 3>());
  if (kmask & 16u) f(std::integral_constant<int, 4>());
}

static int next_pow2(int v) { int p = 1; while (p < v) p <<= 1; return p; }

// Compute threads per CTA (TC, a power of two; the kernel adds one service warp) and nodes per
// thread for the pass kernel.  The chain is latency bound, so prefer many warps with few nodes each.
static void pass_shape(int max_n, int* TC, int* npt) {
  int want = max_n > 512 ? 2 : 1;
  if (max_n > 3968) want = 8;
  int t = next_pow2((std::max(1, max_n) + want - 1) / want);
  if (t < 32) t = 32;
  if (t > 512) t = 512;
  int n = (max_n + t - 1) / t;
  *npt = n <= 1 ? 1 : n <= 2 ? 2 : n <= 4 ? 4 : n <= 8 ? 8 : 16;
  *TC = t;
}

static void run(blance_ctx* ctx, blance_plan* pl) {
  cudaStream_t st = ctx->stream;
  DPool& P = pl->pool;
  const int n = pl->n_inst;
  // restore the mutable state
  if (pl->PT > 0) {
    CUDA(cudaMemcpyAsync(P.rows, pl->rows_init, sizeof(int32_t) * (size_t)pl->RT, cudaMemcpyDeviceToDevice, st));
    CUDA(cudaMemcpyAsync(P.prev_rows, pl->prev_rows_init, sizeof(int32_t) * (size_t)pl->RT, cudaMemcpyDeviceToDevice, st));
    CUDA(cudaMemcpyAsync(P.pmeta, pl->pmeta_init, sizeof(uint32_t) * (size_t)pl->PT, cudaMemcpyDeviceToDevice, st));
    CUDA(cudaMemcpyAsync(P.prev_meta, pl->prev_meta_init, sizeof(uint32_t) * (size_t)pl->PT, cudaMemcpyDeviceToDevice, st));
    CUDA(cudaMemcpyAsync(P.pflags, pl->pflags_init, (size_t)pl->PT, cudaMemcpyDeviceToDevice, st));
  }
  CUDA(cudaMemcpyAsync(P.insts, pl->h_insts.data(), sizeof(DInst) * (size_t)n, cudaMemcpyHostToDevice, st));
  CUDA(cudaEventRecord(ctx->ev[1], st));

  int T = 32, npt = 1;
  pass_shape(pl->max_N, &T, &npt);
  bool any_hier = false;
  for (int i = 0; i < n; ++i) any_hier |= pl->h_insts[i].has_hier_rules != 0;
  int any_active = 0;
  for (int i = 0; i < n; ++i) any_active += pl->h_insts[i].active;
  const int blk = 256;
  const int grid = grid_for(ctx, pl->PT, blk);
  size_t n_ev = 0;
  pl->pass_launches = 0;
  const size_t hist_smem = (size_t)pl->h_insts[0].S * pl->h_insts[0].N * sizeof(int32_t);
  const bool smem_hist = (n == 1) && hist_smem <= 40 * 1024;
  int guard = 0;
  while (any_active > 0) {
    if (++guard > 100000) throw_err(BLANCE_ERR_CUDA, "convergence loop did not terminate");
    if (pl->PT == 0) {          // no partitions at all: the loop of plan.go:32-45 still runs once and matches
      CUDA(cudaMemsetAsync(ctx->d_any_active, 0, sizeof(int), st));
      launch(ctx, k_next_iter, (n + 127) / 128, 128, 0, P, n, ctx->d_any_active);
      break;
    }
    launch(ctx, k_prepare_rows, grid, blk, 0, P, pl->PT);
    CUDA(cudaMemsetAsync(P.counts, 0, sizeof(int32_t) * (size_t)(pl->CT + 1), st));
    if (smem_hist) launch(ctx, k_count_prev<true>, std::min(grid, ctx->sm_count * 2), blk, hist_smem, P, pl->PT);
    else launch(ctx, k_count_prev<false>, grid, blk, 0, P, pl->PT);
    for (int s = 0; s < pl->max_S; ++s) {
      if (!pl->any_state_active[s]) continue;
      launch(ctx, k_build_keys, grid, blk, 0, P, s, pl->PT);
      size_t tmp = ctx->cub_tmp_bytes;
      if (n == 1)
        CUDA(cub::DeviceRadixSort::SortPairs(ctx->cub_tmp, tmp, P.keys_alt, P.keys, P.order_alt, P.order, (int)pl->PT, 0, 64, st));
      else
        CUDA(cub::DeviceSegmentedRadixSort::SortPairs(ctx->cub_tmp, tmp, P.keys_alt, P.keys, P.order_alt, P.order, (int)pl->PT,
                                                      n, pl->d_seg_off, pl->d_seg_off + 1, 0, 64, st));
      launch(ctx, k_gather_stream, grid, blk, 0, P, s, pl->PT);
      unsigned kmask = 0;
      for (int i = 0; i < n; ++i) { const int kk = pl->h_insts[i].S > s ? pl->h_insts[i].state_constraints[s] : 0; if (kk >= 1 && kk <= 4) kmask |= 1u << kk; }
      // speculative kernel: warp 0 leads, 9 scout warps (warps 4 and 8 exit at once: the leader has its scheduler to
      // itself) when the GPU has SMs to spare; leader + 3 scouts per CTA for wide batches
      const bool spec_wide = 2 * n <= ctx->sm_count;
      const int spec_nw = spec_wide ? 12 : 4, spec_sw = spec_wide ? 9 : 3;
      const unsigned spec_idle = spec_wide ? ((1u << 4) | (1u << 8)) : 0u;
      const int spec_shift = 0;
      const int spec_max_n = std::min(2048, 32 * spec_sw * SP_NPTS);
      bool any_auto = false;
      for (int i = 0; i < n; ++i) any_auto |= pl->h_insts[i].engine == BLANCE_ENGINE_AUTO;
      const bool spec_allowed = any_auto && kmask != 0 && pl->pair_end_bit <= 62 && !getenv("BLANCE_NO_SPEC");
      launch(ctx, k_pick_mode, (n + 127) / 128, 128, 0, P, s, n, (npt <= 8 && !getenv("BLANCE_NO_SEQ")) ? 1 : 0,
             spec_allowed ? 1 : 0, spec_max_n);
      if (spec_allowed) {
        // the all-sticky hypothesis counts (qstat) of the instances that picked the speculative kernel
        launch(ctx, k_pair_keys, grid, blk, 0, P, s, pl->PT, pl->pair_inst_shift);
        size_t tmp2 = ctx->cub_tmp_bytes;
        CUDA(cub::DeviceRadixSort::SortPairs(ctx->cub_tmp, tmp2, P.pair_keys_alt, P.pair_keys, P.pair_vals_alt, P.pair_vals,
                                             (int)(4 * pl->PT), 0, pl->pair_end_bit + 1, st));
        launch(ctx, k_pair_rank, grid_for(ctx, 4 * pl->PT, blk), blk, 0, P, 4 * pl->PT);
        CUDA(cudaMemsetAsync(P.n2n_dev, 0, sizeof(int32_t) * (size_t)(pl->N2T + 1), st));
      }
      CUDA(cudaMemsetAsync(P.n2n, 0, sizeof(int32_t) * (size_t)(pl->N2T + 1), st));     // plan.go:266
      cudaEvent_t e0 = get_event(ctx, n_ev), e1 = get_event(ctx, n_ev + 1);
      if (e0 && e1 && n_ev < 256) CUDA(cudaEventRecord(e0, st));
      // sequencer warps per CTA: wide windows when the GPU has SMs to spare, one warp for wide batches
      const int seq_w = (2 * n <= ctx->sm_count) ? SEQ_W_MAX : 1;
      dispatch_npt(npt, [&](auto npt_c) {
        constexpr int NPT = decltype(npt_c)::value;
        launch(ctx, any_hier ? k_assign_pass<NPT, true, 544> : k_assign_pass<NPT, false, 544>, n, T + 32, 0, P, s);
        if constexpr (NPT <= 8) {
          const size_t dyn = seq_dyn_smem_bytes(pl->max_N, seq_w);
          for_each_k(kmask, [&](auto k_c) {
            constexpr int K = decltype(k_c)::value;
            opt_in_smem((const void*)k_assign_pass_seq<NPT, K, 640>, &g_seq_dyn[ctx->device & 63][__builtin_ctz(NPT)][K - 1], dyn);
            launch(ctx, k_assign_pass_seq<NPT, K, 640>, n, T + 32 * seq_w, dyn, P, s, T);
          });
        }
      });
      if (spec_allowed) {
        const size_t sdyn = spec_dyn_smem_bytes(std::min(pl->max_N, spec_max_n), spec_sw);
        for_each_k(kmask, [&](auto k_c) {
          constexpr int K = decltype(k_c)::value;
          opt_in_smem((const void*)k_assign_pass_spec<K>, &g_spec_dyn[ctx->device & 63][K - 1], sdyn);
          launch(ctx, k_assign_pass_spec<K>, n, 32 * spec_nw, sdyn, P, s, spec_sw, spec_idle, spec_shift);
        });
      }
      if (e0 && e1 && n_ev < 256) { CUDA(cudaEventRecord(e1, st)); n_ev += 2; }
      pl->pass_launches++;
      launch(ctx, k_scatter_stream, grid, blk, 0, P, s, pl->PT);
    }
    launch(ctx, k_compare, grid, blk, 0, P, pl->PT);
    launch(ctx, k_commit, grid, blk, 0, P, pl->PT);
    CUDA(cudaMemsetAsync(ctx->d_any_active, 0, sizeof(int), st));
    launch(ctx, k_next_iter, (n + 127) / 128, 128, 0, P, n, ctx->d_any_active);
    CUDA(cudaMemcpyAsync(ctx->h_any_active, ctx->d_any_active, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA(cudaStreamSynchronize(st));
    CUDA(cudaGetLastError());
    any_active = *ctx->h_any_active;
  }
  CUDA(cudaEventRecord(ctx->ev[2], st));
  CUDA(cudaStreamSynchronize(st));
  float ms = 0.f;
  CUDA(cudaEventElapsedTime(&ms, ctx->ev[1], ctx->ev[2]));
  pl->last_kernel_ms = ms;
  float pass = 0.f;
  const bool show = getenv("BLANCE_PASS_TIMES") != nullptr;
  for (size_t i = 0; i + 1 < n_ev; i += 2) {
    float t = 0.f;
    if (cudaEventElapsedTime(&t, ctx->events[i], ctx->events[i + 1]) == cudaSuccess) pass += t;
    if (show) std::fprintf(stderr, "[blance] assign pass %zu: %.3f ms\n", i / 2, t);
  }
  pl->last_pass_ms = pass;
}

static void fetch(blance_ctx* ctx, blance_plan* pl, blance_plan_out* outs) {
  cudaStream_t st = ctx->stream;
  const int n = pl->n_inst;
  if (pl->PT > 0)
    launch(ctx, k_pack, grid_for(ctx, pl->PT, 256), 256, 0, pl->pool, pl->raw_a, pl->rawsh_a, pl->rawsh_b, pl->d_raw_rows_off,
           pl->d_raw_shape_off, pl->PT);
  const bool dir = direct(pl);
  int32_t* h_rows = dir ? outs[0].next_rows : pl->h_rows;
  uint8_t* h_shape = dir ? outs[0].next_shape : pl->h_shape;
  uint8_t* h_warn = dir ? outs[0].warn : pl->h_warn;
  if (pl->RRT && h_rows) CUDA(cudaMemcpyAsync(h_rows, pl->raw_a, sizeof(int32_t) * (size_t)pl->RRT, cudaMemcpyDeviceToHost, st));
  if (pl->RST && h_shape) CUDA(cudaMemcpyAsync(h_shape, pl->rawsh_a, (size_t)pl->RST, cudaMemcpyDeviceToHost, st));
  if (pl->RST && h_warn) CUDA(cudaMemcpyAsync(h_warn, pl->rawsh_b, (size_t)pl->RST, cudaMemcpyDeviceToHost, st));
  std::vector<DInst> fin(n);
  CUDA(cudaMemcpyAsync(fin.data(), pl->pool.insts, sizeof(DInst) * (size_t)n, cudaMemcpyDeviceToHost, st));
  CUDA(cudaStreamSynchronize(st));
  for (int i = 0; i < n; ++i)
    if (fin[i].spec_abort) throw_err(BLANCE_ERR_CUDA, "the speculative pass kernel gave up waiting (internal error; see stderr of the device printf)");
  if (getenv("BLANCE_SPEC_STATS"))
    for (int i = 0; i < n && i < 4; ++i)
      std::fprintf(stderr, "[blance] inst %d: steps %lld accepted %lld | resolved by the leader %lld (stale results %lld) movers %lld team %lld rebuilds %lld waits %lld\n",
                   i, fin[i].steps, fin[i].fast_steps, fin[i].spec_resolved, fin[i].spec_stale, fin[i].spec_movers, fin[i].spec_team,
                   fin[i].spec_rebuilds, fin[i].spec_waits),
      std::fprintf(stderr, "[blance]   leader cycles (-DBLANCE_SPEC_TIMING builds): scans %lld | waits %lld | resolve loads+keys %lld | resolve picks %lld"
                           " | mover mirror %lld | mover list+publish %lld | team %lld | passes total %lld\n",
                   fin[i].spec_cyc[0], fin[i].spec_cyc[1], fin[i].spec_cyc[2], fin[i].spec_cyc[3], fin[i].spec_cyc[4], fin[i].spec_cyc[5],
                   fin[i].spec_cyc[6], fin[i].spec_cyc[7]),
      std::fprintf(stderr, "[blance]   of the resolve loads+keys: waiting for n2n %lld | resolves whose step the previous ballot named next %lld\n",
                   fin[i].spec_cyc_n2n, fin[i].spec_pf_opp),
      std::fprintf(stderr, "[blance]   team: full after a failed proof %lld (%lld cycles) | full, other rows %lld (%lld cycles) | rebuild, list dry %lld"
                           " (%lld cycles) | full that moved %lld (%lld cycles) | extended resolves %lld, too large %lld (%lld cycles)\n",
                   fin[i].spec_path[0], fin[i].spec_cyc_team[0], fin[i].spec_path[1], fin[i].spec_cyc_team[1], fin[i].spec_path[2],
                   fin[i].spec_cyc_team[2], fin[i].spec_path[3], fin[i].spec_cyc_team[3], fin[i].spec_path[4], fin[i].spec_path[5],
                   fin[i].spec_cyc_x);
  for (int i = 0; i < n; ++i) {
    const DInst& D = pl->h_insts[i];
    blance_plan_out& o = outs[i];
    const size_t rr = (size_t)D.PU * D.SL, rs = (size_t)D.PU * D.S;
    if (!dir) {
      if (rr && o.next_rows) std::memcpy(o.next_rows, h_rows + pl->raw_rows_off[i], sizeof(int32_t) * rr);
      if (rs && o.next_shape) std::memcpy(o.next_shape, h_shape + pl->raw_shape_off[i], rs);
      if (rs && o.warn) std::memcpy(o.warn, h_warn + pl->raw_shape_off[i], rs);
    }
    o.iters_run = fin[i].iters_run;
    o.converged = fin[i].converged;
    o.steps = fin[i].steps;
    o.sticky_steps = fin[i].fast_steps;
    o.kernel_ms = pl->last_kernel_ms;
    o.pass_ms = pl->last_pass_ms;
    o.device_ms = 0.f;
  }
}

extern "C" int blance_plan_upload(blance_ctx* ctx, const blance_plan_in* in, blance_plan** plan) {
  return entry(ctx, [&](Device& device) {
    if (!ctx) throw_err(BLANCE_ERR_INVALID_ARG, "ctx is NULL");
    if (!plan) throw_err(BLANCE_ERR_INVALID_ARG, "plan is NULL");
    *plan = nullptr;
    *plan = upload(device(), 1, in).release();
  });
}

extern "C" int blance_plan_run(blance_ctx* ctx, blance_plan* plan) {
  return entry(ctx, [&](Device& device) {
    if (!ctx || !plan) throw_err(BLANCE_ERR_INVALID_ARG, "ctx or plan is NULL");
    run(device(), plan);
  });
}

extern "C" int blance_plan_fetch(blance_ctx* ctx, blance_plan* plan, blance_plan_out* out) {
  return entry(ctx, [&](Device& device) {
    if (!ctx || !plan || !out) throw_err(BLANCE_ERR_INVALID_ARG, "ctx, plan or out is NULL");
    fetch(device(), plan, out);
  });
}

extern "C" int blance_plan_timing(const blance_plan* plan, float* kernel_ms, float* pass_ms, int32_t* pass_launches) {
  if (!plan) return BLANCE_ERR_INVALID_ARG;
  if (kernel_ms) *kernel_ms = plan->last_kernel_ms;
  if (pass_ms) *pass_ms = plan->last_pass_ms;
  if (pass_launches) *pass_launches = plan->pass_launches;
  return BLANCE_OK;
}

extern "C" void blance_plan_free(blance_ctx* ctx, blance_plan* plan) {
  PlanPtr owner(plan);               // freed on the stream it was allocated on, also when ctx is NULL
  if (ctx && plan) entry(ctx, [&](Device& device) { CUDA(cudaStreamSynchronize(device()->stream)); owner.reset(); });
}

static void plan_on_device(blance_ctx* ctx, int n, const blance_plan_in* in, blance_plan_out* out) {
  CUDA(cudaEventRecord(ctx->ev[0], ctx->stream));
  PlanPtr pl = upload(ctx, n, in);
  run(ctx, pl.get());
  fetch(ctx, pl.get(), out);
  cudaEventRecord(ctx->ev[3], ctx->stream);
  cudaEventSynchronize(ctx->ev[3]);
  float ms = 0.f;
  cudaEventElapsedTime(&ms, ctx->ev[0], ctx->ev[3]);
  for (int i = 0; i < n; ++i) out[i].device_ms = ms;
}

// Several GPUs: instance i -> device i mod G, one host thread per device, no collective.
static void plan_batch(blance_ctx* ctx, int32_t n, const blance_plan_in* in, blance_plan_out* out) {
  if (!ctx) throw_err(BLANCE_ERR_INVALID_ARG, "ctx is NULL");
  if (!in || !out) throw_err(BLANCE_ERR_INVALID_ARG, "in or out is NULL");
  if (n <= 0) throw_err(BLANCE_ERR_INVALID_ARG, "batch size must be positive");
  const int G = (int)std::min<size_t>(std::max<size_t>(1, blance_ctx_device_count(ctx)), (size_t)n);
  if (G == 1) return fan_out(ctx, 1, [&](int, blance_ctx* dev) { plan_on_device(dev, n, in, out); });
  std::vector<std::vector<blance_plan_in>> ins((size_t)G);
  std::vector<std::vector<blance_plan_out>> outs((size_t)G);
  for (int i = 0; i < n; ++i) { ins[(size_t)(i % G)].push_back(in[i]); outs[(size_t)(i % G)].push_back(out[i]); }
  fan_out(ctx, G, [&](int d, blance_ctx* dev) {
    plan_on_device(dev, (int)ins[(size_t)d].size(), ins[(size_t)d].data(), outs[(size_t)d].data());
  });
  for (int i = 0; i < n; ++i) out[i] = outs[(size_t)(i % G)][(size_t)(i / G)];
}

extern "C" int blance_plan_next_map(blance_ctx* ctx, const blance_plan_in* in, blance_plan_out* out) {
  return entry(ctx, [&](Device&) { plan_batch(ctx, 1, in, out); });
}

extern "C" int blance_plan_next_map_batch(blance_ctx* ctx, int32_t n, const blance_plan_in* in, blance_plan_out* out) {
  return entry(ctx, [&](Device&) { plan_batch(ctx, n, in, out); });
}

// ---------------------------------------------------------------------------------------
// What-if scenarios of one cluster (blance_plan_scenarios): the base is uploaded once per device, each wave of
// scenarios is a batch whose partition slices are replicated from it on the device.

// The substituted instance of one scenario.  The partition weights of its overrides are not in it: they are
// applied on the device (k_scenario_weights) after the base is replicated.
static blance_plan_in scenario_in(const blance_plan_in& base, const blance_scenario& sc, const blance_scenario_opts* o) {
  blance_plan_in in = base;
  in.node_removed = sc.node_removed; in.node_added = sc.node_added; in.add_is_nil = sc.add_is_nil;
  in.has_node_weights = sc.has_node_weights; in.node_weight = sc.node_weight; in.node_has_weight = sc.node_has_weight;
  if (!o) return in;
  if (o->set & BLANCE_OPT_CONSTRAINTS) in.state_constraints = o->state_constraints;
  if (o->set & BLANCE_OPT_STICKINESS) { in.state_stickiness = o->state_stickiness; in.state_has_stickiness = o->state_has_stickiness; }
  if (o->set & BLANCE_OPT_PART_WEIGHTS) {
    in.has_part_weights = o->has_part_weights;
    if (o->extra_tot_first) in.extra_tot_first = o->extra_tot_first;
    if (o->extra_tot_rest) in.extra_tot_rest = o->extra_tot_rest;
  }
  if (o->set & BLANCE_OPT_HIERARCHY) {
    in.has_hier_rules = o->has_hier_rules; in.n_rules = o->n_rules; in.n_hier_bits = o->n_hier_bits;
    in.rule_off = o->rule_off; in.ie_mask = o->ie_mask;
  }
  return in;
}

static const blance_scenario_opts* opts_of(const blance_scenario_opts* opts, int i) { return opts ? &opts[i] : nullptr; }

static int n_overrides(const blance_scenario_opts* o) {
  return o && (o->set & BLANCE_OPT_PART_WEIGHTS) ? o->n_weight_overrides : 0;
}

// The option checks of one scenario that check_structure cannot make (flags, override lists, the "%10d" rule).
static int check_opts(const blance_plan_in& base, const blance_scenario_opts& o, std::string& why) {
  auto bad = [&](const std::string& what, int st = BLANCE_ERR_INVALID_ARG) { why = what; return st; };
  const uint32_t all = BLANCE_OPT_CONSTRAINTS | BLANCE_OPT_STICKINESS | BLANCE_OPT_PART_WEIGHTS | BLANCE_OPT_HIERARCHY;
  if (o.set & ~all) return bad("opts.set has an unknown bit");
  if ((o.set & BLANCE_OPT_STICKINESS) && o.state_has_stickiness)
    for (int s = 0; s < base.n_states; ++s)
      if (o.state_has_stickiness[s] > 1) return bad("state_has_stickiness is neither 0 nor 1");
  if ((o.set & BLANCE_OPT_HIERARCHY) && o.has_hier_rules != 0 && o.has_hier_rules != 1) return bad("has_hier_rules is neither 0 nor 1");
  if (!(o.set & BLANCE_OPT_PART_WEIGHTS)) return BLANCE_OK;
  if (o.has_part_weights != 0 && o.has_part_weights != 1) return bad("has_part_weights is neither 0 nor 1");
  const int k = o.n_weight_overrides;
  if (k < 0) return bad("n_weight_overrides is negative");
  if (k > 0 && (!o.ow_part || !o.ow_weight || !o.ow_has)) return bad("weight override arrays are NULL");
  std::vector<int32_t> seen(o.ow_part, o.ow_part + k);
  std::sort(seen.begin(), seen.end());
  if (k > 0 && (seen.front() < 0 || seen.back() >= base.n_parts)) return bad("a weight override's partition is outside [0, n_parts)");
  if (std::adjacent_find(seen.begin(), seen.end()) != seen.end()) return bad("a partition has two weight overrides");
  for (int j = 0; j < k; ++j) {
    if (o.ow_has[j] > 1) return bad("ow_has is neither 0 nor 1");
    if (o.ow_has[j] && o.ow_weight[j] > 999999999)      // the "%10d" rule of plan.go:539, as blance_plan_in_check
      return bad("partition weight above 999999999 in override " + std::to_string(j), BLANCE_ERR_UNSUPPORTED);
  }
  return BLANCE_OK;
}

// The count bound (count_bound.hpp) of one scenario's substituted instance `in`, with its weight overrides applied.
// base_sum: sum over the base's partitions of |weight| as if PartitionWeights != nil (1 where it has none), computed
// once by the caller (< 0: not yet).
static int check_counts(const blance_plan_in& base, const blance_plan_in& in, const blance_scenario_opts* o, long long& base_sum,
                        std::string& why) {
  long long sum = in.n_parts;
  if (in.has_part_weights) {
    if (base_sum < 0) {
      blance_plan_in weighted = base;
      weighted.has_part_weights = 1;
      base_sum = count_bound_weight_sum(weighted);
    }
    sum = base_sum;
    for (int j = 0; j < n_overrides(o); ++j) {
      const int32_t p = o->ow_part[j];
      sum += (o->ow_has[j] ? std::llabs((long long)o->ow_weight[j]) : 1) - (base.part_has_weight[p] ? std::llabs((long long)base.part_weight[p]) : 1);
    }
  }
  if (count_bound_fits(sum, in.n_slots, count_bound_max_extra(in.n_nodes, in.extra_tot_first, in.extra_tot_rest))) return BLANCE_OK;
  why = BLANCE_COUNT_BOUND_MSG;
  return BLANCE_ERR_UNSUPPORTED;
}

// uint32 words of one instance's hierarchy masks
static long long mask_words(const blance_plan_in& in) {
  return in.has_hier_rules ? (long long)in.n_rules * (in.n_node_ids + 1) * ((in.n_hier_bits + 31) / 32) : 0;
}

// int64 words of one scenario's summary: node_ops [NU][4] | state_node_load [S][NU] | 3 scalars
static long long summary_stride(const blance_plan_in& base) {
  return 4ll * base.n_node_ids + (long long)base.n_states * base.n_node_ids + 3;
}

// The schedules requested with blance_plan_scenarios_schedule: nc counts (>= 1), the movers ([n_node_ids]) and the
// caller's outputs [n][nc].
struct SchedReq {
  int nc = 0;
  std::vector<int32_t> count;
  std::vector<uint8_t> mover;
  blance_scenario_schedule_out* out = nullptr;
};

// At most 2 x n_slots ops per partition of a scenario: the bound its schedule state is sized by before planning.
static int scenario_ops(const blance_plan_in& base) { return std::max(1, 2 * base.n_slots); }

// The schedule state of nw scenarios x nc counts over PU partitions and NU node ids (wave_schedule.cuh), with room for
// `entries` list entries per instance and PU arrivals per instance.  MO > 0 adds the op table of MO ops per
// partition; MO = 0 leaves the ops to the caller (a moves handle's CSR arrays).  Adds its slices to `a`, the sorts'
// scratch (`tmp`, tmp_bytes) last, and sets W's sizes.
static void sched_slices(Arena& a, int nw, int nc, long long PU, long long NU, int MO, long long entries, WSched& w,
                         void*& tmp, size_t& tmp_bytes, cudaStream_t st) {
  const long long ni = (long long)nw * nc, nseg = ni * NU, cap = ni * entries, nkeys = std::max(1ll, ni * PU);
  size_t sort_tmp = 0, scan_tmp = 0, red_tmp = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, sort_tmp, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)nkeys, 0, 64, st);
  cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, (const int32_t*)nullptr, (long long*)nullptr, (int)(nseg + 1), st);
  cub::DeviceReduce::Sum(nullptr, red_tmp, (const int32_t*)nullptr, (long long*)nullptr, (int)(nseg + 1), st);
  tmp_bytes = std::max(sort_tmp, std::max(scan_tmp, red_tmp)) + 256;
  a.add(w.count, (size_t)nc); a.add(w.mover, (size_t)std::max(1ll, NU));
  if (MO > 0) { a.add(w.op_n, (size_t)(nw * PU)); a.add(w.op_node, (size_t)(nw * PU * MO)); a.add(w.op_kind, (size_t)(nw * PU * MO)); }
  a.add(w.cur, (size_t)(ni * PU)); a.add(w.part_done, (size_t)(ni * PU));
  a.add(w.seg_off, (size_t)(nseg + 1)); a.add(w.len, (size_t)(nseg + 1));
  a.add(w.kcnt, (size_t)(nseg + 1)); a.add(w.poff, (size_t)(nseg + 1));
  a.add(w.astart, (size_t)nseg); a.add(w.aend, (size_t)nseg);
  a.add(w.node_rounds, (size_t)nseg); a.add(w.node_last, (size_t)nseg);
  a.add(w.buf0, (size_t)cap); a.add(w.buf1, (size_t)cap); a.add(w.scratch, (size_t)cap);
  a.add(w.keys_in, (size_t)nkeys); a.add(w.keys_out, (size_t)nkeys);
  a.add(w.scal, (size_t)(4 * ni)); a.add(w.overflow, 1);
  a.add(w.esum, 1); a.add(tmp, tmp_bytes);
  w.nw = nw; w.nc = nc; w.PU = (int32_t)PU; w.NU = (int32_t)NU; w.MO = (int32_t)MO; w.nseg = nseg;
  w.PB = 1;
  while (w.PB < WAVE_PART_BITS && (1ll << w.PB) < PU) ++w.PB;
}

// The wave size of `n_dev` scenarios on one device (0 = one scenario does not fit).  Scenarios differ only in
// their hierarchy masks and weight overrides, so one is priced as in0 with the largest mask and override list of any.
static int wave_size(blance_ctx* ctx, const blance_plan_in& in0, long long max_mask_words, int max_overrides, int n_dev,
                     int max_concurrent, const SchedReq* sr, size_t extra_bytes, size_t* per_scenario) {
  blance_plan probe;
  std::vector<int> seg;
  layout(&probe, 1, &in0, seg);
  Arena one;
  plan_slices(one, &probe, 1);
  size_t per = one.bytes() + sort_scratch_bytes(probe.PT, 1, ctx->stream) +
               sizeof(long long) * (size_t)summary_stride(in0) +
               sizeof(uint32_t) * (size_t)(max_mask_words - mask_words(in0)) + 3 * sizeof(int32_t) * (size_t)max_overrides +
               extra_bytes;
  if (sr) {
    Arena sched;
    WSched w{};
    void* tmp = nullptr;
    size_t tb = 0;
    sched_slices(sched, 1, sr->nc, in0.n_parts, in0.n_node_ids, scenario_ops(in0), (long long)in0.n_parts * scenario_ops(in0), w, tmp, tb,
                 ctx->stream);
    per += sched.bytes();
  }
  *per_scenario = per;
  if (sr)            // the first round's arrival slots (nc x n_parts per scenario) are int32 positions
    n_dev = (int)std::min<long long>(n_dev, std::max(1ll, (long long)INT32_MAX / ((long long)sr->nc * std::max(1, in0.n_parts))));
  if (max_concurrent > 0) return std::min(n_dev, max_concurrent);
  size_t free_b = 0, total_b = 0;
  if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) { cudaGetLastError(); return 1; }
  const size_t headroom = std::max<size_t>(1ull << 30, total_b / 16);     // the device is shared: leave room
  const long long fit = free_b > headroom ? (long long)((free_b - headroom) / std::max<size_t>(per, 1)) : 0;
  int w = (int)std::min<long long>(n_dev, fit);
  // above the 3-scout speculative kernel's node limit a wide batch would drop to lock-step (run(): 2n <= sm_count)
  if (in0.n_nodes > std::min(2048, 32 * 3 * SP_NPTS)) w = std::min(w, std::max(1, ctx->sm_count / 2));
  return w;
}

// grid of a kernel striding over the PU partitions of each of nw scenarios (blockIdx.y = scenario)
static dim3 wave_grid(const blance_ctx* ctx, int PU, int nw) {
  return dim3((unsigned)std::max(1, std::min((PU + 255) / 256, std::max(1, ctx->sm_count * 8 / nw))), (unsigned)nw);
}

// The schedules of nw scenarios x sr.nc counts on W (wave_schedule.cuh), its ops in place: ops[j * NU + q] = the
// ops of scenario j on node q carve the segments.  Rounds are enqueued in blocks of kWaveBlock; after each block the
// host reads the entries left and sizes the next block's sorts by min(picks bound, entries).  Returns the
// instances' scalars [ni][4]: rounds, moves_done, stuck_parts, max_batch.
static const int kWaveBlock = 64;

static std::vector<unsigned long long> wave_schedule(blance_ctx* ctx, const char* name, const SchedReq& sr, const WSched& W,
                                                     void* tmp, size_t tmp_bytes, const long long* ops) {
  cudaStream_t st = ctx->stream;
  const int nc = sr.nc, NU = W.NU, PU = W.PU;
  const long long ni = (long long)W.nw * nc, nseg = W.nseg;
  // segments: capacity = the node's ops in the scenario (0 without a mover: nothing ever waits there)
  std::vector<long long> seg_off((size_t)nseg + 1, 0);
  long long pick_bound = 0, max_ops = 0;
  for (long long i = 0; i < ni; ++i) {
    const int c = sr.count[(size_t)(i % nc)];
    for (int q = 0; q < NU; ++q) {
      const long long s = i * NU + q;
      const long long capq = sr.mover[(size_t)q] ? ops[(i / nc) * NU + q] : 0;
      seg_off[(size_t)s + 1] = seg_off[(size_t)s] + capq;
      pick_bound += std::min<long long>(c, capq);
    }
    max_ops = std::max(max_ops, seg_off[(size_t)(i + 1) * NU] - seg_off[(size_t)i * NU]);
  }
  const long long nkeys = ni * PU;
  const int end_bit = std::min(64, W.PB + [&] { int b = 1; while ((1ll << b) <= nseg) ++b; return b; }());
  CUDA(cudaMemcpyAsync((void*)W.count, sr.count.data(), sizeof(int32_t) * nc, cudaMemcpyHostToDevice, st));
  CUDA(cudaMemcpyAsync((void*)W.mover, sr.mover.data(), (size_t)NU, cudaMemcpyHostToDevice, st));
  CUDA(cudaMemcpyAsync((void*)W.seg_off, seg_off.data(), sizeof(long long) * seg_off.size(), cudaMemcpyHostToDevice, st));
  CUDA(cudaMemsetAsync(W.len, 0, sizeof(int32_t) * (nseg + 1), st));
  CUDA(cudaMemsetAsync(W.kcnt, 0, sizeof(int32_t) * (nseg + 1), st));
  CUDA(cudaMemsetAsync(W.astart, 0, sizeof(int32_t) * nseg, st));
  CUDA(cudaMemsetAsync(W.aend, 0, sizeof(int32_t) * nseg, st));
  CUDA(cudaMemsetAsync(W.node_rounds, 0, sizeof(int32_t) * nseg, st));
  CUDA(cudaMemsetAsync(W.node_last, 0, sizeof(int32_t) * nseg, st));
  CUDA(cudaMemsetAsync(W.scal, 0, sizeof(unsigned long long) * 4 * ni, st));
  CUDA(cudaMemsetAsync(W.overflow, 0, sizeof(int32_t), st));
  if (W.round_off) CUDA(cudaMemsetAsync(W.round_off, 0, sizeof(long long), st));
  const int seg_grid = grid_for(ctx, (nseg + WAVE_THREADS / 32 - 1) / (WAVE_THREADS / 32) * WAVE_THREADS, WAVE_THREADS);
  auto sort = [&](long long n) {
    size_t tb = tmp_bytes;
    if (n > 0) CUDA(cub::DeviceRadixSort::SortKeys(tmp, tb, W.keys_in, const_cast<unsigned long long*>(W.keys_out), (int)n, 0, end_bit, st));
    launch(ctx, k_wave_bounds, grid_for(ctx, std::max(1ll, n), 256), 256, 0, W, n);
  };
  // the lists: every partition's first op, sorted into its segment
  if (PU > 0) {
    launch(ctx, k_wave_first, wave_grid(ctx, PU, W.nw), 256, 0, W);
    sort(nkeys);
    launch(ctx, k_wave_merge, seg_grid, WAVE_THREADS, 0, W, -1);
  }
  long long E = 0;
  int32_t overflow = 0;
  auto entries = [&]() {
    size_t tb = tmp_bytes;
    CUDA(cub::DeviceReduce::Sum(tmp, tb, W.len, W.esum, (int)(nseg + 1), st));
    CUDA(cudaMemcpyAsync(&E, W.esum, sizeof E, cudaMemcpyDeviceToHost, st));
    CUDA(cudaMemcpyAsync(&overflow, W.overflow, sizeof overflow, cudaMemcpyDeviceToHost, st));
    CUDA(cudaStreamSynchronize(st));
    if (overflow) throw_err(BLANCE_ERR_CUDA, std::string(name) + ": a round had more picks than its bound (internal error)");
  };
  entries();
  int32_t r = 0;
  while (E > 0) {
    // every instance with entries picks at least one op per round: no instance has more rounds than ops
    if (r > max_ops + kWaveBlock) throw_err(BLANCE_ERR_CUDA, std::string(name) + ": the schedule did not end (internal error)");
    const long long n_sort = std::min(pick_bound, E);
    for (int b = 0; b < kWaveBlock; ++b, ++r) {
      size_t tb = tmp_bytes;
      CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb, W.kcnt, const_cast<long long*>(W.poff), (int)(nseg + 1), st));
      launch(ctx, k_wave_pick, seg_grid, WAVE_THREADS, 0, W, r, n_sort);
      sort(n_sort);
      launch(ctx, k_wave_merge, seg_grid, WAVE_THREADS, 0, W, r);
    }
    entries();
  }
  std::vector<unsigned long long> scal((size_t)(4 * ni));
  CUDA(cudaMemcpyAsync(scal.data(), W.scal, sizeof(unsigned long long) * scal.size(), cudaMemcpyDeviceToHost, st));
  CUDA(cudaStreamSynchronize(st));
  return scal;
}

// ---------------------------------------------------------------------------------------
// The audit of a partition map (audit.cuh; include/blance_b200.h).

// The audits requested with one call: the checked options and the caller's outputs (one per audited map).
struct AuditReq {
  uint32_t flags = 0;
  int n_domains = 0;
  const int32_t* parent = nullptr;     // host, [n_node_ids + n_domains] or NULL
  blance_audit_out* out = nullptr;
};

// What an audit reads of a model: sizes, the state tables and the hierarchy fields (not the partition tables).
static void check_audit_model(const std::string& name, const blance_plan_in* m) {
  auto bad = [&](const char* what, int st = BLANCE_ERR_INVALID_ARG) { throw_err(st, name + ": " + what); };
  if (!m) bad("model is NULL");
  if (m->n_nodes < 0 || m->n_node_ids < m->n_nodes || m->n_states < 0 || m->n_parts < 0 || m->n_slots < 0)
    bad("negative size or n_node_ids < n_nodes");
  if (m->n_states > BL_S_MAX) bad("more than 8 model states", BLANCE_ERR_UNSUPPORTED);
  if (m->n_slots > BL_SLP_MAX) bad("more than 32 slots per row", BLANCE_ERR_UNSUPPORTED);
  if (m->n_nodes > 8192) bad("more than 8192 nodes", BLANCE_ERR_UNSUPPORTED);
  if (m->n_parts >= (1 << 30)) bad("2^30 or more partitions", BLANCE_ERR_UNSUPPORTED);
  if (m->n_states > 0) {
    if (!m->state_constraints || !m->state_slot_off) bad("state tables are NULL");
    if (m->top_state < 0 || m->top_state >= m->n_states) bad("top_state out of range");
    if (m->state_slot_off[0] != 0 || m->state_slot_off[m->n_states] != m->n_slots) bad("state_slot_off does not span [0, n_slots]");
    for (int s = 0; s < m->n_states; ++s)
      if (m->state_slot_off[s + 1] < m->state_slot_off[s]) bad("state_slot_off not monotone");
  }
  if (!m->has_hier_rules) return;
  if (!m->rule_off) bad("rule_off is NULL");
  if (m->n_rules < 0) bad("n_rules is negative");
  if (m->n_rules > AUDIT_RULES_MAX) bad("more than 256 hierarchy rules", BLANCE_ERR_UNSUPPORTED);
  if (m->n_rules > 0 && !m->ie_mask) bad("ie_mask is NULL");
  if (m->n_hier_bits < m->n_nodes) bad("n_hier_bits < n_nodes");
  if ((m->n_hier_bits + 31) / 32 > 32 * AUDIT_HW_LANE) bad("hierarchy universe above 4096 bits", BLANCE_ERR_UNSUPPORTED);
  for (int s = 0; s <= m->n_states; ++s)
    if (m->rule_off[s] < 0 || m->rule_off[s] > m->n_rules || (s > 0 && m->rule_off[s] < m->rule_off[s - 1]))
      bad("rule_off is not a monotone offset table into the rules");
}

// A fault-domain forest over NU node ids and n_domains inner vertices (parent NULL: none): n_domains in [0, 2^24], no
// cycle, every vertex at most AUDIT_DEPTH_MAX edges below its root.
static void check_forest(const std::string& name, int n_domains, const int32_t* parent, int NU) {
  if (n_domains < 0 || n_domains > (1 << 24)) throw_err(BLANCE_ERR_INVALID_ARG, name + ": n_domains outside [0, 2^24]");
  if (!parent && n_domains != 0) throw_err(BLANCE_ERR_INVALID_ARG, name + ": n_domains without domain_parent");
  if (!parent) return;
  const long long V = (long long)NU + n_domains;
  for (long long v = 0; v < V; ++v)
    if (parent[v] < -1 || parent[v] >= V)
      throw_err(BLANCE_ERR_INVALID_ARG, name + ": domain_parent[" + std::to_string(v) + "] is outside [-1, n_node_ids + n_domains)");
  for (long long v = 0; v < V; ++v) {
    int d = 0;
    for (long long u = parent[v]; u >= 0; u = parent[u])
      if (++d > AUDIT_DEPTH_MAX)
        throw_err(BLANCE_ERR_INVALID_ARG, name + ": domain_parent has a cycle or a vertex more than 16 edges below its root (vertex " + std::to_string(v) + ")");
  }
}

// The options of an audit over NU node ids, checked: flags, and a fault-domain forest without cycles, every vertex
// at most AUDIT_DEPTH_MAX edges below its root.
static AuditReq check_audit_opts(const std::string& name, const blance_audit_opts* o, int NU, blance_audit_out* out) {
  AuditReq ar;
  ar.out = out;
  if (!out) throw_err(BLANCE_ERR_INVALID_ARG, name + ": the audit output is NULL");
  if (!o) return ar;
  if (o->flags & ~(uint32_t)BLANCE_AUDIT_N2N) throw_err(BLANCE_ERR_INVALID_ARG, name + ": audit flags hold an unknown bit");
  ar.flags = o->flags; ar.n_domains = o->n_domains; ar.parent = o->domain_parent;
  check_forest(name, o->n_domains, o->domain_parent, NU);
  return ar;
}

// Without a context there is nothing to run on: BLANCE_ERR_CUDA when that is because the machine has no usable
// device (no context can be created then), an argument error otherwise.
static void need_ctx(const blance_ctx* ctx) {
  if (ctx) return;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0) {
    cudaGetLastError();
    throw_err(BLANCE_ERR_CUDA, "no CUDA device available; libblance_b200 has no CPU fallback");
  }
  throw_err(BLANCE_ERR_INVALID_ARG, "ctx is NULL");
}

// Device buffers of nw audits of maps with P partitions over NU node ids and N nodes: descriptors, the int64
// result blocks (audit_out_words each, Rc rules), and on request the forest, the failover matrices and the
// per-partition flags.  The forest is one array whatever nw; pricing a wave as nw times one audit counts it nw times,
// an over-estimate of V x 4 bytes per scenario.
struct AuditBufs {
  AuditInst* insts = nullptr;
  long long* out = nullptr;
  int32_t* parent = nullptr;
  int32_t* n2n = nullptr;
  uint8_t* flags = nullptr;
  int nw = 0, S = 0, Rc = 0, V = 0, N = 0, P = 0;
  long long words = 0;
};

static void audit_slices(Arena& a, AuditBufs& b, const AuditReq& ar, int nw, int S, int Rc, int NU, int N, int P, bool want_flags) {
  b.nw = nw; b.S = S; b.Rc = Rc; b.V = NU + ar.n_domains; b.N = N; b.P = P;
  b.words = audit_out_words(S, Rc, b.V);
  a.add(b.insts, (size_t)nw);
  a.add(b.out, (size_t)(b.words * nw));
  if (ar.parent) a.add(b.parent, (size_t)b.V);
  if (ar.flags & BLANCE_AUDIT_N2N) a.add(b.n2n, (size_t)nw * N * N);
  if (want_flags) a.add(b.flags, (size_t)nw * P);
}

// The model part of a descriptor, from an instance as laid out for the device / from the caller's tables.
static AuditInst audit_inst(const DInst& D) {
  AuditInst A{};
  A.P = D.PU; A.N = D.N; A.NU = D.NU; A.S = D.S; A.top_state = D.top_state;
  A.HW = D.HW; A.n_rules = D.has_hier_rules ? D.n_rules : 0;
  for (int s = 0; s < D.S; ++s) { A.constraints[s] = D.state_constraints[s]; A.slot_off[s] = D.state_slot_off[s]; A.rule_off[s] = D.rule_off[s]; }
  A.slot_off[D.S] = D.state_slot_off[D.S]; A.rule_off[D.S] = D.rule_off[D.S];
  return A;
}

static AuditInst audit_inst(const blance_plan_in& m) {
  AuditInst A{};
  A.P = m.n_parts; A.N = m.n_nodes; A.NU = m.n_node_ids; A.S = m.n_states; A.top_state = m.top_state;
  A.HW = m.has_hier_rules ? (m.n_hier_bits + 31) / 32 : 0; A.n_rules = m.has_hier_rules ? m.n_rules : 0;
  for (int s = 0; s < m.n_states; ++s) {
    A.constraints[s] = m.state_constraints[s]; A.slot_off[s] = m.state_slot_off[s];
    A.rule_off[s] = m.has_hier_rules ? m.rule_off[s] : 0;
  }
  A.slot_off[m.n_states] = m.n_slots; A.rule_off[m.n_states] = m.has_hier_rules ? m.rule_off[m.n_states] : 0;
  return A;
}

static void audit_kernels(blance_ctx* ctx, const AuditBufs& b, bool any_rules);

// Enqueues the audits `insts` (map and model fields set by the caller) on b's buffers.
static void audit_run(blance_ctx* ctx, const AuditBufs& b, const AuditReq& ar, std::vector<AuditInst>& insts) {
  cudaStream_t st = ctx->stream;
  const int nw = b.nw;
  bool any_rules = false;
  for (int j = 0; j < nw; ++j) {
    AuditInst& A = insts[(size_t)j];
    A.V = b.V; A.Rc = b.Rc; A.dom_parent = b.parent;
    A.out = b.out + (long long)j * b.words;
    A.n2n = b.n2n ? b.n2n + (size_t)j * b.N * b.N : nullptr;
    A.part_flags = b.flags ? b.flags + (size_t)j * b.P : nullptr;
    any_rules |= A.n_rules > 0;
  }
  CUDA(cudaMemcpyAsync(b.insts, insts.data(), sizeof(AuditInst) * (size_t)nw, cudaMemcpyHostToDevice, st));
  if (b.parent) CUDA(cudaMemcpyAsync(b.parent, ar.parent, sizeof(int32_t) * (size_t)b.V, cudaMemcpyHostToDevice, st));
  CUDA(cudaMemsetAsync(b.out, 0, sizeof(long long) * (size_t)(b.words * nw), st));
  if (b.n2n) CUDA(cudaMemsetAsync(b.n2n, 0, sizeof(int32_t) * (size_t)nw * b.N * b.N, st));
  if (b.flags) CUDA(cudaMemsetAsync(b.flags, 0, (size_t)nw * b.P, st));
  CUDA(cudaEventRecord(ctx->ev[4], st));
  audit_kernels(ctx, b, any_rules);
  CUDA(cudaEventRecord(ctx->ev[5], st));
}

static void audit_kernels(blance_ctx* ctx, const AuditBufs& b, bool any_rules) {
  const int nw = b.nw;
  if (b.P <= 0) return;
  const int per_sm = std::max(1, ctx->sm_count * 8 / nw);
  const size_t smem = sizeof(uint32_t) * 3 * (size_t)b.V;
  const dim3 grid((unsigned)std::max(1, std::min((b.P + 255) / 256, per_sm)), (unsigned)nw);
  if (smem <= 44 * 1024) launch(ctx, k_map_audit<true>, grid, 256, smem, b.insts);
  else launch(ctx, k_map_audit<false>, grid, 256, 0, b.insts);
  if (any_rules)         // one warp per partition
    launch(ctx, k_map_audit_rules, dim3((unsigned)std::max(1, std::min((b.P + 7) / 8, per_sm)), (unsigned)nw), 256, 0, b.insts);
  if (b.n2n && b.N > 0)
    launch(ctx, k_audit_n2n_max, dim3((unsigned)std::max(1, (int)std::min<long long>(((long long)b.N * b.N + 255) / 256, per_sm)), (unsigned)nw),
           256, 0, b.insts);
}

// Copies the results of audit j of b into o (the caller synchronises the stream; `host` receives the int64 block
// and must outlive that).
static void audit_fetch(blance_ctx* ctx, const AuditBufs& b, int j, std::vector<long long>& host, blance_audit_out& o) {
  cudaStream_t st = ctx->stream;
  host.assign((size_t)b.words, 0);
  CUDA(cudaMemcpyAsync(host.data(), b.out + (long long)j * b.words, sizeof(long long) * (size_t)b.words, cudaMemcpyDeviceToHost, st));
  if (o.n2n && b.n2n && b.N > 0)
    CUDA(cudaMemcpyAsync(o.n2n, b.n2n + (size_t)j * b.N * b.N, sizeof(int32_t) * (size_t)b.N * b.N, cudaMemcpyDeviceToHost, st));
  if (o.part_flags && b.flags && b.P > 0)
    CUDA(cudaMemcpyAsync(o.part_flags, b.flags + (size_t)j * b.P, (size_t)b.P, cudaMemcpyDeviceToHost, st));
}

// The int64 block of one audit (n_rules of its own) into the caller's arrays and scalars, after the stream was
// synchronised; kernel_ms is the time between the events audit_run recorded.
static void audit_unpack(blance_ctx* ctx, const AuditBufs& b, int n_rules, const std::vector<long long>& host, blance_audit_out& o) {
  o.kernel_ms = 0.f;
  cudaEventElapsedTime(&o.kernel_ms, ctx->ev[4], ctx->ev[5]);
  const long long* h = host.data();
  const int S = b.S, Rc = b.Rc, V = b.V;
  auto put = [](int64_t* dst, const long long* src, int n) { if (dst && n > 0) std::memcpy(dst, src, sizeof(int64_t) * (size_t)n); };
  put(o.short_slots, h, S); put(o.over_slots, h + S, S);
  put(o.rule_miss, h + 2 * S, n_rules); put(o.rule_tested, h + 2 * S + Rc, n_rules);
  const long long* d = h + 2 * S + 2 * Rc;
  put(o.dom_top, d, V); put(o.dom_all, d + V, V); put(o.dom_copies, d + 2ll * V, V);
  const long long* sc = d + 3ll * V;
  o.short_parts = sc[0]; o.rule_miss_parts = sc[1]; o.no_top_parts = sc[2];
  o.n2n_max = o.n2n_max_a = o.n2n_max_b = -1;
  if (b.n2n) {
    const unsigned long long key = (unsigned long long)sc[3];
    o.n2n_max = (int32_t)(key >> 32);
    if (key) {
      const uint32_t idx = 0xFFFFFFFFu - (uint32_t)key;
      o.n2n_max_a = (int32_t)(idx / (uint32_t)b.N); o.n2n_max_b = (int32_t)(idx % (uint32_t)b.N);
    }
  }
}

// The chains requested with blance_plan_chains: T stages per chain, stages [n][T], net [n] or NULL.
struct ChainReq {
  int T = 1;
  const blance_chain_stage* stages = nullptr;
  blance_chain_out* net = nullptr;
};

// The node fields of scenario (or chain) i at stage t.
static const blance_scenario& nodes_of(const blance_scenario* sc, const ChainReq* cr, int i, int t) {
  return cr ? cr->stages[(size_t)i * cr->T + t].nodes : sc[i];
}

// The substituted instance of scenario / chain i at stage t.  A chain stage's node_removed is written in the device
// code into `code` (NR_OUTSIDE for the ids below n_nodes that its node_in_all leaves out), and from stage 2 on the
// non-model counts of iteration 1 are those of the later iterations: the assigned partitions' prevMap entries are
// the previous stage's next rows, which hold model states only.
static blance_plan_in stage_in(const blance_plan_in& base, const blance_scenario* sc, const blance_scenario_opts* opts,
                               const ChainReq* cr, int i, int t, std::vector<uint8_t>& code) {
  blance_plan_in in = scenario_in(base, nodes_of(sc, cr, i, t), opts_of(opts, i));
  if (!cr) return in;
  const blance_chain_stage& st = cr->stages[(size_t)i * cr->T + t];
  code.assign((size_t)std::max(1, base.n_node_ids), 0);
  for (int q = 0; q < base.n_node_ids; ++q)
    code[(size_t)q] = (uint8_t)((st.nodes.node_removed[q] ? NR_REMOVE : 0) | (q < base.n_nodes && !st.node_in_all[q] ? NR_OUTSIDE : 0));
  in.node_removed = code.data();
  if (t > 0) in.extra_tot_first = in.extra_tot_rest;
  return in;
}

// Uploads the node tables (node flags, weights, non-model counts, hierarchy masks) of the wave's instances `ins`
// into pl's pool.
static void upload_nodes(blance_ctx* ctx, blance_plan* pl, const std::vector<blance_plan_in>& ins, bool coded) {
  cudaStream_t st = ctx->stream;
  DPool& P = pl->pool;
  const size_t NT = (size_t)pl->NT, NUT = (size_t)pl->NUT, MT = (size_t)pl->MT;
  std::vector<uint8_t> rm(NUT + 1, 0), ad(NUT + 1, 0), hw(NT + 1, 0);
  std::vector<int32_t> nwt(NT + 1, 0), ef(NT + 1, 0), er(NT + 1, 0);
  std::vector<uint32_t> mask(MT + 1, 0);
  const NodeTables t{rm.data(), ad.data(), hw.data(), nwt.data(), ef.data(), er.data(), mask.data()};
  for (size_t j = 0; j < ins.size(); ++j) stage_nodes(ins[j], pl->h_insts[j], t, coded);
  CUDA(cudaMemcpyAsync((void*)P.node_removed, rm.data(), NUT + 1, cudaMemcpyHostToDevice, st));
  CUDA(cudaMemcpyAsync((void*)P.node_added, ad.data(), NUT + 1, cudaMemcpyHostToDevice, st));
  CUDA(cudaMemcpyAsync((void*)P.node_has_weight, hw.data(), NT + 1, cudaMemcpyHostToDevice, st));
  CUDA(cudaMemcpyAsync((void*)P.node_weight, nwt.data(), sizeof(int32_t) * (NT + 1), cudaMemcpyHostToDevice, st));
  CUDA(cudaMemcpyAsync((void*)P.extra_first, ef.data(), sizeof(int32_t) * (NT + 1), cudaMemcpyHostToDevice, st));
  CUDA(cudaMemcpyAsync((void*)P.extra_rest, er.data(), sizeof(int32_t) * (NT + 1), cudaMemcpyHostToDevice, st));
  CUDA(cudaMemcpyAsync((void*)P.ie_mask, mask.data(), sizeof(uint32_t) * (MT + 1), cudaMemcpyHostToDevice, st));
  CUDA(cudaStreamSynchronize(st));          // the host vectors die here
}

// Scenario summaries (node_ops | state_node_load | 3 scalars per instance, `stride` int64 words) of the wave's plans
// from the beg rows / flags `prev_rows` / `pflags` to the working rows.
static void wave_summary(blance_ctx* ctx, blance_plan* pl, int nw, const int32_t* prev_rows, const uint8_t* pflags, int favor_min,
                         long long stride, long long* d_sum) {
  const DInst& D0 = pl->h_insts[0];
  const int PU = D0.PU, NU = D0.NU, S = D0.S;
  CUDA(cudaMemsetAsync(d_sum, 0, sizeof(long long) * (size_t)(stride * nw), ctx->stream));
  if (PU <= 0) return;
  const size_t smem = align_up(sizeof(uint32_t) * 4 * (size_t)NU, 8) + sizeof(long long) * (size_t)S * NU;
  const int bx = std::max(1, std::min((PU + 255) / 256, std::max(1, ctx->sm_count * 8 / nw)));
  const dim3 grid((unsigned)bx, (unsigned)nw);
  if (smem <= 48 * 1024) launch(ctx, k_scenario_summary<true>, grid, 256, smem, pl->pool, prev_rows, pflags, favor_min, stride, d_sum);
  else launch(ctx, k_scenario_summary<false>, grid, 256, 0, pl->pool, prev_rows, pflags, favor_min, stride, d_sum);
}

// Plans the scenarios idx (of sc / opts) on one device, in waves.  With cr each is a chain of cr->T stages, planned
// in lock step: a stage boundary is an iteration boundary plus the next stage's node tables (DESIGN.md section 12).
static void scenarios_on_device(blance_ctx* ctx, const blance_plan_in* base, const std::vector<int>& idx, const blance_scenario* sc,
                                const blance_scenario_opts* opts, int favor_min, int max_concurrent, blance_scenario_out* out,
                                const SchedReq* sr, const AuditReq* ar, const ChainReq* cr = nullptr) {
  cudaStream_t st = ctx->stream;
  const int n_dev = (int)idx.size();
  const int T = cr ? cr->T : 1;
  const bool coded = cr != nullptr;
  std::vector<uint8_t> code0;
  const blance_plan_in in0 = stage_in(*base, sc, opts, cr, idx[0], 0, code0);
  long long max_mask = 0;
  int max_ow = 0, max_rules = 0;
  bool audit_flags = false;            // any caller wants the per-partition flags
  for (int i : idx) {
    const blance_plan_in in = scenario_in(*base, nodes_of(sc, cr, i, 0), opts_of(opts, i));
    max_mask = std::max(max_mask, mask_words(in));
    max_ow = std::max(max_ow, n_overrides(opts_of(opts, i)));
    max_rules = std::max(max_rules, in.has_hier_rules ? in.n_rules : 0);
    audit_flags |= ar && ar->out[i].part_flags;
  }
  size_t extra_bytes = 0;              // one scenario's audit buffers / one chain's net buffers, priced into the wave
  if (ar) {
    Arena one;
    AuditBufs b;
    audit_slices(one, b, *ar, 1, base->n_states, max_rules, base->n_node_ids, base->n_nodes, base->n_parts, audit_flags);
    extra_bytes = one.bytes();
  }
  {
    cudaMemPool_t pool;                // measure free memory without this context's cached arenas
    if (max_concurrent <= 0 && cudaDeviceGetDefaultMemPool(&pool, ctx->device) == cudaSuccess) {
      cudaStreamSynchronize(st);
      cudaMemPoolTrimTo(pool, 0);
    }
  }
  // the base: one H2D of the caller's layout, then k_unpack (into its *_init slices)
  const PlanPtr pb = upload(ctx, 1, &in0, coded);
  const long long stride = summary_stride(*base);
  const bool want_net = cr && cr->net;
  if (want_net) {                      // the base's prev rows and flags, kept for the net summary, and its result
    Arena one;
    int32_t* r = nullptr;
    uint8_t* f = nullptr;
    long long* d = nullptr;
    one.add(r, (size_t)pb->RT + 4); one.add(f, (size_t)pb->PT + 1); one.add(d, (size_t)stride);
    extra_bytes += one.bytes();
  }
  size_t per = 0;
  int W = wave_size(ctx, in0, max_mask, max_ow, n_dev, max_concurrent, sr, extra_bytes, &per);
  if (W < 1)
    throw_err(BLANCE_ERR_NOMEM, "blance_plan_scenarios: one scenario needs " + std::to_string(per >> 20) + " MiB, more than the free device memory");
  const bool auto_wave = max_concurrent <= 0;
  const bool times = getenv("BLANCE_SCENARIO_TIMES") != nullptr;
  const int PU = base->n_parts, NU = base->n_node_ids, S = base->n_states;
  int n_prev_later = 0;                // len(prevMap) from stage 2 on: the base's prevMap plus every assigned partition
  for (int p = 0; cr && p < PU; ++p) n_prev_later += (base->part_in_prev[p] || base->part_in_assign[p]) ? 1 : 0;
  for (int w0 = 0; w0 < n_dev;) {
    const int nw = std::min(W, n_dev - w0);
    std::vector<blance_plan_in> ins((size_t)nw);
    std::vector<std::vector<uint8_t>> code((size_t)nw);
    for (int j = 0; j < nw; ++j) ins[(size_t)j] = stage_in(*base, sc, opts, cr, idx[(size_t)(w0 + j)], 0, code[(size_t)j]);
    // a device's only scenario is the base upload itself: nothing to replicate (its weight overrides still apply)
    const bool lone = n_dev == 1;
    blance_plan wave_plan;
    blance_plan* pl = lone ? pb.get() : &wave_plan;
    std::vector<int> seg_off;
    if (!lone) layout(pl, nw, ins.data(), seg_off, coded);
    if (!lone && pl->PT >= (1LL << 29)) {
      if (nw > 1) { W = nw / 2; continue; }
      throw_err(BLANCE_ERR_UNSUPPORTED, "2^29 or more partitions in one scenario");
    }
    // the wave's partition-weight overrides over its replicated slices (lone: over the base upload), as
    // wave-global partition indices: ow = index[k] | weight[k] | presence[k]
    std::vector<int32_t> ow;
    for (int pass = 0; pass < 3; ++pass)
      for (int j = 0; j < nw; ++j) {
        const blance_scenario_opts* o = opts_of(opts, idx[(size_t)(w0 + j)]);
        for (int k = 0; k < n_overrides(o); ++k)
          ow.push_back(pass == 0 ? (int32_t)(pl->h_insts[(size_t)j].part_off + o->ow_part[k]) : pass == 1 ? o->ow_weight[k] : (int32_t)o->ow_has[k]);
      }
    // one allocation per wave, so that a plan is never lost for want of its summaries or schedule state: the
    // wave's plan (lone: the base upload is the plan), the summaries, the schedule state, the weight overrides,
    // the chains' net buffers
    Arena wave;
    if (!lone) plan_slices(wave, pl, nw);
    long long* d_sum = nullptr;
    wave.add(d_sum, (size_t)(stride * nw));
    WSched wsch{};
    void* wtmp = nullptr;
    size_t wtmp_bytes = 0;
    if (sr) sched_slices(wave, nw, sr->nc, PU, NU, scenario_ops(*base), (long long)PU * scenario_ops(*base), wsch, wtmp, wtmp_bytes, st);
    int32_t* d_ow = nullptr;
    if (!ow.empty()) wave.add(d_ow, ow.size());
    AuditBufs abuf;
    if (ar) audit_slices(wave, abuf, *ar, nw, S, max_rules, NU, base->n_nodes, PU, audit_flags);
    int32_t* net_prev = nullptr;
    uint8_t* net_flags = nullptr;
    long long* d_net = nullptr;
    if (want_net) { wave.add(net_prev, (size_t)pl->RT + 4); wave.add(net_flags, (size_t)pl->PT + 1); wave.add(d_net, (size_t)(stride * nw)); }
    try {
      wave.alloc(st, "a scenario wave");
    } catch (const Error&) {
      if (auto_wave && nw > 1) { W = nw / 2; continue; }      // the free memory moved
      throw;
    }
    DPool& P = pl->pool;
    // the node tables of the wave's scenarios (small host copies); the hierarchy masks and extra counts of the base
    if (!lone) {
      upload_nodes(ctx, pl, ins, coded);
      CUDA(cudaMemcpyAsync(pl->d_raw_rows_off, pl->raw_rows_off.data(), sizeof(long long) * (size_t)(nw + 1), cudaMemcpyHostToDevice, st));
      CUDA(cudaMemcpyAsync(pl->d_raw_shape_off, pl->raw_shape_off.data(), sizeof(long long) * (size_t)(nw + 1), cudaMemcpyHostToDevice, st));
      CUDA(cudaMemcpyAsync(pl->d_seg_off, seg_off.data(), sizeof(int) * (size_t)(nw + 1), cudaMemcpyHostToDevice, st));
      CUDA(cudaStreamSynchronize(st));          // the host vectors die at the end of this block
    }
    if (!lone && pl->PT > 0)
      launch(ctx, k_scenario_replicate, grid_for(ctx, pl->PT, 256), 256, 0, pl->rows_init, pl->prev_rows_init, pl->pmeta_init,
             pl->prev_meta_init, pl->pflags_init, const_cast<int32_t*>(P.pweight), const_cast<int32_t*>(P.name_rank),
             const_cast<int32_t*>(P.part_inst), pb->rows_init, pb->prev_rows_init, pb->pmeta_init, pb->prev_meta_init,
             pb->pflags_init, pb->pool.pweight, pb->pool.name_rank, PU, pl->h_insts[0].SLP, pl->PT);
    if (!ow.empty()) {
      const int k = (int)(ow.size() / 3);
      CUDA(cudaMemcpyAsync(d_ow, ow.data(), sizeof(int32_t) * ow.size(), cudaMemcpyHostToDevice, st));
      launch(ctx, k_scenario_weights, grid_for(ctx, k, 256), 256, 0, const_cast<int32_t*>(P.pweight), pl->pflags_init, d_ow, k);
    }
    if (want_net && pl->PT > 0) {      // the stage boundary overwrites these (in the lone path, the base upload's own)
      CUDA(cudaMemcpyAsync(net_prev, pl->prev_rows_init, sizeof(int32_t) * (size_t)pl->RT, cudaMemcpyDeviceToDevice, st));
      CUDA(cudaMemcpyAsync(net_flags, pl->pflags_init, (size_t)pl->PT, cudaMemcpyDeviceToDevice, st));
    }
    if (!lone) finish_upload(ctx, pl);
    for (int t = 0; t < T; ++t) {
      if (t > 0) {
        // the stage boundary: what the convergence loop left in the working state is the next stage's input - the
        // assigned partitions' prev and cur rows are their next rows, committed by k_commit (or equal to them when the
        // stage converged) with their flags - then the next stage's node tables and a fresh loop state
        if (pl->PT > 0) {
          CUDA(cudaMemcpyAsync(pl->rows_init, P.rows, sizeof(int32_t) * (size_t)pl->RT, cudaMemcpyDeviceToDevice, st));
          CUDA(cudaMemcpyAsync(pl->prev_rows_init, P.prev_rows, sizeof(int32_t) * (size_t)pl->RT, cudaMemcpyDeviceToDevice, st));
          CUDA(cudaMemcpyAsync(pl->pmeta_init, P.pmeta, sizeof(uint32_t) * (size_t)pl->PT, cudaMemcpyDeviceToDevice, st));
          CUDA(cudaMemcpyAsync(pl->prev_meta_init, P.prev_meta, sizeof(uint32_t) * (size_t)pl->PT, cudaMemcpyDeviceToDevice, st));
          CUDA(cudaMemcpyAsync(pl->pflags_init, P.pflags, (size_t)pl->PT, cudaMemcpyDeviceToDevice, st));
        }
        for (int j = 0; j < nw; ++j) {
          ins[(size_t)j] = stage_in(*base, sc, opts, cr, idx[(size_t)(w0 + j)], t, code[(size_t)j]);
          node_state(pl->h_insts[(size_t)j], ins[(size_t)j], coded, n_prev_later);
        }
        upload_nodes(ctx, pl, ins, coded);
      }
      CUDA(cudaEventRecord(ctx->ev[0], st));
      run(ctx, pl);
      // summaries, then the requested rows
      float sum_ms = 0.f, sched_ms = 0.f;
      CUDA(cudaEventRecord(ctx->ev[1], st));
      wave_summary(ctx, pl, nw, pl->prev_rows_init, pl->pflags_init, favor_min, stride, d_sum);
      if (want_net && t == T - 1) wave_summary(ctx, pl, nw, net_prev, net_flags, favor_min, stride, d_net);
      CUDA(cudaEventRecord(ctx->ev[2], st));
      // the output of wave member j at this stage
      auto out_of = [&](int j) -> blance_scenario_out& { return out[(size_t)idx[(size_t)(w0 + j)] * T + t]; };
      // the audits of the wave's final maps: assigned partitions from the next rows, the others from prevMap as uploaded
      std::vector<AuditInst> a_insts;
      std::vector<std::vector<long long>> a_host((size_t)(ar ? nw : 0));
      if (ar) {
        for (int j = 0; j < nw; ++j) {
          const DInst& D = pl->h_insts[(size_t)j];
          AuditInst A = audit_inst(D);
          A.rows = P.rows + D.rows_off; A.alt_rows = pl->prev_rows_init + D.rows_off;
          A.meta = P.pmeta + D.part_off; A.alt_meta = pl->prev_meta_init + D.part_off;
          A.pflags = pl->pflags_init + D.part_off;
          A.ie_mask = P.ie_mask + D.mask_off;
          A.stride = D.SLP;
          a_insts.push_back(A);
        }
        audit_run(ctx, abuf, *ar, a_insts);
        for (int j = 0; j < nw; ++j) audit_fetch(ctx, abuf, j, a_host[(size_t)j], ar->out[idx[(size_t)(w0 + j)]]);
      }
      bool any_rows = false;
      for (int j = 0; j < nw; ++j) {
        const blance_scenario_out& o = out_of(j);
        any_rows |= o.next_rows || o.next_shape || o.warn;
      }
      if (any_rows && pl->PT > 0)
        launch(ctx, k_pack, grid_for(ctx, pl->PT, 256), 256, 0, P, pl->raw_a, pl->rawsh_a, pl->rawsh_b, pl->d_raw_rows_off,
               pl->d_raw_shape_off, pl->PT);
      std::vector<long long> h_sum((size_t)(stride * nw));
      std::vector<DInst> fin((size_t)nw);
      CUDA(cudaMemcpyAsync(h_sum.data(), d_sum, sizeof(long long) * h_sum.size(), cudaMemcpyDeviceToHost, st));
      CUDA(cudaMemcpyAsync(fin.data(), P.insts, sizeof(DInst) * (size_t)nw, cudaMemcpyDeviceToHost, st));
      for (int j = 0; j < nw; ++j) {
        blance_scenario_out& o = out_of(j);
        const size_t rr = (size_t)PU * base->n_slots, rs = (size_t)PU * S;
        if (rr && o.next_rows) CUDA(cudaMemcpyAsync(o.next_rows, pl->raw_a + pl->raw_rows_off[(size_t)j], sizeof(int32_t) * rr, cudaMemcpyDeviceToHost, st));
        if (rs && o.next_shape) CUDA(cudaMemcpyAsync(o.next_shape, pl->rawsh_a + pl->raw_shape_off[(size_t)j], rs, cudaMemcpyDeviceToHost, st));
        if (rs && o.warn) CUDA(cudaMemcpyAsync(o.warn, pl->rawsh_b + pl->raw_shape_off[(size_t)j], rs, cudaMemcpyDeviceToHost, st));
      }
      CUDA(cudaStreamSynchronize(st));
      cudaEventElapsedTime(&sum_ms, ctx->ev[1], ctx->ev[2]);
      for (int j = 0; j < nw; ++j) {
        if (fin[(size_t)j].spec_abort) throw_err(BLANCE_ERR_CUDA, "the speculative pass kernel gave up waiting (internal error; see stderr of the device printf)");
        blance_scenario_out& o = out_of(j);
        const long long* s = h_sum.data() + (size_t)j * (size_t)stride;
        if (o.node_ops) std::memcpy(o.node_ops, s, sizeof(int64_t) * 4 * (size_t)NU);
        if (o.state_node_load) std::memcpy(o.state_node_load, s + 4ll * NU, sizeof(int64_t) * (size_t)S * NU);
        o.parts_moved = s[stride - 3]; o.ops_total = s[stride - 2]; o.warn_parts = s[stride - 1];
        o.iters_run = fin[(size_t)j].iters_run; o.converged = fin[(size_t)j].converged;
        o.steps = fin[(size_t)j].steps; o.sticky_steps = fin[(size_t)j].fast_steps;
        if (ar) audit_unpack(ctx, abuf, a_insts[(size_t)j].n_rules, a_host[(size_t)j], ar->out[idx[(size_t)(w0 + j)]]);
      }
      if (sr) {
        CUDA(cudaEventRecord(ctx->ev[3], st));
        if (PU > 0) launch(ctx, k_wave_moves, wave_grid(ctx, PU, nw), 256, 0, P, pl->prev_rows_init, pl->pflags_init, favor_min, wsch);
        std::vector<long long> ops((size_t)nw * NU);        // each scenario's ops per node: its node_ops summed over the kinds
        for (size_t x = 0; x < ops.size(); ++x) {
          const long long* s = h_sum.data() + (x / NU) * stride + 4 * (x % NU);
          ops[x] = s[0] + s[1] + s[2] + s[3];
        }
        const std::vector<unsigned long long> scal = wave_schedule(ctx, "blance_plan_scenarios_schedule", *sr, wsch, wtmp, wtmp_bytes, ops.data());
        for (long long i = 0; i < (long long)nw * sr->nc; ++i) {
          blance_scenario_schedule_out& o = sr->out[(size_t)idx[(size_t)(w0 + i / sr->nc)] * sr->nc + (size_t)(i % sr->nc)];
          o.rounds = (int32_t)scal[(size_t)(4 * i)];
          o.moves_done = (int64_t)scal[(size_t)(4 * i + 1)];
          o.stuck_parts = (int64_t)scal[(size_t)(4 * i + 2)];
          o.max_batch = (int32_t)scal[(size_t)(4 * i + 3)];
          if (o.node_rounds && NU) CUDA(cudaMemcpyAsync(o.node_rounds, wsch.node_rounds + i * NU, sizeof(int32_t) * NU, cudaMemcpyDeviceToHost, st));
          if (o.node_last_round && NU) CUDA(cudaMemcpyAsync(o.node_last_round, wsch.node_last + i * NU, sizeof(int32_t) * NU, cudaMemcpyDeviceToHost, st));
          if (o.part_done_round && PU) CUDA(cudaMemcpyAsync(o.part_done_round, wsch.part_done + i * PU, sizeof(int32_t) * PU, cudaMemcpyDeviceToHost, st));
        }
        CUDA(cudaEventRecord(ctx->ev[1], st));
        CUDA(cudaEventSynchronize(ctx->ev[1]));
        cudaEventElapsedTime(&sched_ms, ctx->ev[3], ctx->ev[1]);
      }
      if (times) {
        float wave_ms = 0.f;
        cudaEventElapsedTime(&wave_ms, ctx->ev[0], ctx->ev[2]);
        std::fprintf(stderr, "[blance] scenario wave at %d: %d scenarios (wave size %d, %zu device bytes each), %.3f ms, summary %.3f ms",
                     w0, nw, W, per, wave_ms, sum_ms);
        if (sr) std::fprintf(stderr, ", schedule %.3f ms (%d counts)", sched_ms, sr->nc);
        std::fprintf(stderr, "\n");
      }
    }
    if (want_net) {
      std::vector<long long> h_net((size_t)(stride * nw));
      CUDA(cudaMemcpyAsync(h_net.data(), d_net, sizeof(long long) * h_net.size(), cudaMemcpyDeviceToHost, st));
      CUDA(cudaStreamSynchronize(st));
      for (int j = 0; j < nw; ++j) {
        blance_chain_out& o = cr->net[idx[(size_t)(w0 + j)]];
        const long long* s = h_net.data() + (size_t)j * (size_t)stride;
        if (o.node_ops) std::memcpy(o.node_ops, s, sizeof(int64_t) * 4 * (size_t)NU);
        o.parts_moved = s[stride - 3]; o.ops_total = s[stride - 2];
      }
    }
    w0 += nw;
  }
  cudaStreamSynchronize(st);
}

// The checks of one scenario's substituted instance (base_sum: see check_counts).  Returns a status, `why` the reason.
static int check_scenario(const blance_plan_in& base, const blance_scenario& sc, const blance_scenario_opts* o, long long& base_sum,
                          std::string& why) {
  int st = BLANCE_OK;
  if (sc.add_is_nil != 0 && sc.add_is_nil != 1) why = "add_is_nil is neither 0 nor 1";
  else if (sc.has_node_weights != 0 && sc.has_node_weights != 1) why = "has_node_weights is neither 0 nor 1";
  else {
    const blance_plan_in in = scenario_in(base, sc, o);
    st = check_structure(&in, why);
    if (st == BLANCE_OK && o) st = check_opts(base, *o, why);
    if (st == BLANCE_OK) st = check_counts(base, in, o, base_sum, why);
  }
  if (st == BLANCE_OK && !why.empty()) st = BLANCE_ERR_INVALID_ARG;
  return st;
}

static void plan_scenarios(blance_ctx* ctx, const char* name, const blance_plan_in* base, int32_t n, const blance_scenario* sc,
                           const blance_scenario_opts* opts, int32_t favor_min_nodes, int32_t max_concurrent, blance_scenario_out* out,
                           const SchedReq* sr = nullptr, const AuditReq* ar = nullptr) {
  if (n <= 0) throw_err(BLANCE_ERR_INVALID_ARG, std::string(name) + ": n must be positive");
  if (!base || !sc || !out) throw_err(BLANCE_ERR_INVALID_ARG, std::string(name) + ": base, sc or out is NULL");
  // every scenario is checked before the context is used, so a NULL ctx checks the scenarios without a device
  long long base_sum = -1;                // sum |w_p| of the base (1 without a weight), for the int32 bound
  for (int i = 0; i < n; ++i) {
    std::string why;
    const int st = check_scenario(*base, sc[i], opts_of(opts, i), base_sum, why);
    if (st != BLANCE_OK) throw_err(st, std::string(name) + ": scenario " + std::to_string(i) + ": " + why);
  }
  if (!ctx) throw_err(BLANCE_ERR_INVALID_ARG, "ctx is NULL");
  // several GPUs: scenario i -> device i mod G, one host thread per device, each with its own copy of the base
  const int G = (int)std::min<size_t>((size_t)blance_ctx_device_count(ctx), (size_t)n);
  std::vector<std::vector<int>> idx((size_t)G);
  for (int i = 0; i < n; ++i) idx[(size_t)(i % G)].push_back(i);
  fan_out(ctx, G, [&](int d, blance_ctx* dev) {
    scenarios_on_device(dev, base, idx[(size_t)d], sc, opts, favor_min_nodes, max_concurrent, out, sr, ar);
  });
}

// Chains of stages over one base (blance_plan_chains): chain i -> device i mod G, its stages planned in lock step
// with the other chains of its wave.
static void plan_chains(blance_ctx* ctx, const blance_plan_in* base, int32_t n, int32_t n_stages, const blance_chain_stage* stages,
                        const blance_scenario_opts* opts, int32_t favor_min_nodes, int32_t max_concurrent, blance_scenario_out* out,
                        blance_chain_out* net) {
  const std::string name = "blance_plan_chains";
  if (n <= 0) throw_err(BLANCE_ERR_INVALID_ARG, name + ": n must be positive");
  if (n_stages < 1) throw_err(BLANCE_ERR_INVALID_ARG, name + ": n_stages must be positive");
  if (!base || !stages || !out) throw_err(BLANCE_ERR_INVALID_ARG, name + ": base, stages or out is NULL");
  if (n_stages > 1 && base->max_iters < 1)      // the stage would assign nothing and leave no next map to plan on
    throw_err(BLANCE_ERR_INVALID_ARG, name + ": a chain of several stages needs max_iters >= 1");
  // every stage is checked before the context is used, so a NULL ctx checks the chains without a device
  long long base_sum = -1;
  for (int i = 0; i < n; ++i)
    for (int t = 0; t < n_stages; ++t) {
      const blance_chain_stage& cs = stages[(size_t)i * n_stages + t];
      std::string why;
      int st = check_scenario(*base, cs.nodes, opts_of(opts, i), base_sum, why);
      if (st == BLANCE_OK && base->n_nodes > 0 && !cs.node_in_all) { st = BLANCE_ERR_INVALID_ARG; why = "node_in_all is NULL"; }
      for (int q = 0; st == BLANCE_OK && q < base->n_nodes; ++q)
        if (cs.node_in_all[q] > 1) { st = BLANCE_ERR_INVALID_ARG; why = "node_in_all is neither 0 nor 1"; }
      if (st != BLANCE_OK) throw_err(st, name + ": chain " + std::to_string(i) + ", stage " + std::to_string(t) + ": " + why);
    }
  if (!ctx) throw_err(BLANCE_ERR_INVALID_ARG, "ctx is NULL");
  ChainReq cr;
  cr.T = n_stages; cr.stages = stages; cr.net = net;
  const int G = (int)std::min<size_t>((size_t)blance_ctx_device_count(ctx), (size_t)n);
  std::vector<std::vector<int>> idx((size_t)G);
  for (int i = 0; i < n; ++i) idx[(size_t)(i % G)].push_back(i);
  fan_out(ctx, G, [&](int d, blance_ctx* dev) {
    scenarios_on_device(dev, base, idx[(size_t)d], nullptr, opts, favor_min_nodes, max_concurrent, out, nullptr, nullptr, &cr);
  });
}

extern "C" int blance_plan_chains(blance_ctx* ctx, const blance_plan_in* base, int32_t n, int32_t n_stages,
                                  const blance_chain_stage* stages, const blance_scenario_opts* opts, int32_t favor_min_nodes,
                                  int32_t max_concurrent, blance_scenario_out* out, blance_chain_out* net) {
  return entry(ctx, [&](Device&) {
    plan_chains(ctx, base, n, n_stages, stages, opts, favor_min_nodes, max_concurrent, out, net);
  });
}

extern "C" int blance_plan_scenarios(blance_ctx* ctx, const blance_plan_in* base, int32_t n, const blance_scenario* sc,
                                     int32_t favor_min_nodes, int32_t max_concurrent, blance_scenario_out* out) {
  return entry(ctx, [&](Device&) {
    plan_scenarios(ctx, "blance_plan_scenarios", base, n, sc, nullptr, favor_min_nodes, max_concurrent, out);
  });
}

extern "C" int blance_plan_scenarios_ex(blance_ctx* ctx, const blance_plan_in* base, int32_t n, const blance_scenario* sc,
                                        const blance_scenario_opts* opts, int32_t favor_min_nodes, int32_t max_concurrent,
                                        blance_scenario_out* out) {
  return entry(ctx, [&](Device&) {
    plan_scenarios(ctx, "blance_plan_scenarios_ex", base, n, sc, opts, favor_min_nodes, max_concurrent, out);
  });
}

// The checked schedule request of blance_plan_scenarios_schedule's arguments; the scalars of sched are cleared.
static SchedReq sched_req(const char* name, const blance_plan_in* base, int32_t n, const blance_scenario* sc, const blance_scenario_out* out,
                          int32_t n_move_conc, const int32_t* move_conc, const uint8_t* node_has_mover,
                          blance_scenario_schedule_out* sched) {
  if (n_move_conc < 1 || !move_conc || !sched)
    throw_err(BLANCE_ERR_INVALID_ARG, std::string(name) + ": n_move_conc must be positive and move_conc and sched not NULL");
  if (base && base->n_parts >= (1 << WAVE_PART_BITS))
    throw_err(BLANCE_ERR_UNSUPPORTED, std::string(name) + ": 2^29 or more partitions");
  if (base && (long long)n_move_conc * std::max(0, base->n_parts) > INT32_MAX)
    throw_err(BLANCE_ERR_UNSUPPORTED, std::string(name) + ": n_move_conc x n_parts exceeds 2^31 - 1");
  SchedReq sr;
  sr.nc = n_move_conc;
  sr.out = sched;
  for (int k = 0; k < n_move_conc; ++k) sr.count.push_back(move_conc[k] <= 0 ? 1 : move_conc[k]);   // orchestrate.go:484-487
  if (base && base->n_node_ids > 0) {
    sr.mover.assign((size_t)base->n_node_ids, 0);
    for (int q = 0; q < base->n_node_ids; ++q) sr.mover[(size_t)q] = node_has_mover ? (node_has_mover[q] != 0) : (q < base->n_nodes);
  }
  if (n > 0 && sc && out)
    for (int i = 0; i < n; ++i)
      for (int k = 0; k < n_move_conc; ++k) {
        blance_scenario_schedule_out& o = sched[(size_t)i * n_move_conc + k];
        o.rounds = 0; o.moves_done = 0; o.stuck_parts = 0; o.max_batch = 0;
      }
  return sr;
}

extern "C" int blance_plan_scenarios_schedule(blance_ctx* ctx, const blance_plan_in* base, int32_t n, const blance_scenario* sc,
                                              const blance_scenario_opts* opts, int32_t favor_min_nodes, int32_t max_concurrent,
                                              int32_t n_move_conc, const int32_t* move_conc, const uint8_t* node_has_mover,
                                              blance_scenario_out* out, blance_scenario_schedule_out* sched) {
  return entry(ctx, [&](Device&) {
    const char* name = "blance_plan_scenarios_schedule";
    if (!ctx) throw_err(BLANCE_ERR_INVALID_ARG, "ctx is NULL");
    const SchedReq sr = sched_req(name, base, n, sc, out, n_move_conc, move_conc, node_has_mover, sched);
    plan_scenarios(ctx, name, base, n, sc, opts, favor_min_nodes, max_concurrent, out, &sr);
  });
}

extern "C" int blance_plan_scenarios_audit(blance_ctx* ctx, const blance_plan_in* base, int32_t n, const blance_scenario* sc,
                                           const blance_scenario_opts* opts, int32_t favor_min_nodes, int32_t max_concurrent,
                                           int32_t n_move_conc, const int32_t* move_conc, const uint8_t* node_has_mover,
                                           blance_scenario_out* out, blance_scenario_schedule_out* sched,
                                           const blance_audit_opts* aopts, blance_audit_out* audit) {
  return entry(ctx, [&](Device&) {
    const std::string name = "blance_plan_scenarios_audit";
    if (!base) throw_err(BLANCE_ERR_INVALID_ARG, name + ": base is NULL");
    const AuditReq ar = check_audit_opts(name, aopts, base->n_node_ids, audit);
    const bool no_sched = n_move_conc == 0 && !move_conc && !sched;
    SchedReq sr;
    if (!no_sched) sr = sched_req(name.c_str(), base, n, sc, out, n_move_conc, move_conc, node_has_mover, sched);
    if (n > 0 && sc)
      for (int i = 0; i < n; ++i) {
        const blance_plan_in in = scenario_in(*base, sc[i], opts_of(opts, i));
        check_audit_model(name + ": scenario " + std::to_string(i), &in);
      }
    need_ctx(ctx);
    plan_scenarios(ctx, name.c_str(), base, n, sc, opts, favor_min_nodes, max_concurrent, out, no_sched ? nullptr : &sr, &ar);
  });
}

// blance_map_audit / blance_plan_audit: one audit on buffers of its own.
static void audit_one(blance_ctx* dev, const AuditBufs& b, const AuditReq& ar, const AuditInst& A) {
  std::vector<AuditInst> insts{A};
  audit_run(dev, b, ar, insts);
  std::vector<long long> host;
  audit_fetch(dev, b, 0, host, *ar.out);
  CUDA(cudaStreamSynchronize(dev->stream));
  audit_unpack(dev, b, A.n_rules, host, *ar.out);
}

extern "C" int blance_map_audit(blance_ctx* ctx, const blance_plan_in* model, const int32_t* rows, const uint8_t* shape,
                                const blance_audit_opts* opts, blance_audit_out* out) {
  return entry(ctx, [&](Device& device) {
    const std::string name = "blance_map_audit";
    check_audit_model(name, model);
    const AuditReq ar = check_audit_opts(name, opts, model->n_node_ids, out);
    const size_t P = (size_t)model->n_parts, SL = (size_t)model->n_slots, S = (size_t)model->n_states;
    if (P * SL > 0 && !rows) throw_err(BLANCE_ERR_INVALID_ARG, name + ": rows is NULL");
    if (P * S > 0 && !shape) throw_err(BLANCE_ERR_INVALID_ARG, name + ": shape is NULL");
    need_ctx(ctx);
    blance_ctx* dev = device();
    cudaStream_t st = dev->stream;
    AuditInst A = audit_inst(*model);
    int32_t* d_rows = nullptr;
    uint8_t* d_shape = nullptr;
    uint32_t* d_mask = nullptr;
    const size_t mw = (size_t)mask_words(*model);
    Arena a;
    AuditBufs b;
    a.add(d_rows, P * SL); a.add(d_shape, P * S); a.add(d_mask, mw);
    audit_slices(a, b, ar, 1, model->n_states, A.n_rules, model->n_node_ids, model->n_nodes, model->n_parts, out->part_flags != nullptr);
    a.alloc(st, "the audit");
    if (P * SL) CUDA(cudaMemcpyAsync(d_rows, rows, sizeof(int32_t) * P * SL, cudaMemcpyHostToDevice, st));
    if (P * S) CUDA(cudaMemcpyAsync(d_shape, shape, P * S, cudaMemcpyHostToDevice, st));
    if (mw) CUDA(cudaMemcpyAsync(d_mask, model->ie_mask, sizeof(uint32_t) * mw, cudaMemcpyHostToDevice, st));
    A.rows = d_rows; A.shape8 = d_shape; A.ie_mask = d_mask; A.stride = model->n_slots;
    audit_one(dev, b, ar, A);
  });
}

extern "C" int blance_plan_audit(blance_ctx* ctx, blance_plan* plan, const blance_audit_opts* opts, blance_audit_out* out) {
  return entry(ctx, [&](Device& device) {
    const std::string name = "blance_plan_audit";
    if (!plan) throw_err(BLANCE_ERR_INVALID_ARG, name + ": plan is NULL");
    if (plan->n_inst != 1) throw_err(BLANCE_ERR_INVALID_ARG, name + ": the plan is not a single instance");
    const DInst& D = plan->h_insts[0];
    if (D.has_hier_rules && D.n_rules > AUDIT_RULES_MAX) throw_err(BLANCE_ERR_UNSUPPORTED, name + ": more than 256 hierarchy rules");
    if (D.has_hier_rules && (D.rule_off[0] < 0 || D.rule_off[D.S] > D.n_rules)) throw_err(BLANCE_ERR_INVALID_ARG, name + ": rule_off points outside the rules");
    const AuditReq ar = check_audit_opts(name, opts, D.NU, out);
    need_ctx(ctx);
    blance_ctx* dev = device();
    AuditInst A = audit_inst(D);
    A.rows = plan->pool.rows + D.rows_off; A.meta = plan->pool.pmeta + D.part_off;
    A.ie_mask = plan->pool.ie_mask + D.mask_off; A.stride = D.SLP;
    Arena a;
    AuditBufs b;
    audit_slices(a, b, ar, 1, D.S, A.n_rules, D.NU, D.N, D.PU, out->part_flags != nullptr);
    a.alloc(dev->stream, "the audit");
    audit_one(dev, b, ar, A);
  });
}

extern "C" int blance_calc_partition_moves(blance_ctx* ctx, int32_t n_parts, int32_t n_states, int32_t n_visit_states,
                                           const int32_t* state_slot_off, const int32_t* beg_rows,
                                           const int32_t* end_rows, int32_t favor_min_nodes, int32_t max_ops,
                                           int32_t* op_node, uint8_t* op_state, uint8_t* op_kind, int32_t* op_count) {
  return entry(ctx, [&](Device& device) {
    if (!ctx) throw_err(BLANCE_ERR_INVALID_ARG, "ctx is NULL");
    if (n_parts < 0 || n_states < 0 || n_states >= 255 || n_visit_states < 0 || n_visit_states > n_states || !state_slot_off || max_ops < 0)
      throw_err(BLANCE_ERR_INVALID_ARG, "blance_calc_partition_moves: bad sizes (at most 254 states: 0xFF is the \"\" state of a del op)");
    if (max_ops < 2 * state_slot_off[n_states])
      throw_err(BLANCE_ERR_INVALID_ARG, "blance_calc_partition_moves: max_ops must be at least 2 * n_slots (no op may be dropped)");
    if (n_parts == 0) return;
    const int SL = state_slot_off[n_states];
    if (SL > 0 && (!beg_rows || !end_rows)) throw_err(BLANCE_ERR_INVALID_ARG, "rows are NULL");
    if (!op_node || !op_state || !op_kind || !op_count) throw_err(BLANCE_ERR_INVALID_ARG, "outputs are NULL");
    blance_ctx* dev = device();
    cudaStream_t st = dev->stream;
    const size_t rows = (size_t)n_parts * std::max(SL, 1), ops = (size_t)n_parts * std::max(max_ops, 1);
    int32_t *d_slot, *d_beg, *d_end, *d_node, *d_cnt;
    uint8_t *d_state, *d_kind;
    Arena a;
    a.add(d_slot, (size_t)n_states + 1); a.add(d_beg, rows); a.add(d_end, rows);
    a.add(d_node, ops); a.add(d_state, ops); a.add(d_kind, ops); a.add(d_cnt, (size_t)n_parts);
    a.alloc(st, "the partition moves");
    CUDA(cudaMemcpyAsync(d_slot, state_slot_off, sizeof(int32_t) * (n_states + 1), cudaMemcpyHostToDevice, st));
    if (SL > 0) {
      CUDA(cudaMemcpyAsync(d_beg, beg_rows, sizeof(int32_t) * (size_t)n_parts * SL, cudaMemcpyHostToDevice, st));
      CUDA(cudaMemcpyAsync(d_end, end_rows, sizeof(int32_t) * (size_t)n_parts * SL, cudaMemcpyHostToDevice, st));
    }
    launch(dev, k_calc_moves, grid_for(dev, n_parts, 128), 128, 0, n_parts, n_states, n_visit_states, d_slot, d_beg, d_end,
           favor_min_nodes, max_ops, d_node, d_state, d_kind, d_cnt);
    if (max_ops > 0) {
      CUDA(cudaMemcpyAsync(op_node, d_node, sizeof(int32_t) * (size_t)n_parts * max_ops, cudaMemcpyDeviceToHost, st));
      CUDA(cudaMemcpyAsync(op_state, d_state, (size_t)n_parts * max_ops, cudaMemcpyDeviceToHost, st));
      CUDA(cudaMemcpyAsync(op_kind, d_kind, (size_t)n_parts * max_ops, cudaMemcpyDeviceToHost, st));
    }
    CUDA(cudaMemcpyAsync(op_count, d_cnt, sizeof(int32_t) * (size_t)n_parts, cudaMemcpyDeviceToHost, st));
    CUDA(cudaStreamSynchronize(st));
  });
}

// ---------------------------------------------------------------------------------------
// Move lists for the orchestrator (orchestrate.go:273-287, 749-763, 177-186), resident on the device.

struct blance_moves {
  int32_t n_parts = 0, n_node_ids = 0;
  long long total_ops = 0;
  std::vector<int32_t> slot_off;     // [n_states + 1], host copy of the slot layout
  Arena arena;
  int32_t* d_beg = nullptr;          // [n_parts][n_slots] the beg rows (blance_moves_exposure)
  long long* d_off = nullptr;        // [n_parts + 1]
  int32_t* d_node = nullptr; uint8_t* d_state = nullptr; uint8_t* d_kind = nullptr;   // CSR ops
  int32_t* d_next = nullptr;         // [n_parts] cursors of the current round
  uint32_t *d_key = nullptr, *d_key2 = nullptr; int32_t *d_val = nullptr, *d_val2 = nullptr;   // [n_parts]
  int32_t* d_ncnt = nullptr; int32_t* d_noff = nullptr; unsigned long long* d_nbest = nullptr; int32_t* d_best = nullptr;   // per node
  void* d_tmp = nullptr; size_t tmp_bytes = 0;
  // the last blance_moves_schedule: round_off [rounds + 1] and sched_op [moves_done]
  std::unique_ptr<Arena> sched;
  long long *round_off = nullptr, *sched_op = nullptr;
  int32_t sched_rounds = -1;         // -1: no schedule yet
  long long sched_moves = 0;
};

extern "C" int blance_moves_create(blance_ctx* ctx, int32_t n_parts, int32_t n_states, int32_t n_visit_states,
                                   const int32_t* state_slot_off, const int32_t* beg_rows, const int32_t* end_rows,
                                   int32_t favor_min_nodes, int32_t n_node_ids, blance_moves** out, int64_t* total_ops) {
  return entry(ctx, [&](Device& device) {
    if (!ctx) throw_err(BLANCE_ERR_INVALID_ARG, "ctx is NULL");
    if (!out) throw_err(BLANCE_ERR_INVALID_ARG, "blance_moves_create: out is NULL");
    *out = nullptr;
    if (n_parts < 0 || n_states < 0 || n_states >= 255 || n_visit_states < 0 || n_visit_states > n_states || !state_slot_off || n_node_ids < 0)
      throw_err(BLANCE_ERR_INVALID_ARG, "blance_moves_create: bad sizes");
    const int SL = state_slot_off[n_states];
    if (n_parts > 0 && SL > 0 && (!beg_rows || !end_rows)) throw_err(BLANCE_ERR_INVALID_ARG, "rows are NULL");
    blance_ctx* dev = device();
    cudaStream_t st = dev->stream;
    const int max_ops = std::max(1, 2 * SL);
    const size_t P = (size_t)std::max(n_parts, 1), NN = (size_t)std::max(n_node_ids, 1);
    size_t scan_tmp = 0, sort_tmp = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, (const int32_t*)nullptr, (long long*)nullptr, n_parts + 1, st);
    cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const int32_t*)nullptr, (int32_t*)nullptr, n_parts, 0, 32, st);
    std::unique_ptr<blance_moves> mv(new blance_moves());
    mv->n_parts = n_parts; mv->n_node_ids = n_node_ids;
    mv->slot_off.assign(state_slot_off, state_slot_off + n_states + 1);
    mv->tmp_bytes = std::max(scan_tmp, sort_tmp) + 256;
    // scratch of the construction (end rows, padded ops, counts) lives in the same arena and is simply left unused
    // later; the beg rows stay for blance_moves_exposure
    int32_t *d_slot, *&d_beg = mv->d_beg, *d_end, *p_node, *d_cnt;
    uint8_t *p_state, *p_kind;
    Arena& a = mv->arena;
    a.add(mv->d_off, P + 2); a.add(mv->d_node, P * max_ops);
    a.add(mv->d_state, P * max_ops); a.add(mv->d_kind, P * max_ops); a.add(mv->d_next, P);
    a.add(mv->d_key, P); a.add(mv->d_key2, P); a.add(mv->d_val, P);
    a.add(mv->d_val2, P); a.add(mv->d_ncnt, NN + 1); a.add(mv->d_noff, NN + 2);
    a.add(mv->d_nbest, NN); a.add(mv->d_best, NN); a.add(mv->d_tmp, mv->tmp_bytes);
    a.add(d_slot, (size_t)n_states + 1); a.add(d_beg, P * std::max(SL, 1));
    a.add(d_end, P * std::max(SL, 1)); a.add(p_node, P * max_ops);
    a.add(p_state, P * max_ops); a.add(p_kind, P * max_ops); a.add(d_cnt, P + 1);
    a.alloc(st, "the move lists");
    CUDA(cudaMemcpyAsync(d_slot, state_slot_off, sizeof(int32_t) * (n_states + 1), cudaMemcpyHostToDevice, st));
    if (n_parts > 0 && SL > 0) {
      CUDA(cudaMemcpyAsync(d_beg, beg_rows, sizeof(int32_t) * (size_t)n_parts * SL, cudaMemcpyHostToDevice, st));
      CUDA(cudaMemcpyAsync(d_end, end_rows, sizeof(int32_t) * (size_t)n_parts * SL, cudaMemcpyHostToDevice, st));
    }
    CUDA(cudaMemsetAsync(d_cnt, 0, sizeof(int32_t) * (P + 1), st));
    if (n_parts > 0) {
      launch(dev, k_calc_moves, grid_for(dev, n_parts, 128), 128, 0, n_parts, n_states, n_visit_states, d_slot, d_beg, d_end,
             favor_min_nodes, max_ops, p_node, p_state, p_kind, d_cnt);
      size_t tb = mv->tmp_bytes;
      CUDA(cub::DeviceScan::ExclusiveSum(mv->d_tmp, tb, d_cnt, mv->d_off, n_parts + 1, st));
      launch(dev, k_moves_compact, grid_for(dev, n_parts, 128), 128, 0, n_parts, max_ops, mv->d_off, d_cnt, p_node, p_state,
             p_kind, mv->d_node, mv->d_state, mv->d_kind);
      CUDA(cudaMemcpyAsync(&mv->total_ops, mv->d_off + n_parts, sizeof(long long), cudaMemcpyDeviceToHost, st));
    } else {
      CUDA(cudaMemsetAsync(mv->d_off, 0, sizeof(long long) * (P + 2), st));
    }
    CUDA(cudaStreamSynchronize(st));
    if (total_ops) *total_ops = mv->total_ops;
    *out = mv.release();
  });
}

extern "C" int blance_moves_fetch(blance_ctx* ctx, blance_moves* mv, int64_t* op_off, int32_t* op_node, uint8_t* op_state, uint8_t* op_kind) {
  return entry(ctx, [&](Device& device) {
    if (!ctx || !mv) throw_err(BLANCE_ERR_INVALID_ARG, "ctx or moves is NULL");
    cudaStream_t st = device()->stream;
    if (op_off) CUDA(cudaMemcpyAsync(op_off, mv->d_off, sizeof(long long) * ((size_t)mv->n_parts + 1), cudaMemcpyDeviceToHost, st));
    if (mv->total_ops > 0) {
      if (op_node) CUDA(cudaMemcpyAsync(op_node, mv->d_node, sizeof(int32_t) * (size_t)mv->total_ops, cudaMemcpyDeviceToHost, st));
      if (op_state) CUDA(cudaMemcpyAsync(op_state, mv->d_state, (size_t)mv->total_ops, cudaMemcpyDeviceToHost, st));
      if (op_kind) CUDA(cudaMemcpyAsync(op_kind, mv->d_kind, (size_t)mv->total_ops, cudaMemcpyDeviceToHost, st));
    }
    CUDA(cudaStreamSynchronize(st));
  });
}

extern "C" int blance_moves_available(blance_ctx* ctx, blance_moves* mv, const int32_t* next, int32_t* node_off, int32_t* node_parts,
                                      int32_t* best_part) {
  return entry(ctx, [&](Device& device) {
    if (!ctx || !mv || !next) throw_err(BLANCE_ERR_INVALID_ARG, "ctx, moves or next is NULL");
    blance_ctx* dev = device();
    cudaStream_t st = dev->stream;
    const int P = mv->n_parts, NN = mv->n_node_ids;
    CUDA(cudaMemsetAsync(mv->d_ncnt, 0, sizeof(int32_t) * ((size_t)NN + 1), st));
    CUDA(cudaMemsetAsync(mv->d_nbest, 0xFF, sizeof(unsigned long long) * (size_t)std::max(NN, 1), st));
    if (P > 0) {
      CUDA(cudaMemcpyAsync(mv->d_next, next, sizeof(int32_t) * (size_t)P, cudaMemcpyHostToDevice, st));
      launch(dev, k_moves_next, grid_for(dev, P, 256), 256, 0, P, NN, mv->d_off, mv->d_node, mv->d_kind, mv->d_next, mv->d_key,
             mv->d_val, mv->d_ncnt, mv->d_nbest);
      size_t tb = mv->tmp_bytes;
      CUDA(cub::DeviceRadixSort::SortPairs(mv->d_tmp, tb, mv->d_key, mv->d_key2, mv->d_val, mv->d_val2, P, 0, 32, st));   // stable: partitions stay ascending
    }
    {
      size_t tb = mv->tmp_bytes;
      CUDA(cub::DeviceScan::ExclusiveSum(mv->d_tmp, tb, mv->d_ncnt, mv->d_noff, NN + 1, st));
    }
    if (NN > 0) launch(dev, k_moves_best, (NN + 255) / 256, 256, 0, NN, mv->d_nbest, mv->d_best);
    int32_t n_avail = 0;
    CUDA(cudaMemcpyAsync(&n_avail, mv->d_noff + NN, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    if (node_off) CUDA(cudaMemcpyAsync(node_off, mv->d_noff, sizeof(int32_t) * ((size_t)NN + 1), cudaMemcpyDeviceToHost, st));
    if (best_part && NN > 0) CUDA(cudaMemcpyAsync(best_part, mv->d_best, sizeof(int32_t) * (size_t)NN, cudaMemcpyDeviceToHost, st));
    CUDA(cudaStreamSynchronize(st));
    if (node_parts && n_avail > 0) {
      CUDA(cudaMemcpyAsync(node_parts, mv->d_val2, sizeof(int32_t) * (size_t)n_avail, cudaMemcpyDeviceToHost, st));
      CUDA(cudaStreamSynchronize(st));
    }
  });
}

// The lock-step schedule (include/blance_b200.h) of the handle's CSR ops: one instance of the wave engine
// (wave_schedule.cuh), which also writes round_off and sched_op into the handle.
extern "C" int blance_moves_schedule(blance_ctx* ctx, blance_moves* mv, int32_t max_concurrent_per_node,
                                     const uint8_t* node_has_mover, blance_schedule_out* out) {
  return entry(ctx, [&](Device& device) {
    if (!ctx || !mv || !out) throw_err(BLANCE_ERR_INVALID_ARG, "blance_moves_schedule: ctx, moves or out is NULL");
    std::memset(out, 0, sizeof *out);
    if (mv->n_parts >= (1 << WAVE_PART_BITS)) throw_err(BLANCE_ERR_UNSUPPORTED, "blance_moves_schedule: 2^29 or more partitions");
    blance_ctx* dev = device();
    cudaStream_t st = dev->stream;
    const int32_t P = mv->n_parts, NN = mv->n_node_ids;
    const long long T = mv->total_ops;
    SchedReq sr;
    sr.nc = 1;
    sr.count = {max_concurrent_per_node <= 0 ? 1 : max_concurrent_per_node};   // orchestrate.go:484-487
    sr.mover.assign((size_t)NN, 1);
    if (node_has_mover)
      for (int q = 0; q < NN; ++q) sr.mover[(size_t)q] = node_has_mover[q] != 0;
    WSched W{};
    void* tmp = nullptr;
    size_t tmp_bytes = 0;
    unsigned long long* d_ops = nullptr;
    Arena scratch;
    sched_slices(scratch, 1, 1, P, NN, 0, T, W, tmp, tmp_bytes, st);
    scratch.add(d_ops, (size_t)std::max(NN, 1));
    scratch.alloc(st, "the schedule scratch");
    // results: round_off [T + 2] (R <= T) and sched_op [T], kept in the handle
    mv->sched.reset();
    mv->sched_rounds = -1;
    std::unique_ptr<Arena> res(new Arena());
    res->add(mv->round_off, (size_t)(T + 2));
    res->add(mv->sched_op, (size_t)std::max(T, 1ll));
    res->alloc(st, "the schedule");
    mv->sched = std::move(res);
    W.op_off = mv->d_off; W.op_node = mv->d_node; W.op_kind = mv->d_kind;
    W.round_off = mv->round_off; W.sched_op = mv->sched_op;
    CUDA(cudaEventRecord(dev->ev[0], st));
    // segment capacities: the ops on each node
    std::vector<long long> ops((size_t)NN);
    CUDA(cudaMemsetAsync(d_ops, 0, sizeof(unsigned long long) * (size_t)NN, st));
    if (T > 0 && NN > 0) launch(dev, k_wave_node_ops, grid_for(dev, T, 256), 256, 0, T, mv->d_node, NN, d_ops);
    CUDA(cudaMemcpyAsync(ops.data(), d_ops, sizeof(long long) * (size_t)NN, cudaMemcpyDeviceToHost, st));
    CUDA(cudaStreamSynchronize(st));
    const std::vector<unsigned long long> scal = wave_schedule(dev, "blance_moves_schedule", sr, W, tmp, tmp_bytes, ops.data());
    CUDA(cudaEventRecord(dev->ev[1], st));
    CUDA(cudaStreamSynchronize(st));
    float ms = 0.f;
    cudaEventElapsedTime(&ms, dev->ev[0], dev->ev[1]);
    mv->sched_rounds = (int32_t)scal[0];
    mv->sched_moves = (long long)scal[1];
    out->rounds = (int32_t)scal[0];
    out->moves_done = (int64_t)scal[1];
    out->stuck_parts = (int64_t)scal[2];
    out->max_batch = (int32_t)scal[3];
    out->device_ms = ms;
  });
}

extern "C" int blance_moves_schedule_fetch(blance_ctx* ctx, blance_moves* mv, int64_t* round_off, int64_t* sched_op) {
  return entry(ctx, [&](Device& device) {
    if (!ctx || !mv) throw_err(BLANCE_ERR_INVALID_ARG, "blance_moves_schedule_fetch: ctx or moves is NULL");
    cudaStream_t st = device()->stream;
    if (mv->sched_rounds < 0 || !mv->sched)
      throw_err(BLANCE_ERR_INVALID_ARG, "blance_moves_schedule_fetch: no schedule was computed on this handle");
    if (round_off) CUDA(cudaMemcpyAsync(round_off, mv->round_off, sizeof(long long) * ((size_t)mv->sched_rounds + 1), cudaMemcpyDeviceToHost, st));
    if (sched_op && mv->sched_moves > 0)
      CUDA(cudaMemcpyAsync(sched_op, mv->sched_op, sizeof(long long) * (size_t)mv->sched_moves, cudaMemcpyDeviceToHost, st));
    CUDA(cudaStreamSynchronize(st));
  });
}

// The exposure of the handle's last schedule (exposure.cuh; include/blance_b200.h).
extern "C" int blance_moves_exposure(blance_ctx* ctx, blance_moves* mv, const blance_exposure_in* in, blance_exposure_out* out) {
  return entry(ctx, [&](Device& device) {
    const std::string name = "blance_moves_exposure";
    if (!ctx || !mv || !in || !out) throw_err(BLANCE_ERR_INVALID_ARG, name + ": ctx, moves, in or out is NULL");
    if (mv->sched_rounds < 0 || !mv->sched) throw_err(BLANCE_ERR_INVALID_ARG, name + ": no schedule was computed on this handle");
    const int S = (int)mv->slot_off.size() - 1, SL = mv->slot_off[(size_t)S];
    if (S > BL_S_MAX) throw_err(BLANCE_ERR_UNSUPPORTED, name + ": more than 8 states");
    if (SL > BL_SLP_MAX) throw_err(BLANCE_ERR_UNSUPPORTED, name + ": more than 32 slots per row");
    if (S > 0 && !in->state_constraints) throw_err(BLANCE_ERR_INVALID_ARG, name + ": state_constraints is NULL");
    for (int s = 0; s < S; ++s)
      if (in->state_constraints[s] < 0) throw_err(BLANCE_ERR_INVALID_ARG, name + ": negative state constraint");
    if (in->top_state < -1 || in->top_state >= S) throw_err(BLANCE_ERR_INVALID_ARG, name + ": top_state outside [-1, n_states)");
    const int NU = mv->n_node_ids;
    check_forest(name, in->n_domains, in->domain_parent, NU);
    // a scheduled op emits at most two ancestor chains of AUDIT_DEPTH_MAX + 1 vertices; the event count is an int
    if ((out->dom_peak || out->dom_peak_round) && 2ll * (AUDIT_DEPTH_MAX + 1) * mv->sched_moves >= (1ll << 31))
      throw_err(BLANCE_ERR_UNSUPPORTED, name + ": dom_peak needs 34 x moves_done < 2^31");
    blance_ctx* dev = device();
    cudaStream_t st = dev->stream;
    const int P = mv->n_parts, R = mv->sched_rounds;
    const long long T = mv->total_ops, M = mv->sched_moves, R1 = (long long)R + 1;
    const int V = NU + in->n_domains;
    const bool dom = out->dom_peak || out->dom_peak_round;
    ExpoArgs E{};
    E.op_off = mv->d_off; E.op_node = mv->d_node; E.op_state = mv->d_state; E.op_kind = mv->d_kind; E.beg = mv->d_beg;
    E.P = P; E.SL = SL; E.S = S; E.NU = NU; E.R = R; E.top = in->top_state;
    for (int s = 0; s < S; ++s) { E.constraints[s] = in->state_constraints[s]; E.slot_off[s] = mv->slot_off[(size_t)s]; }
    E.slot_off[S] = SL;
    int32_t* op_round = nullptr;
    long long* stats = nullptr;
    int32_t* parent = nullptr;
    unsigned long long* dom_key = nullptr;
    long long* ev_off = nullptr;
    size_t scan_tmp = 0;
    void* tmp = nullptr;
    CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, (const long long*)nullptr, (long long*)nullptr, P + 1, st));
    Arena a;
    a.add(op_round, (size_t)std::max(T, 1ll)); a.add(E.diff, (size_t)(BLANCE_EXPO_N * R1)); a.add(stats, 3 * BLANCE_EXPO_N);
    if (out->part_min_copies) a.add(E.part_min, (size_t)P);
    if (out->part_no_top) a.add(E.part_notop, (size_t)P);
    if (out->part_flags) a.add(E.part_flags, (size_t)P);
    if (dom) {
      if (in->domain_parent) a.add(parent, (size_t)V);
      a.add(E.dom_base, (size_t)V); a.add(dom_key, (size_t)V);
      a.add(E.ev_count, (size_t)P + 1); a.add(ev_off, (size_t)P + 1); a.add(tmp, scan_tmp);
    }
    a.alloc(st, "the exposure");
    E.op_round = op_round; E.dom_parent = parent;
    CUDA(cudaEventRecord(dev->ev[0], st));
    if (parent) CUDA(cudaMemcpyAsync(parent, in->domain_parent, sizeof(int32_t) * (size_t)V, cudaMemcpyHostToDevice, st));
    CUDA(cudaMemsetAsync(op_round, 0xFF, sizeof(int32_t) * (size_t)std::max(T, 1ll), st));
    CUDA(cudaMemsetAsync(E.diff, 0, sizeof(long long) * (size_t)(BLANCE_EXPO_N * R1), st));
    if (dom && V > 0) CUDA(cudaMemsetAsync(E.dom_base, 0, sizeof(long long) * (size_t)V, st));
    if (M > 0) launch(dev, k_expo_op_round, grid_for(dev, M, 256), 256, 0, M, R, (const long long*)mv->round_off, (const long long*)mv->sched_op, op_round);
    if (P > 0) launch(dev, k_expo_walk<0>, grid_for(dev, P, 256), 256, 0, E);
    launch(dev, k_expo_series, BLANCE_EXPO_N, 512, 0, E.diff, R, stats);
    // fault domains: (vertex, t, +-1) events where a partition's deepest common ancestor changes, sized exactly by a
    // counting walk, sorted by (vertex, t), merged per key, scanned per vertex; dom_key keeps each vertex's maximum
    std::unique_ptr<Arena> ev;
    if (dom && V > 0) {
      launch(dev, k_expo_dom_init, grid_for(dev, V, 256), 256, 0, V, (const long long*)E.dom_base, dom_key);
      long long n_ev = 0;
      if (P > 0 && M > 0) {
        CUDA(cudaMemsetAsync(E.ev_count + P, 0, sizeof(long long), st));
        launch(dev, k_expo_walk<1>, grid_for(dev, P, 256), 256, 0, E);
        CUDA(cub::DeviceScan::ExclusiveSum(tmp, scan_tmp, E.ev_count, ev_off, P + 1, st));
        CUDA(cudaMemcpyAsync(&n_ev, ev_off + P, sizeof(long long), cudaMemcpyDeviceToHost, st));
        CUDA(cudaStreamSynchronize(st));
        E.ev_off = ev_off;
      }
      if (n_ev > 0) {
        const int NE = (int)n_ev;
        int vbits = 1;
        while ((1ll << vbits) < V) ++vbits;
        unsigned long long *k2, *uk;
        int32_t *v2, *uv, *run;
        int* n_runs;
        size_t sort_b = 0, red_b = 0, scan_b = 0;
        CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_b, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                             (const int32_t*)nullptr, (int32_t*)nullptr, NE, 0, 32 + vbits, st));
        CUDA(cub::DeviceReduce::ReduceByKey(nullptr, red_b, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                            (const int32_t*)nullptr, (int32_t*)nullptr, (int*)nullptr, ExpoSum(), NE, st));
        CUDA(cub::DeviceScan::InclusiveScanByKey(nullptr, scan_b, (const unsigned long long*)nullptr, (const int32_t*)nullptr,
                                                 (int32_t*)nullptr, ExpoSum(), NE, ExpoSameVertex(), st));
        size_t ev_tmp_b = std::max(sort_b, std::max(red_b, scan_b));
        void* ev_tmp = nullptr;
        ev.reset(new Arena());
        ev->add(E.ev_key, (size_t)NE); ev->add(E.ev_val, (size_t)NE); ev->add(k2, (size_t)NE); ev->add(v2, (size_t)NE);
        ev->add(uk, (size_t)NE); ev->add(uv, (size_t)NE); ev->add(run, (size_t)NE); ev->add(n_runs, 1); ev->add(ev_tmp, ev_tmp_b);
        ev->alloc(st, "the exposure's fault-domain events");
        launch(dev, k_expo_walk<2>, grid_for(dev, P, 256), 256, 0, E);
        size_t b = ev_tmp_b;
        CUDA(cub::DeviceRadixSort::SortPairs(ev_tmp, b, E.ev_key, k2, E.ev_val, v2, NE, 0, 32 + vbits, st));
        b = ev_tmp_b;
        CUDA(cub::DeviceReduce::ReduceByKey(ev_tmp, b, k2, uk, v2, uv, n_runs, ExpoSum(), NE, st));
        int h_runs = 0;                            // only the merged runs are scanned
        CUDA(cudaMemcpyAsync(&h_runs, n_runs, sizeof(int), cudaMemcpyDeviceToHost, st));
        CUDA(cudaStreamSynchronize(st));
        b = ev_tmp_b;
        CUDA(cub::DeviceScan::InclusiveScanByKey(ev_tmp, b, uk, uv, run, ExpoSum(), h_runs, ExpoSameVertex(), st));
        launch(dev, k_expo_dom_max, grid_for(dev, h_runs, 256), 256, 0, h_runs, (const unsigned long long*)uk,
               (const int32_t*)run, (const long long*)E.dom_base, dom_key);
      }
    }
    CUDA(cudaEventRecord(dev->ev[1], st));
    std::vector<long long> h_stats(3 * BLANCE_EXPO_N);
    std::vector<unsigned long long> h_key(dom ? (size_t)V : 0);
    CUDA(cudaMemcpyAsync(h_stats.data(), stats, sizeof(long long) * h_stats.size(), cudaMemcpyDeviceToHost, st));
    if (out->series) CUDA(cudaMemcpyAsync(out->series, E.diff, sizeof(long long) * (size_t)(BLANCE_EXPO_N * R1), cudaMemcpyDeviceToHost, st));
    if (P > 0) {
      if (out->part_min_copies) CUDA(cudaMemcpyAsync(out->part_min_copies, E.part_min, sizeof(int32_t) * (size_t)P, cudaMemcpyDeviceToHost, st));
      if (out->part_no_top) CUDA(cudaMemcpyAsync(out->part_no_top, E.part_notop, sizeof(int32_t) * (size_t)P, cudaMemcpyDeviceToHost, st));
      if (out->part_flags) CUDA(cudaMemcpyAsync(out->part_flags, E.part_flags, (size_t)P, cudaMemcpyDeviceToHost, st));
    }
    if (dom && V > 0) CUDA(cudaMemcpyAsync(h_key.data(), dom_key, sizeof(unsigned long long) * (size_t)V, cudaMemcpyDeviceToHost, st));
    CUDA(cudaStreamSynchronize(st));
    out->kernel_ms = 0.f;
    cudaEventElapsedTime(&out->kernel_ms, dev->ev[0], dev->ev[1]);
    out->rounds = R;
    for (int m = 0; m < BLANCE_EXPO_N; ++m) {
      out->peak[m] = h_stats[(size_t)(3 * m)];
      out->peak_round[m] = (int32_t)h_stats[(size_t)(3 * m + 1)];
      out->area[m] = h_stats[(size_t)(3 * m + 2)];
    }
    for (int v = 0; v < (dom ? V : 0); ++v) {
      if (out->dom_peak) out->dom_peak[v] = (int64_t)(h_key[(size_t)v] >> 32);
      if (out->dom_peak_round) out->dom_peak_round[v] = (int32_t)(0xFFFFFFFFu - (uint32_t)h_key[(size_t)v]);
    }
  });
}

extern "C" void blance_moves_free(blance_ctx* ctx, blance_moves* mv) {
  std::unique_ptr<blance_moves> owner(mv);   // freed on the stream it was allocated on, also when ctx is NULL
  if (ctx && mv)
    entry(ctx, [&](Device& device) {
      blance_ctx* dev = device();
      owner.reset();
      CUDA(cudaStreamSynchronize(dev->stream));
    });
}
