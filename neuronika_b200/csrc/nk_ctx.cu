// Context, buffers, copies: the device-side replacement of cuda::Device / cuda::CuArray
// (reference: neuronika-variable/src/cuda/device.rs:11-75, cuda/cuarray.rs:10-171).
#include <stdarg.h>

#include <new>

#include "nk_internal.cuh"

static thread_local std::string g_null_ctx_error;

int nk_set_error(nk_ctx* ctx, int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  if (ctx)
    ctx->last_error = buf;
  else
    g_null_ctx_error = buf;
  return code;
}

// ---- arena of the step being captured
static inline size_t arena_round(size_t b) { return (b + 255) & ~size_t(255); }

static bool in_arena(nk_ctx* ctx, const void* p, nk_graph** owner) {
  const char* c = static_cast<const char*>(p);
  for (nk_graph* g : ctx->graphs)
    if (c >= g->arena && c < g->arena + g->arena_bytes) {
      if (owner) *owner = g;
      return true;
    }
  return false;
}

static int arena_alloc(nk_ctx* ctx, size_t bytes, void** out) {
  nk_graph* g = ctx->capturing;
  const size_t need = arena_round(bytes ? bytes : 16);
  auto it = ctx->arena_free.find(need);  // a block of exactly this size freed earlier in the same capture
  if (it != ctx->arena_free.end()) {
    *out = it->second;
    ctx->arena_free.erase(it);
    return NK_OK;
  }
  if (g->arena_used + need > g->arena_bytes)
    return nk_set_error(ctx, NK_ERR_OOM, "capture arena exhausted (%zu of %zu bytes used, %zu more requested): pass a larger "
                        "arena to nk_capture_begin", g->arena_used, g->arena_bytes, need);
  *out = g->arena + g->arena_used;
  g->arena_used += need;
  ctx->capturing_sizes[*out] = need;
  return NK_OK;
}

int nk_workspace(nk_ctx* ctx, size_t bytes, void** out) {
  if (bytes > ctx->workspace_bytes && ctx->capturing)
    return nk_set_error(ctx, NK_ERR_UNSUPPORTED, "the scratch workspace would have to grow (%zu -> %zu bytes) inside a "
                        "capture: run the step once before capturing it", ctx->workspace_bytes, bytes);
  if (bytes > ctx->workspace_bytes) {
    if (ctx->workspace) {
      NK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
      NK_CUDA(ctx, cudaFree(ctx->workspace));
      ctx->workspace = nullptr;
      ctx->workspace_bytes = 0;
    }
    size_t want = bytes < (size_t(8) << 20) ? (size_t(8) << 20) : bytes;
    NK_CUDA(ctx, cudaMalloc(&ctx->workspace, want));
    ctx->workspace_bytes = want;
  }
  *out = ctx->workspace;
  return NK_OK;
}

extern "C" {

const char* nk_version(void) { return "neuronika_b200 0.1 (sm_90a)"; }

int nk_ctx_create(int device, nk_ctx** out) {
  if (!out) return nk_set_error(nullptr, NK_ERR_INVALID_ARG, "nk_ctx_create: out is NULL");
  *out = nullptr;
  nk_ctx* ctx = new (std::nothrow) nk_ctx();
  if (!ctx) return NK_ERR_OOM;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) {
    int rc = nk_set_error(nullptr, NK_ERR_CUDA, "nk_ctx_create: no CUDA device (%s); this library has no CPU fallback",
                          cudaGetErrorString(e));
    delete ctx;
    return rc;
  }
  if (device < 0 || device >= count) {
    delete ctx;
    return nk_set_error(nullptr, NK_ERR_INVALID_ARG, "nk_ctx_create: device %d out of range [0,%d)", device, count);
  }
  ctx->device = device;
  if ((e = cudaSetDevice(device)) != cudaSuccess) {
    delete ctx;
    return nk_set_error(nullptr, NK_ERR_CUDA, "cudaSetDevice(%d): %s", device, cudaGetErrorString(e));
  }
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, device);
  if (prop.major != 9 || prop.minor != 0) {   // sm_90a code (wgmma, setmaxnreg) loads on compute capability 9.0 only
    delete ctx;
    return nk_set_error(nullptr, NK_ERR_UNSUPPORTED, "device %d is sm_%d%d; this library is built for sm_90a only",
                        device, prop.major, prop.minor);
  }
  ctx->sm_count = prop.multiProcessorCount;
  ctx->smem_optin = prop.sharedMemPerBlockOptin;
  cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
  ctx->own_stream = true;
  cudaEventCreate(&ctx->ev0);
  cudaEventCreate(&ctx->ev1);
  // keep freed blocks cached in the stream-ordered pool: the reference rebuilds its graph (and
  // re-allocates every node output and gradient) each step, examples/quickstart.rs:216-227
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
    uint64_t thr = UINT64_MAX;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
  }
  cudaDriverEntryPointQueryResult qres;
  void* fn = nullptr;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess &&
      qres == cudaDriverEntryPointSuccess)
    ctx->encode_tiled = fn;
  cudaGetLastError();
  *out = ctx;
  return NK_OK;
}

int nk_ctx_destroy(nk_ctx* ctx) {
  if (!ctx) return NK_OK;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  nk_comm_destroy(ctx);
  while (!ctx->graphs.empty()) {
    nk_graph* g = ctx->graphs.back();
    if (g == ctx->capturing) {
      cudaGraph_t tmp = nullptr;
      cudaStreamEndCapture(ctx->stream, &tmp);
      if (tmp) cudaGraphDestroy(tmp);
      ctx->capturing = nullptr;
    }
    nk_graph_destroy(ctx, g);
  }
  if (ctx->workspace) cudaFree(ctx->workspace);
  if (ctx->rng_state) cudaFree(ctx->rng_state);
  if (ctx->ev0) cudaEventDestroy(ctx->ev0);
  if (ctx->ev1) cudaEventDestroy(ctx->ev1);
  if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
  return NK_OK;
}

int nk_ctx_set_stream(nk_ctx* ctx, void* cuda_stream) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
  ctx->stream = static_cast<cudaStream_t>(cuda_stream);
  ctx->own_stream = false;
  return NK_OK;
}

void* nk_ctx_stream(nk_ctx* ctx) { return ctx ? ctx->stream : nullptr; }

const char* nk_last_error(nk_ctx* ctx) { return ctx ? ctx->last_error.c_str() : g_null_ctx_error.c_str(); }

int nk_sync(nk_ctx* ctx) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return NK_OK;
}

uint64_t nk_launch_count(nk_ctx* ctx) { return ctx ? ctx->launches : 0; }
int nk_sm_count(nk_ctx* ctx) { return ctx ? ctx->sm_count : 0; }

int nk_gemm_config(nk_ctx* ctx, int engine) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, engine >= NK_GEMM_AUTO && engine <= NK_GEMM_TC, "nk_gemm_config: bad engine %d", engine);
  ctx->gemm_engine = engine;
  return NK_OK;
}
int nk_gemm_f32_config(nk_ctx* ctx, int mode) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, mode >= NK_F32_GEMM_IEEE && mode <= NK_F32_GEMM_TF32X3, "nk_gemm_f32_config: bad mode %d", mode);
  ctx->f32_gemm = mode;
  return NK_OK;
}
int nk_conv_config(nk_ctx* ctx, int engine) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, engine >= NK_CONV_AUTO && engine <= NK_CONV_DIRECT, "nk_conv_config: bad engine %d", engine);
  ctx->conv_engine = engine;
  return NK_OK;
}
int nk_conv_f32_config(nk_ctx* ctx, int mode) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, mode >= NK_F32_GEMM_IEEE && mode <= NK_F32_GEMM_TF32X3, "nk_conv_f32_config: bad mode %d", mode);
  ctx->f32_conv = mode;
  return NK_OK;
}
const char* nk_last_gemm_kernel(nk_ctx* ctx) { return ctx ? ctx->last_gemm_kernel : "none"; }
const char* nk_last_conv_kernel(nk_ctx* ctx) { return ctx ? ctx->last_conv_kernel : "none"; }

int nk_alloc(nk_ctx* ctx, size_t bytes, void** dptr) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, dptr != nullptr, "nk_alloc: dptr is NULL");
  *dptr = nullptr;
  if (bytes == 0) bytes = 16;
  if (ctx->capturing) {
    int rc = arena_alloc(ctx, bytes, dptr);
    if (rc) return rc;
  } else {
    NK_CUDA(ctx, cudaMallocAsync(dptr, bytes, ctx->stream));
  }
  NK_CUDA(ctx, cudaMemsetAsync(*dptr, 0, bytes, ctx->stream));
  return NK_OK;
}

int nk_alloc_uninit(nk_ctx* ctx, size_t bytes, void** dptr) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, dptr != nullptr, "nk_alloc_uninit: dptr is NULL");
  *dptr = nullptr;
  if (bytes == 0) bytes = 16;
  if (ctx->capturing) return arena_alloc(ctx, bytes, dptr);
  NK_CUDA(ctx, cudaMallocAsync(dptr, bytes, ctx->stream));
  return NK_OK;
}

int nk_free(nk_ctx* ctx, void* dptr) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  if (!dptr) return NK_OK;
  nk_graph* owner = nullptr;
  if (in_arena(ctx, dptr, &owner)) {
    // arena memory belongs to its graph: recycled inside the capture that allocated it, otherwise left alone
    if (ctx->capturing && owner == ctx->capturing) {
      auto it = ctx->capturing_sizes.find(dptr);
      if (it != ctx->capturing_sizes.end()) ctx->arena_free.emplace(it->second, dptr);
    }
    return NK_OK;
  }
  if (ctx->capturing) {  // memory from before the capture: a free node for it cannot be recorded; release it afterwards
    ctx->deferred_frees.push_back(dptr);
    return NK_OK;
  }
  cudaError_t e = cudaFreeAsync(dptr, ctx->stream);
  if (e == cudaErrorInvalidValue) {
    // a block of a graph that has been destroyed in the meantime (a handle outlived nk_graph_destroy): its memory went
    // with the arena
    const char* c = static_cast<const char*>(dptr);
    for (auto& r : ctx->retired_arenas)
      if (c >= r.first && c < r.first + r.second) {
        cudaGetLastError();
        return NK_OK;
      }
  }
  NK_CUDA(ctx, e);
  return NK_OK;
}

int nk_h2d(nk_ctx* ctx, void* dst, const void* src, size_t bytes) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  if (bytes == 0) return NK_OK;
  NK_REQUIRE(ctx, dst && src, "nk_h2d: NULL pointer");
  NK_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
  return NK_OK;
}

int nk_d2h(nk_ctx* ctx, void* dst, const void* src, size_t bytes) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  if (bytes == 0) return NK_OK;
  NK_REQUIRE(ctx, dst && src, "nk_d2h: NULL pointer");
  NK_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  NK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return NK_OK;
}

int nk_d2d(nk_ctx* ctx, void* dst, const void* src, size_t bytes) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  if (bytes == 0) return NK_OK;
  NK_REQUIRE(ctx, dst && src, "nk_d2d: NULL pointer");
  NK_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
  return NK_OK;
}

int nk_memset0(nk_ctx* ctx, void* dptr, size_t bytes) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  if (bytes == 0) return NK_OK;
  NK_REQUIRE(ctx, dptr, "nk_memset0: NULL pointer");
  NK_CUDA(ctx, cudaMemsetAsync(dptr, 0, bytes, ctx->stream));
  return NK_OK;
}

int nk_host_alloc(nk_ctx* ctx, size_t bytes, void** hptr) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, hptr != nullptr, "nk_host_alloc: hptr is NULL");
  NK_CUDA(ctx, cudaMallocHost(hptr, bytes ? bytes : 16));
  return NK_OK;
}

int nk_host_free(nk_ctx* ctx, void* hptr) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  if (hptr) NK_CUDA(ctx, cudaFreeHost(hptr));
  return NK_OK;
}

// ---- whole-step capture ---------------------------------------------------------------------------------------
// The reference rebuilds its define-by-run graph every iteration (examples/quickstart.rs:216-227); a training step's
// tape is the same every time, so the kernels it launches can be recorded once and replayed: between begin and end
// every launch, copy and memset this library enqueues on the context stream (and on streams that join it through
// events) goes into a CUDA graph instead of executing, and nk_graph_launch replays the step with ONE driver call.
int nk_capture_begin(nk_ctx* ctx, size_t arena_bytes) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, !ctx->capturing, "nk_capture_begin: a capture is already running on this context");
  NK_REQUIRE(ctx, arena_bytes > 0, "nk_capture_begin: the arena needs a size");
  nk_graph* g = new (std::nothrow) nk_graph();
  if (!g) return NK_ERR_OOM;
  g->ctx = ctx;
  g->arena_bytes = arena_round(arena_bytes);
  cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&g->arena), g->arena_bytes);
  if (e != cudaSuccess) {
    delete g;
    return nk_set_error(ctx, NK_ERR_OOM, "nk_capture_begin: cudaMalloc of a %zu-byte arena failed: %s", arena_bytes,
                        cudaGetErrorString(e));
  }
  e = cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeRelaxed);
  if (e != cudaSuccess) {
    cudaFree(g->arena);
    delete g;
    return nk_set_error(ctx, NK_ERR_CUDA, "cudaStreamBeginCapture failed: %s", cudaGetErrorString(e));
  }
  ctx->graphs.push_back(g);
  ctx->capturing = g;
  ctx->arena_free.clear();
  ctx->capturing_sizes.clear();
  return NK_OK;
}

int nk_capture_end(nk_ctx* ctx, nk_graph** out) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, ctx->capturing && out, "nk_capture_end: no capture is running");
  nk_graph* g = ctx->capturing;
  ctx->capturing = nullptr;
  ctx->arena_free.clear();
  ctx->capturing_sizes.clear();
  *out = nullptr;
  auto drop = [&] {
    for (size_t i = 0; i < ctx->graphs.size(); ++i)
      if (ctx->graphs[i] == g) ctx->graphs.erase(ctx->graphs.begin() + i);
    if (g->exec) cudaGraphExecDestroy(g->exec);
    if (g->graph) cudaGraphDestroy(g->graph);
    cudaFree(g->arena);
    delete g;
  };
  cudaError_t e = cudaStreamEndCapture(ctx->stream, &g->graph);
  for (void* p : ctx->deferred_frees) cudaFreeAsync(p, ctx->stream);
  ctx->deferred_frees.clear();
  if (e != cudaSuccess || !g->graph) {
    drop();
    cudaGetLastError();
    return nk_set_error(ctx, NK_ERR_CUDA, "cudaStreamEndCapture failed: %s (an operation that cannot be captured ran "
                        "inside the step: a synchronous copy, a synchronize, a first-use allocation)", cudaGetErrorString(e));
  }
  size_t n = 0;
  cudaGraphGetNodes(g->graph, nullptr, &n);
  std::vector<cudaGraphNode_t> nodes(n);
  if (n) cudaGraphGetNodes(g->graph, nodes.data(), &n);
  for (size_t i = 0; i < n; ++i) {
    cudaGraphNodeType t;
    if (cudaGraphNodeGetType(nodes[i], &t) == cudaSuccess && t == cudaGraphNodeTypeKernel) g->kernel_nodes++;
  }
  e = cudaGraphInstantiate(&g->exec, g->graph, 0);
  if (e != cudaSuccess) {
    drop();
    return nk_set_error(ctx, NK_ERR_CUDA, "cudaGraphInstantiate failed: %s", cudaGetErrorString(e));
  }
  *out = g;
  return NK_OK;
}

int nk_graph_launch(nk_ctx* ctx, nk_graph* g) {
  if (!ctx || !g) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, g->ctx == ctx && g->exec, "nk_graph_launch: the graph belongs to another context");
  NK_CUDA(ctx, cudaGraphLaunch(g->exec, ctx->stream));
  ctx->launches += g->kernel_nodes;
  return NK_OK;
}

int64_t nk_graph_kernel_count(nk_graph* g) { return g ? int64_t(g->kernel_nodes) : 0; }
size_t nk_graph_arena_used(nk_graph* g) { return g ? g->arena_used : 0; }

int nk_graph_destroy(nk_ctx* ctx, nk_graph* g) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  if (!g) return NK_OK;
  NK_REQUIRE(ctx, g->ctx == ctx && g != ctx->capturing, "nk_graph_destroy: bad graph");
  cudaStreamSynchronize(ctx->stream);
  for (size_t i = 0; i < ctx->graphs.size(); ++i)
    if (ctx->graphs[i] == g) {
      ctx->graphs.erase(ctx->graphs.begin() + i);
      break;
    }
  if (g->exec) cudaGraphExecDestroy(g->exec);
  if (g->graph) cudaGraphDestroy(g->graph);
  if (g->arena) {
    cudaFree(g->arena);
    ctx->retired_arenas.emplace_back(g->arena, g->arena_bytes);
  }
  delete g;
  return NK_OK;
}

int nk_timer_start(nk_ctx* ctx) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_CUDA(ctx, cudaEventRecord(ctx->ev0, ctx->stream));
  return NK_OK;
}

int nk_timer_stop(nk_ctx* ctx, float* ms) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, ms != nullptr, "nk_timer_stop: ms is NULL");
  NK_CUDA(ctx, cudaEventRecord(ctx->ev1, ctx->stream));
  NK_CUDA(ctx, cudaEventSynchronize(ctx->ev1));
  NK_CUDA(ctx, cudaEventElapsedTime(ms, ctx->ev0, ctx->ev1));
  return NK_OK;
}

}  // extern "C"
