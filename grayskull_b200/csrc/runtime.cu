// runtime.cu -- host runtime of libgrayskull_b200.so: error text, launch counter and shared-memory opt-in, workspace
// arenas, tensor-map construction (driver entry point fetched at run time, so the library links
// against cudart only and loads on machines without a GPU driver), memory helpers of the C ABI.
#include <atomic>
#include <map>
#include <mutex>
#include <string.h>
#include <tuple>

#include "common.cuh"

namespace gsb {

static thread_local char t_last_error[512] = "no error";
static std::atomic<unsigned long long> g_launches{0};

int record_error(cudaError_t e, const char *file, int line) {
  snprintf(t_last_error, sizeof(t_last_error), "%s (%s) at %s:%d", cudaGetErrorName(e),
           cudaGetErrorString(e), file, line);
  return static_cast<int>(e);
}

// largest dynamic shared memory each (device, kernel) has been opted in to
static std::mutex g_smem_mutex;
static std::map<std::pair<int, const void *>, size_t> g_smem_optin;

int opt_in_smem(const void *k, size_t smem, const char *file, int line) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return record_error(e, file, line);
  std::lock_guard<std::mutex> lock(g_smem_mutex);
  size_t &have = g_smem_optin[std::make_pair(dev, k)];
  if (have >= smem) return 0;
  e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (e != cudaSuccess) return record_error(e, file, line);
  have = smem;
  return 0;
}
int launched(const char *file, int line) {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : record_error(e, file, line);
}

static int g_force_generic = -1;
bool force_generic() {
  if (g_force_generic < 0) {
    const char *e = getenv("GS_B200_FORCE_GENERIC");
    g_force_generic = (e && e[0] && e[0] != '0') ? 1 : 0;
  }
  return g_force_generic == 1;
}

int sm_count() {
  static std::atomic<int> counts[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  int n = counts[dev].load(std::memory_order_relaxed);
  if (!n) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    counts[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}

// ---- workspace arenas ---------------------------------------------------------------------
struct Arena {
  void *ptr = nullptr;
  size_t bytes = 0;
};
static std::mutex g_ws_mutex;
static std::map<std::tuple<int, cudaStream_t, int>, Arena> g_ws;

// cudaStreamPerThread is one handle for a different stream in each host thread, so its arenas cannot be keyed by the
// handle: each thread keeps its own, and frees them at thread exit once that thread's stream has drained.
struct ThreadArenas {
  std::map<std::pair<int, int>, Arena> m;   // (device, slot)
  ~ThreadArenas() {
    int cur = 0;
    if (cudaGetDevice(&cur) != cudaSuccess) return;   // runtime already shut down
    for (auto &kv : m) {
      if (!kv.second.ptr) continue;
      if (cudaSetDevice(kv.first.first) != cudaSuccess) continue;
      cudaStreamSynchronize(cudaStreamPerThread);
      cudaFree(kv.second.ptr);
    }
    cudaSetDevice(cur);
  }
};
static thread_local ThreadArenas t_ws;
static thread_local int t_ws_error = cudaErrorMemoryAllocation;

bool capturing(cudaStream_t s) {
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(s, &cs) != cudaSuccess) {
    cudaGetLastError();
    return true;   // e.g. the legacy stream while another stream captures: no allocation or sync is legal either
  }
  return cs != cudaStreamCaptureStatusNone;
}

int workspace_error() { return t_ws_error; }

int upload(void *dst, const void *src, size_t bytes, const char *file, int line) {
  cudaStream_t st = nullptr;
  cudaError_t e = cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (st) cudaStreamDestroy(st);
  return e == cudaSuccess ? 0 : record_error(e, file, line);
}

void *workspace(cudaStream_t s, int slot, size_t bytes) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  const bool per_thread = s == cudaStreamPerThread;
  std::unique_lock<std::mutex> lock(g_ws_mutex, std::defer_lock);
  if (!per_thread) lock.lock();
  Arena &a = per_thread ? t_ws.m[std::make_pair(dev, slot)] : g_ws[std::make_tuple(dev, s, slot)];
  if (a.bytes >= bytes && a.ptr) return a.ptr;
  if (capturing(s)) {
    // growing would synchronise, free and allocate inside the capture; the arena stays as it is
    t_ws_error = record_error(cudaErrorStreamCaptureUnsupported, __FILE__, __LINE__);
    snprintf(t_last_error, sizeof(t_last_error),
             "cudaErrorStreamCaptureUnsupported: workspace slot %d must grow to %zu bytes while the stream is capturing; "
             "run the call once at this geometry on this stream before capturing it", slot, bytes);
    return nullptr;
  }
  if (a.ptr) {
    // the old arena may still be in use by work queued on `s`
    cudaStreamSynchronize(s);
    cudaFree(a.ptr);
    a.ptr = nullptr, a.bytes = 0;
  }
  size_t want = bytes + bytes / 4 + 256;
  if (cudaMalloc(&a.ptr, want) != cudaSuccess) {
    a.ptr = nullptr;
    t_ws_error = record_error(cudaGetLastError(), __FILE__, __LINE__);
    return nullptr;
  }
  a.bytes = want;
  return a.ptr;
}

// ---- tensor maps --------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *,
                                  const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                                  const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void *p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

static bool encode3(CUtensorMap *m, const void *base, cuuint64_t d0, cuuint64_t d1, cuuint64_t d2,
                    cuuint64_t stride1_bytes, cuuint64_t stride2_bytes, unsigned b0, unsigned b1) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return false;
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {stride1_bytes, stride2_bytes};
  cuuint32_t box[3] = {b0, b1, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, const_cast<void *>(base), dims, strides, box,
                  estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

bool make_tmap_u8frames(CUtensorMap *m, const void *base, unsigned w, unsigned h, unsigned n,
                        unsigned box_words, unsigned box_rows) {
  if (w % 16u || reinterpret_cast<uintptr_t>(base) % 16u || box_words > 256 || box_rows > 256 ||
      (box_words * 4u) % 16u)
    return false;
  return encode3(m, base, w / 4, h, n, w, static_cast<cuuint64_t>(w) * h, box_words, box_rows);
}

bool make_tmap_u32frames(CUtensorMap *m, const void *base, unsigned w, unsigned h, unsigned n,
                         unsigned box_w, unsigned box_h) {
  if (w % 4u || reinterpret_cast<uintptr_t>(base) % 16u || box_w > 256 || box_h > 256 || box_w % 4u)
    return false;
  return encode3(m, base, w, h, n, static_cast<cuuint64_t>(w) * 4, static_cast<cuuint64_t>(w) * h * 4,
                 box_w, box_h);
}

}  // namespace gsb

// ---- C ABI: runtime + memory helpers --------------------------------------------------------
extern "C" {

int gs_b200_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}
int gs_b200_set_device(int device) {
  GSB_CHECK(cudaSetDevice(device));
  GSB_CHECK(cudaFree(0));
  return 0;
}
const char *gs_b200_last_error(void) { return gsb::t_last_error; }
const char *gs_b200_version(void) { return "grayskull-b200 0.1 (sm_90a)"; }
int gs_b200_uses_tma(unsigned w, unsigned h, const void *ptr) {
  (void)h;
  return gsb::tma_ok(ptr, w) ? 1 : 0;
}
unsigned long long gs_b200_launch_count(void) { return gsb::g_launches.load(); }
void gs_b200_force_generic(int on) { gsb::g_force_generic = on ? 1 : 0; }

void *gs_b200_malloc(size_t bytes) {
  void *p = nullptr;
  if (cudaMalloc(&p, bytes ? bytes : 1) != cudaSuccess) {
    gsb::record_error(cudaGetLastError(), __FILE__, __LINE__);
    return nullptr;
  }
  return p;
}
void gs_b200_free(void *p) { cudaFree(p); }
void *gs_b200_malloc_host(size_t bytes) {
  void *p = nullptr;
  if (cudaMallocHost(&p, bytes ? bytes : 1) != cudaSuccess) {
    gsb::record_error(cudaGetLastError(), __FILE__, __LINE__);
    return nullptr;
  }
  return p;
}
void gs_b200_free_host(void *p) { cudaFreeHost(p); }
int gs_b200_memcpy_h2d(void *dst, const void *src, size_t bytes, gs_b200_stream s) {
  GSB_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, static_cast<cudaStream_t>(s)));
  return 0;
}
int gs_b200_memcpy_d2h(void *dst, const void *src, size_t bytes, gs_b200_stream s) {
  GSB_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, static_cast<cudaStream_t>(s)));
  return 0;
}
int gs_b200_memset(void *dst, int value, size_t bytes, gs_b200_stream s) {
  GSB_CHECK(cudaMemsetAsync(dst, value, bytes, static_cast<cudaStream_t>(s)));
  return 0;
}
int gs_b200_stream_sync(gs_b200_stream s) {
  GSB_CHECK(cudaStreamSynchronize(static_cast<cudaStream_t>(s)));
  return 0;
}

struct gs_image gs_b200_alloc(unsigned w, unsigned h) {
  struct gs_image img = {0, 0, nullptr};
  if (w == 0 || h == 0) return img;
  void *p = nullptr;
  size_t bytes = static_cast<size_t>(w) * h;
  if (cudaMallocManaged(&p, bytes) != cudaSuccess) {
    gsb::record_error(cudaGetLastError(), __FILE__, __LINE__);
    return img;
  }
  memset(p, 0, bytes);  // calloc semantics of the reference's gs_alloc (grayskull.h:103-107)
  img.w = w, img.h = h, img.data = static_cast<uint8_t *>(p);
  return img;
}
void gs_b200_image_free(struct gs_image img) { cudaFree(img.data); }

}  // extern "C"
