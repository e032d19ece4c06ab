// Tensor-core operand ("weight image") cache shared by the tensor-core convolution kernels.
//
// The kernels read their B operand from a UMMA-ready image built once per layer from the
// caller's packed weights ([27][Cin][Cout], casmvs_pack_conv3d_weights).  Images are cached by
// (packed-weight pointer, kernel tag, size); their lifetime is tied to the packed buffer:
//   * casmvs_release_weight_images(ptr, bytes) drops every image whose key lies inside
//     [ptr, ptr + bytes) -- the Python binding calls it whenever it (re)creates a packed buffer,
//     so an address that the allocator hands out again can never hit a stale image;
//   * a captured CUDA graph holds raw image pointers: GraphedCascade records, per packed buffer
//     of its model, casmvs_weight_image_count() and re-checks it before each replay (releases
//     that concern other buffers do not invalidate it; casmvs_weight_cache_generation() counts
//     all releases).
// Thread-safe (one mutex); entries carry the stream + event of their builder kernel so that a
// hit from another stream waits for the build, and programmatic dependent launch (whose
// prologue reads the image BEFORE griddepcontrol.wait) is only allowed once the build is known
// to have completed.
#include <mutex>
#include <vector>

#include "tc_common.cuh"

namespace casmvs {
namespace tc {

struct CacheEntry {
  const void* key;
  int tag;
  size_t bytes;
  float* img;
  cudaStream_t built_on;
  cudaEvent_t built;     // recorded after the builder kernel
  bool settled;          // the build is known to have completed
};
static std::vector<CacheEntry> g_cache;
static std::mutex g_cache_mu;
static std::atomic<uint64_t> g_generation{0};

// cudaEventQuery / cudaStreamWaitEvent on an event from outside a capture are "unsafe" calls that
// INVALIDATE a stream capture (torch captures in global mode): while `st` is capturing the cache
// touches no event.  An image that is not known to be built then relies on the caller having
// synchronised between its warm-up and the capture -- GraphedCascade does, and marks everything
// built with casmvs_settle_weight_images() -- and is used without programmatic dependent launch.
static bool is_capturing(cudaStream_t st) {
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(st, &cs) != cudaSuccess) { cudaGetLastError(); return false; }
  return cs != cudaStreamCaptureStatusNone;
}

ImageRef image_cache_get(const void* wpk, int tag, size_t bytes, cudaStream_t st) {
  std::lock_guard<std::mutex> lock(g_cache_mu);
  const bool capturing = is_capturing(st);
  for (auto& e : g_cache) {
    if (e.key != wpk || e.tag != tag || e.bytes != bytes) continue;
    if (capturing) return ImageRef{e.img, true, e.settled};
    if (!e.settled && e.built && cudaEventQuery(e.built) == cudaSuccess) e.settled = true;
    if (!e.settled && e.built && e.built_on != st) {
      // built on another stream and possibly still running there: order this stream after it
      if (cudaStreamWaitEvent(st, e.built, 0) != cudaSuccess) {
        set_error("weight image: cannot order stream after the image build: %s",
                  cudaGetErrorString(cudaGetLastError()));
        return ImageRef{nullptr, false, false};
      }
    }
    return ImageRef{e.img, true, e.settled};
  }
  float* img = nullptr;
  if (cudaMalloc(&img, bytes) != cudaSuccess) {
    set_error("weight image: cudaMalloc(%zu) failed: %s", bytes,
              cudaGetErrorString(cudaGetLastError()));
    return ImageRef{nullptr, false, false};
  }
  g_cache.push_back(CacheEntry{wpk, tag, bytes, img, st, nullptr, false});
  return ImageRef{img, false, false};
}

void image_cache_built(const float* img, cudaStream_t st) {
  std::lock_guard<std::mutex> lock(g_cache_mu);
  for (auto& e : g_cache) {
    if (e.img != img) continue;
    e.built_on = st;
    if (is_capturing(st)) return;      // built inside a capture: never marked settled (no PDL)
    if (!e.built) cudaEventCreateWithFlags(&e.built, cudaEventDisableTiming);
    if (e.built && cudaEventRecord(e.built, st) != cudaSuccess) {
      cudaGetLastError();          // e.g. a capturing stream: leave the entry unsettled
      cudaEventDestroy(e.built);
      e.built = nullptr;
    }
    return;
  }
}

// frees the images keyed inside [lo, hi); returns how many were dropped
static int release_range(const char* lo, const char* hi) {
  std::lock_guard<std::mutex> lock(g_cache_mu);
  int n = 0;
  for (size_t i = 0; i < g_cache.size();) {
    const char* k = static_cast<const char*>(g_cache[i].key);
    if (k >= lo && k < hi) {
      cudaFree(g_cache[i].img);            // synchronises with every kernel still reading it
      if (g_cache[i].built) cudaEventDestroy(g_cache[i].built);
      g_cache[i] = g_cache.back();
      g_cache.pop_back();
      ++n;
    } else {
      ++i;
    }
  }
  if (n) g_generation.fetch_add(1);
  return n;
}

}  // namespace tc
}  // namespace casmvs

using namespace casmvs;

extern "C" int casmvs_release_weight_images(const void* w_packed, size_t bytes) {
  const char* lo = static_cast<const char*>(w_packed);
  tc::release_range(lo, lo + bytes);
  return 0;
}

extern "C" int casmvs_invalidate_weight_cache(void) {
  tc::release_range(nullptr, reinterpret_cast<const char*>(~uintptr_t(0)));
  return 0;
}

extern "C" uint64_t casmvs_weight_cache_generation(void) { return tc::g_generation.load(); }

extern "C" int casmvs_settle_weight_images(void) {
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    set_error("settle_weight_images: %s", cudaGetErrorString(e));
    return -2;
  }
  std::lock_guard<std::mutex> lock(tc::g_cache_mu);
  for (auto& en : tc::g_cache) en.settled = true;      // every builder enqueued so far has finished
  return 0;
}

extern "C" int casmvs_weight_image_count(const void* w_packed, size_t bytes) {
  std::lock_guard<std::mutex> lock(tc::g_cache_mu);
  const char* lo = static_cast<const char*>(w_packed);
  int n = 0;
  for (auto& e : tc::g_cache) {
    const char* k = static_cast<const char*>(e.key);
    if (k >= lo && k < lo + bytes) ++n;
  }
  return n;
}
