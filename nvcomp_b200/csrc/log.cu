// log.cu -- call logging controlled by NVCOMP_LOG_LEVEL / NVCOMP_LOG_FILE, as documented for the reference
// (README.md:79-88): level 0 (default) = off, 3 = every low-level API call, 4-5 = more detail;
// NVCOMP_LOG_FILE = path | "stdout" | "stderr" (default file name nvcomp_yyyy-mm-dd_hh-mm.log).
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <mutex>

#include "common.cuh"

namespace b200 {

static int g_level = -1;
static FILE* g_file = nullptr;
static std::mutex g_mu;

static void log_init() {
  const char* lv = getenv("NVCOMP_LOG_LEVEL");
  g_level = lv ? atoi(lv) : 0;
  if (g_level <= 0) return;
  const char* f = getenv("NVCOMP_LOG_FILE");
  if (f && strcmp(f, "stdout") == 0) g_file = stdout;
  else if (f && strcmp(f, "stderr") == 0) g_file = stderr;
  else {
    char name[64];
    if (!f) {
      time_t t = time(nullptr);
      struct tm tmv;
      localtime_r(&t, &tmv);
      strftime(name, sizeof(name), "nvcomp_%Y-%m-%d_%H-%M.log", &tmv);
      f = name;
    }
    g_file = fopen(f, "a");
    if (!g_file) g_file = stderr;
  }
}

int log_level() {
  if (g_level < 0) {
    std::lock_guard<std::mutex> lk(g_mu);
    if (g_level < 0) log_init();
  }
  return g_level;
}

void log_call(const char* fn, size_t batch, size_t max_chunk, const void* stream) {
  if (log_level() < 3) return;
  std::lock_guard<std::mutex> lk(g_mu);
  fprintf(g_file, "[nvcomp][info] %s(batch_size=%zu, max_chunk_bytes=%zu, stream=%p)\n", fn, batch, max_chunk, stream);
  fflush(g_file);
}

}  // namespace b200

namespace b200 {

int sm_count_for_current_device() {
  static std::atomic<int> counts[64];   // zero until the device is first seen
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 0;
  int n = counts[dev].load(std::memory_order_relaxed);
  if (n == 0 && cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess)
    counts[dev].store(n, std::memory_order_relaxed);
  return n;
}

// one non-blocking side stream per device, created on first use and kept for the process (see StreamFork)
cudaError_t side_stream_for_current_device(cudaStream_t* side) {
  static std::mutex mu;
  static cudaStream_t streams[64] = {nullptr};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
  std::lock_guard<std::mutex> lk(mu);
  if (!streams[dev]) {
    e = cudaStreamCreateWithFlags(&streams[dev], cudaStreamNonBlocking);
    if (e != cudaSuccess) return e;
  }
  *side = streams[dev];
  return cudaSuccess;
}

}  // namespace b200
