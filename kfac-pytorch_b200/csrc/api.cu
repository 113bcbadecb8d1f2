// Library-level entry points: version, thread-local error string, device probe.
#include <stdarg.h>
#include <string.h>

#include <algorithm>

#include "common.cuh"

namespace kfac {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
static long long g_launches = 0;
void count_launch(int n) { __atomic_fetch_add(&g_launches, (long long)n, __ATOMIC_RELAXED); }

int HostStage::begin() {
  if (pending) KFAC_CUDA(cudaEventSynchronize(done));
  pending = false;
  if (nbuf > 1) {                  // the last call needed more than one block: one block of the total from now on
    size_t total = 0;
    for (int i = 0; i < nbuf; ++i) { total += size[i]; KFAC_CUDA(cudaFreeHost(buf[i])); buf[i] = nullptr; }
    KFAC_CUDA(cudaHostAlloc((void**)&buf[0], total, cudaHostAllocPortable));
    size[0] = total;
    nbuf = 1;
  }
  used = 0;
  return KFAC_OK;
}

int HostStage::send(void* dst, const void* src, size_t bytes, cudaStream_t s) {
  if (bytes == 0) return KFAC_OK;
  if (nbuf == 0 || used + bytes > size[nbuf - 1]) {
    if (nbuf == 8) { set_error("host stage: more than 8 blocks in one call"); return KFAC_ERR_WORKSPACE; }
    size[nbuf] = std::max<size_t>(size_t(1) << 20, 2 * bytes);
    KFAC_CUDA(cudaHostAlloc((void**)&buf[nbuf], size[nbuf], cudaHostAllocPortable));
    ++nbuf;
    used = 0;
  }
  char* p = buf[nbuf - 1] + used;
  memcpy(p, src, bytes);
  used = align_up(used + bytes, 64);
  KFAC_CUDA(cudaMemcpyAsync(dst, p, bytes, cudaMemcpyHostToDevice, s));
  return KFAC_OK;
}

int HostStage::end(cudaStream_t s) {
  if (!done) KFAC_CUDA(cudaEventCreateWithFlags(&done, cudaEventDisableTiming));
  KFAC_CUDA(cudaEventRecord(done, s));
  pending = true;
  return KFAC_OK;
}

int send_table(HostStage* stage, void* dst, const void* src, size_t bytes, cudaStream_t s) {
  if (stage) return stage->send(dst, src, bytes, s);
  KFAC_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s));
  return KFAC_OK;
}
}  // namespace kfac

extern "C" int kfac_version(void) { return 100; /* 0.1.0 */ }
extern "C" const char* kfac_last_error(void) { return kfac::g_err; }
extern "C" int kfac_device_arch(void) {
  int dev = 0;
  cudaDeviceProp p;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&p, dev) != cudaSuccess) {
    kfac::set_error("no CUDA device available");
    return KFAC_ERR_CUDA;
  }
  return p.major * 10 + p.minor;
}

extern "C" long long kfac_launch_count(void) { return __atomic_load_n(&kfac::g_launches, __ATOMIC_RELAXED); }
