// C-ABI plumbing: version, thread-local error string, launch checking.
#include "common.cuh"
#include <stdarg.h>
#include <string.h>

static thread_local char g_err[512] = {0};

void zsb_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int zsb_check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    zsb_set_error("%s: CUDA launch failed: %s", what, cudaGetErrorString(e));
    return ZSB_ERR_CUDA;
  }
  return ZSB_OK;
}

// Device-resident draw epoch (see zsb_random_set_device_epoch): added to the `iter` word of every
// in-kernel Philox draw of the distribution samplers, so that a sampling step captured once in a
// CUDA graph draws fresh numbers on every replay.
static const uint32_t* g_epoch = nullptr;
const uint32_t* zsb_epoch_ptr() { return g_epoch; }

namespace {
__global__ void epoch_bump_kernel(uint32_t* e, uint32_t by) {
  if (threadIdx.x == 0 && blockIdx.x == 0) *e += by;
}
}  // namespace

extern "C" {

int zsb_version(void) { return 102; }  // 0.1.2

// Registers (or, with NULL, removes) a device uint32 that the samplers add to their Philox
// iteration word: draws become a function of (seed, iter + *epoch, ...).  The stand-in for the
// op-level counters of tf.random_* (hmc.py:22, univariate.py:161-172) when the step that contains
// the draw is replayed from a CUDA graph; zsb_random_bump_epoch advances it on the stream.
int zsb_random_set_device_epoch(const uint32_t* epoch) {
  g_epoch = epoch;
  return ZSB_OK;
}
int zsb_random_bump_epoch(uint32_t* epoch, uint32_t by, void* stream) {
  ZSB_REQUIRE(epoch, "zsb_random_bump_epoch: null epoch");
  epoch_bump_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(epoch, by);
  return zsb_check_launch("random_bump_epoch");
}

// Copies the calling thread's last error message (NUL-terminated) into buf; returns its length.
int zsb_last_error(char* buf, size_t n) {
  if (buf && n) {
    strncpy(buf, g_err, n - 1);
    buf[n - 1] = 0;
  }
  return (int)strlen(g_err);
}

// Number of CUDA devices visible (0 when there is no GPU: every compute entry point then fails
// with ZSB_ERR_CUDA -- there is no CPU fallback in this library).
int zsb_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

// Blocks until `stream` drains; surfaces asynchronous kernel faults as an error code.
int zsb_stream_sync(void* stream) {
  cudaError_t e = cudaStreamSynchronize((cudaStream_t)stream);
  if (e != cudaSuccess) {
    zsb_set_error("zsb_stream_sync: %s", cudaGetErrorString(e));
    return ZSB_ERR_CUDA;
  }
  return ZSB_OK;
}

}  // extern "C"
