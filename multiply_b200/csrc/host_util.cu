// Host-side utilities of the C ABI: error text, device info, torch-exact linspace.
#include "common.cuh"
#include <stdarg.h>

namespace mp {
thread_local char g_err[512] = {0};
std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int Arena::fits(const char* who, const char* what) const {
  MP_REQUIRE(((uintptr_t)base & 255) == 0, "%s: %s base %p is not 256-byte aligned", who, what, (void*)base);
  MP_REQUIRE(ok, "%s: %s too small (%zu needed, %zu given)", who, what, off, cap);
  return 0;
}

// SM count of the CURRENT device (cached per device ordinal)
int sm_count() {
  static std::atomic<int> cache[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  int n = cache[dev].load();
  if (n <= 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) return 132;
    cache[dev].store(n);
  }
  return n;
}
}  // namespace mp

extern "C" {

int mp_version(void) { return 103; }

const char* mp_last_error(void) { return mp::g_err; }

int mp_device_sm_count(void) { return mp::sm_count(); }

long long mp_launch_count(int reset) {
  return reset ? mp::g_launches.exchange(0) : mp::g_launches.load();
}

// torch.linspace CPU kernel (ATen RangeFactoriesKernel): step = (end-start)/(n-1);
// i < n/2 : fma(step, i, start) ; else fma(-step, n-1-i, end).  Verified bit-exact in
// tests/test_host_logic.py against torch.linspace for every size the sampler uses.
int mp_linspace_host(float start, float end, int n, float* out) {
  if (n <= 0 || out == nullptr) {
    mp::set_error("mp_linspace_host: bad arguments");
    return -1;
  }
  if (n == 1) {
    out[0] = start;
    return 0;
  }
  float step = (end - start) / (float)(n - 1);
  int half = n / 2;
  for (int i = 0; i < n; ++i) {
    if (i < half)
      out[i] = fmaf(step, (float)i, start);
    else
      out[i] = fmaf(-step, (float)(n - 1 - i), end);
  }
  return 0;
}

}  // extern "C"
