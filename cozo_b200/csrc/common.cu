// common.cu — lifecycle, error string, options (see include/cozo_gpu.h).
#include <map>
#include <mutex>

#include "common.cuh"

namespace cozo {

std::string& last_error() {
  thread_local std::string e;
  return e;
}

int set_error(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  last_error() = buf;
  return code;
}

static std::mutex g_mu;
static std::map<std::string, int64_t> g_opts;
static DeviceInfo g_dev;

int64_t get_option(const char* name, int64_t dflt) {
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_opts.find(name);
  return it == g_opts.end() ? dflt : it->second;
}

const DeviceInfo& device_info() { return g_dev; }

static int do_init(int device) {
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0)
    return set_error(COZO_GPU_ENODEV, "no CUDA device: %s (there is no CPU fallback)",
                     e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
  if (device < 0 || device >= count) return set_error(COZO_GPU_EINVAL, "device %d out of range [0,%d)", device, count);
  cudaDeviceProp prop;
  COZO_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)
    return set_error(COZO_GPU_ENODEV, "device %d is sm_%d%d; this library is built for sm_90a only", device,
                     prop.major, prop.minor);
  COZO_CUDA(cudaSetDevice(device));
  COZO_CUDA(cudaFree(0));
  g_dev.device = device;
  g_dev.sm_count = prop.multiProcessorCount;
  g_dev.cc_major = prop.major;
  g_dev.cc_minor = prop.minor;
  g_dev.smem_optin = prop.sharedMemPerBlockOptin;
  g_dev.ok = true;
  return 0;
}

int ensure_init() {
  if (g_dev.ok) {
    // calls may come from any host thread (Rayon workers, eval.rs:199-202)
    int cur = -1;
    if (cudaGetDevice(&cur) != cudaSuccess || cur != g_dev.device) COZO_CUDA(cudaSetDevice(g_dev.device));
    return 0;
  }
  std::lock_guard<std::mutex> lk(g_mu);
  if (g_dev.ok) return 0;
  int dev = 0;
  cudaGetDevice(&dev);
  return do_init(dev);
}

}  // namespace cozo

using namespace cozo;

extern "C" int cozo_gpu_init(int device) {
  std::lock_guard<std::mutex> lk(g_mu);
  return do_init(device);
}

extern "C" void cozo_gpu_shutdown(void) {
  std::lock_guard<std::mutex> lk(g_mu);
  g_dev = DeviceInfo();
}

extern "C" const char* cozo_gpu_last_error(void) { return last_error().c_str(); }

extern "C" int cozo_gpu_device_count(void) {
  int c = 0;
  if (cudaGetDeviceCount(&c) != cudaSuccess) return 0;
  return c;
}

extern "C" int cozo_gpu_set_option(const char* name, int64_t value) {
  if (!name) return set_error(COZO_GPU_EINVAL, "null option name");
  std::lock_guard<std::mutex> lk(g_mu);
  g_opts[name] = value;
  return 0;
}

extern "C" int64_t cozo_gpu_get_option(const char* name) {
  if (!name) return 0;
  return get_option(name, 0);
}
