// Context management and shared host helpers of libcurate_b200 (C ABI in include/curate_b200.h).
#include <cudaTypedefs.h>

#include <cstdlib>
#include <cstring>

#include "common.h"

namespace cb {

static std::mutex g_err_mu;
static std::string g_last_error;
// A failing call and the cb_last_error() that follows it run on the same host thread (ctypes: check() right after the call),
// so the message is kept per thread: concurrent decode sessions on one cb_ctx never see (or tear) each other's strings.
static thread_local std::string t_last_error;
static thread_local std::string t_copy;

void set_global_error(const char* msg) {
  std::lock_guard<std::mutex> lk(g_err_mu);
  g_last_error = msg;
}

int fail(cb_ctx* ctx, int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  t_last_error = buf;
  if (ctx) {
    std::lock_guard<std::mutex> lk(ctx->mu);
    ctx->last_error = buf;
  }
  set_global_error(buf);
  return code;
}

int make_tensor_map(cb_ctx* ctx, CUtensorMap* out, CUtensorMapDataType dtype, int rank, const void* base, const uint64_t* dims,
                    const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swizzle) {
  if (!ctx->encode_tiled) return fail(ctx, CB_ERR_CUDA, "cuTensorMapEncodeTiled unavailable");
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bdim[5], estr[5];
  for (int i = 0; i < rank; ++i) gdim[i] = dims[i], bdim[i] = box[i], estr[i] = 1;
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  CUresult r = ctx->encode_tiled(out, dtype, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                 swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(ctx, CB_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d): rank %d dims %llu,%llu box %u,%u stride0 %llu", (int)r, rank,
                (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0), box[0], rank > 1 ? box[1] : 0,
                (unsigned long long)(rank > 1 ? strides_bytes[0] : 0));
  return CB_OK;
}

void mark_launch(cb_ctx* ctx, int category, cudaStream_t stream) {
  ctx->launches.fetch_add(1, std::memory_order_relaxed);
  if (!ctx->prof_on) return;
  std::lock_guard<std::mutex> lk(ctx->mu);  // decode threads (thumbnail kernel) may launch while the tower thread profiles
  if (ctx->prof_n >= ctx->prof_ev.size()) {
    cudaEvent_t e;
    if (cudaEventCreate(&e) != cudaSuccess) return;
    ctx->prof_ev.push_back(e);
    ctx->prof_cat.push_back(0);
  }
  ctx->prof_cat[ctx->prof_n] = category;
  cudaEventRecord(ctx->prof_ev[ctx->prof_n], stream);
  ctx->prof_n++;
}

}  // namespace cb

extern "C" {

int cb_profile_begin(cb_ctx* ctx) {
  if (!ctx) return CB_ERR_ARG;
  ctx->prof_on = true;
  ctx->prof_n = 0;
  return CB_OK;
}

int cb_profile_end(cb_ctx* ctx, void* stream, float* ms_by_category, int* launches_by_category, int n_categories) {
  if (!ctx) return CB_ERR_ARG;
  if (!ctx->prof_on) return cb::fail(ctx, CB_ERR_STATE, "profile_end without profile_begin");
  if (!ms_by_category || !launches_by_category || n_categories < CB_PROF_CATEGORIES) return cb::fail(ctx, CB_ERR_ARG, "profile_end: need %d categories", CB_PROF_CATEGORIES);
  cb::mark_launch(ctx, -1, (cudaStream_t)stream);  // closing event
  ctx->launches.fetch_sub(1, std::memory_order_relaxed);
  ctx->prof_on = false;
  CB_CUDA(ctx, cudaEventSynchronize(ctx->prof_ev[ctx->prof_n - 1]));
  for (int i = 0; i < n_categories; ++i) ms_by_category[i] = 0.f, launches_by_category[i] = 0;
  for (size_t i = 0; i + 1 < ctx->prof_n; ++i) {
    float ms = 0.f;
    CB_CUDA(ctx, cudaEventElapsedTime(&ms, ctx->prof_ev[i], ctx->prof_ev[i + 1]));
    const int c = ctx->prof_cat[i];
    if (c >= 0 && c < n_categories) ms_by_category[c] += ms, launches_by_category[c]++;
  }
  ctx->prof_n = 0;
  return CB_OK;
}

int cb_abi_version(void) { return CB_ABI_VERSION; }

int cb_init(int device, cb_ctx** out) {
  if (!out) return CB_ERR_ARG;
  *out = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0)
    return cb::fail(nullptr, CB_ERR_CUDA, "no CUDA device (%s); libcurate_b200 has no CPU fallback", cudaGetErrorString(e));
  if (device < 0 || device >= count) return cb::fail(nullptr, CB_ERR_ARG, "device %d out of range (0..%d)", device, count - 1);
  if ((e = cudaSetDevice(device)) != cudaSuccess) return cb::fail(nullptr, CB_ERR_CUDA, "cudaSetDevice: %s", cudaGetErrorString(e));
  cudaDeviceProp p;
  if ((e = cudaGetDeviceProperties(&p, device)) != cudaSuccess) return cb::fail(nullptr, CB_ERR_CUDA, "cudaGetDeviceProperties: %s", cudaGetErrorString(e));
  if (p.major != 9 || p.minor != 0)
    return cb::fail(nullptr, CB_ERR_UNSUPPORTED, "device %d is sm_%d%d; this library is built for sm_90a (H100) only", device, p.major, p.minor);
  cb_ctx* ctx = new cb_ctx();
  ctx->device = device;
  ctx->sm_count = p.multiProcessorCount;
  ctx->cc_major = p.major, ctx->cc_minor = p.minor;
  ctx->total_mem = p.totalGlobalMem;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q);
  if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !fn) {
    delete ctx;
    return cb::fail(nullptr, CB_ERR_CUDA, "cuTensorMapEncodeTiled not found in the driver");
  }
  ctx->encode_tiled = (PFN_cuTensorMapEncodeTiled_v12000)fn;
  *out = ctx;
  return CB_OK;
}

void cb_nvdec_release(cb_ctx* ctx);  // nvdec.cpp

void cb_destroy(cb_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cb_nvdec_release(ctx);
  for (auto& kv : ctx->taps) {
    cudaFree(kv.second.d_min);
    cudaFree(kv.second.d_size);
    cudaFree(kv.second.d_w);
  }
  for (auto& kv : ctx->resize_taps) {
    cudaFree(kv.second.d_first);
    cudaFree(kv.second.d_wq);
    cudaFree(kv.second.d_wf);
  }
  cb::release_tc_plans(ctx);
  if (ctx->d_tmp_u8) cudaFree(ctx->d_tmp_u8);
  if (ctx->d_norm_lut) cudaFree(ctx->d_norm_lut);
  if (ctx->d_slots) cudaFree(ctx->d_slots);
  for (cudaEvent_t e : ctx->prof_ev) cudaEventDestroy(e);
  delete ctx;
}

const char* cb_last_error(cb_ctx* ctx) {
  if (!cb::t_last_error.empty()) return cb::t_last_error.c_str();  // this thread's own last failure
  if (ctx) {
    std::lock_guard<std::mutex> lk(ctx->mu);
    cb::t_copy = ctx->last_error;
  } else {
    std::lock_guard<std::mutex> lk(cb::g_err_mu);
    cb::t_copy = cb::g_last_error;
  }
  return cb::t_copy.c_str();
}

int cb_device_info(cb_ctx* ctx, int* sm_count, int* cc_major, int* cc_minor, size_t* total_mem) {
  if (!ctx) return CB_ERR_ARG;
  if (sm_count) *sm_count = ctx->sm_count;
  if (cc_major) *cc_major = ctx->cc_major;
  if (cc_minor) *cc_minor = ctx->cc_minor;
  if (total_mem) *total_mem = ctx->total_mem;
  return CB_OK;
}

int cb_device_pci_bus_id(cb_ctx* ctx, char* buf, int len) {
  if (!ctx) return CB_ERR_ARG;
  if (!buf || len < 16) return cb::fail(ctx, CB_ERR_ARG, "device_pci_bus_id: buffer of at least 16 bytes needed");
  CB_CUDA(ctx, cudaDeviceGetPCIBusId(buf, len, ctx->device));
  return CB_OK;
}

unsigned long long cb_launch_count(cb_ctx* ctx) { return ctx ? ctx->launches.load(std::memory_order_relaxed) : 0ull; }

}  // extern "C"
