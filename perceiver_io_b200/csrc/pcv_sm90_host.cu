// pcv_sm90_host.cu — host side shared by the wgmma kernels (see the host section of pcv_sm90.cuh).
#include "pcv_sm90.cuh"

#include <cudaTypedefs.h>

#include <mutex>
#include <set>
#include <utility>

namespace pcv {
namespace sm90 {
namespace {

PFN_cuTensorMapEncodeTiled_v12000 encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(ptr);
  });
  return fn;
}

int encode(CUtensorMap* tm, int dtype, int rank, const void* base, const cuuint64_t* dims, const cuuint64_t* strides,
           const cuuint32_t* box) {
  auto fn = encode_fn();
  PCV_REQUIRE(fn != nullptr, PCV_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  const CUtensorMapDataType dt = dtype == PCV_BF16   ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                 : dtype == PCV_E4M3 ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                                     : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  CUresult r = fn(tm, dt, rank, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  PCV_REQUIRE(r == CUDA_SUCCESS, PCV_ERR_CUDA, "cuTensorMapEncodeTiled (%d-D) failed with CUresult %d", rank, (int)r);
  return PCV_OK;
}

uint32_t* g_diag_host = nullptr;  // the watchdog record: 16 words of mapped pinned host memory
std::mutex g_diag_mu;
std::set<std::pair<const void*, int>> g_diag_attached;  // (symbol, device)

std::mutex g_smem_mu;
std::set<std::pair<const void*, int>> g_smem_set;  // (kernel, device)

}  // namespace

const char* device_problem() {
  int dev = 0, major = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess)
    return "no CUDA device";
  return major == 9 ? nullptr : "device is not sm_90";
}

int make_tmap_4d(CUtensorMap* tm, const void* base, int dtype, int channels, int rows, int heads, int batch,
                 int64_t stride_row, int64_t stride_head, int64_t stride_batch, int box_rows) {
  const cuuint64_t dims[4] = {(cuuint64_t)channels, (cuuint64_t)rows, (cuuint64_t)heads, (cuuint64_t)batch};
  if (stride_batch == 0) stride_batch = (int64_t)rows * stride_row;  // broadcast batch: dim is 1, stride unused
  const int es = dtype == PCV_E4M3 ? 1 : 2;  // bytes per element
  const cuuint64_t strides[3] = {(cuuint64_t)stride_row * es, (cuuint64_t)stride_head * es, (cuuint64_t)stride_batch * es};
  const cuuint32_t box[4] = {(cuuint32_t)(128 / es), (cuuint32_t)box_rows, 1, 1};
  return encode(tm, dtype, 4, base, dims, strides, box);
}

int make_tmap_2d(CUtensorMap* tm, const void* base, int dtype, int64_t inner, int64_t rows, int64_t stride_row,
                 int box_rows) {
  const cuuint64_t dims[2] = {(cuuint64_t)inner, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)stride_row * 2};
  const cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
  return encode(tm, dtype, 2, base, dims, strides, box);
}

int attach_wait_diag(const void* symbol) {
  int dev = 0;
  PCV_CHECK_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lk(g_diag_mu);
  if (g_diag_attached.count({symbol, dev})) return PCV_OK;
  if (g_diag_host == nullptr) {
    PCV_CHECK_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&g_diag_host), 64, cudaHostAllocMapped | cudaHostAllocPortable));
    for (int i = 0; i < 16; ++i) g_diag_host[i] = 0;
  }
  uint32_t* dptr = nullptr;
  PCV_CHECK_CUDA(cudaHostGetDevicePointer(reinterpret_cast<void**>(&dptr), g_diag_host, 0));
  PCV_CHECK_CUDA(cudaMemcpyToSymbol(symbol, &dptr, sizeof(dptr)));
  g_diag_attached.insert({symbol, dev});
  return PCV_OK;
}

int set_smem_limit(const void* kernel, int smem) {
  int dev = 0;
  PCV_CHECK_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lk(g_smem_mu);
  if (g_smem_set.count({kernel, dev})) return PCV_OK;
  PCV_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  g_smem_set.insert({kernel, dev});
  return PCV_OK;
}

}  // namespace sm90

int debug_read(uint32_t* out, int n) {
  std::lock_guard<std::mutex> lk(sm90::g_diag_mu);
  for (int i = 0; i < n; ++i) out[i] = (sm90::g_diag_host != nullptr && i < 16) ? sm90::g_diag_host[i] : 0u;
  return PCV_OK;
}

}  // namespace pcv
