// Host-side helpers shared by the C-ABI translation units: error codes, TMA tensor-map encoding.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/aria_b200.h"

namespace aria {

#define ARIA_CHECK_ARG(cond)                                                             \
  do {                                                                                   \
    if (!(cond)) {                                                                       \
      fprintf(stderr, "aria_b200: bad argument: %s (%s:%d)\n", #cond, __FILE__, __LINE__); \
      return ARIA_ERR_BAD_ARG;                                                           \
    }                                                                                    \
  } while (0)

inline int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    fprintf(stderr, "aria_b200: launch of %s failed: %s\n", what, cudaGetErrorString(e));
    return ARIA_ERR_CUDA;
  }
  return ARIA_OK;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

// bf16 tensor map, 128B swizzle (or the given one), zero OOB fill.  dims/strides innermost-first; strides[i] is the byte stride
// of dim i+1 (rank-1 entries).  `dtype`: UINT8 for the e4m3 expert weights (fp8 grouped GEMM).
inline int make_tmap_bf16_swz(CUtensorMap* tm, const void* ptr, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                              const uint32_t* box, CUtensorMapSwizzle swizzle,
                              CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
inline int make_tmap_bf16(CUtensorMap* tm, const void* ptr, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                          const uint32_t* box) {
  return make_tmap_bf16_swz(tm, ptr, rank, dims, strides_bytes, box, CU_TENSOR_MAP_SWIZZLE_128B);
}
inline int make_tmap_bf16_swz(CUtensorMap* tm, const void* ptr, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                              const uint32_t* box, CUtensorMapSwizzle swizzle, CUtensorMapDataType dtype) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) {
    fprintf(stderr, "aria_b200: cuTensorMapEncodeTiled unavailable\n");
    return ARIA_ERR_CUDA;
  }
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
  }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  // cuTensorMapEncodeTiled is a DRIVER entry point: it needs a CUDA context bound to the calling thread.  The runtime binds
  // the primary context lazily, on a thread's first runtime call that needs it — and a fresh thread whose current device is
  // already the wanted one (PyTorch's autograd worker: its device guard skips cudaSetDevice when cudaGetDevice() matches)
  // has none.  The first C-ABI call of such a thread then failed with CUDA_ERROR_INVALID_CONTEXT (201): the round-1
  // "nondeterministic LoRA test" (a backward whose first node is one of our GEMMs).  cudaFree(0) binds the primary context.
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) {
    cudaFree(0);
    ctx_bound = true;
  }
  CUresult r = enc(tm, dtype, rank, const_cast<void*>(ptr), gdim, gstr, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r == CUDA_ERROR_INVALID_CONTEXT || r == CUDA_ERROR_NOT_INITIALIZED) {  // e.g. the context was popped by another library
    cudaFree(0);
    r = enc(tm, dtype, rank, const_cast<void*>(ptr), gdim, gstr, bx, es,
            CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "aria_b200: cuTensorMapEncodeTiled failed (%d): rank %d ptr %p dims %llu,%llu stride %llu box %u,%u\n",
            (int)r, rank, ptr, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
            (unsigned long long)(rank > 1 ? strides_bytes[0] : 0), box[0], rank > 1 ? box[1] : 0);
    return ARIA_ERR_CUDA;
  }
  return ARIA_OK;
}

// Row-major 2-D tensor map; e4m3 operands are UINT8 maps
inline int make_tmap_2d(CUtensorMap* tm, const void* ptr, uint64_t inner, uint64_t outer, uint64_t row_stride_bytes,
                        uint32_t box_inner, uint32_t box_outer, CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B,
                        CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16) {
  uint64_t dims[2] = {inner, outer};
  uint64_t str[1] = {row_stride_bytes};
  uint32_t box[2] = {box_inner, box_outer};
  return make_tmap_bf16_swz(tm, ptr, 2, dims, str, box, swizzle, dtype);
}

// Per-device state: one process may drive several GPUs (the reference's device_map="auto", aria/inference.py:55-57), and
// both the SM count and cudaFuncSetAttribute opt-ins belong to the CURRENT device.
constexpr int kMaxDevices = 64;
inline int current_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return (dev >= 0 && dev < kMaxDevices) ? dev : 0;
}
inline int sm_count() {
  static int n[kMaxDevices] = {};
  const int dev = current_device();
  if (!n[dev]) {
    int v = 0;
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    n[dev] = v > 0 ? v : 132;
  }
  return n[dev];
}
// `flags` is a function-local `static bool flags[kMaxDevices]`: true once the dynamic-smem opt-in was done on that device.
template <typename Kernel>
inline cudaError_t ensure_dynamic_smem(bool* flags, Kernel kern, int bytes) {
  const int dev = current_device();
  if (flags[dev]) return cudaSuccess;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess) flags[dev] = true;
  else fprintf(stderr, "aria_b200: cudaFuncSetAttribute(smem=%d) failed: %s\n", bytes, cudaGetErrorString(e));
  return e;
}

// Launches a persistent kernel: one CTA per SM, fewer when there are fewer than `max_tiles` tiles, with `smem` bytes of
// dynamic shared memory.  Each kernel instantiates this template once, so each has its own opt-in flags.
template <auto kernel, typename... Args>
inline int launch_persistent(const char* name, int threads, int smem, int64_t max_tiles, cudaStream_t stream,
                             const Args&... args) {
  static bool attr_set[kMaxDevices] = {};
  if (ensure_dynamic_smem(attr_set, kernel, smem) != cudaSuccess) return ARIA_ERR_CUDA;
  int grid = sm_count();
  if (max_tiles < grid) grid = static_cast<int>(max_tiles);
  if (grid < 1) grid = 1;
  kernel<<<grid, threads, smem, stream>>>(args...);
  return check_launch(name);
}

// Launches a persistent kernel as clusters of two CTAs along x (one CTA per SM): as many clusters as the device holds at once,
// fewer when there are fewer than `max_pairs` tile pairs.  How many fit is asked once per device: a GPC with an odd number of
// free SMs can leave one of them out.
template <auto kernel, typename... Args>
inline int launch_persistent_pairs(const char* name, int threads, int smem, int64_t max_pairs, cudaStream_t stream,
                                   const Args&... args) {
  static bool attr_set[kMaxDevices] = {};
  static int max_clusters[kMaxDevices] = {};
  if (ensure_dynamic_smem(attr_set, kernel, smem) != cudaSuccess) return ARIA_ERR_CUDA;
  cudaLaunchAttribute attr{};
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = 2;
  attr.val.clusterDim.y = 1;
  attr.val.clusterDim.z = 1;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(2);
  cfg.blockDim = dim3(threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  const int dev = current_device();
  if (!max_clusters[dev]) {
    int n = 0;
    const cudaError_t e = cudaOccupancyMaxActiveClusters(&n, kernel, &cfg);
    if (e != cudaSuccess || n < 1) {
      fprintf(stderr, "aria_b200: cudaOccupancyMaxActiveClusters(%s) = %d: %s\n", name, n, cudaGetErrorString(e));
      return ARIA_ERR_CUDA;
    }
    max_clusters[dev] = n;
  }
  const int64_t clusters = max_pairs < max_clusters[dev] ? (max_pairs > 1 ? max_pairs : 1) : max_clusters[dev];
  cfg.gridDim = dim3(static_cast<unsigned>(2 * clusters));
  cudaLaunchKernelEx(&cfg, kernel, args...);  // its error, if any, is the one check_launch reads
  return check_launch(name);
}

// Grouped expert GEMM (gemm.cu): out[rows, n] = a[rows, k] x b[g] for the rows of group g (`offsets`), b = [groups, k, n]
// bf16, or e4m3 with one fp32 scale per (group, column) when b_scale is given.  `epilogue`: LINEAR or SWIGLU.
int grouped_gemm(const void* a, const void* b, const float* b_scale, void* out, const int32_t* offsets, int64_t rows,
                 int64_t k, int64_t n, int32_t groups, int32_t epilogue, cudaStream_t stream);

#ifdef __CUDACC__
// Packed sequences: n_seg segments along one row axis, segment b = rows [cu[b], cu[b + 1]) (cu nondecreasing, device).
// The segment holding row q: the last b < n_seg with cu[b] <= q.
__device__ __forceinline__ int packed_segment(const int32_t* cu, int n_seg, int q) {
  int lo = 0, hi = n_seg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (cu[mid] <= q) lo = mid; else hi = mid - 1;
  }
  return lo;
}
#endif

}  // namespace aria
