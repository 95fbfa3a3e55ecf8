// C ABI glue: library state, error reporting, tensor-map encoding, extern "C" wrappers.
#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstring>
#include "d3_internal.h"

namespace d3 {

static thread_local char g_err[512] = "";
static int g_sm_count = 0;
static std::atomic<long long> g_launches{0};
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn g_encode = nullptr;

int set_error(int code, const char* msg) {
  snprintf(g_err, sizeof(g_err), "%s", msg ? msg : "");
  return code;
}
int sm_count() { return g_sm_count > 0 ? g_sm_count : 132; }
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int encode_tensor_map_2d_bf16(CUtensorMap* map, const void* ptr, const cuuint64_t dims[2],
                              const cuuint64_t strides[1], const cuuint32_t box[2], const cuuint32_t estr[2]) {
  if (!g_encode) return set_error(D3_ERR_CUDA, "d3_init() was not called (cuTensorMapEncodeTiled unresolved)");
  CUresult r = g_encode(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[160];
    snprintf(buf, sizeof(buf), "cuTensorMapEncodeTiled failed (%d): dims=(%llu,%llu) stride=%llu box=(%u,%u)", (int)r,
             (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)strides[0], box[0], box[1]);
    return set_error(D3_ERR_CUDA, buf);
  }
  return D3_OK;
}

int encode_tensor_map_2d_u8(CUtensorMap* map, const void* ptr, cuuint64_t cols, cuuint64_t rows, cuuint64_t ld_bytes,
                            cuuint32_t box_cols, cuuint32_t box_rows) {
  if (!g_encode) return set_error(D3_ERR_CUDA, "d3_init() was not called (cuTensorMapEncodeTiled unresolved)");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld_bytes};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[160];
    snprintf(buf, sizeof(buf), "cuTensorMapEncodeTiled(e4m3) failed (%d): dims=(%llu,%llu) stride=%llu", (int)r,
             (unsigned long long)cols, (unsigned long long)rows, (unsigned long long)ld_bytes);
    return set_error(D3_ERR_CUDA, buf);
  }
  return D3_OK;
}

int encode_tensor_map_2d(CUtensorMap* map, const void* ptr, int elt_bytes, cuuint64_t cols, cuuint64_t rows,
                         cuuint64_t row_stride_bytes, cuuint32_t box_cols, cuuint32_t box_rows, int swizzle_bytes) {
  if (!g_encode) return set_error(D3_ERR_CUDA, "d3_init() was not called (cuTensorMapEncodeTiled unresolved)");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {row_stride_bytes};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                          : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE;
  CUresult r = g_encode(map, elt_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                        const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                        CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[160];
    snprintf(buf, sizeof(buf), "cuTensorMapEncodeTiled(epilogue) failed (%d): dims=(%llu,%llu) stride=%llu", (int)r,
             (unsigned long long)cols, (unsigned long long)rows, (unsigned long long)row_stride_bytes);
    return set_error(D3_ERR_CUDA, buf);
  }
  return D3_OK;
}

float* slab_workspace(size_t floats, cudaStream_t st) {
  void* p = nullptr;
  cudaError_t e = cudaMallocAsync(&p, floats * sizeof(float), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(p, 0, floats * sizeof(float), st);
  if (e != cudaSuccess) { set_error(D3_ERR_CUDA, cudaGetErrorString(e)); return nullptr; }
  return static_cast<float*>(p);
}
void slab_release(float* ws, cudaStream_t st) {
  if (ws) cudaFreeAsync(ws, st);
}

__global__ void slab_combine_kernel(const float* __restrict__ ws, int slabs, long long stride, long long rows, int cols,
                                    float* __restrict__ dst, long long ld) {
  const long long n = rows * cols;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols, c = i - r * cols;
    float tot = 0.f;
    for (int k = 0; k < slabs; ++k) tot += ws[k * stride + i];
    dst[r * ld + c] += tot;
  }
}
int slab_combine(const float* ws, int slabs, long long stride, long long rows, int cols, float* dst, long long ld,
                 cudaStream_t st) {
  if (!dst || rows <= 0 || cols <= 0) return D3_OK;
  const long long n = rows * cols;
  const int blocks = (int)std::min<long long>((n + 255) / 256, (long long)sm_count() * 8);
  slab_combine_kernel<<<blocks, 256, 0, st>>>(ws, slabs, stride, rows, cols, dst, ld);
  cudaError_t e = cudaPeekAtLastError();
  if (e != cudaSuccess) return set_error(D3_ERR_CUDA, cudaGetErrorString(e));
  count_launch();
  return D3_OK;
}

}  // namespace d3

using namespace d3;

extern "C" {

int d3_abi_version(void) { return 7; }   // 2: d3_gemm_epilogue gained the sc_* scatter fields; 3: round-2 entry points (swiglu, ema, colmax, deterministic Sinkhorn sums, koleo rows, augmentation); 4: two entry points removed (the plain LayerNorm backward is d3_layernorm_bwd_ls without a tail; d3_sinkhorn_colsum is deterministic for every K); 5: d3_debug_attn_trace removed (the attention clock64() trace); 6: d3_koleo_fwd_bwd removed (it is d3_koleo_fwd_bwd_rows with row0 = 0, nrows = B); 7: the scatter-mode and SM-limit setters removed (the peer push is always one device-scope vector red; the persistent grids always cover every SM)
const char* d3_last_error(void) { return g_err; }
long long d3_launch_count(void) { return g_launches.load(); }
void d3_reset_launch_count(void) { g_launches.store(0); }

int d3_init(int device) {
  cudaError_t e = cudaSetDevice(device);
  if (e != cudaSuccess) return set_error(D3_ERR_CUDA, cudaGetErrorString(e));
  cudaDeviceProp prop;
  e = cudaGetDeviceProperties(&prop, device);
  if (e != cudaSuccess) return set_error(D3_ERR_CUDA, cudaGetErrorString(e));
  if (prop.major != 9 || prop.minor != 0) {
    char buf[128];
    snprintf(buf, sizeof(buf), "device %d is sm_%d%d; this library only has sm_90a code (no fallback)", device,
             prop.major, prop.minor);
    return set_error(D3_ERR_DEVICE, buf);
  }
  g_sm_count = prop.multiProcessorCount;
  {  // keep the stream-ordered workspaces of the deterministic reductions cached instead of returning them at every sync
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
      uint64_t keep = UINT64_MAX;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    }
  }
  if (!g_encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q);
    if (e != cudaSuccess || !fn) return set_error(D3_ERR_CUDA, "cannot resolve cuTensorMapEncodeTiled");
    g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  }
  return D3_OK;
}

// the public epilogue description -> the kernels' GemmEpilogue, with the flag / pointer checks both GEMM entry points make
static int epilogue_from_abi(const d3_gemm_epilogue* ep, GemmEpilogue& g) {
  if ((ep->flags & D3_EP_ACCUM) && !(ep->flags & D3_EP_OUT_F32)) return set_error(D3_ERR_ARG, "ACCUM needs fp32 out");
  g.bias = ep->bias; g.gamma = ep->gamma; g.resid = ep->resid;
  g.aux_in = reinterpret_cast<const __nv_bfloat16*>(ep->aux_in);
  g.aux_out = reinterpret_cast<__nv_bfloat16*>(ep->aux_out);
  g.out = ep->out; g.ld_out = ep->ld_out; g.ld_aux = ep->ld_aux; g.ld_resid = ep->ld_resid;
  g.flags = ep->flags & 0x3FF; g.alpha = ep->alpha;
  for (int i = 0; i < 8; ++i) g.sc_peer[i] = ep->sc_peer[i];
  g.sc_off = ep->sc_off; g.sc_shard = ep->sc_shard; g.sc_world = ep->sc_world;
  if (g.flags & EP_SCATTER)
    for (int i = 0; i < g.sc_world && i < 8; ++i)
      if (!g.sc_peer[i]) return set_error(D3_ERR_ARG, "scatter flag without peer pointers");
  if ((g.flags & EP_BIAS) && !g.bias) return set_error(D3_ERR_ARG, "bias flag without pointer");
  if ((g.flags & EP_GAMMA) && !g.gamma) return set_error(D3_ERR_ARG, "gamma flag without pointer");
  if ((g.flags & EP_RESID) && !g.resid) return set_error(D3_ERR_ARG, "resid flag without pointer");
  if ((g.flags & EP_STORE_PRE) && !g.aux_out) return set_error(D3_ERR_ARG, "store_pre flag without pointer");
  if ((g.flags & EP_MUL_DGELU) && !g.aux_in) return set_error(D3_ERR_ARG, "mul_dgelu flag without pointer");
  return D3_OK;
}

int d3_gemm_bf16(const void* A, int lda, int a_major, const void* B, int ldb, int b_major, int M, int N, int K,
                 const d3_gemm_epilogue* ep, int tile_n, int split_k, void* stream) {
  if (!A || !B || !ep || !ep->out) return set_error(D3_ERR_ARG, "d3_gemm_bf16: null pointer");
  if (tile_n != 0 && tile_n != 64 && tile_n != 128 && tile_n != 256 && tile_n != 512) return set_error(D3_ERR_ARG, "tile_n");
  if (split_k < 0) return set_error(D3_ERR_ARG, "split_k");
  GemmEpilogue g;
  const int rc = epilogue_from_abi(ep, g);
  if (rc) return rc;
  return gemm_bf16(A, lda, a_major, B, ldb, b_major, M, N, K, g, tile_n, split_k, reinterpret_cast<cudaStream_t>(stream));
}

int d3_gemm_e4m3(const void* A_u8, int lda, const float* sa, const void* B_u8, int ldb, const float* sb, int M, int N,
                 int K, const d3_gemm_epilogue* ep, void* stream) {
  if (!A_u8 || !B_u8 || !sa || !sb || !ep || !ep->out) return set_error(D3_ERR_ARG, "d3_gemm_e4m3: null pointer");
  GemmEpilogue g;
  const int rc = epilogue_from_abi(ep, g);
  if (rc) return rc;
  return gemm_e4m3(A_u8, lda, sa, B_u8, ldb, sb, M, N, K, g, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
