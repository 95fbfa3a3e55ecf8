// Internal declarations shared by the kernels behind the C ABI in include/dinov3_b200.h.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include "../../include/dinov3_b200.h"

namespace d3 {

// epilogue flag bits mirror D3_EP_* in the public header
enum : int {
  EP_BIAS = D3_EP_BIAS,
  EP_GELU = D3_EP_GELU,
  EP_STORE_PRE = D3_EP_STORE_PRE,
  EP_MUL_DGELU = D3_EP_MUL_DGELU,
  EP_GAMMA = D3_EP_GAMMA,
  EP_RESID = D3_EP_RESID,
  EP_OUT_F32 = D3_EP_OUT_F32,
  EP_ACCUM = D3_EP_ACCUM,
  EP_SCATTER = D3_EP_SCATTER,
  EP_GELU_ERF = D3_EP_GELU_ERF,
  EP_SLOW = 1 << 30,      // internal: force the bounds-checked scalar epilogue
  EP_SLABS = 1 << 27,     // internal: split-K slice s stores its partial tile at rows [s*M, s*M + M) of `out`
};

struct GemmEpilogue {
  const float* bias;             // [N] fp32
  const float* gamma;            // [N] fp32 (LayerScale)
  const float* resid;            // [M, ld_resid] fp32 residual stream (may alias out)
  const __nv_bfloat16* aux_in;   // [M, ld_aux] bf16 pre-activation for GELU'
  __nv_bfloat16* aux_out;        // [M, ld_aux] bf16 pre-activation stash
  void* out;                     // [M, ld_out] bf16 or fp32
  int ld_out, ld_aux, ld_resid;
  int flags;
  float alpha;
  // EP_SCATTER: the fp32 result is not stored at `out` but added (red.add over NVLink peer mappings) into the rank
  // that owns it: element e of the output ([row*ld_out + col]) has global index g = sc_off + e inside a flat range cut
  // into sc_world slices of sc_shard elements; it goes to sc_peer[g / sc_shard][g % sc_shard].
  float* sc_peer[8];
  long long sc_off;
  int sc_shard, sc_world;
};

int set_error(int code, const char* msg);
int sm_count();
void count_launch(int n = 1);
int encode_tensor_map_2d_bf16(CUtensorMap* map, const void* ptr, const cuuint64_t dims[2],
                              const cuuint64_t strides[1], const cuuint32_t box[2], const cuuint32_t estr[2]);
// generic 2-D map: elt_bytes 2 (bf16) or 4 (fp32); swizzle_bytes 0 / 64 / 128
int encode_tensor_map_2d(CUtensorMap* map, const void* ptr, int elt_bytes, cuuint64_t cols, cuuint64_t rows,
                         cuuint64_t row_stride_bytes, cuuint32_t box_cols, cuuint32_t box_rows, int swizzle_bytes);
// e4m3 (uint8) operand map: `cols` bytes per row, SWIZZLE_128B, boxes of box_cols x box_rows
int encode_tensor_map_2d_u8(CUtensorMap* map, const void* ptr, cuuint64_t cols, cuuint64_t rows, cuuint64_t ld_bytes,
                            cuuint32_t box_cols, cuuint32_t box_rows);

// Deterministic reductions.  A kernel that would add one partial per (slab, element) into a destination with a float
// atomic (whose order, and so whose rounding, changes from run to run) writes it into slab s of a zeroed, stream-ordered
// workspace instead; slab_combine then adds the slabs to the destination in slab order, the same bits every run.
float* slab_workspace(size_t floats, cudaStream_t st);          // nullptr (error set) on failure
void slab_release(float* ws, cudaStream_t st);
// dst[r * ld + c] += sum_s ws[s * stride + r * cols + c] for r < rows, c < cols (dst == nullptr: nothing)
int slab_combine(const float* ws, int slabs, long long stride, long long rows, int cols, float* dst, long long ld,
                 cudaStream_t st);

int gemm_bf16(const void* A, int lda, int a_mn, const void* B, int ldb, int b_mn, int M, int N, int K,
              GemmEpilogue ep, int tile_n, int split_k, cudaStream_t stream);
int gemm_e4m3(const void* A, int lda, const float* sa, const void* B, int ldb, const float* sb, int M, int N, int K,
              GemmEpilogue ep, cudaStream_t stream);

#define D3_CHECK_LAUNCH()                                               \
  do {                                                                  \
    cudaError_t e__ = cudaPeekAtLastError();                            \
    if (e__ != cudaSuccess) return d3::set_error(D3_ERR_CUDA, cudaGetErrorString(e__)); \
    d3::count_launch();                                                 \
  } while (0)

}  // namespace d3
