// On-GPU DINO multi-crop augmentation (SURVEY §8f.3): the step BEFORE the training hot path.  Replaces the per-sample
// torchvision / PIL host pipeline of dinov3_jax/data/augmentations.py:23-230 (RandomResizedCrop(bicubic) + flip,
// ColorJitter(0.4, 0.4, 0.2, 0.1) in random order, RandomGrayscale, GaussianBlur(9, sigma 0.1..2), RandomSolarize(128),
// ToTensor + Normalize) for a whole batch of decoded uint8 images resident in HBM; the random parameters are drawn on the
// host (a few scalars per crop, dinov3_jax/data/gpu_augment.py) so that the kernels are deterministic functions that can
// be checked against torchvision's float implementations.  Output: crop-major NHWC bf16, i.e. exactly the
// `collated_global_crops` / `collated_local_crops` tensors of data/collate.py:72-93.
//
// All kernels are HBM / L2 streaming work (one thread per output pixel, channels innermost); arithmetic is fp32 on
// [0, 1] images like torchvision.transforms.v2.functional on float tensors (PIL's per-op uint8 re-quantisation is not
// reproduced).
#include "ptx.cuh"
#include "d3_internal.h"
#include "resample.cuh"

#include <cstdio>
#include <type_traits>

namespace d3 {

// one record per output crop (host-filled, 64 bytes)
struct AugCrop {
  int img;                 // source image index
  int x0, y0, w, h;        // crop box in the source (RandomResizedCrop.get_params)
  int flip;                // horizontal flip
  int order[4];            // ColorJitter op order: 0 brightness, 1 contrast, 2 saturation, 3 hue; -1 = jitter not applied
  float fb, fc, fs, fh;    // factors
  int gray;                // RandomGrayscale applied
  int solarize;            // RandomSolarize applied (threshold 128/255)
};
struct AugBlur { float sigma; };   // <= 0: no blur

// one row per source image of a ragged batch (host-filled, 16 bytes): the images' HWC pixels are packed one after the
// other in one buffer, image i starting at pixel `off`.  A dense [n, H, W, 3] batch has no table (nullptr) and the
// geometry of image i is computed: a dense batch is a ragged batch of equal sizes.
struct AugImage {
  long long off;           // first pixel of the image in the packed buffer (element offset / 3)
  int h, w;
};
static_assert(sizeof(AugImage) == 16, "AugImage is the 16-byte row of the host-filled image table");
__device__ __forceinline__ AugImage image_of(const AugImage* __restrict__ imgs, int i, int H, int W) {
  if (imgs) return imgs[i];
  return AugImage{(long long)i * H * W, H, W};
}

// out[n, S, S, 3] (fp32, [0,1]) = antialiased bicubic resize of src[img, y0:y0+h, x0:x0+w] (+ horizontal flip).
// Same definition as torch's _upsample_bicubic2d_aa (align_corners = False): per axis, scale = in/out,
// support = 2 * max(scale, 1), taps j in [floor(center - support + 0.5), ...), weight cubic((j + 0.5 - center) / max(scale, 1)),
// normalised; taps are clipped to the crop box.
// T = uint8_t reads a decoded image (/255); T = float reads an fp32 [0,1] image (the colour-jittered source of
// share_color_jitter, or a base crop resized to the global / gram size).  CLAMP = false is the Resize of a normalised
// tensor, which torchvision does not clamp.
template <typename T, bool CLAMP>
__global__ void aug_resized_crop_kernel(const T* __restrict__ src, const AugImage* __restrict__ imgs, int H, int W,
                                        const AugCrop* __restrict__ crops, float* __restrict__ out, int S) {
  const int n = blockIdx.z;
  const int ox = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y * blockDim.y + threadIdx.y;
  if (ox >= S || oy >= S) return;
  const AugCrop c = crops[n];
  const AugImage im = image_of(imgs, c.img, H, W);
  const int sx_out = c.flip ? (S - 1 - ox) : ox;        // flip after resize == sample the mirrored column
  const float scx = (float)c.w / S, scy = (float)c.h / S;
  const float isx = 1.f / fmaxf(scx, 1.f), isy = 1.f / fmaxf(scy, 1.f);
  const float supx = 2.f * fmaxf(scx, 1.f), supy = 2.f * fmaxf(scy, 1.f);
  const float cx = scx * (sx_out + 0.5f), cy = scy * (oy + 0.5f);
  int xmin, xmax, ymin, ymax;
  const float wxs = aa_window(cx, supx, isx, c.w, c.w, xmin, xmax);
  const float wys = aa_window(cy, supy, isy, c.h, c.h, ymin, ymax);
  const T* base = src + ((size_t)im.off + (size_t)c.y0 * im.w) * 3 + (size_t)c.x0 * 3;
  float r = 0.f, g = 0.f, b = 0.f;
  for (int y = ymin; y < ymax; ++y) {
    const float wy = cubic_aa<float>((y - cy + 0.5f) * isy);
    const T* row = base + (size_t)y * im.w * 3;
    float rr = 0.f, gg = 0.f, bb = 0.f;
    for (int x = xmin; x < xmax; ++x) {
      const float wx = cubic_aa<float>((x - cx + 0.5f) * isx);
      rr += wx * row[3 * x]; gg += wx * row[3 * x + 1]; bb += wx * row[3 * x + 2];
    }
    r += wy * rr; g += wy * gg; b += wy * bb;
  }
  const float norm = 1.f / ((std::is_same_v<T, uint8_t> ? 255.f : 1.f) * wxs * wys);
  float* o = out + (((size_t)n * S + oy) * S + ox) * 3;
  if constexpr (CLAMP) {
    // bicubic overshoots are clamped like a uint8 image would (PIL result is uint8)
    o[0] = fminf(fmaxf(r * norm, 0.f), 1.f); o[1] = fminf(fmaxf(g * norm, 0.f), 1.f); o[2] = fminf(fmaxf(b * norm, 0.f), 1.f);
  } else {
    o[0] = r * norm; o[1] = g * norm; o[2] = b * norm;
  }
}

// torchvision _rgb_to_grayscale_image weights
__device__ __forceinline__ float gray_of(float r, float g, float b) { return 0.2989f * r + 0.587f * g + 0.114f * b; }
__device__ __forceinline__ float clamp01(float x) { return fminf(fmaxf(x, 0.f), 1.f); }

// torchvision _rgb2hsv / _hsv2rgb on one pixel, hue shifted by fh (adjust_hue)
__device__ __forceinline__ void hue_shift(float& r, float& g, float& b, float fh) {
  const float maxc = fmaxf(r, fmaxf(g, b)), minc = fminf(r, fminf(g, b));
  const bool eqc = maxc == minc;
  const float cr = maxc - minc;
  const float s = cr / (eqc ? 1.f : maxc);
  const float crd = eqc ? 1.f : cr;
  const float rc = (maxc - r) / crd, gc = (maxc - g) / crd, bc = (maxc - b) / crd;
  float h = 0.f;
  if (maxc == r) h = bc - gc;
  else if (maxc == g) h = 2.f + rc - bc;
  else h = 4.f + gc - rc;
  h = h / 6.f + 1.f;
  h = h - floorf(h);
  h = h + fh;
  h = h - floorf(h);
  const float v = maxc;
  const float i = floorf(h * 6.f);
  const float f = h * 6.f - i;
  const int ii = ((int)i) % 6;
  const float p = clamp01(v * (1.f - s)), q = clamp01(v * (1.f - s * f)), t = clamp01(v * (1.f - s * (1.f - f)));
  switch (ii) {
    case 0: r = v; g = t; b = p; break;
    case 1: r = q; g = v; b = p; break;
    case 2: r = p; g = v; b = t; break;
    case 3: r = p; g = q; b = v; break;
    case 4: r = t; g = p; b = v; break;
    default: r = v; g = p; b = q; break;
  }
}

__device__ __forceinline__ void jitter_op(int op, const AugCrop& c, float mean_gray, float& r, float& g, float& b) {
  if (op == 0) { r = clamp01(r * c.fb); g = clamp01(g * c.fb); b = clamp01(b * c.fb); }
  else if (op == 1) { const float m = (1.f - c.fc) * mean_gray; r = clamp01(c.fc * r + m); g = clamp01(c.fc * g + m); b = clamp01(c.fc * b + m); }
  else if (op == 2) { const float m = (1.f - c.fs) * gray_of(r, g, b); r = clamp01(c.fs * r + m); g = clamp01(c.fs * g + m); b = clamp01(c.fs * b + m); }
  else if (op == 3) hue_shift(r, g, b, c.fh);
}

// Pass A: the jitter ops that come BEFORE contrast in this crop's order, plus the sum of the gray values of the result
// (contrast blends with the mean gray of the image it is applied to).  Pass B: contrast and what follows, then
// RandomGrayscale.  A crop without jitter / without a pending contrast simply passes through pass A untouched.
// x holds n images of `npix` pixels each (S x S crops, or whole H x W sources), or with an image table the ragged
// sources of a batch, each jittered with its own pixel count.
__device__ __forceinline__ void color_geometry(const AugImage* __restrict__ imgs, int n, int npix, long long& off,
                                               int& count) {
  if (imgs) { const AugImage im = imgs[n]; off = im.off; count = im.h * im.w; }
  else { off = (long long)n * npix; count = npix; }
}
__global__ void aug_color_a_kernel(float* __restrict__ x, const AugImage* __restrict__ imgs,
                                   const AugCrop* __restrict__ crops, float* __restrict__ gray_sum, int npix_dense) {
  const int n = blockIdx.y;
  const AugCrop c = crops[n];
  long long off;
  int npix;
  color_geometry(imgs, n, npix_dense, off, npix);
  float local = 0.f;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += gridDim.x * blockDim.x) {
    float* px = x + ((size_t)off + p) * 3;
    float r = px[0], g = px[1], b = px[2];
    if (c.order[0] >= 0)
      for (int k = 0; k < 4 && c.order[k] != 1; ++k) jitter_op(c.order[k], c, 0.f, r, g, b);
    px[0] = r; px[1] = g; px[2] = b;
    local += gray_of(r, g, b);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(&gray_sum[n], local);
}
__global__ void aug_color_b_kernel(float* __restrict__ x, const AugImage* __restrict__ imgs,
                                   const AugCrop* __restrict__ crops, const float* __restrict__ gray_sum, int npix_dense) {
  const int n = blockIdx.y;
  const AugCrop c = crops[n];
  long long off;
  int npix;
  color_geometry(imgs, n, npix_dense, off, npix);
  const float mean_gray = gray_sum[n] / npix;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += gridDim.x * blockDim.x) {
    float* px = x + ((size_t)off + p) * 3;
    float r = px[0], g = px[1], b = px[2];
    if (c.order[0] >= 0) {
      int k = 0;
      while (k < 4 && c.order[k] != 1) ++k;
      for (; k < 4; ++k) jitter_op(c.order[k], c, mean_gray, r, g, b);
    }
    if (c.gray) { const float y = gray_of(r, g, b); r = g = b = y; }
    px[0] = r; px[1] = g; px[2] = b;
  }
}

// torchvision _get_gaussian_kernel1d(9, sigma) taps, unnormalised; returns their sum
__device__ __forceinline__ float blur_taps(float sigma, float (&w)[9]) {
  float ws = 0.f;
#pragma unroll
  for (int k = 0; k < 9; ++k) { const float d = (float)(k - 4) / sigma; w[k] = __expf(-0.5f * d * d); ws += w[k]; }
  return ws;
}
// reflect padding (no edge repeat) of index t into [0, S), S >= 5
__device__ __forceinline__ int reflect(int t, int S) { return t < 0 ? -t : (t >= S ? 2 * S - 2 - t : t); }

// separable 9-tap Gaussian (torchvision gaussian_blur: kernel_size 9, reflect padding), one axis per launch
__global__ void aug_blur_kernel(const float* __restrict__ x, float* __restrict__ y, const AugBlur* __restrict__ blur, int S,
                                int vertical) {
  const int n = blockIdx.z;
  const int ox = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y * blockDim.y + threadIdx.y;
  if (ox >= S || oy >= S) return;
  const float sigma = blur[n].sigma;
  const float* xi = x + (size_t)n * S * S * 3;
  float* yo = y + (((size_t)n * S + oy) * S + ox) * 3;
  if (sigma <= 0.f) {
    const float* p = xi + ((size_t)oy * S + ox) * 3;
    yo[0] = p[0]; yo[1] = p[1]; yo[2] = p[2];
    return;
  }
  float w[9];
  const float ws = blur_taps(sigma, w);
  float r = 0.f, g = 0.f, b = 0.f;
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    int t = (vertical ? oy : ox) + k - 4;
    t = t < 0 ? -t : (t >= S ? 2 * S - 2 - t : t);           // reflect(); written out, the kernel keeps its schedule
    const float* p = xi + (vertical ? ((size_t)t * S + ox) : ((size_t)oy * S + t)) * 3;
    r += w[k] * p[0]; g += w[k] * p[1]; b += w[k] * p[2];
  }
  const float inv = 1.f / ws;
  yo[0] = r * inv; yo[1] = g * inv; yo[2] = b * inv;
}

// RandomSolarize(threshold 128): pixels >= 128/255 inverted
__device__ __forceinline__ float solarize(float v) { return v >= 128.f / 255.f ? 1.f - v : v; }

// RandomSolarize (pixels >= 128/255 inverted), Normalize(mean, std), cast to bf16 NHWC
__global__ void aug_finish_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ out,
                                  const AugCrop* __restrict__ crops, int S, float m0, float m1, float m2, float is0,
                                  float is1, float is2) {
  const int n = blockIdx.y;
  const int sol = crops[n].solarize;
  const int npix = S * S;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += gridDim.x * blockDim.x) {
    const float* px = x + ((size_t)n * npix + p) * 3;
    float r = px[0], g = px[1], b = px[2];
    if (sol) { r = solarize(r); g = solarize(g); b = solarize(b); }
    __nv_bfloat16* o = out + ((size_t)n * npix + p) * 3;
    o[0] = __float2bfloat16((r - m0) * is0); o[1] = __float2bfloat16((g - m1) * is1); o[2] = __float2bfloat16((b - m2) * is2);
  }
}

// RandomSolarize in place, for crops that are resized after their distortions (gram crops with distortions: the
// reference normalises, then resizes; Resize commutes with Normalize but not with Solarize)
__global__ void aug_solarize_kernel(float* __restrict__ x, const AugCrop* __restrict__ crops, int S) {
  const int n = blockIdx.y;
  if (!crops[n].solarize) return;
  const int npix = S * S;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += gridDim.x * blockDim.x) {
    float* px = x + ((size_t)n * npix + p) * 3;
    px[0] = solarize(px[0]); px[1] = solarize(px[1]); px[2] = solarize(px[2]);
  }
}

// uint8 [n, npix, 3] -> fp32 [0, 1] copy (share_color_jitter transforms the whole source image before any crop)
__global__ void aug_u8_to_f32_kernel(const uint8_t* __restrict__ src, float* __restrict__ x, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    x[i] = src[i] * (1.f / 255.f);
}

// Local crops cut from a global base crop (local_crops_subset_of_global_crops): the reference jitters and blurs the
// WHOLE M x M base, then slices an L x L window at (y0, x0).  Per window record (img = base index):
//  gray   pass A of aug_color over the whole base without writing it: the contrast mean of the whole image;
//  gather the window plus a 4-pixel halo, reflected at the base's border, through the full jitter and grayscale;
//  blur   valid-mode 9-tap Gaussian over the halo (what the whole-image blur gives inside the window).
__global__ void aug_window_gray_kernel(const float* __restrict__ base, int M, const AugCrop* __restrict__ crops,
                                       float* __restrict__ gray_sum) {
  const int n = blockIdx.y;
  const AugCrop c = crops[n];
  if (c.order[0] < 0) return;                                // no jitter: the mean is never read
  const int npix = M * M;
  const float* xi = base + (size_t)c.img * npix * 3;
  float local = 0.f;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += gridDim.x * blockDim.x) {
    const float* px = xi + (size_t)p * 3;
    float r = px[0], g = px[1], b = px[2];
    for (int k = 0; k < 4 && c.order[k] != 1; ++k) jitter_op(c.order[k], c, 0.f, r, g, b);
    local += gray_of(r, g, b);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(&gray_sum[n], local);
}
__global__ void aug_window_gather_kernel(const float* __restrict__ base, int M, const AugCrop* __restrict__ crops,
                                         const float* __restrict__ gray_sum, float* __restrict__ win, int L) {
  const int n = blockIdx.z, E = L + 8;
  const int ox = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y * blockDim.y + threadIdx.y;
  if (ox >= E || oy >= E) return;
  const AugCrop c = crops[n];
  const int sx = reflect(c.x0 - 4 + ox, M), sy = reflect(c.y0 - 4 + oy, M);
  const float* px = base + (((size_t)c.img * M + sy) * M + sx) * 3;
  float r = px[0], g = px[1], b = px[2];
  if (c.order[0] >= 0) {
    const float mean_gray = gray_sum[n] / (M * M);
    for (int k = 0; k < 4; ++k) jitter_op(c.order[k], c, mean_gray, r, g, b);
  }
  if (c.gray) { const float y = gray_of(r, g, b); r = g = b = y; }
  float* o = win + (((size_t)n * E + oy) * E + ox) * 3;
  o[0] = r; o[1] = g; o[2] = b;
}
// x [n, Hin, Win, 3] -> y [n, Hin, Win - 8, 3] (horizontal) or [n, Hin - 8, Win, 3] (vertical)
__global__ void aug_blur_valid_kernel(const float* __restrict__ x, float* __restrict__ y, const AugBlur* __restrict__ blur,
                                      int Hin, int Win, int vertical) {
  const int n = blockIdx.z;
  const int Ho = vertical ? Hin - 8 : Hin, Wo = vertical ? Win : Win - 8;
  const int ox = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y * blockDim.y + threadIdx.y;
  if (ox >= Wo || oy >= Ho) return;
  const float sigma = blur[n].sigma;
  const float* xi = x + (size_t)n * Hin * Win * 3;
  float* yo = y + (((size_t)n * Ho + oy) * Wo + ox) * 3;
  if (sigma <= 0.f) {
    const float* p = xi + (vertical ? ((size_t)(oy + 4) * Win + ox) : ((size_t)oy * Win + ox + 4)) * 3;
    yo[0] = p[0]; yo[1] = p[1]; yo[2] = p[2];
    return;
  }
  float w[9];
  const float ws = blur_taps(sigma, w);
  float r = 0.f, g = 0.f, b = 0.f;
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    const float* p = xi + (vertical ? ((size_t)(oy + k) * Win + ox) : ((size_t)oy * Win + ox + k)) * 3;
    r += w[k] * p[0]; g += w[k] * p[1]; b += w[k] * p[2];
  }
  const float inv = 1.f / ws;
  yo[0] = r * inv; yo[1] = g * inv; yo[2] = b * inv;
}

}  // namespace d3

using namespace d3;
#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

extern "C" {

// One launch of aug_resized_crop_kernel for every entry point: imgs = nullptr reads a dense [n_img, H, W, 3] batch.
static int launch_resized_crop(const void* src, bool f32, int clamp, const AugImage* imgs, int H, int W,
                               const void* crops, int n_crops, float* out, int S, void* stream) {
  dim3 block(32, 8), grid((S + 31) / 32, (S + 7) / 8, n_crops);
  const AugCrop* c = (const AugCrop*)crops;
  if (!f32)
    aug_resized_crop_kernel<uint8_t, true><<<grid, block, 0, STREAM(stream)>>>((const uint8_t*)src, imgs, H, W, c, out, S);
  else if (clamp)
    aug_resized_crop_kernel<float, true><<<grid, block, 0, STREAM(stream)>>>((const float*)src, imgs, H, W, c, out, S);
  else
    aug_resized_crop_kernel<float, false><<<grid, block, 0, STREAM(stream)>>>((const float*)src, imgs, H, W, c, out, S);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

// Argument checks of the ragged entry points, before any CUDA call.  The crop records are read from their host copy:
// every crop must name a row of the image table (its box is checked against that image's size by the caller, which
// drew it).
static int check_ragged(const char* what, const void* src, const void* imgs, int n_img, const void* crops,
                        const void* crops_host, int n_crops, const void* out, int S) {
  char buf[160];
  if (!src || !imgs || !crops || !crops_host || !out) snprintf(buf, sizeof(buf), "%s: null pointer", what);
  else if (n_img < 1) snprintf(buf, sizeof(buf), "%s: n_img < 1", what);
  else if (S < 5) snprintf(buf, sizeof(buf), "%s: S < 5", what);
  else {
    const AugCrop* c = (const AugCrop*)crops_host;
    int i = 0;
    while (i < n_crops && c[i].img >= 0 && c[i].img < n_img) ++i;
    if (i == n_crops) return D3_OK;
    snprintf(buf, sizeof(buf), "%s: crop %d reads image %d of a %d-image table", what, i, c[i].img, n_img);
  }
  return set_error(D3_ERR_ARG, buf);
}

int d3_aug_resized_crop(const void* src_u8, int n_img, int H, int W, const void* crops, int n_crops, float* out, int S,
                        void* stream) {
  if (n_crops <= 0) return D3_OK;
  if (S < 5 || H <= 0 || W <= 0 || n_img <= 0) return set_error(D3_ERR_ARG, "d3_aug_resized_crop: bad geometry");
  return launch_resized_crop(src_u8, false, 1, nullptr, H, W, crops, n_crops, out, S, stream);
}

int d3_aug_resized_crop_ragged(const void* src_u8, const void* imgs, int n_img, const void* crops, const void* crops_host,
                               int n_crops, float* out, int S, void* stream) {
  if (n_crops <= 0) return D3_OK;
  if (int rc = check_ragged("d3_aug_resized_crop_ragged", src_u8, imgs, n_img, crops, crops_host, n_crops, out, S))
    return rc;
  return launch_resized_crop(src_u8, false, 1, (const AugImage*)imgs, 0, 0, crops, n_crops, out, S, stream);
}

int d3_aug_color(float* x, const void* crops, int n_crops, int S, float* gray_sum /* [n_crops] zeroed */, void* stream) {
  if (n_crops <= 0) return D3_OK;
  dim3 grid(min((S * S + 255) / 256, 64), n_crops);
  aug_color_a_kernel<<<grid, 256, 0, STREAM(stream)>>>(x, nullptr, (const AugCrop*)crops, gray_sum, S * S);
  aug_color_b_kernel<<<grid, 256, 0, STREAM(stream)>>>(x, nullptr, (const AugCrop*)crops, gray_sum, S * S);
  D3_CHECK_LAUNCH();
  count_launch(1);
  return D3_OK;
}

int d3_aug_blur(const float* x, float* tmp, float* y, const void* blur, int n_crops, int S, void* stream) {
  if (n_crops <= 0) return D3_OK;
  if (S < 5) return set_error(D3_ERR_ARG, "d3_aug_blur: S < 5");
  dim3 block(32, 8), grid((S + 31) / 32, (S + 7) / 8, n_crops);
  aug_blur_kernel<<<grid, block, 0, STREAM(stream)>>>(x, tmp, (const AugBlur*)blur, S, 0);
  aug_blur_kernel<<<grid, block, 0, STREAM(stream)>>>(tmp, y, (const AugBlur*)blur, S, 1);
  D3_CHECK_LAUNCH();
  count_launch(1);
  return D3_OK;
}

int d3_aug_finish(const float* x, void* out_bf16, const void* crops, int n_crops, int S, const float* mean3,
                  const float* std3, void* stream) {
  if (n_crops <= 0) return D3_OK;
  dim3 grid(min((S * S + 255) / 256, 64), n_crops);
  aug_finish_kernel<<<grid, 256, 0, STREAM(stream)>>>(x, (__nv_bfloat16*)out_bf16, (const AugCrop*)crops, S, mean3[0], mean3[1],
                                                     mean3[2], 1.f / std3[0], 1.f / std3[1], 1.f / std3[2]);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_aug_resized_crop_f32(const float* src, int n_img, int H, int W, const void* crops, int n_crops, float* out, int S,
                            int clamp, void* stream) {
  if (n_crops <= 0) return D3_OK;
  if (S < 5 || H <= 0 || W <= 0 || n_img <= 0) return set_error(D3_ERR_ARG, "d3_aug_resized_crop_f32: bad geometry");
  return launch_resized_crop(src, true, clamp, nullptr, H, W, crops, n_crops, out, S, stream);
}

int d3_aug_resized_crop_ragged_f32(const float* src, const void* imgs, int n_img, const void* crops,
                                   const void* crops_host, int n_crops, float* out, int S, int clamp, void* stream) {
  if (n_crops <= 0) return D3_OK;
  if (int rc = check_ragged("d3_aug_resized_crop_ragged_f32", src, imgs, n_img, crops, crops_host, n_crops, out, S))
    return rc;
  return launch_resized_crop(src, true, clamp, (const AugImage*)imgs, 0, 0, crops, n_crops, out, S, stream);
}

// share_color_jitter: fp32 copy of the n_pix packed source pixels, then the jitter of each whole image with its record
static int color_images(const uint8_t* src, long long n_pix, const AugImage* imgs, int n_img, int npix_dense,
                        const void* recs, float* x, float* gray_sum, int blocks_per_image, void* stream) {
  const long long n = n_pix * 3;
  aug_u8_to_f32_kernel<<<(int)std::min<long long>((n + 255) / 256, 4096), 256, 0, STREAM(stream)>>>(src, x, n);
  dim3 grid(blocks_per_image, n_img);
  aug_color_a_kernel<<<grid, 256, 0, STREAM(stream)>>>(x, imgs, (const AugCrop*)recs, gray_sum, npix_dense);
  aug_color_b_kernel<<<grid, 256, 0, STREAM(stream)>>>(x, imgs, (const AugCrop*)recs, gray_sum, npix_dense);
  D3_CHECK_LAUNCH();
  count_launch(2);
  return D3_OK;
}

int d3_aug_color_images(const void* src_u8, int n_img, int H, int W, const void* recs, float* x, float* gray_sum,
                        void* stream) {
  if (n_img <= 0) return D3_OK;
  if (H <= 0 || W <= 0) return set_error(D3_ERR_ARG, "d3_aug_color_images: bad geometry");
  return color_images((const uint8_t*)src_u8, (long long)n_img * H * W, nullptr, n_img, H * W, recs, x, gray_sum,
                      min((H * W + 255) / 256, 64), stream);
}

int d3_aug_color_images_ragged(const void* src_u8, long long n_pix, const void* imgs, int n_img, const void* recs,
                               const void* recs_host, float* x, float* gray_sum, void* stream) {
  if (int rc = check_ragged("d3_aug_color_images_ragged", src_u8, imgs, n_img, recs, recs_host, n_img, x, 5)) return rc;
  if (!gray_sum || n_pix < 1) return set_error(D3_ERR_ARG, "d3_aug_color_images_ragged: null gray_sum or n_pix < 1");
  return color_images((const uint8_t*)src_u8, n_pix, (const AugImage*)imgs, n_img, 0, recs, x, gray_sum, 64, stream);
}

int d3_aug_solarize(float* x, const void* crops, int n_crops, int S, void* stream) {
  if (n_crops <= 0) return D3_OK;
  dim3 grid(min((S * S + 255) / 256, 64), n_crops);
  aug_solarize_kernel<<<grid, 256, 0, STREAM(stream)>>>(x, (const AugCrop*)crops, S);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_aug_local_windows(const float* base, int n_base, int M, const void* crops, const void* blur, int n_crops, int L,
                         float* win, float* tmp, float* y, float* gray_sum, void* stream) {
  if (n_crops <= 0) return D3_OK;
  if (M < 5 || L < 1 || L > M || n_base <= 0) return set_error(D3_ERR_ARG, "d3_aug_local_windows: bad geometry");
  const int E = L + 8;
  aug_window_gray_kernel<<<dim3(min((M * M + 255) / 256, 64), n_crops), 256, 0, STREAM(stream)>>>(
      base, M, (const AugCrop*)crops, gray_sum);
  dim3 block(32, 8);
  aug_window_gather_kernel<<<dim3((E + 31) / 32, (E + 7) / 8, n_crops), block, 0, STREAM(stream)>>>(
      base, M, (const AugCrop*)crops, gray_sum, win, L);
  aug_blur_valid_kernel<<<dim3((L + 31) / 32, (E + 7) / 8, n_crops), block, 0, STREAM(stream)>>>(
      win, tmp, (const AugBlur*)blur, E, E, 0);
  aug_blur_valid_kernel<<<dim3((L + 31) / 32, (L + 7) / 8, n_crops), block, 0, STREAM(stream)>>>(
      tmp, y, (const AugBlur*)blur, E, L, 1);
  D3_CHECK_LAUNCH();
  count_launch(3);
  return D3_OK;
}

}  // extern "C"
