/* dinov3_b200.h — C ABI of libdinov3_b200.so: the H100 (sm_90a) kernels behind the DINOv3 SSL training hot path.
 *
 * The reference (Dhia-naouali/dinov3-jax) has no FFI: its hot path is Flax modules traced by jax.jit.  Each entry
 * point below therefore cites the reference *module call site* (path:line under dinov3_jax/) whose arithmetic it
 * replaces; INTEGRATION.md shows the ctypes binding a maintainer would add.
 *
 * Conventions
 *   - every pointer is a caller-owned DEVICE pointer (torch.Tensor.data_ptr()); the library allocates nothing
 *     persistent; `stream` is a cudaStream_t passed as void*; every call is asynchronous on that stream.
 *   - return value: D3_OK (0) or a negative d3_status; d3_last_error() gives the message for the calling thread.
 *     Launch-configuration errors are reported synchronously, asynchronous faults surface at the next sync.
 *   - one process per GPU, calls come from that process' single training thread.
 *   - there is NO CPU fallback: without an sm_90 (Hopper) GPU d3_init() fails.
 */
#ifndef DINOV3_B200_H
#define DINOV3_B200_H
#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  D3_OK = 0,
  D3_ERR_ARG = -1,     /* bad shape / alignment / null pointer */
  D3_ERR_CUDA = -2,    /* CUDA runtime or driver error (message has the CUDA string) */
  D3_ERR_DEVICE = -3,  /* not an sm_90 device */
} d3_status;

/* ---- library ------------------------------------------------------------------------------------------------ */
int d3_init(int device);                /* bind to device, cache SM count, resolve cuTensorMapEncodeTiled */
const char* d3_last_error(void);
int d3_abi_version(void);
/* Cap the grid of the persistent kernels (GEMMs) to n SMs (0 = all).  Multi-GPU runs leave a few SMs to the NCCL
 * kernels of the FSDP all-gather / reduce-scatter so they run under the GEMMs instead of between them.              */
int d3_set_sm_limit(int n);
long long d3_launch_count(void);        /* kernels launched by this library since the last reset (bench: gpu_launches) */
void d3_reset_launch_count(void);

/* ---- dense contraction (wgmma / TMA) -----------------------------------------------------------------------------
 * D[M,N] = epilogue( alpha * A[M,K] . B[K,N] ), bf16 operands, fp32 accumulation in registers.
 *   a_major = 0: A stored [M][K] (row stride lda)      a_major = 1: A stored [K][M]
 *   b_major = 0: B stored [N][K] (row stride ldb)      b_major = 1: B stored [K][N]   (reference kernel layout [in,out])
 * Replaces nn.Dense / nn.Conv(stride=kernel) at layers/attention.py:63-65,94,101, layers/ffn_layers.py:36-47,
 * layers/patch_embed.py:38-51, layers/dino_head.py:20-43,65-85, and their jax.grad transposes (train/train.py:504-513).
 * Epilogue order: +bias -> [store bf16 pre-activation] -> [tanh-GELU] -> [* GELU'(aux_in)] -> [* gamma] -> [+ resid]
 *                 -> [+= out] -> store (bf16 or fp32).   (layers/block.py:198-199, layers/layer_scale.py:17-21)     */
enum {
  D3_EP_BIAS = 1,       /* v += bias[n]                       (fp32 [N]) */
  D3_EP_GELU = 2,       /* v = gelu_tanh(v)                   flax nn.gelu, approximate=True */
  D3_EP_STORE_PRE = 4,  /* aux_out[m,n] = bf16(v) before the activation (stash for backward) */
  D3_EP_MUL_DGELU = 8,  /* v *= gelu_tanh'(aux_in[m,n])       backward through an activation */
  D3_EP_GAMMA = 16,     /* v *= gamma[n]                      LayerScale */
  D3_EP_RESID = 32,     /* v += resid[m,n]                    fp32 residual stream */
  D3_EP_OUT_F32 = 64,   /* out is fp32 (default bf16) */
  D3_EP_ACCUM = 128,    /* out += v (fp32 out only; weight-gradient accumulation over crop sets) */
  D3_EP_SCATTER = 256, /* add the result into peer-mapped shard slices (see d3_gemm_epilogue.sc_*) */
};
typedef struct {
  const float* bias;
  const float* gamma;
  const float* resid;
  const void* aux_in;   /* bf16 [M, ld_aux] */
  void* aux_out;        /* bf16 [M, ld_aux] */
  void* out;            /* bf16 or fp32 [M, ld_out] */
  int ld_out, ld_aux, ld_resid;
  int flags;
  float alpha;
  /* D3_EP_SCATTER (fused weight-gradient reduce-scatter, replaces jax.lax.psum_scatter at fsdp/utils.py:61-64): the fp32
   * result, scaled by alpha (= 1/world for the mean), is ADDED into the rank that owns each element instead of being
   * stored at `out`: output element e = row*ld_out + col has index g = sc_off + e in a flat range split into sc_world
   * slices of sc_shard elements; it is accumulated at sc_peer[g / sc_shard] + g % sc_shard, where sc_peer[r] is rank
   * r's (peer-mapped, zero-initialised) shard slice for that range.  `out` is only used for its alignment.           */
  float* sc_peer[8];
  long long sc_off;
  int sc_shard, sc_world;
} d3_gemm_epilogue;
/* tile_n : 0 = auto; 64 / 128 = 128-row tiles of that width; 256 and 512 (wider tiles) are taken as 128.
 * split_k: 0 = auto (used only for plain fp32 outputs with D3_EP_ACCUM, i.e. weight gradients: the slices' partial sums
 *          are added to `out`, which the caller zeroes or wants accumulated into, in slice order); >= 1 = forced.  */
int d3_gemm_bf16(const void* A, int lda, int a_major, const void* B, int ldb, int b_major, int M, int N, int K,
                 const d3_gemm_epilogue* ep, int tile_n, int split_k, void* stream);

/* ---- patch embedding / token assembly ---------------------------------------------------------------------------
 * layers/patch_embed.py:38-51: the stride==kernel conv is im2col + GEMM (d3_gemm_bf16 with the kernel viewed as
 * [p*p*3, D]); models/vision_transformer.py:173-203: where(mask, mask_token, x), prepend cls.                        */
int d3_im2col(const void* img_bf16 /*[n,H,W,3]*/, void* out_bf16 /*[n*Hp*Wp, ld_out >= p*p*3], padding zeroed*/,
              int ld_out, int n, int H, int W, int p, void* stream);
int d3_assemble_tokens(const float* tok /*[n*P,D]*/, const float* cls /*[D]*/, const float* storage /*[R,D] or NULL*/,
                       const float* mask_token /*[D]*/, const unsigned char* masks /*[n*P] or NULL*/,
                       float* X /*[n,1+R+P,D]: cls, R storage tokens, patches*/, int n, int P, int R, int D, void* stream);
int d3_assemble_tokens_bwd(const float* dX, const unsigned char* masks, void* dTok_bf16 /*[n*P,D]*/,
                           float* dcls /*[D] +=*/, float* dstorage /*[R,D] += or NULL*/, float* dmask_token /*[D] +=*/,
                           int n, int P, int R, int D, void* stream);

/* ---- LayerNorm (models/vision_transformer.py:40: eps 1e-6, biased variance E[x^2]-E[x]^2, fp32 statistics) ------- */
int d3_layernorm_fwd(const float* x /*[T,D]*/, const float* scale, const float* bias, void* y, int y_is_f32,
                     float* mean /*[T] or NULL*/, float* rstd, int T, int D, float eps, void* stream);
/* LayerNorm backward: dx = LN'(dy) (+ dx_add), dscale += colsum(dy * xhat), dbias += colsum(dy); with ls_gamma == NULL
 * that is all it does (the plain LayerNorm backward).  With ls_gamma it is fused with the LayerScale (+GELU) backward
 * of the branch upstream of it (layers/block.py:198-199 x_out = x_in + gamma * act(u); layers/layer_scale.py:17-21):
 * with dx the row gradient it has just produced it also writes du = bf16(dx * gamma * act'(u)), ls_dbias += colsum(du)
 * and, when the stash `ls_u` is given, ls_dgamma += colsum(dx * act(u)) (act = tanh-GELU if ls_gelu else identity).
 * ls_u == NULL: act = identity, dgamma comes from d3_ls_gamma_from_wgrad.                                           */
int d3_layernorm_bwd_ls(const void* dy, int dy_is_f32, const float* x, const float* mean, const float* rstd,
                        const float* scale, const float* dx_add /*residual-stream gradient or NULL*/, float* dx,
                        float* dscale /*[D] += or NULL*/, float* dbias /*[D] +=*/, int T, int D,
                        const float* ls_gamma /*[D] or NULL*/, const void* ls_u_bf16 /*[T,D] or NULL*/, int ls_gelu,
                        void* ls_du_bf16 /*[T,D]*/, float* ls_dgamma /*[D] += or NULL*/, float* ls_dbias /*[D] +=*/,
                        void* stream);
/* LayerScale gradient of a linear branch x + gamma * (a W + b) from that layer's weight gradient:
 * dgamma_j += (sum_i W_ij dW_ij + b_j db_j) / gamma_j   (W bf16 [K,N] as used by the forward, dW fp32 [K,N]).        */
int d3_ls_gamma_from_wgrad(const void* W_bf16, const float* dW, const float* bias, const float* dbias,
                           const float* gamma, float* dgamma, int K, int N, void* stream);

/* ---- FSDP gradient reduce-scatter without NCCL (fsdp/utils.py:61-64 psum_scatter/n, :108 pmean) ---------------------
 * adds alpha * src[i] into the rank owning flat index off + i of a range split into `world` slices of `shard` elements;
 * peers[r] = rank r's zero-initialised slice (a pointer valid in THIS process: NVLink peer mapping, peers[rank] local).
 * The caller orders the step with a cross-rank barrier before the slices are consumed.                               */
/* 0 (default): one device-scope vector red per float4; 1: four scalar system-scope atomics (also env D3_FSDP_PUSH_SYS=1).
 * Applies to D3_EP_SCATTER and d3_scatter_add_peers.                                                                   */
int d3_set_scatter_mode(int mode);
int d3_scatter_add_peers(const float* src, long long n, float* const* peers /*host array [world]*/, int world,
                         long long off, int shard, float alpha, void* stream);

/* Small all-reduce over NVLink peer mappings: out[i] = reduce over r (in rank order: identical bits on every rank) of
 * peers[r][i]; op 0 = sum (jax.lax.psum: loss/dino_clstoken_loss.py:53, loss/ibot_patch_loss.py:99, the gradient norms of
 * train/train.py:516-541), 1 = max.  peers[r] = rank r's staged input (pointer valid in THIS process); the caller
 * brackets the call with a cross-rank barrier after the inputs were written (and re-uses an input buffer no earlier than
 * two barriers later).                                                                                                 */
int d3_allreduce_peers(const float* const* peers /*host array [world]*/, int world, float* out, long long n, int op,
                       void* stream);

/* ---- RoPE (layers/attention.py:14-20,69-90; tables from layers/rope_position_encoding.py:117-123) -----------------
 * in place on the q and k thirds of qkv bf16 [T,3D]; tokens t < prefix of every crop are left untouched.             */
int d3_rope(void* qkv_bf16, const float* sin_t /*[P,hd]*/, const float* cos_t, long long T, int tokens_per_crop,
            int prefix, int D, int head_dim, int inverse, void* stream);

/* ---- attention (layers/attention.py:116 nn.dot_product_attention; head_dim 64, N <= 448 fwd / 384 bwd) ------------ */
int d3_attn_fwd(const void* qkv_bf16 /*[n*N,3D] post-RoPE*/, void* o_bf16 /*[n*N,D]*/, float* lse /*[n,H,N] or NULL*/,
                int n_crops, int N, int D, int H, void* stream);
/* rope_sin / rope_cos ([P,64] fp32, or NULL): when given, the inverse rotation (transpose of layers/attention.py:19-20)
 * is applied to dq / dk of tokens >= rope_prefix before they are stored, i.e. dqkv is the gradient w.r.t. the
 * pre-RoPE qkv projection output.                                                                                  */
int d3_attn_bwd(const void* qkv_bf16, const void* o_bf16, const void* do_bf16, const float* lse,
                float* delta_scratch /*[n,H,N]*/, void* dqkv_bf16 /*[n*N,3D]*/, int n_crops, int N, int D, int H,
                const float* rope_sin, const float* rope_cos, int rope_prefix, void* stream);

/* diagnostics: when buf != NULL, CTA (0,0) of d3_attn_bwd writes clock64() marks (2 threads x 32 slots) into it */
int d3_debug_attn_trace(long long* buf);

/* ---- row gather / scatter (train/ssl_meta_arch.py:377,432 patch.reshape(-1,D)[mask_indices_list]; cls = token 0) --- */
int d3_token_rows(const long long* mask_indices /*int64 [count] (mode 0)*/, int* rows /*int32 [count]*/, int count,
                  int P, int prefix /*tokens before the patches: 1 + n_storage_tokens*/,
                  int mode /*0: masked patch -> token row, 1: cls row of crop i*/, void* stream);
int d3_gather_rows(const float* src /*[*,D]*/, const int* rows, void* dst_bf16 /*or NULL*/, float* dst_f32 /*or NULL*/,
                   int R, int D, void* stream);
int d3_scatter_add_rows(const void* src, int src_is_f32, const int* rows, float* dst /*+=*/, int R, int D, void* stream);

/* ---- DINO head pieces (layers/dino_head.py:78-85) ----------------------------------------------------------------- */
int d3_l2norm_fwd(const float* u /*[R,C]*/, void* y_bf16, float* nrm /*[R]*/, int R, int C, float eps, void* stream);
int d3_l2norm_bwd(const void* g_bf16, const float* u, const float* nrm, void* du_bf16, int R, int C, float eps,
                  void* stream);

/* ---- backward helpers ----------------------------------------------------------------------------------------------
 * d3_ls_act_bwd: x_out = x_in + gamma * act(u) (layers/block.py:198-199): du = dX*gamma*act'(u) (bf16),
 * dgamma += colsum(dX*act(u)), dbias += colsum(du).  d3_colsum_bf16: bias gradients.                                 */
int d3_ls_act_bwd(const float* dX /*[T,D]*/, const void* u_bf16, const float* gamma, void* du_bf16, float* dgamma,
                  float* dbias, int T, int D, int use_gelu, void* stream);
int d3_colsum_bf16(const void* x_bf16 /*[T,N], row stride ld*/, float* out /*[N] +=*/, long long T, int N, int ld,
                   void* stream);
int d3_cast_f32_bf16(const float* src, void* dst_bf16, long long n, void* stream);

/* ---- SwiGLU FFN gate (layers/ffn_layers.py:52-76, the 7B recipe's ffn_layer: swiglu64): x12 = [x1 | x2] is the [T, 2*Hs]
 * bf16 output of the w1 / w2 projections; h = silu(x1) * x2; backward dx1 = dh*x2*silu'(x1), dx2 = dh*silu(x1).     */
int d3_swiglu_fwd(const void* x12_bf16 /*[T,2Hs]*/, void* h_bf16 /*[T,Hs]*/, long long T, int Hs, void* stream);
int d3_swiglu_bwd(const void* x12_bf16, const void* dh_bf16 /*[T,Hs]*/, void* dx12_bf16 /*[T,2Hs]*/, long long T, int Hs,
                  void* stream);

/* ---- Sinkhorn-Knopp (loss/dino_clstoken_loss.py:35-62, loss/ibot_patch_loss.py:77-109) ----------------------------
 * Q[b,k] = Btot * exp((L[b,k]-mx[k])/temp) * r[k] * a[b],  r = 1/(K * E^T a),  a = 1/(Btot * E r); the caller alternates
 * colsum (-> all-reduce over ranks of s[K]) and rowsum three times.  mx is a [K] vector of per-prototype shifts that
 * cancel exactly in E*r: d3_colmax (column maxima, all-reduce MAX over ranks) for Sinkhorn, so that a prototype far
 * below the batch maximum keeps its mass 1/K as in the reference's unshifted exp (:39); the softmax-centering path
 * fills it with the global maximum from d3_absmax.                                                                 */
int d3_absmax(const float* L, long long n, float* out /*pre-set to -inf*/, void* stream);
int d3_colmax(const float* L /*[R,K]*/, float* cm /*[K] pre-set to -inf*/, int R, int K, void* stream);
int d3_sinkhorn_colsum(const float* L /*[R,K]*/, const float* mx, float temp, const float* a /*[R] or NULL (=1)*/,
                       float* s /*[K] zeroed, +=*/, int R, int K, void* stream);
int d3_sinkhorn_rowsum(const float* L, const float* mx, float temp, const float* s, const float* btot /*device*/,
                       float* a /*[R]*/, int R, int K, void* stream);
int d3_sinkhorn_probs(const float* L, const float* mx, float temp, const float* s, const float* a, const float* btot,
                      float* Q /*[R,K]*/, int R, int K, void* stream);

/* ---- softmax centering (optional teacher normalisation; loss/dino_clstoken_loss.py:24-33,91-95, ibot :28-36,69-73) ----
 * center <- m*center + (1-m)*colsum/total_rows; s_out[k] = exp((center[k]-max center)/temp)/K.  One d3_sinkhorn_rowsum
 * with this s then gives a[] such that the teacher probabilities are softmax((L-center)/temp) for d3_ce_fwd_bwd.   */
int d3_colsum_f32(const float* L /*[R,K]*/, float* out /*[K] zeroed, +=*/, int R, int K, void* stream);
int d3_center_update(float* center /*[K]*/, const float* colsum /*[K] (all-reduced)*/, const float* total_rows /*device*/,
                     float momentum, float temp, float* s_out /*[K]*/, int K, void* stream);

/* ---- cross-entropy over prototypes, forward + backward fused (loss/dino_clstoken_loss.py:66-89,
 * loss/ibot_patch_loss.py:13-14,55-67; weights train/ssl_meta_arch.py:480-525) ---------------------------------------
 * per student row i with teacher rows t0[i], t1[i] (-1 = none): metric[slot[i]] += wm[i] * CE_i;
 * dS[i,:] = wg[i]/student_temp * (npairs*softmax(S_i/student_temp) - sum_p Q_p)  (bf16; NULL = forward only).
 * s_t == NULL: the rows of Lt are already teacher probabilities (mx / a_t / btot ignored); mx is the [K] shift vector
 * of the Sinkhorn section above.                                                                                   */
int d3_ce_fwd_bwd(const float* S /*[Rs,K]*/, float student_temp, const float* Lt /*[Rt,K] teacher logits*/,
                  const float* mx, float teacher_temp, const float* s_t /*[K]*/, const float* a_t /*[Rt]*/,
                  const float* btot, const int* t0, const int* t1, const float* wm, const float* wg, const int* slot,
                  float* metric, void* dS_bf16, int Rs, int K, void* stream);

/* ---- Gram-anchoring loss (loss/gram_loss.py:13-50; SURVEY 8f.2), elementwise stage: given the similarity matrices
 * Ss = Xs Xs^T, St = Xt Xt^T (fp32 [n*n], produced by d3_gemm_bf16 on the L2-normalised patch features) applies the
 * negative-removal mode (0 none | 1 remove_neg | 2 remove_only_teacher_neg, lines 40-48), accumulates
 * *loss += inv_count * sum (s' - t')^2 (line 50: mean) and writes G = (s' - t') * ds'/ds as bf16 (or skips it when
 * G_bf16 is NULL), the left operand of the backward GEMM dXs = (4 w / n^2) G Xs.
 * block > 0 (gram.img_level: true): Ss / St are [n, n] and only the diagonal blocks of block x block tokens (one image
 * each) count; the rest contributes nothing and gets G = 0.                                                           */
int d3_gram_diff(const float* Ss, const float* St, void* G_bf16, long long n_elems, int mode, float inv_count, float* loss,
                 int n, int block, void* stream);

/* Gram teacher features at crops.gram_teacher_crops_size -> the student's patch grid (gram.global_teacher_resize_method:
 * bicubic, gram.global_teacher_resize_antialias; configs/ssl_default_config.yaml:71-72): fp32 token maps
 * [n, Hs, Ws, D] -> [n, Hd, Wd, D], torch's upsample_bicubic2d (antialias 0) / _upsample_bicubic2d_aa (1) arithmetic. */
int d3_resize_tokens_bicubic(const float* src, float* dst, int n, int Hs, int Ws, int Hd, int Wd, int D, int antialias,
                             void* stream);

/* ---- KoLeo (loss/koleo_loss.py:16-35), forward + backward: metric += w_metric * loss; dx += w_grad * dloss/dx ------ */
int d3_koleo_fwd_bwd(const float* x /*[B,D]*/, float* xn_scratch /*[B,D]*/, float* nrm_scratch /*[B]*/,
                     int* nn_scratch /*[B]*/, float* coef_scratch /*[B]*/, float* metric, float* dx /*[B,D] +=*/, int B,
                     int D, float eps, float w_metric, float w_grad, void* stream);
/* KoLeoLossDistributed (loss/koleo_loss.py:39-70): x holds the all-gathered rows of every rank; only the local rows
 * [row0, row0+nrows) contribute loss terms (mean over nrows), neighbours are searched over all B rows; dx gets the
 * gradient for all B rows (the caller reduce-scatters the other ranks' parts).                                     */
int d3_koleo_fwd_bwd_rows(const float* x /*[B,D]*/, float* xn_scratch, float* nrm_scratch, int* nn_scratch,
                          float* coef_scratch, float* metric, float* dx /*[B,D] +=*/, int B, int D, int row0, int nrows,
                          float eps, float w_metric, float w_grad, void* stream);

/* ---- optimiser (train/train.py:516-541 clip, :95-106,562-563 optax.adamw; train/ssl_meta_arch.py:650-652 EMA) -------
 * flat fp32 buffers; segs = array of {int64 start; float lr_mult, wd_mult; int is_last_layer, pad} sorted by start.  */
int d3_sumsq(const float* g, long long n, float* out /*+=*/, void* stream);
int d3_adamw_ema(float* p, const float* g, float* m, float* v, float* teacher, void* p_bf16, void* t_bf16,
                 long long n_bf16, const void* segs, int nseg, long long n, const float* sumsq /*device, clip*/,
                 float max_norm, float lr, float last_layer_lr, float wd, float b1, float b2, float eps, int step,
                 float momentum, void* stream);
/* Stand-alone teacher EMA (train/ssl_meta_arch.py:644-660, the fn(ema_params, params, mom) returned by update_ema()):
 * teacher <- momentum*teacher + (1-momentum)*student over a flat fp32 shard; the leading n_bf16 elements (matrix
 * region) are re-cast into the teacher's bf16 compute copy.                                                        */
int d3_ema(float* teacher, const float* student, void* t_bf16, long long n_bf16, long long n, float momentum,
           void* stream);

/* ---- On-GPU DINO multi-crop augmentation (SURVEY §8f.3; replaces the per-sample torchvision host pipeline of
 * dinov3_jax/data/augmentations.py:23-230 for a batch of decoded uint8 images resident in HBM).  Random parameters are
 * drawn on the host and passed as one 64-byte record per output crop:
 *   struct { int img, x0, y0, w, h, flip; int order[4]; float fb, fc, fs, fh; int gray, solarize; }
 * (order[] = ColorJitter op order: 0 brightness 1 contrast 2 saturation 3 hue; order[0] = -1: jitter not applied).
 * Images are fp32 in [0,1] between the stages, like torchvision.transforms.v2.functional on float tensors.           */
int d3_aug_resized_crop(const void* src_u8 /*[n_img,H,W,3]*/, int n_img, int H, int W, const void* crops /*device*/,
                        int n_crops, float* out /*[n_crops,S,S,3]*/, int S, void* stream);   /* RandomResizedCrop(bicubic, antialias) + flip */
int d3_aug_color(float* x /*[n_crops,S,S,3] in place*/, const void* crops, int n_crops, int S,
                 float* gray_sum /*[n_crops] zeroed*/, void* stream);                      /* ColorJitter + RandomGrayscale */
int d3_aug_blur(const float* x, float* tmp, float* y, const void* blur /*device float sigma[n_crops], <= 0: none*/,
                int n_crops, int S, void* stream);                                          /* GaussianBlur(9, sigma) */
int d3_aug_finish(const float* x, void* out_bf16 /*[n_crops,S,S,3]*/, const void* crops, int n_crops, int S,
                  const float* mean3 /*host*/, const float* std3 /*host*/, void* stream);     /* Solarize(128) + Normalize + bf16 */

#ifdef __cplusplus
}
#endif
#endif
