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
long long d3_launch_count(void);        /* kernels launched by this library since the last reset (bench: gpu_launches) */
void d3_reset_launch_count(void);

/* ---- dense contraction (wgmma / TMA) -----------------------------------------------------------------------------
 * D[M,N] = epilogue( alpha * A[M,K] . B[K,N] ), bf16 operands, fp32 accumulation in registers.
 *   a_major = 0: A stored [M][K] (row stride lda)      a_major = 1: A stored [K][M]
 *   b_major = 0: B stored [N][K] (row stride ldb)      b_major = 1: B stored [K][N]   (reference kernel layout [in,out])
 * Replaces nn.Dense / nn.Conv(stride=kernel) at layers/attention.py:63-65,94,101, layers/ffn_layers.py:36-47,
 * layers/patch_embed.py:38-51, layers/dino_head.py:20-43,65-85, and their jax.grad transposes (train/train.py:504-513).
 * Epilogue order: +bias -> [store bf16 pre-activation] -> [tanh-GELU] -> [erf-GELU] -> [* GELU'(aux_in)] -> [* gamma]
 *                 -> [+ resid] -> [+= out] -> store (bf16 or fp32).   (layers/block.py:198-199, layers/layer_scale.py:17-21,
 *                 the ConvNeXt block's pwconv1 -> nn.GELU(), models/convnext.py:70-72)                               */
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
  D3_EP_GELU_ERF = 512, /* v = 0.5 v (1 + erf(v / sqrt 2))  exact GELU (torch nn.GELU()), forward only */
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
/* tile_n : 0 = auto (256 when both operands are MN-major, else 64 or 128); 64 / 128 / 256 = 128-row tiles of that
 *          width; 512 is taken as 256.
 * split_k: 0 = auto (used only for plain fp32 outputs with D3_EP_ACCUM, i.e. weight gradients: the slices' partial sums
 *          are added to `out`, which the caller zeroes or wants accumulated into, in slice order); >= 1 = forced.  */
int d3_gemm_bf16(const void* A, int lda, int a_major, const void* B, int ldb, int b_major, int M, int N, int K,
                 const d3_gemm_epilogue* ep, int tile_n, int split_k, void* stream);

/* ---- FP8 (e4m3) block linears: row-wise power-of-two scales -----------------------------------------------------
 * d3_quant_rows_e4m3: dst[r, c] = e4m3(src[r, c] / scale[r]) for a bf16 [R, C] view (row stride ld elements), with
 *   scale[r] = 2^e, e the smallest integer with max_c |src[r, c]| <= 448 * 2^e over the row's finite elements (1 for a
 *   row with none but zeros).  Round to nearest even; x / 2^e is exact and never exceeds 448.  A non-finite element
 *   becomes the e4m3 NaN.  The same bits on every run.
 * d3_quant_cols_e4m3_t: the same per column of a bf16 W [R = in, C = out], written transposed: dst [C, R] e4m3 (row
 *   stride ld_dst bytes), scale [C].
 * d3_gemm_e4m3: out = epilogue(alpha * sum_k A[m, k] B[n, k] * sa[m] * sb[n]) with A [M, K] and B [N, K] e4m3, both
 *   K-major (row strides lda / ldb bytes, multiples of 16, 16-byte aligned; K % 16 == 0), the tensor core's
 *   sum of every 64 k-elements added into the fp32 accumulator on its own.  Every epilogue flag but SCATTER and GELU_ERF; no split-K.  */
int d3_quant_rows_e4m3(const void* src_bf16, int ld, int R, int C, void* dst_u8, int ld_dst, float* scale,
                       void* stream);
int d3_quant_cols_e4m3_t(const void* src_bf16, int ld, int R, int C, void* dst_u8, int ld_dst, float* scale,
                         void* stream);
int d3_gemm_e4m3(const void* A_u8, int lda, const float* sa, const void* B_u8, int ldb, const float* sb, int M, int N,
                 int K, const d3_gemm_epilogue* ep, void* stream);

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

/* ---- LayerNorm (models/vision_transformer.py:40: eps 1e-6, biased variance E[x^2]-E[x]^2, fp32 statistics) -------
 * D % 4 == 0.  Alignment (else D3_ERR_ARG): d3_layernorm_fwd: x, scale, bias and an fp32 y 16 bytes, a bf16 y 8 bytes;
 * d3_layernorm_bwd_ls: every row operand and parameter vector (dy, x, scale, dx_add, dx, ls_gamma, ls_u, ls_du) 16 bytes. */
int d3_layernorm_fwd(const float* x /*[T,D]*/, const float* scale, const float* bias, void* y, int y_is_f32,
                     float* mean /*[T] or NULL*/, float* rstd, int T, int D, float eps, void* stream);
/* One block output -> the dense features of models/vision_transformer.py:280-313 (get_intermediate_layers), one launch:
 * X fp32 [n, N, D] with N = 1 + R + Hp*Wp (cls, R storage tokens, patches) -> cls [n, D], storage [n, R, D] (NULL when
 * R == 0) and patches, channels-last [n, Hp*Wp, D] (channels_first = 0) or channels-first [n, D, Hp, Wp] (reshape=True),
 * all three fp32 (out_f32 = 1) or bf16 (round to nearest even).  Each row is LayerNorm-ed with the statistics and
 * arithmetic of d3_layernorm_fwd (the same bits as d3_layernorm_fwd on that row): the 1 + R prefix rows with
 * (pre_scale, pre_bias), the patch rows with (scale, bias); pass the same pointers for tied norms and four NULLs for
 * norm=False (values only copied / converted).  Any D % 4 == 0; channels-first stores are 16 bytes wide where a channel
 * plane's byte stride and base allow it, narrower otherwise.  Alignment (else D3_ERR_ARG): X and the norm vectors 16
 * bytes; cls, storage and channels-last patches 16 (fp32) / 8 (bf16) bytes; channels-first patches one element.      */
int d3_layernorm_tokens_out(const float* X, const float* scale, const float* bias, const float* pre_scale,
                            const float* pre_bias, float eps, int n, int N, int R, int Hp, int Wp, int D, void* cls,
                            void* storage, void* patches, int out_f32, int channels_first, void* stream);
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

/* ---- attention (layers/attention.py:116 nn.dot_product_attention; head_dim D/H = 64 or 128, any N up to 32768) ---- */
/* N > 32768, n_crops * N >= 2^31 or another head_dim returns D3_ERR_ARG before any CUDA call.  Scale head_dim^-0.5.
 * head_dim 64: crops of up to 448 tokens (forward) / 256 tokens (backward) run on kernels that hold a whole crop in
 * shared memory, longer ones on streamed kernels.  head_dim 128 (vit_7b): streamed kernels at every N.             */
int d3_attn_fwd(const void* qkv_bf16 /*[n*N,3D] post-RoPE*/, void* o_bf16 /*[n*N,D]*/, float* lse /*[n,H,N] or NULL*/,
                int n_crops, int N, int D, int H, void* stream);
/* rope_sin / rope_cos ([P,head_dim] fp32, or NULL): when given, the inverse rotation (transpose of layers/attention.py:19-20)
 * is applied to dq / dk of tokens >= rope_prefix before they are stored, i.e. dqkv is the gradient w.r.t. the
 * pre-RoPE qkv projection output.                                                                                  */
int d3_attn_bwd(const void* qkv_bf16, const void* o_bf16, const void* do_bf16, const float* lse,
                float* delta_scratch /*[n,H,N]*/, void* dqkv_bf16 /*[n*N,3D]*/, int n_crops, int N, int D, int H,
                const float* rope_sin, const float* rope_cos, int rope_prefix, void* stream);

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
 * dgamma += colsum(dX*act(u)), dbias += colsum(bf16 du), the same arithmetic as the tail of d3_layernorm_bwd_ls;
 * D % 4 == 0, dX and gamma 16-byte, u and du 8-byte aligned.  d3_colsum_bf16: bias gradients, any N, ld and
 * alignment, the same sums whatever the layout.                                                                      */
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

/* ---- ConvNeXt backbone (models/convnext.py:45-335, upstream DINOv3's ConvNeXt; forward only) -----------------------
 * A block is d3_dwconv7_layernorm -> d3_gemm_bf16 (pwconv1, D3_EP_BIAS | D3_EP_GELU_ERF, bf16 out) -> d3_gemm_bf16
 * (pwconv2, D3_EP_BIAS | D3_EP_GAMMA | D3_EP_RESID | D3_EP_OUT_F32 into the residual stream).  The stem is d3_im2col
 * (p = 4) + d3_gemm_bf16 + d3_layernorm_fwd; a downsampling layer is d3_layernorm_patchify2 + d3_gemm_bf16 (K = 4C).
 * Every LayerNorm here has the statistics and arithmetic of d3_layernorm_fwd (the same bits on each pixel's row).
 * d3_dwconv7_layernorm: Y = LayerNorm(dwconv7x7(X) + wb) per pixel; X fp32 NHWC [n, H, W, C] (zero padding 3 at every
 * border, any H, W >= 1), w fp32 [49, C] tap-major (the HWIO kernel [7, 7, 1, C]), Y bf16 [n*H*W, C].  C % 8 == 0,
 * C <= 1536.  Alignment: X, Y, scale, bias 16 bytes.                                                                */
int d3_dwconv7_layernorm(const float* X, const float* w, const float* wb, const float* scale, const float* bias, float eps,
                         void* Y_bf16, int n, int H, int W, int C, void* stream);
/* Y bf16 [n * H/2 * W/2, 4C]: row (b, i, j), column (kh * 2 + kw) * C + c = LayerNorm(X[b, 2i + kh, 2j + kw])[c], the
 * operand of the 2x2 stride-2 conv GEMM (HWIO kernel viewed as [4C, C']).  Even H, W; C % 4 == 0; X, scale, bias
 * 16-byte, Y 8-byte aligned.                                                                                        */
int d3_layernorm_patchify2(const float* X, const float* scale, const float* bias, float eps, void* Y_bf16, int n, int H,
                           int W, int C, void* stream);
/* out fp32 [n, rows, C]: row 0 of image b = mean over the P rows of X[b] ([n, P, C] fp32), summed in a fixed order (the
 * same bits every run); copy_tokens (rows == 1 + P): rows 1..P = X[b].  Otherwise rows 1.. are left untouched (for
 * d3_resize_tokens_bilinear_aa).  The result is the X of d3_layernorm_tokens_out with R = 0.  C % 4 == 0, 16-byte
 * aligned.                                                                                                          */
int d3_pool_tokens(const float* X, float* out, int n, int P, int C, int rows, int copy_tokens, void* stream);
/* fp32 maps [n, Hs, Ws, C] -> rows prefix .. prefix + Hd*Wd - 1 of each image's [prefix + Hd*Wd, C] block of dst:
 * torch F.interpolate(mode="bilinear", antialias=True, align_corners=False) arithmetic (models/convnext.py:256-261).
 * Down-scaling factors up to 7; C % 4 == 0; 16-byte aligned.                                                        */
int d3_resize_tokens_bilinear_aa(const float* src, float* dst, int n, int Hs, int Ws, int Hd, int Wd, int C, int prefix,
                                 void* stream);

/* ---- KoLeo (loss/koleo_loss.py:16-35), forward + backward: metric += w_metric * loss; dx += w_grad * dloss/dx ------
 * Only the rows [row0, row0+nrows) contribute loss terms (mean over nrows); neighbours are searched over all B rows.
 * row0 = 0, nrows = B is KoLeoLoss.  A sub-range is KoLeoLossDistributed (loss/koleo_loss.py:39-70): x holds the
 * all-gathered rows of every rank, and dx gets the gradient for all B rows (the caller reduce-scatters the other ranks'
 * parts).                                                                                                          */
int d3_koleo_fwd_bwd_rows(const float* x /*[B,D]*/, float* xn_scratch /*[B,D]*/, float* nrm_scratch /*[B]*/,
                          int* nn_scratch /*[B]*/, float* coef_scratch /*[B]*/, float* metric, float* dx /*[B,D] +=*/,
                          int B, int D, int row0, int nrows, float eps, float w_metric, float w_grad, void* stream);
/* ---- Top-k KoLeo over gathered rows (dino.koleo_loss_distributed, loss/koleo_loss.py:39-70; parity unpinned) -------
 * x holds the rows of every rank in rank order.  The loss group is rows [g0, g0+gn); this rank's rows [row0, row0+B)
 * lie inside it.  Each row is normalised, xn = x/(||x||+eps); local row i takes the topk largest fp32 dots xn_i.xn_j
 * over the group's other rows (ties to the lower j), and
 *   metric += w_metric * L,  L = -1/(B topk) sum_{i,s} log(||xn_i - xn_nbr(i,s)|| + eps + eps)
 *   dx[j]  += w_grad * dL/dx_j for every row j of the group (this rank's contribution; rows outside it untouched).
 * 1 <= topk <= min(16, gn - 1); D % 4 == 0, D <= 6144; x, dx, scratch 16-byte aligned; scratch holds
 * N*D + N + 2*B*topk floats.  No atomics: the same bits on every run.                                              */
int d3_koleo_topk_rows(const float* x /*[N,D]*/, int N, int D, int g0, int gn, int row0, int B, int topk, float eps,
                       float w_metric, float w_grad, float* scratch, long long scratch_floats, float* metric,
                       float* dx /*[N,D] +=*/, void* stream);

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
/* The remaining DataAugmentationDINO options (augmentations.py:70-230):
 *  - share_color_jitter (:156-175): ColorJitter + RandomGrayscale of each whole [H, W] source image, one record per image
 *    (img = image index); x = the jittered fp32 copy, which d3_aug_resized_crop_f32 (clamp 1) then crops.
 *  - gram_teacher_crops_size (:70-113, :197-205): the global "base" crops are taken at max(global, gram) and resized to
 *    the global and gram sizes with d3_aug_resized_crop_f32 over the whole base (x0 = y0 = 0, w = h = base size).
 *    Before the distortions (gram_teacher_no_distortions) the Resize acts on a PIL image: clamp 1.  After them the
 *    reference resizes the normalised tensor: clamp 0, run after d3_aug_solarize and before d3_aug_finish (Resize
 *    commutes with Normalize, not with Solarize), and d3_aug_finish is given records with solarize = 0.
 *  - local_crops_subset_of_global_crops (:208-223): each local crop is the L x L window at (y0, x0) = (rx, ry) of its
 *    whole base crop (img = base index in [n_base, M, M, 3]) after the base's own jitter and 9-tap blur; y = the
 *    un-normalised window for d3_aug_finish.  Scratch: win [n_crops, L+8, L+8, 3], tmp [n_crops, L+8, L, 3].         */
int d3_aug_resized_crop_f32(const float* src /*[n_img,H,W,3] in [0,1]*/, int n_img, int H, int W, const void* crops,
                            int n_crops, float* out /*[n_crops,S,S,3]*/, int S, int clamp, void* stream);
int d3_aug_color_images(const void* src_u8 /*[n_img,H,W,3]*/, int n_img, int H, int W, const void* recs /*[n_img]*/,
                        float* x /*[n_img,H,W,3]*/, float* gray_sum /*[n_img] zeroed*/, void* stream);
int d3_aug_solarize(float* x /*[n_crops,S,S,3] in place*/, const void* crops, int n_crops, int S, void* stream);
int d3_aug_local_windows(const float* base /*[n_base,M,M,3]*/, int n_base, int M, const void* crops, const void* blur,
                         int n_crops, int L, float* win, float* tmp, float* y /*[n_crops,L,L,3]*/,
                         float* gray_sum /*[n_crops] zeroed*/, void* stream);
/* Ragged sources: B decoded images of their own sizes, their HWC pixels packed one after the other in one buffer,
 * with a device table of one 16-byte row per image,
 *   struct { long long off; int h, w; }   (off = the image's first pixel in the buffer, in pixels),
 * and crops drawn from each image's own size.  The crops are the same kernel as the dense entries above (a dense batch
 * is a ragged batch of equal sizes); everything after the first crop works on dense base crops.  `crops_host` /
 * `recs_host` are the host copies of the device records: a record whose img is outside the table is refused with
 * D3_ERR_ARG before any CUDA call, as are null pointers and n_img < 1.  That each box lies inside its own image is
 * the caller's to check (it drew the boxes from the sizes).
 *  - d3_aug_resized_crop_ragged / _f32: RandomResizedCrop of uint8, or of fp32 [0,1] (clamp as above), sources.
 *  - d3_aug_color_images_ragged: share_color_jitter on ragged sources; x is the fp32 copy of the n_pix packed pixels
 *    with the same offsets, and contrast blends with the mean gray of each image's own h * w pixels.               */
int d3_aug_resized_crop_ragged(const void* src_u8 /*packed HWC*/, const void* imgs /*device [n_img]*/, int n_img,
                               const void* crops /*device*/, const void* crops_host, int n_crops,
                               float* out /*[n_crops,S,S,3]*/, int S, void* stream);
int d3_aug_resized_crop_ragged_f32(const float* src /*packed HWC in [0,1]*/, const void* imgs, int n_img,
                                   const void* crops, const void* crops_host, int n_crops, float* out, int S, int clamp,
                                   void* stream);
int d3_aug_color_images_ragged(const void* src_u8 /*packed HWC*/, long long n_pix, const void* imgs, int n_img,
                               const void* recs /*device [n_img]*/, const void* recs_host, float* x /*packed HWC*/,
                               float* gray_sum /*[n_img] zeroed*/, void* stream);

/* ---- k-NN evaluation (the DINO / DINOv2 / DINOv3 k-NN protocol on the teacher's normalised class token) ---------
 * The similarities of a query tile with a bank chunk are d3_gemm_bf16 (fp32 out) of L2-normalised bf16 rows; these
 * entry points are the rest of the search and the vote.  Every one is deterministic (the same bits on every run).
 * d3_eval_resize_crop: n uint8 HWC images of any sizes packed in one buffer, desc[3i .. 3i+2] = (byte offset, H, W)
 *   (device, int64).  torchvision Resize(resize, BICUBIC, antialias=True) on the short side (long side
 *   int(resize * long / short)) with torch's uint8 arithmetic, then CenterCrop(crop); only the crop is computed.  out:
 *   bf16 NHWC [n, crop, crop, 3] = (u8 / 255 - mean) / std, or (out_u8) the uint8 crop.  max_taps >= 2 ceil(2 max(s, 1))
 *   + 1 over both axes of every image, s = input / resized length (the filter taps of the widest window).
 * d3_knn_normalize: y = x / max(||x||, 1e-12) per row (F.normalize), into y_f32 and / or y_bf16 (both NULL: error).
 * d3_topk_merge: per query row q, the running top-k (top_sim fp32 / top_idx int32 [Q, ldk], sorted by similarity desc,
 *   index asc; fresh = 1: start from an empty list) merged with sims[q, 0:valid] (bank indices offset + column) into
 *   the new sorted top-k.  1 <= k <= 1024; chunks must come in increasing offset; empty slots are (-inf, -1).
 * d3_knn_vote: per query and per k in nb_knn (host, <= 16 entries, each <= ldk): weights softmax(sims[:k] / T) (fp32,
 *   max subtracted), class scores (labels[top_idx]) summed in neighbour order, the 5 best classes (score desc, class
 *   asc) into preds int32 [Q, n_k, 5].  num_classes <= 32768.                                                        */
int d3_eval_resize_crop(const void* src_u8, const long long* desc, int n, int resize, int crop, int max_taps,
                        const float* mean3 /*host*/, const float* std3 /*host*/, void* out, int out_u8, void* stream);
int d3_knn_normalize(const float* x, int ldx, int R, int D, float* y_f32, void* y_bf16, int ldy, void* stream);
int d3_topk_merge(const float* sims, long long lds, int Q, int valid, int offset, float* top_sim, int* top_idx, int ldk,
                  int k, int fresh, void* stream);
int d3_knn_vote(const float* top_sim, const int* top_idx, int ldk, int Q, const int* bank_labels, int n_bank,
                const int* nb_knn /*host*/, int n_k, float temperature, int num_classes, int* preds, void* stream);

/* ---- linear-probe evaluation (the DINOv2 / DINOv3 linear protocol: many linear classifiers on frozen features) ------
 * Every entry point is deterministic.  The logits are d3_gemm_bf16 (fp32 out, bias epilogue) of one column window of
 * the input rows per classifier group, the weight gradients d3_gemm_bf16 of dZ^T and the same window, the bias
 * gradients d3_colsum_bf16 of dZ.
 * d3_train_resized_crop: torchvision RandomResizedCrop's resized_crop + RandomHorizontalFlip of n packed uint8 images
 *   (desc as d3_eval_resize_crop): boxes int32 [n, 5] (device) = (top, left, height, width, flip); the box is resized
 *   to crop x crop with torch's uint8 bicubic antialias arithmetic (the int16 weights of d3_eval_resize_crop), then
 *   mirrored when flip != 0.  out: bf16 NHWC (u8 / 255 - mean) / std, or (out_u8) uint8.  max_taps >= 2 ceil(2
 *   max(box / crop, 1)) + 1 over both axes of every box.
 * d3_linear_inputs: out[b, s * D + c] = bf16(srcs[s][b * D + c]) for the n_src fp32 [B, D] sources (host array of
 *   device pointers, 16-byte aligned, n_src <= 32): [cls of the last n blocks | patch mean] in one row of stride ld_out.
 * d3_linear_xent_fwd_bwd: logits fp32 [B, ld >= G * Cp], classifier g in columns [g * Cp, g * Cp + C) (the padding
 *   columns are not read); labels int32 [B] in [0, C).  loss fp32 [G] = batch-mean cross-entropy per classifier (rows
 *   summed in order); dz bf16 [B, ld_dz] = (softmax - onehot) / B, 0 in the padding columns.  2 <= C <= 32768,
 *   Cp % 8 == 0.
 * d3_sgd_momentum: torch SGD(momentum, dampening 0, weight_decay 0) on fp32 p / g / m [rows, cols]: m = first ? g :
 *   momentum * m + g; p -= lr[(row) / Cp] * lr_scale * m (lr device fp32, one per classifier of Cp rows); p_bf16
 *   (optional) receives the bf16 copy of p.  rows * cols % 4 == 0.                                                    */
int d3_train_resized_crop(const void* src_u8, const long long* desc, const int* boxes, int n, int crop, int max_taps,
                          const float* mean3 /*host*/, const float* std3 /*host*/, void* out, int out_u8, void* stream);
int d3_linear_inputs(const float* const* srcs /*host*/, int n_src, int B, int D, void* out_bf16, int ld_out,
                     void* stream);
int d3_linear_xent_fwd_bwd(const float* logits, int ld, const int* labels, int B, int G, int C, int Cp, float* loss,
                           void* dz_bf16, int ld_dz, void* stream);
int d3_sgd_momentum(float* p, const float* g, float* m, void* p_bf16, long long rows, int cols, const float* lr, int Cp,
                    float lr_scale, float momentum, int first, void* stream);

/* ---- linear segmentation probe (BatchNorm without affine + a 1x1 convolution on frozen patch features) ---------------
 * Every entry point is deterministic (integer atomics only).  The head's logits are d3_gemm_bf16 (fp32 out, bias
 * epilogue), its weight gradient d3_gemm_bf16 of dZ^T and the normalised rows, its bias gradient d3_colsum_bf16 of dZ,
 * its update d3_adamw_ema.  Upsampling is torch's bilinear F.interpolate(align_corners=False) at any ratio.
 * d3_seg_crop: n packed uint8 images (desc as d3_eval_resize_crop) with uint8 label maps of the same sizes (packed at
 *   desc offset / 3 of labels_u8); boxes int32 [n, 6] (device) = (rh, rw, top, left, flip, unused): the image is resized
 *   to rh x rw with d3_eval_resize_crop's arithmetic, and the out_h x out_w window at (top, left) is written (mirrored
 *   within the part inside the resized image when flip != 0; outside it: 0 in the normalised image, 255 in the labels,
 *   at the bottom / right).  out: bf16 NHWC (u8 / 255 - mean) / std, or (out_u8) uint8; label_out (optional) uint8
 *   [n, out_h, out_w], torch 'nearest' from the label map.  max_taps as d3_eval_resize_crop for in / out = H / rh, W / rw.
 * d3_seg_bn_stats: per column of bf16 x [M, N] (row stride ld): mean and biased var (fp32 [N]), as torch's BatchNorm in
 *   training mode; run_mean / run_var (both or neither) <- (1 - momentum) run + momentum (mean, unbiased var).
 * d3_seg_bn_apply: out[r, c] = bf16((x[r, c] - mean[c]) * rsqrt(var[c] + eps)).  N, ld, ld_out even.
 * d3_seg_xent_fwd_bwd: logits fp32 [B * h * w, ld] (patch cells row-major, C <= ld classes), labels uint8 [B, Hl, Wl]
 *   (>= C: ignored; 255 is the ignore label).  loss fp32 [1] = mean over the valid pixels of the cross-entropy of the
 *   upsampled logits (0 when none is valid); count int32 [1] = the valid pixels; dz (fp32 and / or bf16 [B * h * w,
 *   ld_dz], optional) = d loss / d logits in columns [0, C), 0 in [C, Cp).  2 <= C <= 256.  No full-resolution buffer.
 * d3_seg_predict_confusion: conf int64 [C, C] += the (label, argmax of the upsampled logits) counts over the pixels with
 *   label < C (argmax ties to the lower class).                                                                       */
int d3_seg_crop(const void* src_u8, const long long* desc, const void* labels_u8, const int* boxes, int n, int out_h,
                int out_w, int max_taps, const float* mean3 /*host*/, const float* std3 /*host*/, void* out, int out_u8,
                void* label_out, void* stream);
int d3_seg_bn_stats(const void* x_bf16, int ld, int M, int N, float* mean, float* var, float* run_mean, float* run_var,
                    float momentum, void* stream);
int d3_seg_bn_apply(const void* x_bf16, int ld, long long M, int N, const float* mean, const float* var, float eps,
                    void* out_bf16, int ld_out, void* stream);
int d3_seg_xent_fwd_bwd(const float* logits, int ld, const void* labels_u8, int B, int h, int w, int Hl, int Wl, int C,
                        int Cp, float* loss, int* count, float* dz_f32, void* dz_bf16, int ld_dz, void* stream);
int d3_seg_predict_confusion(const float* logits, int ld, const void* labels_u8, int B, int h, int w, int Hl, int Wl,
                             int C, long long* conf, void* stream);

/* ---- linear depth probe (the segmentation probe's BatchNorm and 1x1 convolution to n_bins "linear" depth bins) -------
 * Deterministic (no atomics).  Bin centres c_k = linspace(min_depth, max_depth, n_bins); per cell q_k = relu(z_k) + 0.1
 * and depth d = sum_k q_k c_k / sum_k q_k; d is upsampled as d3_seg_xent_fwd_bwd's logits.  A ground-truth pixel is
 * valid when min_depth < gt <= max_depth.
 * d3_depth_crop: d3_seg_crop's image (the same bits) and, when depth_out != NULL, the fp32 depth planes of the same
 *   sizes (packed at desc offset / 3 floats of depth_src) cropped from the same boxes by torch 'nearest' into
 *   depth_out [n, out_h, out_w], 0 outside the resized image.
 * d3_depth_head_fwd_bwd: logits fp32 [B * h * w, ld] (n_bins <= ld), gt fp32 [B, Hl, Wl].  loss fp32 [1] = the
 *   scale-invariant log loss sqrt(var(g) + 0.15 mean(g)^2), g = log(d_hat + 1e-3) - log(gt + 1e-3) over the valid
 *   pixels (unbiased var; 0 with fewer than 2); count int32 [1] = the valid pixels; dz (fp32 and / or bf16
 *   [B * h * w, ld_dz], optional) = d loss / d logits in columns [0, n_bins), 0 in [n_bins, Cp).  No full-resolution
 *   buffer.
 * d3_depth_predict_metrics: sums fp64 [B, 9] = per image, over the valid pixels in rows [crop_top, crop_bottom) and
 *   columns [crop_left, crop_right), with p = d_hat clamped to [min_depth, max_depth] and t = gt: the count, and the
 *   sums of |p - t| / t, (p - t)^2 / t, (p - t)^2, (ln p - ln t)^2, |log10 p - log10 t|, and 1[max(p/t, t/p) < 1.25^k]
 *   for k = 1, 2, 3 (fp32 within a tile, fp64 across tiles).                                                        */
int d3_depth_crop(const void* src_u8, const long long* desc, const float* depth_src, const int* boxes, int n, int out_h,
                  int out_w, int max_taps, const float* mean3 /*host*/, const float* std3 /*host*/, void* out,
                  int out_u8, float* depth_out, void* stream);
int d3_depth_head_fwd_bwd(const float* logits, int ld, const float* gt, int B, int h, int w, int Hl, int Wl,
                          int n_bins, int Cp, float min_depth, float max_depth, float* loss, int* count, float* dz_f32,
                          void* dz_bf16, int ld_dz, void* stream);
int d3_depth_predict_metrics(const float* logits, int ld, const float* gt, int B, int h, int w, int Hl, int Wl,
                             int n_bins, float min_depth, float max_depth, int crop_top, int crop_bottom,
                             int crop_left, int crop_right, double* sums, void* stream);

/* ---- video object segmentation by label propagation (DINO's eval_video_segmentation.py; see csrc/video.cu) -------
 * d3_video_resize: n packed uint8 HWC frames (desc int64 [n, 3] = (byte offset, H, W)) -> bf16 NHWC [n, out_h, out_w, 3]:
 *   torch bilinear (align_corners = False, antialias = False) of frame / 255 in fp32, then (v - mean) / std.
 * d3_video_propagate: the soft labels out fp32 [h w, C] of one target frame.  sim0 fp32 [h w, ld0] = the target rows'
 *   similarities to frame 0's rows; simr fp32 [h w, ldr] = those to the n_recent recent frames, frame c at columns
 *   [c h w, (c + 1) h w); lab0 fp32 [h w, C] and labr fp32 [n_recent h w, C] their label rows.  Per target patch: the
 *   candidates within radius rows and columns in every context frame (frame 0 first, then row, then column), the k-th
 *   largest similarity as threshold (ties kept), weights exp((x - x_max) / temperature) normalised to sum 1, the
 *   weighted sum of the kept label rows.  C <= 32, topk <= 32.  Deterministic (no atomics).
 * d3_video_label_map: labels uint8 [out_h, out_w] = argmax over channels (lowest index on ties) of the soft map
 *   fp32 [h, w, C] upsampled bilinearly by patch (align_corners = False), each channel with maximum > 0 min-max
 *   normalised over the upsampled frame, sampled by torch nearest-exact at out_h x out_w.  No full-resolution buffer.
 * d3_video_jf_counts: pred, gt uint8 [F, H, W] (gt 255 = void); counts int64 [F, K, 6] (zeroed here) per frame and
 *   object k = 1..K: intersection and union outside void, the boundary pixels of pred and of gt (void cleared first),
 *   and the boundary pixels of each with a boundary pixel of the other within the disk of radius `radius`.        */
int d3_video_resize(const void* src_u8, const long long* desc, int n, int out_h, int out_w, const float* mean3 /*host*/,
                    const float* std3 /*host*/, void* out, void* stream);
int d3_video_propagate(const float* sim0, int ld0, const float* simr, int ldr, const float* lab0, const float* labr,
                       int n_recent, int h, int w, int C, int radius, int topk, float temperature, float* out,
                       void* stream);
int d3_video_label_map(const float* soft, int h, int w, int C, int patch, int out_h, int out_w, void* labels_u8,
                       void* stream);
int d3_video_jf_counts(const void* pred_u8, const void* gt_u8, int F, int H, int W, int K, int radius,
                       long long* counts, void* stream);

/* ---- keypoint correspondence over bilinearly upsampled patch features (see csrc/correspondence.cu) ---------------
 * U(y, x) is torch's bilinear F.interpolate (align_corners = False) of an [h, w, D] bf16 patch map (rows of ld
 * elements, map m at rows [m h w, (m + 1) h w)) to out_h x out_w.
 * d3_corr_descriptors: out bf16 [K, ldo] row k = U_{map_k}(y_k, x_k) L2-normalised in fp32, rounded to bf16; qnorm
 *   fp32 [K] the norm of each rounded row.  kp (host) int [K, 3] = (map, x, y), each checked against n_maps and
 *   [0, out_w) x [0, out_h) before anything is launched.
 * d3_corr_gram: gram fp32 [n_maps h w, 5] per patch (i, j): <f_ij, f_ij> and its dot products with the right, lower,
 *   lower-right and lower-left neighbours (0 where the neighbour does not exist), fp32 in a fixed order.
 * d3_corr_argmax: for each keypoint k, the pixel (x, y) of the target map that maximises the cosine of q_k with U(y, x),
 *   from sim fp32 [K, lds] (row k = <q_k, f_p> over the target's h w patches, from d3_gemm_bf16), the target's gram
 *   and qnorm; ties go to the lowest y out_w + x.  xy int [K, 2], cosine fp32 [K] the cosine there.  Nothing of
 *   full resolution is written; deterministic (no atomics).                                                        */
int d3_corr_descriptors(const void* feats, int ld, int n_maps, int h, int w, int D, int out_h, int out_w,
                        const int* kp /*host*/, int K, void* out, int ldo, float* qnorm, void* stream);
int d3_corr_gram(const void* feats, int ld, int n_maps, int h, int w, int D, float* gram, void* stream);
int d3_corr_argmax(const float* sim, int lds, const float* gram, const float* qnorm, int K, int h, int w, int out_h,
                   int out_w, int* xy, float* cosine, void* stream);

/* ---- unsupervised object discovery: TokenCut's normalized cut (see csrc/discovery.cu) -----------------------------
 * A launch covers n images with one grid of N = h w patches (2 <= N <= 4096); sim fp32 [n, N, lds] holds each image's
 * patch similarities (d3_gemm_bf16).  Deterministic (no atomics).
 * d3_od_graph: bits uint32 [n, N, ceil(N / 32)] with bit j % 32 of word j / 32 of row i set when sim_ij > tau; degree
 *   fp32 [n, N] = c_i + (N - c_i) eps from the count c_i of set bits (A_ij = 1 above tau, else eps).
 * d3_od_fiedler: per image the eigenvector x [n, N] of (D - A) x = lambda D x at the second-smallest lambda (lambda2
 *   [n]), by deflated Lanczos on D^-1/2 A D^-1/2 with full reorthogonalisation, one CTA per image; x^T D x = 1.  It
 *   stops when the residual bound falls to 1e-6 or after k_max <= 256 steps: iters [n] the steps taken, converged [n]
 *   0 when k_max was reached first.
 * d3_od_box: per image the bipartition fg_u8 [n, N] (x_i > mean(x), complemented when the seed argmax |x_i| is not in
 *   it), the pixel box [n, 4] = (x0, y0, x1, y1) of the seed's 4-connected component clipped to the image, its best IoU
 *   [n] with the image's ground-truth boxes gt fp32 [n, b_max, 4] (x1 y1 x2 y2) and hit [n] = best IoU >= 0.5.  sizes
 *   (host) int [n, 2] = (H, W) must give the grid (ceil(H / patch) = h, ceil(W / patch) = w); n_gt (host) int [n] in
 *   [0, b_max]; both checked before anything is launched.                                                        */
int d3_od_graph(const float* sim, int lds, int n, int N, float tau, float eps, void* bits, float* degree, void* stream);
int d3_od_fiedler(const void* bits, const float* degree, int n, int N, float eps, int k_max, float* x, float* lambda2,
                  int* iters, int* converged, void* stream);
int d3_od_box(const float* x, int n, int h, int w, int patch, const int* sizes /*host*/, const int* n_gt /*host*/,
              const float* gt, int b_max, void* fg_u8, int* box, float* best_iou, int* hit, void* stream);

/* ---- instance retrieval: revisited Oxford / Paris (see csrc/retrieval.cu) --------------------------------------------
 * Deterministic (no float atomics).
 * d3_ret_resize: n packed uint8 HWC images, desc (host) int64 [n, 7] = (byte offset, H, W, x0, y0, x1, y1) inside a
 *   source buffer of src_bytes bytes; the crop box [x0, x1) x [y0, y1) of each image is resized to out_h x out_w with
 *   torch's antialiased bicubic (align_corners = False) on float values and normalised, (v / 255 - mean) / std, into
 *   bf16 NHWC [n, out_h, out_w, 3].  desc is checked before anything is launched.
 * d3_ret_scale_sum: out[i] = x[i] + x[stride + i] + ... + x[(S - 1) stride + i] (scale order) for i < count, fp32.
 * d3_ret_rank_ap: per query q of the fp32 similarities sim [Q, lds] (N columns), the exact 0-based rank of every
 *   listed image j, #{i : s_qi > s_qj or (s_qi == s_qj and i < j)}, into ranks (device int [n_easy + n_hard +
 *   n_junk], the easy entries, then the hard, then the junk, as in the index arrays), and for the Easy, Medium and
 *   Hard protocols of the revisited benchmark ap [Q, 3] and pk [Q, 3, 3] (P@1, P@5, P@10) in fp64, n_ok [Q, 3] the ok
 *   images (AP and P@k are NaN where it is 0).  The lists are host CSR pairs (ptr [Q + 1] from 0, idx in [0, N)),
 *   at most 8192 entries per query over the three lists; all are checked before anything is launched.           */
int d3_ret_resize(const void* src_u8, long long src_bytes, const long long* desc /*host*/, int n, int out_h, int out_w,
                  const float* mean3 /*host*/, const float* std3 /*host*/, void* out, void* stream);
int d3_ret_scale_sum(const float* x, int S, long long stride, long long count, float* out, void* stream);
int d3_ret_rank_ap(const float* sim, long long lds, int Q, int N, const int* easy_ptr /*host*/,
                   const int* easy_idx /*host*/, const int* hard_ptr /*host*/, const int* hard_idx /*host*/,
                   const int* junk_ptr /*host*/, const int* junk_idx /*host*/, int* ranks, double* ap, double* pk,
                   int* n_ok, void* stream);

/* ---- logistic-regression evaluation: L-BFGS over a grid of regularisation strengths (see csrc/logreg.cu) ---------
 * Problem g's parameters are theta[g] = [W (Cp x K, row-major) | b (Cp)], P = Cp K + Cp floats, in [G, P] buffers
 * indexed by slot; act (device int [Ga]) lists the slots a launch covers.  Deterministic (no float atomics).
 * d3_logreg_split_x: x fp32 [n, ldx] -> xa bf16 [rows, 3K] = [Xh | Xh | Xl] and (when xg is given) xg bf16 [3 rows, K],
 *   chunk c holding [Xh; Xl; Xh] of its rows; rows = n rounded up to whole chunks, padding rows zero.
 * d3_logreg_weights: wcat bf16 [Ga Cp, 3K] = [Wh | Wl | Wh] per class row, bias fp32 [Ga Cp] (the logits GEMM operand).
 * d3_logreg_xent: per (row, problem) of a chunk of `rows` rows (the first n real), z = logits + bias: loss[a] (double,
 *   +=) gets sum_i (lse - z_y) inv_n; r bf16 [3 rows, ld_r] gets the residual (softmax - onehot) inv_n as hi, hi, lo.
 * d3_logreg_finish: grad[g] = [gw_a + W icn_g | gb_a] (gw fp32 [Ga Cp, K], gb fp32 [Ga Cp]); out double [Ga, 4] = (loss
 *   + icn ||W||^2 / 2, grad . d (0 without d), max |grad|, ||grad||^2).
 * d3_logreg_trial: theta_t[g] = theta[g] + alpha[g] d[g] (alpha device fp32 [G]).
 * d3_logreg_direction: d[g] = -H_g grad[g] by the L-BFGS two-loop recursion over count[g] pairs of S, Y [G, m, P]
 *   (newest in slot newest[g]), rho [G, m] = 1 / s.y, gamma [G] = s.y / y.y of the newest pair; gd double [Ga] = grad.d.
 * d3_logreg_accept: S, Y [g, slot[g]] = theta_t - theta, grad_t - grad; theta = theta_t, grad = grad_t; out double
 *   [Ga, 3] = (s.y, y.y, s.s).  1 <= m <= 64.                                                                       */
int d3_logreg_split_x(const float* x, int ldx, int n, int K, int chunk, void* xa, void* xg, void* stream);
int d3_logreg_weights(const float* theta, long long P, const int* act, int Ga, int Cp, int K, void* wcat, float* bias,
                      void* stream);
int d3_logreg_xent(const float* logits, int ld, const float* bias, const int* labels, int n, int rows, int Ga, int C,
                   int Cp, float inv_n, double* loss, void* r, int ld_r, void* stream);
int d3_logreg_finish(const float* theta, const float* gw, const float* gb, const double* loss, const float* icn,
                     const float* d, const int* act, int Ga, int Cp, int K, float* grad, double* out, void* stream);
int d3_logreg_trial(const float* theta, const float* d, const float* alpha, const int* act, int Ga, long long P,
                    float* theta_t, void* stream);
int d3_logreg_direction(const float* grad, const float* S, const float* Y, const float* rho, const float* gamma,
                        const int* count, const int* newest, const int* act, int Ga, long long P, int m, float* d,
                        double* gd, void* stream);
int d3_logreg_accept(float* theta, float* grad, const float* theta_t, const float* grad_t, float* S, float* Y,
                     const int* slot, const int* act, int Ga, long long P, int m, double* out, void* stream);

/* ---- attentive-probe video classification: the probe's single-query pooling folded over the tokens (csrc/attentive.cu)
 * One learnable query q0 [D] and H heads (dh = D / H): q = Wq q0 + bq, kt [H, D] = Wk_h^T q_h / sqrt(dh) per head (the
 * keys folded into the query).  Clip tokens x bf16 [B, T * P, D] (T frames of P tokens, frame-major), temporal
 * embedding e fp32 [T, D], LN1 scale g1 / bias b1 fp32 [D] (eps 1e-6).  Deterministic (no float atomics).
 * d3_atp_query_fwd: q fp32 [D], kt fp32 [H, D] from fp32 q0, Wq [D, D], bq [D], Wk [D, D] (rows are outputs).
 * d3_atp_query_bwd: from dkt [H, D]: dWk, dWq [D, D] and dbq [D] written; dq0 [D] += Wq^T dq.
 * d3_atp_pool_fwd: ybar fp32 [B, H, D] = sum_n p_{n,h} LN1(x_n + e_t(n)), p = softmax_n((LN1(u_n) - b1) . kt_h);
 *   lse fp32 [B, H] the softmax's log-sum-exp.  8 <= D <= 1536, D % 8 == 0, H | D, x 16-byte aligned.
 * d3_atp_pool_bwd: from dybar fp32 [B, H, D] (and the forward's ybar, lse): dkt [H, D], dg1, db1 [D] and de [T, D]
 *   written (summed over the clips).
 * d3_atp_gelu_erf_bwd: out bf16 [rows, ld_out] = dh fp32 * GELU_erf'(pre bf16).                                     */
int d3_atp_query_fwd(const float* q0, const float* Wq, const float* bq, const float* Wk, int D, int H, float* q,
                     float* kt, void* stream);
int d3_atp_query_bwd(const float* q0, const float* Wq, const float* Wk, const float* q, const float* dkt, int D, int H,
                     float* dWq, float* dbq, float* dWk, float* dq0, void* stream);
int d3_atp_pool_fwd(const void* x, const float* e, const float* g1, const float* b1, const float* kt, int B, int T,
                    int P, int D, int H, float* ybar, float* lse, void* stream);
int d3_atp_pool_bwd(const void* x, const float* e, const float* g1, const float* b1, const float* kt, const float* lse,
                    const float* ybar, const float* dybar, int B, int T, int P, int D, int H, float* dkt, float* dg1,
                    float* db1, float* de, void* stream);
int d3_atp_gelu_erf_bwd(const float* dh, int ld_dh, const void* pre, int ld_pre, int rows, int cols, void* out,
                        int ld_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif
