/* libeat_b200 -- C ABI of the H100-native EfficientAT hot path (mel front end + MobileNetV3 /
 * DyMN forward & backward).  sm_90a only; no CPU fallback.
 *
 * The reference (fschmid56/EfficientAT) has no FFI: its hot path is Python nn.Modules calling
 * cuFFT / cuDNN / cuBLAS through PyTorch.  Each entry point below therefore cites the reference
 * *module code* (file:line under the reference tree) whose library calls it replaces.  The host
 * side (efficientat_b200/models/...) mirrors the reference's nn.Module surface and reaches these
 * functions through ctypes with raw device pointers + the current CUDA stream.
 *
 * Conventions
 *   - every function returns 0 (EAT_OK) or an EAT_ERR_* code; eat_last_error() has the text.
 *   - all pointers are DEVICE pointers unless stated; the caller owns all memory.
 *   - work is enqueued on `stream` and is asynchronous; no function synchronises or allocates.
 *   - activations are NHWC: [B, F, T, C] with C innermost, dtype EAT_F32 or EAT_BF16;
 *     parameters, BatchNorm vectors, statistics and gates are always fp32 (statistics: fp64).
 *   - "in_scale/in_shift/in_act": optional per-channel affine + activation applied to the input
 *     operand as it is loaded (the BatchNorm+activation of the producing layer);  NULL = none.
 *   - "scale/shift/act": optional per-channel affine + activation applied to the result.
 *   - "stat_sum/stat_sq": optional fp64 per-channel sum / sum of squares of the RAW result
 *     (BatchNorm batch statistics), accumulated with atomics; caller zeroes them.
 */
#ifndef EAT_B200_H
#define EAT_B200_H

#ifndef __CUDA_RUNTIME_H__
typedef struct CUstream_st* cudaStream_t;
#endif

#ifdef __cplusplus
extern "C" {
#endif

#define EAT_OK 0
#define EAT_ERR_ARG 1
#define EAT_ERR_CUDA 2
#define EAT_ERR_UNSUPPORTED 3

#define EAT_ACT_NONE 0
#define EAT_ACT_RELU 1
#define EAT_ACT_HSWISH 2
#define EAT_ACT_SIGMOID 3   /* forward-only (DyMN coordinate attention / DyReLU coefficient nets) */

#define EAT_F32 0
#define EAT_BF16 1

const char* eat_last_error(void);
int eat_abi_version(void);

/* Host-only (no GPU work): the launch plan of the sliding-window depthwise kernels (csrc/dw_slide.cu) for a layer.
 * kind: 0 forward, 1 weight gradient, 2 stride-2 data gradient, 3 fused backward (eat_dw_conv_bwd_fused, fp32; its
 * channel vectors are 4 channels for 3x3 and 2 for 5x5).  per_sample != 0: blockIdx.y must be the sample
 * (squeeze-excitation pooling, DynamicConv per-sample weights; ignored by kind 3).  plan[6] = {channel chunks, channel
 * vectors per chunk, output rows (row pairs for kind 2; din rows, or row pairs for stride 2, for kind 3) per segment,
 * CTA groups per chunk, gridDim.y, strip width}.
 * kind 4: the shared-memory tile kernel (csrc/conv_kernels.cu: the 5x5 eval forward and the 5x5 stride-1 data gradient
 * above 256 channels; k must be 5, per_sample is ignored since blockIdx.y is always the sample).  plan[6] = {channel
 * chunks, 32 channels per chunk, output tiles of FR x (32 / stride) pixels per chunk and sample, CTA groups per chunk
 * (each CTA strides over tiles / groups of them), gridDim.y = B, FR}.  Exposed so the
 * host logic is testable without a device (tests/test_cabi.py). */
int eat_dw_plan(int kind, int dtype, int B, int F, int T, int C, int k, int stride, int per_sample, int* plan);
/* Host-only: the cp.async prefetch-ring depth in input rows (0: ring off) that the sliding-window kernel of
 * eat_dw_conv_fwd / the stride-1 eat_dw_conv_dgrad takes for C channels, k x k, stride; EAT_DW_RING overrides it. */
int eat_dw_ring_depth(int dtype, int C, int k, int stride, int* depth);
int eat_device_check(int device);

/* Fused log-mel front end.  Replaces AugmentMelSTFT.forward, models/preprocess.py:40-67
 * (conv1d pre-emphasis :41, torch.stft :42-43, power :44, mel matmul :56-57, log :59, affine :65).
 * wave [B,N] fp32 -> out [B, n_mels, 1+(N-1)/hop] fp32.  n_fft in {256, 512, 1024, 2048, 4096}, anything
 * else returns EAT_ERR_UNSUPPORTED; win_length <= n_fft, n_mels <= 512, N - 1 > n_fft/2, else EAT_ERR_ARG; a hop
 * whose signal slice does not fit in shared memory returns EAT_ERR_UNSUPPORTED.  All checks precede any device call.
 * twiddle: n_fft float2 (exp(-2 pi i m/M), m<M, then exp(-2 pi i k/n_fft), k<M, with M = n_fft/2).
 * Filterbank as bands: fb_start/fb_len [n_mels], fb_w [max_len][n_mels] (tap-major). */
int eat_mel_fwd(const float* wave, int B, int N, const float* window, int win_length, int hop, int n_fft,
                const float* twiddle, const int* fb_start, const int* fb_len, const float* fb_w, int max_len,
                int n_mels, float preemph, float* out, cudaStream_t stream);

/* eat_mel_fwd on clips of different lengths in one batch: clip b is wave[b, :n_valid[b]] (n_valid: B int32 on the
 * device).  Its frames t < 1 + (n_valid[b] - 1) / hop equal eat_mel_fwd on that clip alone (pre-emphasis and reflect
 * padding end at its own last sample; the same per-frame arithmetic); frames up to T = 1 + (N - 1) / hop are 0.
 * Samples at or past n_valid[b] are never read.  The caller guarantees n_fft / 2 + 2 <= n_valid[b] <= N.  Checks as
 * eat_mel_fwd, and n_valid is required when B > 0. */
int eat_mel_fwd_len(const float* wave, int B, int N, const float* window, int win_length, int hop, int n_fft,
                    const float* twiddle, const int* fb_start, const int* fb_len, const float* fb_w, int max_len,
                    int n_mels, float preemph, float* out, const int* n_valid, cudaStream_t stream);

/* Adjoint of eat_mel_fwd (with eat_mel_mask's bands): dspec [B, n_mels, T] fp32 -> dwave [B, N] fp32 (overwritten), the
 * gradient through the affine, the masks (zero where the forward masked), log(mel + 1e-5), the banded filterbank, the
 * power spectrum, the real FFT, the window, the overlap-add of the frames, the reflect padding and the pre-emphasis.
 * wave, window, twiddle and the filterbank are the forward call's; the frame spectra are recomputed.  f_start, f_end,
 * t_start, t_end [B] int32: the forward's SpecAugment bands, all four or none.  work: eat_mel_bwd_workspace floats of
 * scratch.  Bitwise repeatable (no floating-point atomics).  Geometry checks as eat_mel_fwd; a hop whose slice does not
 * fit in shared memory -> EAT_ERR_UNSUPPORTED, a short work -> EAT_ERR_ARG.  All checks precede any launch; B = 0 is a
 * no-op. */
int eat_mel_bwd(const float* dspec, const float* wave, int B, int N, const float* window, int win_length, int hop,
                int n_fft, const float* twiddle, const int* fb_start, const int* fb_len, const float* fb_w, int max_len,
                int n_mels, float preemph, const int* f_start, const int* f_end, const int* t_start, const int* t_end,
                float* work, long long work_floats, float* dwave, cudaStream_t stream);
/* Host-only: the floats of scratch eat_mel_bwd needs for B clips of N samples. */
int eat_mel_bwd_workspace(int B, int N, int hop, int n_fft, long long* floats);

/* Kaldi mel filterbank in banded form, built on the device (training-mode fmin/fmax jitter,
 * models/preprocess.py:45-55 + torchaudio.compliance.kaldi.get_mel_banks).  fb_w holds cap x n_mels floats. */
int eat_mel_filterbank(int n_mels, int n_fft, float sample_rate, double fmin, double fmax, int* fb_start,
                       int* fb_len, float* fb_w, int cap, cudaStream_t stream);

/* SpecAugment masking of the log-mel (training only): torchaudio Frequency/TimeMasking with
 * iid_masks=True, models/preprocess.py:31-38,61-63.  spec [B,F,T]; band [start,end) per example. */
int eat_mel_mask(float* spec, int B, int F, int T, const int* f_start, const int* f_end, const int* t_start,
                 const int* t_end, float fill, cudaStream_t stream);

/* Stem 3x3 conv on the 1-channel spectrogram.  Replaces ConvNormActivation(1, C, k=3, s=2) at
 * models/mn/model.py:125-133 (dymn/model.py:80-87).  x [B,F,T] fp32 -> out [B,Fo,To,C]. */
int eat_stem_fwd(const float* x, const float* w, void* out, int out_dtype, int B, int F, int T, int C, int stride,
                 const float* scale, const float* shift, int act, double* stat_sum, double* stat_sq,
                 cudaStream_t stream);

/* Depthwise weights [C,1,k,k] -> tap-major [k*k][C]. */
int eat_dw_repack(const float* w, float* wt, int C, int k, cudaStream_t stream);

/* Depthwise k x k conv (k in {3,5}, stride in {1,2}, pad (k-1)/2) + BN/act (+ SE squeeze sums).
 * Replaces the depthwise ConvNormActivation at models/mn/block_types.py:150-162 and the mean of
 * SqueezeExcitation._scale :73 (pool [B,C] += per-sample channel sums of the result). */
int eat_dw_conv_fwd(const void* in, const float* wt, void* out, int dtype, int B, int F, int T, int C, int k,
                    int stride, const float* in_scale, const float* in_shift, int in_act, const float* scale,
                    const float* shift, int act, float* pool, double* stat_sum, double* stat_sq,
                    cudaStream_t stream);

/* Eval-mode BatchNorm folding: scale = gamma / sqrt(rvar + eps), shift = beta - rmean * scale. */
int eat_bn_fold(const float* gamma, const float* beta, const float* rmean, const float* rvar, float eps,
                float* scale, float* shift, int C, cudaStream_t stream);

/* Training-mode BatchNorm: batch statistics -> scale/shift, saved mean/invstd, running-stat update
 * (nn.BatchNorm2d(eps=1e-3, momentum=0.01), models/mn/model.py:114-115). rmean/rvar/nbt may be NULL. */
int eat_bn_finalize(const double* sum, const double* sq, double count, const float* gamma, const float* beta,
                    float eps, float momentum, float* rmean, float* rvar, long long* nbt, float* scale,
                    float* shift, float* save_mean, float* save_invstd, int C, cudaStream_t stream);

/* y = act(z * scale + shift) (+ res), elementwise on [rows, C]  (BN apply + residual,
 * models/mn/block_types.py:177-181). */
int eat_bn_apply(const void* z, const float* scale, const float* shift, int act, const void* res, void* y,
                 int dtype, long long rows, int C, cudaStream_t stream);

/* pool[b,c] += mul * sum_p act(z[b,p,c] * scale[c] + shift[c])   (SE squeeze / global average pool,
 * models/mn/block_types.py:73, models/mn/model.py:220). */
int eat_bn_act_pool(const void* z, const float* scale, const float* shift, int act, float* pool, float mul,
                    int dtype, int B, int P, int C, cudaStream_t stream);

/* Squeeze-excitation MLP: gate = sigmoid(W2 relu(W1 (pool*inv_count) + b1) + b2)
 * (models/mn/block_types.py:72-83).  hidden_out [B,S] optional (saved for backward). */
int eat_se_fc_fwd(const float* pool, float inv_count, const float* w1, const float* b1, const float* w2,
                  const float* b2, float* gate, float* hidden_out, int B, int C, int S, cudaStream_t stream);

/* Exact-fp32 CUDA-core GEMM: C[M,N] = epi(xf(A)[M,K] . W[N,K]^T).  1x1 convs on NHWC rows
 * (models/mn/block_types.py:140-147,167-171) and the classifier Linear layers
 * (models/mn/model.py:187-194).  gate [B,K]: SE gate of sample row/rows_per_sample.
 * w_trans = 1 reads W as [K,N] (data gradient: dA[M,Cin] = G[M,Cout] . W[Cout,Cin]). */
int eat_gemm_simt_fwd(const void* A, int a_dtype, const float* W, int w_trans, void* C, int c_dtype, long long M,
                      int N, int K, const float* in_scale, const float* in_shift, int in_act, const float* gate,
                      int rows_per_sample, const float* scale, const float* shift, int act, const void* residual,
                      double* stat_sum, double* stat_sq, cudaStream_t stream);

/* wgmma tensor-core version of the same GEMM contract (w_trans must be 0; A and C share the dtype;
 * K, N multiples of 8).  bf16 storage: one bf16 MMA per product; fp32 storage: hi/lo split, three MMAs
 * (fp32-grade products, ~2^-16 relative).  Same reference call sites as eat_gemm_simt_fwd. */
int eat_pw_tc_fwd(const void* A, int a_dtype, const float* W, int w_trans, void* C, int c_dtype, long long M, int N,
                  int K, const float* in_scale, const float* in_shift, int in_act, const float* gate,
                  int rows_per_sample, const float* scale, const float* shift, int act, const void* residual,
                  double* stat_sum, double* stat_sq, cudaStream_t stream);
/* fp32-storage version of the same contract, fed by TMA (cp.async.bulk.tensor tiles of A, W and the residual) with
 * bf16x3 wgmma products (hi/lo split on chip, ~2^-16 relative) and TMA stores; w_trans = 0, K and N multiples of 4.
 * The residual is accumulated before shift/activation, so residual != NULL requires act == EAT_ACT_NONE (the only
 * combination the reference has: block_types.py:167-171,179-180).  w_ws (optional, 128-byte aligned, at least
 * N * ceil(K/32) * 128 bytes): scratch into which the weights are pre-split once per launch (bf16 hi|lo rows, epilogue
 * scale folded, transposed when w_trans = 1, i.e. W given as [K, N]) so that no CTA repeats that work per tile; without
 * it the split happens on chip per tile and w_trans must be 0.  eat_pw_tc_fwd forwards fp32 launches here (without
 * workspace) unless the environment says EAT_PW_IMPL=tc. */
int eat_pw_tma_fwd(const float* A, const float* W, int w_trans, float* C, long long M, int N, int K,
                   const float* in_scale, const float* in_shift, int in_act, const float* gate, int rows_per_sample,
                   const float* scale, const float* shift, int act, const float* residual, double* stat_sum,
                   double* stat_sq, void* w_ws, long long w_ws_bytes, cudaStream_t stream);
/* DynamicConv 1x1 (models/dymn/dy_block.py:103-131) on the same TMA kernel: W = dyn_k kernels [dyn_k][N][K] ([dyn_k][K][N]
 * with w_trans = 1), sample b uses sum_j att[b, j] * W[j]; the per-sample kernels are mixed + pre-split once per launch
 * into w_ws (>= B * N * ceil(K/32) * 128 bytes, 128-byte aligned).  M = B * rows_per_sample. */
int eat_pw_tma_dyn_fwd(const float* A, const float* W, const float* att, int dyn_k, int w_trans, float* C, long long M,
                       int N, int K, int rows_per_sample, const float* scale, const float* shift, int act,
                       const float* residual, double* stat_sum, double* stat_sq, void* w_ws, long long w_ws_bytes,
                       cudaStream_t stream);
/* Host-only (no GPU work): the tile walk eat_pw_tma_fwd (rows_per_sample = 0) / eat_pw_tma_dyn_fwd (rows_per_sample > 0:
 * M tiles never straddle samples) launch on a GPU of sms SMs; raw != 0: the raw-output variant (training forward with
 * batch statistics, data gradients), else an epilogue variant.  plan[5] = {N tile width, N tiles, M tiles, CTAs, M tiles
 * of the CTA that takes the most}. */
int eat_pw_tma_plan(long long M, int N, int K, int rows_per_sample, int raw, int sms, int* plan);
/* out[cols, rows] = in[rows, cols]^T (fp32); used to feed W^T to the data-gradient GEMM. */
int eat_transpose_f32(const float* in, float* out, int rows, int cols, cudaStream_t stream);

/* ---- DyMN (reference models/dymn/dy_block.py) ---- */

/* DynamicConv 1x1 on tensor cores (dy_block.py:103-131): W = dyn_k kernels [dyn_k][N][K]; sample b uses
 * sum_k att[b,k]*W[k], mixed while the weight tile is staged (never materialised).  M = B*rows_per_sample. */
int eat_pw_tc_dyn_fwd(const void* A, int dtype, const float* W, const float* att, int dyn_k, void* C, long long M,
                      int N, int K, int rows_per_sample, const float* in_scale, const float* in_shift, int in_act,
                      const float* scale, const float* shift, int act, const void* residual, double* stat_sum,
                      double* stat_sq, cudaStream_t stream);
/* DynamicConv depthwise + BN affine + DyReLU-B (dy_block.py:172-188) + CoordAtt (:195-201) in one kernel.
 * wt: per-sample tap-major weight tables (stride wt_bstride floats); theta [B,C,4] = sigmoid(coef_net(h_c));
 * lam/init: DyReLU buffers; ca_f [B,Fo,C], ca_t [B,To,C] = sigmoid(g_cf), sigmoid(g_ct). */
int eat_dw_conv_fwd_dy(const void* in, const float* wt, long long wt_bstride, void* out, int dtype, int B, int F, int T,
                       int C, int k, int stride, const float* in_scale, const float* in_shift, int in_act,
                       const float* scale, const float* shift, const float* theta, const float* lam,
                       const float* init, const float* ca_f, const float* ca_t, double* stat_sum, double* stat_sq,
                       cudaStream_t stream);
/* eat_dw_conv_fwd_dy with M = `pieces` DyReLU-B linear pieces, 1..4 (dy_block.py:142-188, dyrelu_k):
 * theta [B, C, 2M] channel-major, lam / init [2M]; out = max_m (a_m u + b_m) * ca_f * ca_t with
 * a_m = (2 theta[m] - 1) lam[m] + init[m], b_m = (2 theta[M+m] - 1) lam[M+m] + init[M+m], u = BN(conv).  The training
 * form (in_scale/in_shift, stat_sum/stat_sq, no theta) does not depend on M.  Before any launch: pieces outside 1..4,
 * k outside {3,5}, stride outside {1,2} -> EAT_ERR_UNSUPPORTED; bad dtype or sizes, C not a multiple of the vector
 * width (4 fp32, 8 bf16), pointers that come in sets given partly, the training transform or statistics together with
 * the eval epilogue -> EAT_ERR_ARG.  B = 0 is a no-op. */
int eat_dw_conv_fwd_dy_m(const void* in, const float* wt, long long wt_bstride, void* out, int dtype, int B, int F, int T,
                         int C, int k, int stride, const float* in_scale, const float* in_shift, int in_act,
                         const float* scale, const float* shift, const float* theta, const float* lam,
                         const float* init, const float* ca_f, const float* ca_t, int pieces, double* stat_sum,
                         double* stat_sq, cudaStream_t stream);
/* ContextGen pooling (dy_block.py:236-240): out [B, F+T, C] fp32 = [mean over T | mean over F]. */
int eat_ctx_pool(const void* x, int dtype, float* out, int B, int F, int T, int C, cudaStream_t stream);
/* Sequence pooling of ContextGen (dy_block.py:227-233,249): AvgPool(3, stride, pad 1) or copy (stride 1) of rows
 * [row0, row0+L) of each sample of in [B, Ltot, H] -> out [B, Lo, H].  stride >= 1 and row0 + L <= Ltot, else EAT_ERR_ARG
 * (also for eat_seq_pool_bwd). */
int eat_seq_pool(const float* in, float* out, int B, int Ltot, int row0, int L, int H, int stride, const float* scale,
                 const float* shift, int act, cudaStream_t stream);   /* optional affine+act applied to `in` on load */
/* att [B,k] = softmax((Wr h_c + br)/temperature)  (dy_block.py:104-107). */
int eat_dyconv_att(const float* hc, const float* wr, const float* br, float temperature, float* att, int B, int H, int k,
                   cudaStream_t stream);
/* per-sample depthwise weight tables wt [B][ksize^2][C] = sum_j att[b,j] * W[j] (dy_block.py:111-117). */
int eat_dyconv_mix_dw(const float* w, const float* att, float* wt, int B, int C, int ksize, int k, cudaStream_t stream);

/* DyMN training path.  p = DyReLU-B(BN(z)) * ca_f * ca_t materialised for the projection conv, and its backward:
 * du = d/d(BN output), dcaf [B,Fo,C] / dcoef [B,C,4] accumulated (caller zeroes), dcat [B,To,C] overwritten. */
int eat_dy_act_fwd(const void* z, void* out, int dtype, const float* scale, const float* shift, const float* theta,
                   const float* lam, const float* init, const float* ca_f, const float* ca_t, int B, int Fo, int To,
                   int C, cudaStream_t stream);
int eat_dy_act_bwd(const void* dp, const void* z, void* du, int dtype, const float* scale, const float* shift,
                   const float* theta, const float* lam, const float* init, const float* ca_f, const float* ca_t,
                   float* dcaf, float* dcat, float* dcoef, int B, int Fo, int To, int C, cudaStream_t stream);
/* dpre = dcoef * lam * 2 s (1-s) with s = theta (DyReLU coefficient net); out = g * s * (1-s) (sigmoid backward). */
int eat_dyrelu_coef_bwd(const float* dcoef, const float* theta, const float* lam, float* dpre, long long n,
                        cudaStream_t stream);
/* The three above with M = `pieces` DyReLU-B linear pieces, 1..4: theta [B, C, 2M], lam / init [2M], dcoef [B, C, 2M]
 * (accumulated; da_m = sum du x [m = argmax], db_m = sum du [m = argmax]).  The pixel's gradient goes to the one piece
 * that attains the max; on a tie, to the lowest piece index (M = 2 included).  n = B * C * 2M.  Before any launch: pieces
 * outside 1..4 -> EAT_ERR_UNSUPPORTED; bad dtype or sizes, C not a multiple of 4, n not a multiple of 2M, a null
 * pointer -> EAT_ERR_ARG.  B = 0 (n = 0) is a no-op. */
int eat_dy_act_fwd_m(const void* z, void* out, int dtype, const float* scale, const float* shift, const float* theta,
                     const float* lam, const float* init, const float* ca_f, const float* ca_t, int pieces, int B, int Fo,
                     int To, int C, cudaStream_t stream);
int eat_dy_act_bwd_m(const void* dp, const void* z, void* du, int dtype, const float* scale, const float* shift,
                     const float* theta, const float* lam, const float* init, const float* ca_f, const float* ca_t,
                     float* dcaf, float* dcat, float* dcoef, int pieces, int B, int Fo, int To, int C, cudaStream_t stream);
int eat_dyrelu_coef_bwd_m(const float* dcoef, const float* theta, const float* lam, float* dpre, long long n, int pieces,
                          cudaStream_t stream);
int eat_sigmoid_bwd(const float* g, const float* s, float* out, long long n, cudaStream_t stream);
/* softmax(Linear(h_c)/T) backward: dWr/dbr accumulated, dh_c[b,:] += dlogit . Wr.  k in 1..4, as eat_dyconv_att. */
int eat_dyconv_att_bwd(const float* datt, const float* att, float temperature, const float* hc, const float* wr,
                       float* dwr, float* dbr, float* dhc, int B, int H, int k, cudaStream_t stream);
int eat_seq_pool_bwd(const float* dout, float* dsrc, int B, int Ltot, int row0, int L, int H, int stride,
                     cudaStream_t stream);
int eat_ctx_pool_bwd(const float* dg, void* dx, int dtype, int B, int F, int T, int C, cudaStream_t stream);
/* Per-sample weight gradients S [B,N,K] of a 1x1 conv on tensor cores, and the DynamicConv bank / attention
 * gradients derived from per-sample gradients S [B,n]: dW[k] += sum_b att[b,k] S[b]; datt[b,k] = <S[b], W[k]>. */
int eat_pw_tc_wgrad_persample(const void* G, const void* A, int dtype, float* S, long long M, int N, int K,
                              int rows_per_sample, cudaStream_t stream);
int eat_dyn_wgrad_mix(const float* S, const float* att, const float* W, float* dW, float* datt, int B, long long n, int k,
                      cudaStream_t stream);

/* ---- backward (training step: ex_audioset.py:197 loss.backward() over the modules above) ---- */

/* Weight gradient of a 1x1 conv / Linear: dW[N,K] += G[M,N]^T . xf(A)[M,K]; db[N] += colsum(G) (db may be
 * NULL).  dW/db are fp32 and must be zeroed by the caller once per step (atomically accumulated). */
int eat_gemm_simt_wgrad(const void* G, int g_dtype, const void* A, int a_dtype, float* dW, float* db, long long M,
                        int N, int K, const float* in_scale, const float* in_shift, int in_act, const float* gate,
                        int rows_per_sample, cudaStream_t stream);

/* wgmma version of the weight gradient (db must be NULL; G and A share the dtype; K, N multiples of 8):
 * MN-major wgmma operands, reduction over pixels split across CTAs, vector atomics into dW. */
int eat_pw_tc_wgrad(const void* G, int g_dtype, const void* A, int a_dtype, float* dW, float* db, long long M, int N,
                    int K, const float* in_scale, const float* in_shift, int in_act, const float* gate,
                    int rows_per_sample, cudaStream_t stream);

/* fp32-storage successor of eat_pw_tc_wgrad, fed by TMA (cp.async.bulk.tensor boxes of G and X, bf16 hi/lo split in
 * place on chip, MN-major wgmma, one CTA per SM).  per_sample != 0: S[b] = G_b^T . X_b for DynamicConv (M = B *
 * rows_per_sample, dW = S [B, N, K]).  eat_pw_tc_wgrad / eat_pw_tc_wgrad_persample forward fp32 launches here unless the
 * environment says EAT_WG_IMPL=tc. */
int eat_pw_tma_wgrad(const float* G, const float* X, float* dW, long long M, int N, int K, const float* in_scale,
                     const float* in_shift, int in_act, const float* gate, int rows_per_sample, int per_sample,
                     cudaStream_t stream);
/* Host-only: the launch plan of eat_pw_tma_wgrad for the same M, N, K, rows_per_sample, per_sample on a GPU of sms SMs.
 * plan[6] = {reduction rows per pipeline stage (64 or 128), (64 x 64) dW tiles, reduction splits (CTAs per dW tile),
 * rows per split, splits per sample (per-sample mode; 0 otherwise), pipeline stages}. */
int eat_pw_wgrad_plan(long long M, int N, int K, int rows_per_sample, int per_sample, int sms, int* plan);

/* BatchNorm backward, pass 1: s1[c] += sum dy, s2[c] += sum dy*xhat with dy = g * act'(z*scale+shift),
 * g = gA * gate[b,c] + dpool[b,c] (gA / gate / dpool each optional).  z, gA: [B, P, C]. */
int eat_bn_bwd_reduce(const void* gA, const float* gate, const float* dpool, const void* z, const float* scale,
                      const float* shift, const float* mean, const float* invstd, int act, int dtype, int B, int P,
                      int C, double* s1, double* s2, cudaStream_t stream);
/* dgamma += s2, dbeta += s1 (either may be NULL), c1 = s1/count, c2 = s2/count. */
int eat_bn_bwd_finalize(const double* s1, const double* s2, double count, float* dgamma, float* dbeta, float* c1,
                        float* c2, int C, cudaStream_t stream);
/* pass 2: dz = scale * (dy - c1 - xhat * c2). */
int eat_bn_bwd_apply(const void* gA, const float* gate, const float* dpool, const void* z, const float* scale,
                     const float* shift, const float* mean, const float* invstd, int act, const float* c1,
                     const float* c2, void* dz, int dtype, int B, int P, int C, cudaStream_t stream);

/* SE backward: dgate[b,c] += sum_p dp[b,p,c] * act(z[b,p,c]*scale[c]+shift[c]). */
int eat_se_bwd_reduce(const void* dp, const void* z, const float* scale, const float* shift, int act, float* dgate,
                      int dtype, int B, int P, int C, cudaStream_t stream);
/* SE block (block_types.py:72-83,177-181; autograd of `scale * input` and of the BatchNorm in front of it): the
 * squeeze-excitation reduce and the BatchNorm-backward reduce of the depthwise output in ONE pass over (dp, z).
 * dgate as eat_se_bwd_reduce; part [parts][4][B][C] fp32 (no zero fill needed) receives, per slice of the pixels,
 * sum dp*act'(v), sum dp*act'(v)*(z-mean), sum act'(v), sum act'(v)*(z-mean) with v = z*scale+shift.  Grid = parts x B. */
int eat_se_bn_bwd_reduce(const void* dp, const void* z, const float* scale, const float* shift, const float* mean, int act,
                         float* dgate, float* part, int parts, int dtype, int B, int P, int C, cudaStream_t stream);
/* ... and, once the SE MLP backward has produced dpool: s1[c] += sum_b gate*part0 + dpool*part2,
 * s2[c] += invstd[c] * sum_b gate*part1 + dpool*part3 -- the sums eat_bn_bwd_reduce(gA = dp, gate, dpool) yields. */
int eat_se_bn_bwd_combine(const float* part, int parts, const float* gate, const float* dpool, const float* invstd, int B,
                          int C, double* s1, double* s2, cudaStream_t stream);
/* SE MLP backward (per sample): du2 = dgate*gate*(1-gate), du1 = (W2^T du2)*(hidden>0),
 * dpool = (W1^T du1) * inv_count.  Weight gradients follow from du2/du1 via eat_gemm_simt_wgrad. */
int eat_se_fc_bwd(const float* dgate, const float* gate, const float* hidden, const float* w1, const float* w2,
                  float inv_count, float* du2, float* du1, float* dpool, int B, int C, int S, cudaStream_t stream);

/* Depthwise conv backward: data gradient (+ optional residual add into din) and weight gradient
 * (dw [C,1,k,k] fp32, atomically accumulated; in may carry the producing layer's BN+act as in_*). */
int eat_dw_conv_dgrad(const void* dz, const float* wt, long long wt_bstride, const void* res, void* din, int dtype, int B,
                      int F, int T, int C, int k, int stride, cudaStream_t stream);
int eat_dw_conv_dgrad_s1(const void* dz, const float* wt, long long wt_bstride, const void* res, void* din, int dtype,
                         int B, int F, int T, int C, int k, cudaStream_t stream);   /* stride-1 fast path */
/* Stride-2 data gradient whose output din [B,F,T,C] is the upstream gradient of a BatchNorm + activation with raw input
 * z [B,F,T,C] (the expand stage of an InvertedResidual, block_types.py:140-147): the BatchNorm-backward reduce
 * (s1[c] += sum g, s2[c] += invstd[c] * sum g*(z-mean[c]), g = din * act'(z*scale+shift) -- what eat_bn_bwd_reduce(gA = din)
 * yields) is taken in the epilogue while din is still in registers.  fp32 storage, k in {3,5}; anything else returns
 * EAT_ERR_UNSUPPORTED and the caller runs eat_dw_conv_dgrad + eat_bn_bwd_reduce. */
int eat_dw_conv_dgrad_bnred(const void* dz, const float* wt, const void* res, void* din, const void* z, const float* zscale,
                            const float* zshift, const float* zmean, const float* zinvstd, int zact, double* s1, double* s2,
                            int dtype, int B, int F, int T, int C, int k, int stride, cudaStream_t stream);
int eat_dw_conv_wgrad(const void* dz, const void* in, const float* in_scale, const float* in_shift, int in_act,
                      float* dw, long long dw_bstride, int dtype, int B, int F, int T, int C, int k, int stride,
                      cudaStream_t stream);   /* wt_bstride / dw_bstride: floats between per-sample tables (0: shared) */
/* Dilated depthwise k x k conv, the tail of get_model(dilated=True) (models/mn/block_types.py:150-162 with
 * cnf.dilation = 2): dilation 2, stride 1, padding (k-1)/2 * 2, so the output has the input's size [B,F,T,C].  The three
 * entry points mirror eat_dw_conv_fwd (training forward with in_* applied on load and fp64 batch statistics, or the eval
 * epilogue with folded BatchNorm + act and the SE squeeze sums into pool), the stride-1 data gradient of eat_dw_conv_dgrad
 * (mirrored taps, din = data gradient of dz (+ res)) and eat_dw_conv_wgrad (dw [C,1,k,k] += weight gradient of dz against
 * xf(in)).  wt is the tap-major table of eat_dw_repack.  dilation must be 2, stride 1, k 3 or 5, dtype fp32 or bf16, and
 * C a multiple of 4 (fp32) or 8 (bf16); anything else returns EAT_ERR_ARG or EAT_ERR_UNSUPPORTED before any launch.
 * B = 0 is a no-op. */
int eat_dw_conv_fwd_dil(const void* in, const float* wt, void* out, int dtype, int B, int F, int T, int C, int k, int stride,
                        int dilation, const float* in_scale, const float* in_shift, int in_act, const float* scale,
                        const float* shift, int act, float* pool, double* stat_sum, double* stat_sq, cudaStream_t stream);
int eat_dw_conv_dgrad_dil(const void* dz, const float* wt, const void* res, void* din, int dtype, int B, int F, int T,
                          int C, int k, int stride, int dilation, cudaStream_t stream);
int eat_dw_conv_wgrad_dil(const void* dz, const void* in, const float* in_scale, const float* in_shift, int in_act,
                          float* dw, int dtype, int B, int F, int T, int C, int k, int stride, int dilation,
                          cudaStream_t stream);
/* The depthwise stage's backward in one pass, from the upstream gradient dp [B,Fo,To,C] of its BatchNorm + activation
 * (BN2, raw output z2 [B,Fo,To,C]) down to the input: dz = eat_bn_bwd_apply(dp, gate, dpool, z2, scale ... c2) is
 * computed on load and never stored; din [B,F,T,C] = data gradient of dz (+ res); dw [C,1,k,k] += weight gradient of
 * dz against xf(in) = act(in*in_scale+in_shift) (identity when in_scale is NULL; in_act must equal act); and, unless s1 is
 * NULL, the BatchNorm-backward reduce of the expand stage behind din (s1[c] += sum g, s2[c] += zinvstd[c] *
 * sum g*(in-zmean[c]), g = din * act'(in*in_scale+in_shift)), as eat_dw_conv_dgrad_bnred.  c1/c2 come from
 * eat_bn_bwd_finalize of BN2's sums.  fp32 storage, k in {3,5}, stride in {1,2}, act relu or hardswish, C a multiple of
 * 4 (3x3) or 2 (5x5); anything else returns EAT_ERR_UNSUPPORTED before any launch. */
int eat_dw_conv_bwd_fused(const float* dp, const float* gate, const float* dpool, const float* z2, const float* scale,
                          const float* shift, const float* mean, const float* invstd, int act, const float* c1,
                          const float* c2, const float* wt, const float* in, const float* in_scale, const float* in_shift,
                          int in_act, const float* res, float* din, float* dw, const float* zmean, const float* zinvstd,
                          double* s1, double* s2, int dtype, int B, int F, int T, int C, int k, int stride,
                          cudaStream_t stream);
/* The expand stage's backward (1x1 conv + BatchNorm + activation, models/mn/block_types.py:140-147) in one pass, from
 * the gradient da [M, cexp] at its output and its raw output z [M, cexp]: dz = eat_bn_bwd_apply(da, NULL, NULL, z, scale
 * ... c2) is computed on load and never stored; dX [M, cin] = dz . W (+ res [M, cin]) with W the expand weight
 * [cexp, cin]; dW [cexp, cin] += dz^T . X (zeroed by the caller, atomically accumulated).  c1/c2 come from
 * eat_bn_bwd_finalize of the BatchNorm's backward sums.  bf16x3 tensor-core products (~2^-16 relative, as eat_pw_tma_fwd
 * and eat_pw_tma_wgrad).  fp32 storage, act relu or hardswish, cin <= 32 and cexp <= 128, both multiples of 4;
 * anything else returns EAT_ERR_UNSUPPORTED / EAT_ERR_ARG before any launch.  M == 0 is a no-op. */
int eat_pw_conv_bwd_fused(const float* da, const float* z, const float* scale, const float* shift, const float* mean,
                          const float* invstd, int act, const float* c1, const float* c2, const float* X, const float* W,
                          const float* res, float* dX, float* dW, int dtype, long long M, int cexp, int cin,
                          cudaStream_t stream);
/* Host-only (no GPU work): whether eat_pw_conv_bwd_fused takes a shape (EAT_OK) or not (EAT_ERR_UNSUPPORTED /
 * EAT_ERR_ARG), and its launch on a 132-SM H100: plan[4] = {CTAs (one per SM at most, each a contiguous range of
 * 128-row tiles), rows per CTA at most, pipeline stages, dynamic shared-memory bytes}. */
int eat_pw_bwd_plan(long long M, int cexp, int cin, int* plan);
/* Backward of an InvertedResidual's project stage (1x1 conv + BatchNorm, no activation) for a block without
 * squeeze-excitation, in one pass over its tensors: from the gradient dy [M, cout] at the BatchNorm's output, its raw
 * output z3 [M, cout] and the depthwise stage's raw output z2 [M, cexp]: dz3 = eat_bn_bwd_apply(dy, NULL, NULL, z3,
 * scale3 ... c2, act none) is computed on load and never stored; dp [M, cexp] = dz3 . W with W the project weight
 * [cout, cexp]; dW [cout, cexp] += dz3^T . act(z2 * scale2 + shift2) (zeroed by the caller, atomically accumulated);
 * and the depthwise BatchNorm's backward sums s1[c] += sum g, s2[c] += invstd2[c] * sum g * (z2 - mean2[c]) with
 * g = dp * act'(z2 * scale2 + shift2) -- what eat_bn_bwd_reduce(dp, NULL, NULL, z2, ...) adds.  c1/c2 come from
 * eat_bn_bwd_finalize of BN3's sums.  bf16x3 tensor-core products as eat_pw_conv_bwd_fused.  fp32 storage, act relu or
 * hardswish, cout <= 32 and cexp <= 128, both multiples of 4; anything else returns EAT_ERR_UNSUPPORTED / EAT_ERR_ARG
 * before any launch.  M == 0 is a no-op. */
int eat_pw_proj_bwd_fused(const float* dy, const float* z3, const float* scale3, const float* shift3, const float* mean3,
                          const float* invstd3, const float* c1, const float* c2, const float* z2, const float* scale2,
                          const float* shift2, const float* mean2, const float* invstd2, int act, const float* W, float* dp,
                          float* dW, double* s1, double* s2, int dtype, long long M, int cexp, int cout,
                          cudaStream_t stream);
/* Host-only: whether eat_pw_proj_bwd_fused takes a shape, and its launch plan, as eat_pw_bwd_plan. */
int eat_pw_proj_bwd_plan(long long M, int cexp, int cout, int* plan);
/* Stem weight gradient (the spectrogram itself needs no gradient).  z == NULL: dz is the gradient at the conv output.
 * z != NULL: dz is the gradient dy at the stem BatchNorm + activation's output and z the raw conv output, and the conv
 * output's gradient eat_bn_bwd_apply(dy, NULL, NULL, z, scale, shift, mean, invstd, act, c1, c2) is computed on load and
 * never stored (fp32 storage, C <= 64, stride 1 or 2; otherwise EAT_ERR_UNSUPPORTED before any launch). */
int eat_stem_wgrad(const void* dz, int dtype, const float* x, float* dw, int B, int F, int T, int C, int stride,
                   const float* z, const float* scale, const float* shift, const float* mean, const float* invstd, int act,
                   const float* c1, const float* c2, cudaStream_t stream);
/* Stem data gradient, the adjoint of eat_stem_fwd's 3x3 conv: dy [B,Fo,To,C] (dtype) is the gradient at the stem
 * BatchNorm + activation's output and z [B,Fo,To,C] (dtype) the raw conv output; the conv output's gradient
 * eat_bn_bwd_apply(dy, NULL, NULL, z, scale, shift, mean, invstd, act, c1, c2) is computed on load and never stored.
 * c1 = c2 = 0 with the running statistics' scale, shift, mean and invstd is the backward of a BatchNorm in eval mode.
 * w [C,1,3,3] fp32 -> dx [B,F,T] fp32 (overwritten).  Bitwise repeatable (no atomics).  C as eat_stem_fwd (a multiple
 * of 4 (fp32) or 8 (bf16), at most 256 vectors), F, T >= 1, act none/relu/hardswish and every pointer given, else
 * EAT_ERR_ARG; stride other than 1 or 2 -> EAT_ERR_UNSUPPORTED.  All checks precede any launch; B = 0 is a no-op. */
int eat_stem_dgrad(const void* dy, int dtype, const void* z, const float* scale, const float* shift, const float* mean,
                   const float* invstd, int act, const float* c1, const float* c2, const float* w, float* dx, int B, int F,
                   int T, int C, int stride, cudaStream_t stream);
/* The gradient of a returned feature map into NHWC storage (the reference's return_fmaps maps, models/mn/model.py:212-230,
 * models/dymn/model.py:157-200, in training): dst[b,f,t,c] (+)= src[b,c,f,t] in fp32 arithmetic, one rounding to
 * dst_dtype.  src is a [B, C, F, T] tensor with element strides sB, sC, sF, sT (any of them 0: an expanded broadcast);
 * dst is contiguous [B, F, T, C].  accumulate != 0 adds to dst, else overwrites it.  src_dtype and dst_dtype are EAT_F32
 * or EAT_BF16 each.  A source fastest along T or F goes through a shared-memory tiled transpose, one fastest along C
 * through a vectorised direct pass.  A bad dtype, negative sizes or strides, or a null pointer -> EAT_ERR_ARG; all checks
 * precede any launch; B = 0 (any size 0) is a no-op. */
int eat_fmap_grad_nhwc(const void* src, int src_dtype, long long sB, long long sC, long long sF, long long sT, void* dst,
                       int dst_dtype, int B, int C, int F, int T, int accumulate, cudaStream_t stream);
/* dpre = dh * mask * act'(pre), fp32 vectors (classifier Hardswish + Dropout backward). */
int eat_act_bwd(const float* dh, const float* pre, const float* mask, int act, float* dpre, long long n,
                cudaStream_t stream);

/* ---- multi-head attention pooling classifier head (reference models/mn/attention_pooling.py:9-56, MN with
 * head_type='multihead_attention_pooling', mn/model.py:170-172).  The projection P = m . W^T + b [B*T, 2*H*K] between
 * the two halves below runs on the 1x1-conv GEMMs; column j of P is s*H*K + h*K + k (s = 0 attention, 1 value).
 * Every check precedes any device call; B == 0 is a no-op. ---- */

/* Frequency mean, collapse_dim(x, dim=2) at attention_pooling.py:43 (mn/utils.py:29-41): x [B,F,T,C] (dtype) ->
 * m [B,T,C] fp32 = mean over f of xf(x); feat [B,C] fp32 (optional, overwritten) = mean over (f, t) of xf(x), the
 * `features` output of mn/model.py:220.  xf = act(x*scale+shift) when scale is given (the last conv's BatchNorm +
 * Hardswish, mn/model.py:160-166, in training), identity otherwise.  C a multiple of 4 (fp32) or 8 (bf16); x, m and
 * feat 16-byte aligned. */
int eat_freq_pool(const void* x, int dtype, const float* scale, const float* shift, int act, float* m, float* feat, int B,
                  int F, int T, int C, cudaStream_t stream);
/* Backward of the frequency mean: dx[b,f,t,c] = dm[b,t,c] * mul for every f (mul = 1/F), dx in the storage dtype. */
int eat_freq_pool_bwd(const float* dm, float mul, void* dx, int dtype, int B, int F, int T, int C, cudaStream_t stream);
/* attention_pooling.py:45-55: a = clamp(sigmoid(P_att), eps, 1-eps), v = P_val,
 * out[b,k] = sum_h hw[h] * sum_t a v / sum_t a  (out [B,K] overwritten).  sa, r [B,H,K] (optional together, saved for
 * backward): sa = sum_t a, r = sum_t a v / sa.  T, H, K >= 1, 0 < eps < 0.5. */
int eat_att_pool_fwd(const float* P, const float* hw, float eps, float* out, float* sa, float* r, int B, int T, int H, int K,
                     cudaStream_t stream);
/* eat_att_pool_fwd where sample b's sums over t stop at t_valid[b] (B int32 on the device, 1 <= t_valid[b] <= T, which
 * the caller guarantees): clips of different lengths in one eval batch.  No saved tensors.  Checks as eat_att_pool_fwd. */
int eat_att_pool_fwd_len(const float* P, const float* hw, float eps, float* out, int B, int T, int H, int K,
                         const int* t_valid, cudaStream_t stream);
/* Its backward from dout [B,K]: dP [B*T, 2*H*K] overwritten (may alias P) with dP_val = dout hw a / sa and
 * dP_att = dout hw (v - r) / sa * sigmoid'(P_att), zero where the clamp is active (torch.clamp's gradient);
 * dhw [H] += sum_{b,k} dout r; dbias [2*H*K] += sum over rows of dP (the projection's bias gradient). */
int eat_att_pool_bwd(const float* dout, const float* P, float* dP, const float* hw, const float* sa, const float* r, float eps,
                     float* dhw, float* dbias, int B, int T, int H, int K, cudaStream_t stream);

/* ---- clips of different lengths in one eval batch (csrc/packed.cu).  x is NHWC [B, F, T, C] in dtype; sample b holds
 * its clip in t < t_valid[b] and padding beyond.  t_valid: B int32 on the device, 1 <= t_valid[b] <= T, which the caller
 * guarantees (the values are not read on the host).  A bad dtype, B outside [0, 65535], F outside [1, 65535], T or C
 * below 1, or a missing pointer -> EAT_ERR_ARG before any launch; B = 0 is a no-op.  No atomics: bitwise repeatable. ---- */

/* x[b, f, t, c] = 0 for t >= t_valid[b], in place; nothing else is written.  One CTA per (f, b) clears that row's
 * contiguous (T - t_valid[b]) * C padding elements: the work is proportional to the padding. */
int eat_time_pad_zero(void* x, int dtype, int B, int F, int T, int C, const int* t_valid, cudaStream_t stream);
/* out[b, c] (fp32, overwritten) = mean over f < F, t < t_valid[b] of x[b, f, t, c]; the padding is never read. */
int eat_mean_len(const void* x, int dtype, float* out, int B, int F, int T, int C, const int* t_valid, cudaStream_t stream);
/* eat_ctx_pool with the mean over time taken over t < t_valid[b]: out [B, F+T, C] fp32 = [mean over t < t_valid[b] |
 * mean over F for t < t_valid[b], 0 beyond].  C a multiple of 4 (fp32) or 8 (bf16). */
int eat_ctx_pool_len(const void* x, int dtype, float* out, int B, int F, int T, int C, const int* t_valid,
                     cudaStream_t stream);

/* ---- training step around the network (ex_audioset.py:135-199) ---- */

/* Spectrogram mixup, ex_audioset.py:145-146: out[b] = x[b]*lam[b] + x[perm[b]]*(1-lam[b]). */
int eat_mixup(const float* x, const int* perm, const float* lam, float* out, int B, long long per_sample,
              cudaStream_t stream);
/* Hard-label + knowledge-distillation BCE-with-logits and its gradient, ex_audioset.py:149-189.
 * loss_acc (fp64[2], caller-zeroed) += {kd*label_loss, (1-kd)*distillation_loss}; teacher/perm/lam optional
 * (NULL teacher: plain BCE, weight 1).  teacher_known [B] (optional, 1/0): 0 zeroes the distillation loss of a clip
 * without teacher predictions, ex_audioset.py:166-178.  dlogits = d(total loss)/d(logits), may be NULL. */
int eat_bce_kd_loss(const float* logits, const float* y, const float* teacher, const float* teacher_known,
                    const int* perm, const float* lam, float kd_lambda, int B, int C, float* dlogits,
                    double* loss_acc, cudaStream_t stream);
/* torch.optim.Adam (adamw = 0) / AdamW (adamw = 1) on flat fp32 arenas, ex_audioset.py:86-91,198;
 * grad_scale multiplies the gradient first (1/world_size after a sum all-reduce). step counts from 1. */
int eat_adam_step(float* p, const float* g, float* m, float* v, long long n, float lr, float beta1, float beta2,
                  float eps, float weight_decay, int adamw, int step, float grad_scale, cudaStream_t stream);

/* ---- fine-tuning step (ex_esc50.py:96-118, ex_dcase20.py:98-123, ex_openmic.py:97-121; FSD50K, ex_fsd50k.py:97-115,
 * is eat_bce_kd_loss without a teacher).  Every check precedes any device call; B == 0 is a no-op. ---- */

/* Softmax cross-entropy, F.cross_entropy(logits, y, reduction="none").mean(), and its gradient.  Exactly one of
 * y_index (int32 [B], class indices) and y_prob (fp32 [B, C], probability rows) is given.  perm/lam (optional,
 * together): the mixup blend lam*CE(z, y) + (1-lam)*CE(z, y[perm]) as one CE against the blended target y_mix.
 * loss_acc[0] (fp64, caller-zeroed) += mean over b of sum_c y_mix * (lse(z_b) - z_bc);
 * dlogits (optional) = (S * softmax(z) - y_mix) / B with S = sum_c y_mix per row.  Any C >= 1.  An index outside
 * [0, C) makes the loss NaN. */
int eat_ce_loss(const float* logits, const int* y_index, const float* y_prob, const int* perm, const float* lam, int B,
                int C, float* dlogits, double* loss_acc, cudaStream_t stream);
/* OpenMIC's masked multi-label BCE, ex_openmic.py:101-121: y [B, *] (row stride y_stride) is binarised (> 0.5) before
 * the optional mixup blend; mask [B, *] (row stride mask_stride) is row b's own, not blended.
 * loss_acc[0] += mean over all B*C elements of mask * BCE(z, y_mix); dlogits (optional) = mask * (sigmoid(z) - y_mix) / (B*C).
 * y_stride, mask_stride >= C (y = batch[:, :C] and mask = batch[:, C:] of one [B, 2C] tensor: stride 2C). */
int eat_bce_masked_loss(const float* logits, const float* y, int y_stride, const float* mask, int mask_stride,
                        const int* perm, const float* lam, int B, int C, float* dlogits, double* loss_acc,
                        cudaStream_t stream);
/* Frequency-wise MixStyle, helpers/utils.py:101-121, on x [B, 1, F, T] fp32 (out of place, out [B, 1, F, T]):
 * mu, sig = mean and sqrt(unbiased variance + eps) over T per (b, f) (two passes over each row, fp32);
 * out = (x - mu_b) / sig_b * (lam_b sig_b + (1 - lam_b) sig_pb) + lam_b mu_b + (1 - lam_b) mu_pb with pb = perm[b].
 * stats: workspace of 2*B*F floats (mu, sig per row).  Two launches: statistics, then apply.  T >= 2, else EAT_ERR_ARG. */
int eat_mixstyle(const float* x, const int* perm, const float* lam, float eps, float* stats, float* out, int B, int F,
                 int T, cudaStream_t stream);

/* ---- waveform augmentation of the training datasets (csrc/wave_aug.cu): gain, datasets/helpers/audiodatasets.py:45-51
 * and esc50.py:39-44 (pydub_augment, also audioset.py:58-63, fsd50k.py:62-67, openmic.py:56-61); roll,
 * audiodatasets.py:26-38; waveform mixing, esc50.py:47-69, dcase20.py:100-118, fsd50k.py:70-92, openmic.py:74-95,
 * audioset.py:66-88.  The random draws are made on the host (efficientat_b200/augment.py) and passed as B-vectors on
 * the device: idx1 (int32, the primary clip, in [0, S)), idx2 (int32, the partner clip in [0, S), or -1 for a row that
 * is not mixed), shift1/shift2 (int32 roll shifts, any value: taken mod N), gain1/gain2 (fp32 amplitudes 10^(dB/20)),
 * lam (fp32 mixing weight).  These values are not read on the host: an index out of range makes its output row NaN.
 * Every check precedes any launch; B == 0 is a no-op.  No atomics: bitwise repeatable. ---- */

#define EAT_LABEL_PLAIN 0     /* lam y[p] + (1 - lam) y[q] over fp32 label rows (ESC-50, FSD50K, AudioSet) */
#define EAT_LABEL_ONEHOT 1    /* the same over one-hot rows of int32 class indices (DCASE20, dcase20.py:101-114) */
#define EAT_LABEL_OPENMIC 2   /* rows of scores | masks (C = 2H): scores masked (> 0.5) then blended, masks max-ed
                                 (openmic.py:84-94) */

/* sums[s] (fp64, overwritten) = sum over n < N of x[s, n], x [S, N] fp32: one CTA per clip, a fixed-order sum. */
int eat_clip_sum(const float* x, int S, int N, double* sums, cudaStream_t stream);
/* out [B, N] fp32 (overwritten, must not alias src) from src [S, N] fp32, row b with p = idx1[b], q = idx2[b]:
 *   q < 0:   out[b, n] = gain1[b] * src[p, (n - shift1[b]) mod N]
 *   q >= 0:  out[b, n] = l g1 src[p, (n - shift1[b]) mod N] + (1 - l) g2 src[q, (n - shift2[b]) mod N] - c0,
 *            l = lam[b], c0 = (l g1 sums[p] + (1 - l) g2 sums[q]) / N, which is the reference's
 *            x = l (x1 - mean x1) + (1 - l)(x2 - mean x2), x -= mean x, with x1, x2 gained and rolled.
 * sums: eat_clip_sum of src; may be NULL when no row is mixed (a mixed row without sums is NaN).
 * 1 <= N <= 2^30, S >= 1, B <= 65535.  Reads each source sample once per output sample; bandwidth-bound. */
int eat_wave_aug(const float* src, const double* sums, int S, int N, const int* idx1, const int* idx2, const int* shift1,
                 const int* shift2, const float* gain1, const float* gain2, const float* lam, float* out, int B,
                 cudaStream_t stream);
/* out [B, C] fp32 (overwritten) = the labels of the rows eat_wave_aug made, rule EAT_LABEL_*: y_prob [S, C] fp32 for
 * PLAIN and OPENMIC (C even), y_index [S] int32 class indices for ONEHOT (exactly one of the two).  A row with q < 0
 * is row p as it is (one-hot for ONEHOT; OpenMIC's scores unmasked, as the reference returns them).  A class index
 * outside [0, C) makes its row NaN. */
int eat_label_mix(int rule, const float* y_prob, const int* y_index, int S, int C, const int* idx1, const int* idx2,
                  const float* lam, int B, float* out, cudaStream_t stream);

/* ---- polyphase resampling (csrc/resample.cu): scipy.signal.resample_poly(x, up, down) with its defaults
 * (window ('kaiser', 5.0), padtype 'constant'), the step the reference leaves to librosa.core.load(path, sr=32000) in
 * inference.py:45, windowed_inference.py:89 and datasets/esc50.py:115.  up / down is reduced by its gcd; h is the
 * centred filter of 2 hl + 1 taps (hl = 10 max(up, down)), so that
 *   y[b, m] = sum_i x[b, i] h[m down - i up + hl],  m < n_out = ceil(N up / down).
 * The filter is designed on the host (efficientat_b200/resample.py) and passed as a polyphase table [taps][rows] fp32,
 * tap-major over the output residue: table[k][r] = h[p + (taps - 1 - k) up] with p = (r down + offset) mod up, r < up,
 * taps = ceil((2 hl + 1) / up), and 0 where the index passes 2 hl; offset = hl.  up, down <= EAT_RESAMPLE_MAX_RATE and
 * taps x rows <= 43008 floats, else EAT_ERR_UNSUPPORTED; n_out other than ceil(N up / down), or beyond int32, a
 * negative offset or a missing pointer -> EAT_ERR_ARG.  All checks precede any launch; B = 0 is a no-op.  fp32
 * accumulation, no atomics: bitwise repeatable. ---- */

#define EAT_RESAMPLE_MAX_RATE 2048

/* x [B, N] fp32 -> y [B, n_out] fp32 (overwritten, must not alias x).  lengths: NULL, or B int32 on the device, each
 * clip's sample count in [1, N] (the caller checks the range): row b's outputs m < ceil(lengths[b] up / down) then equal
 * the resampling of x[b, :lengths[b]] alone and later outputs are 0; samples at or past lengths[b] are never read. */
int eat_resample_poly_fwd(const float* x, int B, int N, const int* lengths, int up, int down, const float* table, int taps,
                          int offset, float* y, int n_out, cudaStream_t stream);
/* Adjoint of eat_resample_poly_fwd without lengths: dy [B, n_out] fp32 -> dx [B, N] fp32 (overwritten),
 * dx[b, i] = sum_m dy[b, m] h[m down - i up + hl].  table_adj is the forward's table for the exchanged pair (down, up)
 * over h reversed: [taps_adj][down], taps_adj = ceil((2 hl + 1) / down), rows the input residue i mod down. */
int eat_resample_poly_bwd(const float* dy, int B, int N, int up, int down, const float* table_adj, int taps_adj,
                          int offset, float* dx, int n_out, cudaStream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* EAT_B200_H */
