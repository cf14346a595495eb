/* holocron_b200 — C ABI of the H100 (sm_90a) kernels behind the holocron.nn / holocron.ops / holocron.optim
 * hot path of frgfm/Holocron.
 *
 * The reference is pure Python/PyTorch and has no FFI of its own (SURVEY.md §8b): every entry point below replaces
 * the chain of ATen/cuDNN kernels that a reference *Python* function launches; the reference file:line each one
 * stands in for is cited per declaration (paths relative to the reference repository root).
 *
 * Conventions
 *   - plain pointers and sizes only; no torch / C++ types cross this boundary;
 *   - every pointer is a DEVICE pointer unless stated otherwise; `stream` is a cudaStream_t;
 *   - return value: 0 on success, otherwise a cudaError_t (launch-configuration errors included);
 *   - re-entrant, no global mutable state apart from one-time kernel attribute setup;
 *   - dtype codes: 0 = float32, 1 = bfloat16, 2 = float16;
 *   - window geometry: every entry point that slides a K-tap window (dilation dil, 1 where it takes none) over H input
 *     pixels computes Ho = (H + 2*pad - dil*(K-1) - 1) / stride + 1, and Wo likewise. It refuses the call with
 *     cudaErrorInvalidValue (a size query returns 0) before any device call unless H, K, stride, dil >= 1, pad >= 0,
 *     H + 2*pad >= dil*(K-1) + 1 (the dilated window fits the padded input) and Ho fits an int;
 *   - activation tensors of the convolution / BatchNorm entry points are NHWC bf16 ("channels_last"),
 *     filters are KRSC ([Cout][R][S][Cin]).
 */
#ifndef HOLOCRON_B200_H
#define HOLOCRON_B200_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- activations: holocron/nn/functional.py:30-41 (hard_mish), :44-56 (nl_relu) ------------------------ */
int hb_hard_mish_fwd(const void* x, void* y, size_t n, int dtype, void* stream);
int hb_hard_mish_bwd(const void* x, const void* dy, void* dx, size_t n, int dtype, void* stream);
int hb_nl_relu_fwd(const void* x, void* y, size_t n, float beta, int dtype, void* stream);
int hb_nl_relu_bwd(const void* x, const void* dy, void* dx, size_t n, float beta, int dtype, void* stream);
/* backward of the in-place variant, from the OUTPUT y = log(1 + beta*relu(x)) */
int hb_nl_relu_bwd_from_out(const void* y, const void* dy, void* dx, size_t n, float beta, int dtype, void* stream);

/* ---- dense convolutions (wgmma implicit GEMM): nn.Conv2d call sites of holocron/models/utils.py:71-76
 *      (conv_sequence), models/classification/repvgg.py:55-73 (RepBlock) and their autograd backward -------- */
/* y[N,Ho,Wo,Cout] = act(conv(x[N,H,W,Cin], w[Cout,R,S,Cin]) + bias + residual); Cin % 8 == 0, Cout % 16 == 0.
 * bias: fp32 [Cout] or NULL; residual: bf16 like y or NULL; act: 0 none, 1 relu; num_ctas: 0 = one per SM. */
int hb_conv2d_fprop_bf16(const void* x, const void* w, void* y, const float* bias, const void* residual, int N, int H,
                         int W, int Cin, int Cout, int R, int S, int stride, int pad, int dil, int act, int num_ctas,
                         void* stream);
/* General form of the above (one kernel launch), used by the fused RepVGG block (repvgg.py:71-73) and by every
 * conv -> BatchNorm2d unit of conv_sequence (utils.py:71-76) in training mode:
 *   K extension   xe != NULL: y += conv1x1(xe [N,Ho,Wo,Ce], we [Cout,1,1,Ce]) in the SAME accumulator (stride-1 layers:
 *                 the input gradient of both RepVGG branches, dX = dgrad3x3(dY3) + dgrad1x1(dY1) (+ residual));
 *   dual output   w2 != NULL: y2 [N,Ho,Wo,Cout] = conv1x1(x, w2 [Cout,1,1,Cin]; same stride, pad 0) from the centre-tap
 *                 loads of the RxS convolution (pad must be (R/2)*dil): x is read once for both RepVGG branches;
 *   statistics    stats / stats2 != NULL: per-channel (sum, sum of squares) partials of the bf16 outputs y / y2 as
 *                 float [*stat_slots][Cout][2]; the caller allocates hb_conv_stat_slots_max() slots, the launch writes
 *                 the first *stat_slots (host int) completely; summing the slots in order is deterministic. This replaces
 *                 the separate statistics pass of training-mode BatchNorm2d.
 *   patch norm    norm_mean != NULL (NormConv2d, holocron/nn/functional.py:322-413): y = norm_rstd[m] * (acc - norm_mean[m] *
 *                 norm_wsum[co]) + bias, m = output pixel: the per-patch standardisation of the im2col rows folded
 *                 algebraically into the epilogue (statistics from hb_patch_stats_bf16).
 * bias / residual / act apply to y only. Fields not used must be zero. */
typedef struct hb_conv_args {
  const void* x; const void* w; void* y; const float* bias; const void* residual;
  int N, H, W, Cin, Cout, R, S, stride, pad, dil, act, num_ctas;
  const void* xe; const void* we; int Ce;
  const void* w2; void* y2;
  float* stats; float* stats2;
  const float* norm_mean; const float* norm_rstd; const float* norm_wsum;
} hb_conv_args;
int hb_conv2d_fused_bf16(const hb_conv_args* args, int* stat_slots, void* stream);
int hb_conv_stat_slots_max(void);
/* Per-patch statistics of the im2col rows of x [N,H,W,C] bf16 (zero padding included, like F.unfold): for every output
 * pixel m, mean[m] and rstd[m] = 1/sqrt(biased var + eps) over its K = k_logical = Cin*kh*kw patch values (channels
 * beyond the logical ones are zero padding of the layout and do not count). scratch: float [2*N*H*W]. */
int hb_patch_stats_bf16(const void* x, float* mean, float* rstd, float* scratch, int N, int H, int W, int C, int kh, int kw,
                        int stride, int pad, int dil, int k_logical, float eps, void* stream);
/* y = conv3x3(x, w; stride 1, pad 1) + sum_{e<nextra} conv1x1(xe_e, we_e), one accumulator (nextra <= 2; all inputs
 * [N,H,W,Cin] bf16, w [Cout,3,3,Cin], we_e [Cout,1,1,Cin]). Input gradient of a RepVGG block in one kernel
 * (holocron/models/classification/repvgg.py:71-73). Returns cudaErrorNotSupported (801) when the filter does not fit the
 * shared-memory-resident scheme (Cin, Cout <= 64 typically) - fall back to separate convolutions then. */
int hb_conv3x3_accum_bf16(const void* x, const void* w, const void* xe0, const void* we0, const void* xe1, const void* we1,
                          int nextra, void* y, int N, int H, int W, int Cin, int Cout, int num_ctas, void* stream);
/* dw[Cout,R,S,Cin] (fp32, overwritten) = sum over pixels of dy[N,Ho,Wo,Cout] x im2col(x[N,H,W,Cin]).
 * workspace: optional fp32 scratch of hb_conv2d_wgrad_workspace_bytes(...) bytes: the per-pixel-range partial sums are
 * then reduced in a fixed order (deterministic); with NULL they are accumulated with fp32 atomics. */
size_t hb_conv2d_wgrad_workspace_bytes(int N, int H, int W, int Cin, int Cout, int R, int S, int stride, int pad, int dil,
                                       int num_ctas);
int hb_conv2d_wgrad_bf16(const void* x, const void* dy, float* dw, float* workspace, size_t workspace_bytes, int N, int H,
                         int W, int Cin, int Cout, int R, int S, int stride, int pad, int dil, int num_ctas, void* stream);
/* Both weight gradients of a stride-1 RepVGG block in ONE pass over x (the 1x1 branch reads x through the centre-tap
 * window of the rows the 3x3 branch already holds in shared memory; holocron/models/classification/repvgg.py:55-73):
 * dw = [dW3 (Cout,3,3,Cin) | dW1 (Cout,Cin)] fp32, overwritten. hb_repvgg_wgrad_workspace_bytes == 0 / return code
 * cudaErrorNotSupported (801): shape outside the row-window scheme, use hb_conv2d_wgrad_bf16 per branch. */
size_t hb_repvgg_wgrad_workspace_bytes(int N, int H, int W, int Cin, int Cout, int num_ctas);
int hb_repvgg_wgrad_bf16(const void* x, const void* dy3, const void* dy1, float* dw, float* workspace, size_t workspace_bytes,
                         int N, int H, int W, int Cin, int Cout, int num_ctas, void* stream);
/* Accumulating forms: the fixed-order reduction ADDS onto dw / dw3 / dw1 (the parameters' .grad storage, e.g. views of
 * the flat data-parallel gradient bucket) instead of overwriting - what autograd's AccumulateGrad does with one more
 * element-wise kernel per parameter and step. hb_conv2d_wgrad_acc_bf16 returns cudaErrorNotSupported (801), dw untouched,
 * for shapes that run as a single pixel range. */
int hb_conv2d_wgrad_acc_bf16(const void* x, const void* dy, float* dw, float* workspace, size_t workspace_bytes, int N, int H,
                             int W, int Cin, int Cout, int R, int S, int stride, int pad, int dil, int num_ctas,
                             void* stream);
int hb_repvgg_wgrad_acc_bf16(const void* x, const void* dy3, const void* dy1, float* dw3, float* dw1, float* workspace,
                             size_t workspace_bytes, int N, int H, int W, int Cin, int Cout, int num_ctas, void* stream);
/* fp32 KRSC master filter -> bf16 KRSC [CoutF][R][S][CinP] (zero-padded rows / channels) and, if wd != NULL, the
 * flipped + transposed bf16 filter [CinD][R][S][CoutP] used by the data-gradient pass */
int hb_pack_conv_weights(const float* w, void* wf, void* wd, int Cout, int Cin, int R, int S, int CinP, int CinD,
                         int CoutP, int CoutF, void* stream);
/* The same for a whole network in ONE launch. metas: device array of hb_pack_meta_bytes()-byte rows
 * {const float* w; bf16* wf; bf16* wd (NULL allowed); int32 Cout, Cin, R, S, CinP, CinD, CoutP, CoutF}; chunks: device array
 * of int32 pairs (row index, chunk index), hb_pack_chunk_elems() output elements (wf then wd) per chunk. */
int hb_pack_conv_weights_multi(const void* metas, const void* chunks, int num_chunks, void* stream);
int hb_pack_chunk_elems(void);
int hb_pack_meta_bytes(void);
/* Data gradient of a stride-2 3x3 pad-1 convolution (the backward of the stride-2 nn.Conv2d at the head of every
 * RepVGG / Darknet / ReXNet stage, holocron/models/classification/repvgg.py:55-73, utils.py:28-86) without zero insertion:
 * the 4 parity classes of dx [N,H,W,Cd] are 1/2/2/4-tap correlations over dy [N,Ho,Wo,C] written to their sub-grids.
 * wcls: class filters from hb_pack_dgrad_s2_weights. dy1/wd1 (may be NULL): output gradient and [Cd,1,1,C] filter of a
 * parallel 1x1 stride-2 branch, accumulated into class (0,0). Ho = (H-1)/2+1, Wo = (W-1)/2+1. */
int hb_conv2d_dgrad_s2_bf16(const void* dy, const void* wcls, const void* dy1, const void* wd1, void* dx, int N, int H, int W,
                            int Ho, int Wo, int C, int Cd, int num_ctas, void* stream);
/* fp32 KRSC master filter [Cout,3,3,Cin] -> the four bf16 class filters [CinD][1+a][1+b][CoutP], (a,b) = (0,0), (0,1),
 * (1,0), (1,1), stored back to back (9*CinD*CoutP elements) */
int hb_pack_dgrad_s2_weights(const float* w, void* out, int Cout, int Cin, int CinD, int CoutP, void* stream);
/* y[N,Ho,Wo,C] = zeros, y[n, sp*p, sp*q, :] = x[n,p,q,:]  (input of a stride-sp transposed convolution) */
int hb_zero_insert_bf16(const void* x, void* y, int N, int Hi, int Wi, int Ho, int Wo, int C, int sp, void* stream);
/* NCHW image (dtype code) -> NHWC bf16 with channels zero-padded to CP (CP % 8 == 0) */
int hb_nchw_to_nhwc_pad_bf16(const void* x, void* y, int N, int C, int H, int W, int CP, int dtype, void* stream);

/* explicit im2col for stems (Cin <= 4): x NCHW (dtype code) -> col [N*Ho*Wo, Kp] bf16 with k = (r*S + s)*C + c, zero
 * padded to Kp (multiple of 8); the stem then runs as a 1x1 convolution over Kp channels */
int hb_im2col_smallc_bf16(const void* x, void* col, int N, int C, int H, int W, int R, int S, int stride, int pad, int Kp,
                          int dtype, void* stream);

/* ---- BatchNorm2d + branch sum + activation, fused: BatchNorm2d/act emitted by conv_sequence
 *      (holocron/models/utils.py:73-78) and the branch sum of RepBlock.forward (repvgg.py:71-73) ------------- */
/* Training-mode statistics are carried as PARTIALS: float [slots][C][2] = per-channel (sum, sum of squares) of a
 * subset of the rows, written by the producer of the tensor (hb_conv2d_fused_bf16's stats/stats2, hb_bn_act_fwd_bf16's
 * out_stats) or by this stand-alone pass over u [M,C] bf16 (capacity hb_bn_stat_slots_max() slots, *slots = host int
 * out). hb_bn_finalize adds the slots of each branch in a fixed order in fp64: no floating-point atomics anywhere, two
 * runs give bit-identical statistics. */
int hb_bn_stats_partials_bf16(const void* u, int M, int C, float* parts, int* slots, void* stream);
int hb_bn_stat_slots_max(void);
/* parts, slots, gamma, beta, running_mean/var, num_batches_tracked: HOST arrays of B entries (device pointers / ints;
 * pointer entries other than parts may be NULL). Outputs fp32 [B][C]. Updates the running statistics with `momentum`
 * (unbiased variance) and increments the int64 num_batches_tracked counters, like nn.BatchNorm2d in training mode. */
int hb_bn_finalize(const float* const* parts, const int* slots, const float* const* gamma, const float* const* beta,
                   float* const* running_mean, float* const* running_var, long long* const* num_batches_tracked,
                   float* mean, float* rstd, float* scale, float* shift, int B, int C, int C_logical, int M, float eps,
                   float momentum, void* stream);
/* Synchronised BatchNorm (nn.SyncBatchNorm), forward in two steps around a SUM all-reduce of `sums` over the ranks:
 * hb_bn_partials_sums folds each branch's partial slots in hb_bn_finalize's fixed order into double sums[B][C][2]
 * (sum, sum of squares; 0 on the padding channels) and writes the row count M as a double at sums[B*C*2] (B*C*2 + 1
 * doubles). hb_bn_finalize_sums then writes what hb_bn_finalize writes, from the (all-reduced) sums and count: same
 * arithmetic, the running variance unbiased over the summed count. Arguments as hb_bn_finalize. */
int hb_bn_partials_sums(const float* const* parts, const int* slots, int B, int C, int C_logical, int M, double* sums,
                        void* stream);
int hb_bn_finalize_sums(const double* sums, const float* const* gamma, const float* const* beta,
                        float* const* running_mean, float* const* running_var, long long* const* num_batches_tracked,
                        float* mean, float* rstd, float* scale, float* shift, int B, int C, int C_logical, float eps,
                        float momentum, void* stream);
/* channels in [C_logical, C) are zero padding (the parameter arrays hold C_logical entries): scale = shift = 0 */
int hb_bn_eval_affine(const float* gamma, const float* beta, const float* running_mean, const float* running_var,
                      float eps, int C, int C_logical, float* scale, float* shift, float* mean, float* rstd,
                      void* stream);
/* out = act(sum_b (scale_b * u_b + shift_b) + residual)  [res_after = 1: act(sum_b ...) + residual, the shortcut of
 * holocron/models/classification/resnet.py:75-87 (_ResBlock.forward) used by the Darknet ResBlocks]; act: 0 none 1 relu 2 relu6 3 silu 4 leaky(slope) 5 mish
 * 6 hard_mish, 7 funnel: out = max(sum_b(...), residual) (FReLU, holocron/nn/modules/activation.py:58-82) */
/* out_stats (optional): (sum, sum of squares) partials of the bf16 OUTPUT, float [*out_stat_slots][C][2] (capacity
 * hb_bn_stat_slots_max()): the statistics of the identity-branch BatchNorm of the next RepVGG block, for free. */
int hb_bn_act_fwd_bf16(const void* u0, const void* u1, const void* u2, int B, const float* scale, const float* shift,
                       const void* residual, void* out, int M, int C, int act, float slope, int res_after,
                       float* out_stats, int* out_stat_slots, void* stream);
/* backward of the above; scratch: double [hb_bn_bwd_scratch_doubles(M, C, B)] (uninitialised); du_b/dres/dgamma/dbeta may
 * be NULL; gamma_grad_acc / beta_grad_acc: optional HOST arrays of B device pointers (entries may be NULL) to the fp32
 * [C_logical] gradient buffers of the BatchNorm weight / bias, which dgamma_b / dbeta_b are ADDED to (deterministic
 * fixed-order reductions, no atomics). */
size_t hb_bn_bwd_scratch_doubles(int M, int C, int B);
int hb_bn_act_bwd_bf16(const void* dout, const void* u0, const void* u1, const void* u2, int B, const float* scale,
                       const float* shift, const float* mean, const float* rstd, const void* residual, double* scratch,
                       void* du0, void* du1, void* du2, void* dres, float* dgamma, float* dbeta,
                       float* const* gamma_grad_acc, float* const* beta_grad_acc, int C_logical, int M, int C, int act,
                       float slope, int train, int res_after, void* stream);
/* hb_bn_act_bwd_bf16 (train = 1) in two steps around a SUM all-reduce of scratch[0 .. (1+B)*C) over the ranks of a
 * synchronised BatchNorm. reduce: scratch[0][c] = sum dz, scratch[1+b][c] = sum dz*u_b over these M rows, and the LOCAL
 * dgamma/dbeta written / added exactly as hb_bn_act_bwd_bf16 does. apply: du_b and dres from the (all-reduced) sums
 * (scratch of the reduce step) over `count` rows (device double, e.g. hb_bn_partials_sums' count after its all-reduce). */
int hb_bn_act_bwd_reduce_bf16(const void* dout, const void* u0, const void* u1, const void* u2, int B, const float* scale,
                              const float* shift, const float* mean, const float* rstd, const void* residual,
                              double* scratch, float* dgamma, float* dbeta, float* const* gamma_grad_acc,
                              float* const* beta_grad_acc, int C_logical, int M, int C, int act, float slope, int res_after,
                              void* stream);
int hb_bn_act_bwd_apply_bf16(const void* dout, const void* u0, const void* u1, const void* u2, int B, const float* scale,
                             const float* shift, const float* mean, const float* rstd, const void* residual,
                             const double* sums, const double* count, void* du0, void* du1, void* du2, void* dres, int M,
                             int C, int act, float slope, int res_after, void* stream);

/* ---- depth-wise k x k convolution (NHWC bf16; weights fp32 [C,K,K]): FReLU's conv (activation.py:71-73) and the
 *      ReXNet depth-wise stage (holocron/models/classification/rexnet.py:112-125) -------------------------
 * Ho = (H + 2*pad - K) / stride + 1, Wo likewise. All three entry points return cudaErrorInvalidValue, before any launch
 * or device query, unless N, H, W, C, K, stride >= 1, pad >= 0, C % 8 == 0 and K <= H + 2*pad, K <= W + 2*pad (so
 * Ho, Wo >= 1). hb_dwconv_wgrad_scratch_doubles returns 0 for C < 1, C % 8 != 0 or K outside {1,3,5,7}. */
int hb_dwconv_fwd_bf16(const void* x, const float* w, const float* bias, void* y, int N, int H, int W, int C, int K,
                       int stride, int pad, void* stream);
int hb_dwconv_bwd_data_bf16(const void* dy, const float* w, void* dx, int N, int H, int W, int C, int K, int stride,
                            int pad, void* stream);
/* dw fp32 [C,K,K], db fp32 [C] or NULL; scratch: double[hb_dwconv_wgrad_scratch_doubles(C, K)] (per-block partial sums,
 * folded in a fixed order: deterministic); K in {1,3,5,7} */
size_t hb_dwconv_wgrad_scratch_doubles(int C, int K);
int hb_dwconv_bwd_weight_bf16(const void* x, const void* dy, float* dw, float* db, double* scratch, int N, int H, int W,
                              int C, int K, int stride, int pad, void* stream);

/* ---- involution: holocron/nn/modules/conv.py:441-499 (Involution2d: the unfold, the product with the generated kernel
 *      and the sum over the taps) -------------------------------------------------------------------------------
 * x NHWC bf16 [N,H,W,Cp], ker NHWC bf16 [N,Ho,Wo,Kp] with channel g*K*K + t for group g and tap t (Kp >= G*K*K: the
 * zero-padded span output), y / dy NHWC bf16 [N,Ho,Wo,Cp], Ho = (H + 2*pad - dil*(K-1) - 1) / stride + 1. C % G == 0,
 * Cp >= C with Cp % 8 == 0 (channels C..Cp-1 of y and dx are written as zeros), K in {1,3,5,7}. dker: every column
 * of [N,Ho,Wo,Kp] is written, the padding columns G*K*K..Kp-1 as zeros. Deterministic (fixed-order sums, no atomics). */
int hb_involution_fwd_bf16(const void* x, const void* ker, void* y, int N, int H, int W, int C, int Cp, int Kp, int K,
                           int G, int stride, int pad, int dil, void* stream);
int hb_involution_bwd_data_bf16(const void* dy, const void* ker, void* dx, int N, int H, int W, int C, int Cp, int Kp,
                                int K, int G, int stride, int pad, int dil, void* stream);
int hb_involution_bwd_kernel_bf16(const void* x, const void* dy, void* dker, int N, int H, int W, int C, int Cp, int Kp,
                                  int K, int G, int stride, int pad, int dil, void* stream);

/* ---- lambda layer: holocron/nn/modules/lambda_layer.py:15-108 (LambdaLayer.forward :70-108: the key softmax :90, the
 *      content lambda :93-94, the position lambda :97-104 and the output :106-108) ----------------------------------
 * Every entry takes the same geometry: B samples of H x W positions, dim_k dk in {8,16,32}, dim_u u in 1..4, heads in
 * 1..8, dim_v dv >= 1, r = the odd local receptive field (1..23, lambda_layer.py:60-64) or 0 for the global variant
 * (pos_emb, :66-68), and the padded NHWC widths (multiples of 8) of q (channel h*dk+k, Cqp >= heads*dk), k (k*u+u',
 * Ckp >= dk*u), v (v*u+u', Cvp >= dv*u) and y / dy (h*dv+v, Cop >= heads*dv); every channel past the logical ones of an
 * output is written as zero. stats [B][dk*u][2] fp32 (row max, sum of exponentials of the key softmax); lc / dlc
 * [B][dk][dv] fp32; Rt [r*r][u][dk] fp32 (R transposed tap-major); lp [B][HW][dk][dv] fp32 (global only, the GEMM of
 * pos_emb and v); dlp [B][HW][dk][dvp] bf16, dvp = dv rounded up to 8 (sum_h q * dy, the per-position gradient of lp);
 * dvpos [B][HW][dv*u] fp32 (global only, pos_emb^T dlp). Deterministic (fixed-order sums, no atomics), no host sync. */
int hb_lambda_content_fwd_bf16(const void* k, const void* v, float* stats, float* lc, int B, int H, int W, int dk,
                               int u, int heads, int dv, int r, int Cqp, int Ckp, int Cvp, int Cop, void* stream);
int hb_lambda_out_fwd_bf16(const void* q, const void* v, const float* Rt, const float* lc, const float* lp, void* y,
                           int B, int H, int W, int dk, int u, int heads, int dv, int r, int Cqp, int Ckp, int Cvp,
                           int Cop, void* stream);
int hb_lambda_bwd_content_bf16(const void* q, const void* k, const void* v, const void* dy, const float* stats,
                               float* dlc, void* dk_out, int B, int H, int W, int dk, int u, int heads, int dv, int r,
                               int Cqp, int Ckp, int Cvp, int Cop, void* stream);
int hb_lambda_dlp_bf16(const void* q, const void* dy, void* dlp, int B, int H, int W, int dk, int u, int heads, int dv,
                       int r, int Cqp, int Ckp, int Cvp, int Cop, void* stream);
int hb_lambda_bwd_q_bf16(const void* dy, const void* v, const float* Rt, const float* lc, const float* lp, void* dq,
                         int B, int H, int W, int dk, int u, int heads, int dv, int r, int Cqp, int Ckp, int Cvp,
                         int Cop, void* stream);
int hb_lambda_bwd_v_bf16(const void* k, const float* stats, const float* dlc, const void* dlp, const float* Rt,
                         const float* dvpos, void* dv_out, int B, int H, int W, int dk, int u, int heads, int dv, int r,
                         int Cqp, int Ckp, int Cvp, int Cop, void* stream);
/* dR [dk][u][r*r] fp32 (R's own layout); scratch: B*dk*u*r*r floats of per-sample partials */
int hb_lambda_bwd_r_bf16(const void* dlp, const void* v, float* scratch, float* dR, int B, int H, int W, int dk, int u,
                         int heads, int dv, int r, int Cqp, int Ckp, int Cvp, int Cop, void* stream);

/* ---- global average pooling: holocron/nn/modules/downsample.py:58-74 ----------------------------------- */
int hb_gap_fwd_bf16(const void* x, void* y, int N, int HW, int C, void* stream);
int hb_gap_bwd_bf16(const void* dy, void* dx, int N, int HW, int C, void* stream);

/* ---- blur pooling: holocron/nn/modules/downsample.py:106-151 (BlurPool2d: ReflectionPad2d(p) then a depth-wise
 *      conv2d with the binomial filter, :148-151) ------------------------------------------------------------------
 * x / dx NHWC [N,H,W,Cp], y / dy NHWC [N,Ho,Wo,Cp] of dtype 0 (fp32) or 1 (bf16), fp32 accumulation; Cp >= C with
 * Cp * sizeof(dtype) % 16 == 0 (channels C..Cp-1 of y and dx are written as zeros). taps: HOST pointer to the K*K
 * filter (row-major fp32 values, copied into the launch), K in 2..7, stride >= 1, p = ((stride-1) + (K-1)) / 2 < H, W
 * (ReflectionPad2d's limit), Ho = (H + 2p - K) / stride + 1. The reflection is folded into the indices (no padded
 * copy); the backward pass is the gather-form adjoint (each dx element written once). */
int hb_blurpool_fwd(const void* x, void* y, const float* taps, int N, int H, int W, int C, int Cp, int K, int stride,
                    int dtype, void* stream);
int hb_blurpool_bwd(const void* dy, void* dx, const float* taps, int N, int H, int W, int C, int Cp, int K, int stride,
                    int dtype, void* stream);

/* ---- max / mean reductions: holocron/nn/modules/downsample.py:80-99 (GlobalMaxPool2d), :170-183 (ZPool) and
 *      holocron/nn/functional.py:139-147 (z_pool: cat(max(dim), mean(dim))) -------------------------------------
 * mid: x [A,L,M] reduced over L (GlobalMaxPool2d: A=N, L=H*W, M=Cp; z_pool dim 2: A=N, L=H, M=W*Cp; dim 3: A=N*H,
 * L=W, M=Cp); y [A][1 + with_mean][M] holds the max plane, then the mean plane when with_mean; idx int32 [A,M] the
 * index along L of the max. last: x [R,Cp] reduced over its first C channels (z_pool dim 1: R=N*H*W); y [R][2] =
 * (max, mean), idx int32 [R]. Index order: NaN first, then larger, then lower index (torch's max(dim).indices).
 * Backward: dx = dmax at the saved index + dmean / L (L = C for last), each element written once. dtype 0 (fp32) or 1
 * (bf16), Cp * sizeof(dtype) % 16 == 0, M % Cp == 0; channels C..Cp-1 of y, idx and dx are written as zeros.
 * Deterministic (fixed-order combination, no atomics), no host sync. */
int hb_pool_mid_fwd(const void* x, void* y, int* idx, int A, int L, int M, int C, int Cp, int with_mean, int dtype,
                    void* stream);
int hb_pool_mid_bwd(const void* dy, const int* idx, void* dx, int A, int L, int M, int C, int Cp, int with_mean,
                    int dtype, void* stream);
int hb_pool_last_fwd(const void* x, void* y, int* idx, int R, int C, int Cp, int dtype, void* stream);
int hb_pool_last_bwd(const void* dy, const int* idx, void* dx, int R, int C, int Cp, int dtype, void* stream);

/* ---- attention: holocron/nn/modules/attention.py:17-30 (SAM: x * sigmoid(conv1x1(x))), :33-56 (DimAttention: x gated by
 *      sigmoid(BN(conv7x7(z_pool(x)))) along one dim), :59-77 (TripletAttention: the mean of the C, H and W branches) -
 * x / y / dy / dx NHWC [N,H,W,Cp] of dtype 0 (fp32) or 1 (bf16), Cp * sizeof(dtype) % 16 == 0; channels C..Cp-1 are
 * never read into a result and are written as zeros. Gates, planes, statistics and parameter gradients are fp32.
 * Deterministic (fixed-order partial sums, no atomics), no host sync: graph-capturable. */
/* SAM over R = N*H*W pixel rows, C <= 128 vectors of 16 bytes. w fp32 [C], b fp32 [1]; gate fp32 [R] (saved for the
 * backward pass). Backward: part fp32 [hb_sam_bwd_slots()][Cp + 1] scratch; dwdb fp32 [C + 1] = (dw, db). */
int hb_sam_bwd_slots(int R, int C, int Cp, int dtype);
int hb_sam_fwd(const void* x, const float* w, const float* b, void* y, float* gate, int R, int C, int Cp, int dtype,
               void* stream);
int hb_sam_bwd(const void* x, const void* dy, const float* w, const float* gate, void* dx, float* part, float* dwdb,
               int R, int C, int Cp, int dtype, void* stream);
/* Triplet pool, Cp <= 2048: one read of x gives the z_pool planes of the branches whose pointers are set: pc [N][2][H][W]
 * (max, mean over C) + ic [N][H][W]; pw [N][2][H][C] (over W) + iw [N][H][C]; ph [N][2][C][W] (over H) + ih [N][C][W],
 * through the row-block partials hp_* [N][nHB][W][C], nHB = ceil(H / hb_triplet_row_block()). Indices follow
 * max(dim).indices (NaN first, then larger, then lower index). Backward: the same traversal of x and dy gives the sums
 * of dy * x over C (dgc [N][H][W]), W (dgw [N][H][C]) and H (dgh [N][C][W], through hp_sum). */
int hb_triplet_row_block(int H, int C, int Cp, int dtype);
int hb_triplet_pool_fwd(const void* x, float* pc, int* ic, float* pw, int* iw, float* hp_max, float* hp_sum,
                        int* hp_idx, float* ph, int* ih, int N, int H, int W, int C, int Cp, int dtype, void* stream);
int hb_triplet_pool_bwd(const void* x, const void* dy, float* dgc, float* dgw, float* hp_sum, float* dgh, int N, int H,
                        int W, int C, int Cp, int dtype, void* stream);
/* Per-branch planes: HOST arrays of 3 entries (device pointers, NULL = branch disabled; rows / cols = R / S of each
 * [N][R][S] plane). conv: z = conv2d(plane [N][2][R][S], weight [2][7][7], padding 3) and parts [slots][2] = per-CTA
 * (sum z, sum z^2) for hb_bn_finalize (slots: HOST int[3] out). gate: g = sigmoid(z * stats[2] + stats[3]), stats =
 * (mean, rstd, scale, shift) as hb_bn_finalize / hb_bn_eval_affine write them. bn_bwd: dz = (dg * inv_nb) g (1 - g)
 * through the BatchNorm (batch statistics when train, else the affine map), dgamma / dbeta fp32 [1] written; parts
 * [slots][2] scratch. conv_bwd: dplane [N][2][R][S] (gather form) and dweight [2][7][7]; parts [slots][98] scratch. */
int hb_triplet_conv_fwd(const float* const* plane, const float* const* weight, float* const* z, float* const* parts,
                        int* slots, const int* rows, const int* cols, int N, void* stream);
int hb_triplet_gate(const float* const* z, const float* const* stats, float* const* gate, const int* rows,
                    const int* cols, int N, void* stream);
int hb_triplet_bn_bwd(const float* const* dg, const float* const* z, const float* const* gate,
                      const float* const* stats, float* const* dz, float* const* parts, float* const* dgamma,
                      float* const* dbeta, const int* rows, const int* cols, int N, float inv_nb, int train,
                      void* stream);
int hb_triplet_conv_bwd(const float* const* plane, const float* const* weight, const float* const* dz,
                        float* const* dplane, float* const* parts, float* const* dweight, const int* rows,
                        const int* cols, int N, void* stream);
/* y = (x g_c + x g_h + x g_w) / (number of set gates), in that order; gates fp32 [N][H][W], [N][C][W], [N][H][C].
 * dx = dy (g_c + g_h + g_w) / nb + per branch: the plane's dmax at the saved index + dmean / (reduced length). */
int hb_triplet_apply(const void* x, void* y, const float* gc, const float* gh, const float* gw, int N, int H, int W,
                     int C, int Cp, int dtype, void* stream);
int hb_triplet_dx(const void* dy, void* dx, const float* gc, const float* gh, const float* gw, const float* dpc,
                  const float* dph, const float* dpw, const int* ic, const int* ih, const int* iw, int N, int H, int W,
                  int C, int Cp, int dtype, void* stream);

/* ---- squeeze-excite gate: SEBlock.forward `x * y` followed by the block's activation,
 *      holocron/models/classification/rexnet.py:63-66, 125-131 --------------------------------------------- */
/* out[n,p,c] = act(x[n,p,c] * gate[n,c]);  x/out [N,HW,C] bf16, gate fp32 [N,C]; act codes as hb_bn_act_fwd_bf16 (0-6) */
int hb_gate_act_fwd_bf16(const void* x, const float* gate, void* out, int N, int HW, int C, int act, float slope,
                         void* stream);
/* dz = dout * act'(x*gate); dx = dz * gate (bf16); dgate[n,c] = sum_p dz * x (fp32, overwritten, deterministic) */
int hb_gate_act_bwd_bf16(const void* dout, const void* x, const float* gate, void* dx, float* dgate, int N, int HW, int C,
                         int act, float slope, void* stream);

/* ---- box operators: holocron/ops/boxes.py:16-211 (+ torchvision.ops.boxes.box_iou, boxes.py:11) ---------- */
/* mode: 0 IoU, 1 GIoU, 2 DIoU penalty rho^2/c^2, 3 DIoU loss (== the reference's ciou_loss, boxes.py:208-209),
 * 4 aspect-ratio consistency. boxes fp32 [M,4]/[N,4] xyxy; out fp32 [M,N]. */
int hb_box_pairwise(const float* boxes1, const float* boxes2, float* out, int M, int N, int mode, void* stream);
/* sets *flag (device int) to 1 when a box has x2 < x1 or y2 < y1 (box_giou's AssertionError, boxes.py:56-57) */
int hb_box_degenerate(const float* boxes, int n, int* flag, void* stream);
/* g1 [M,4], g2 [N,4] (either may be NULL) = gradients of sum(gout * op) for modes 0-3 */
int hb_box_pairwise_bwd(const float* boxes1, const float* boxes2, const float* gout, float* g1, float* g2, int M, int N,
                        int mode, void* stream);

/* ---- NormConv2d / Add2d: holocron/nn/functional.py:322-462 (_xcorr2d, norm_conv2d, add2d) ---------------- */
/* x fp32 NCHW, w fp32 [Cout,Cin,KH,KW], out fp32 [N,Cout,Ho,Wo]; mode 0 multiply-accumulate, 1 adder (-L1);
 * normalize: standardise every im2col patch (biased var + eps); mean/rstd: fp32 [N*Ho*Wo] (written when normalize). */
int hb_xcorr2d_fwd(const float* x, const float* w, const float* bias, float* out, float* mean, float* rstd, int N, int Cin,
                   int H, int W, int Cout, int KH, int KW, int stride, int pad, int dil, int mode, int normalize,
                   float eps, void* stream);
int hb_xcorr2d_wgrad(const float* x, const float* w, const float* g, const float* mean, const float* rstd, float* dw,
                     int N, int Cin, int H, int W, int Cout, int KH, int KW, int stride, int pad, int dil, int mode,
                     int normalize, float eps, void* stream);
int hb_add2d_dgrad(const float* x, const float* w, const float* g, float* dx, int N, int Cin, int H, int W, int Cout,
                   int KH, int KW, int stride, int pad, int dil, void* stream);

/* ---- DropBlock: holocron/nn/functional.py:465-500, nn/modules/dropblock.py:14-41 ------------------------ */
/* mask[N,H,W] = 1 - maxpool_bs(noise <= gamma); *kept (device 64-bit integer) = sum(mask), exact. block_size must be
   odd. */
int hb_dropblock_mask(const float* noise, float* mask, unsigned long long* kept, int N, int H, int W, int block_size,
                      float gamma, void* stream);
/* out = x * mask * scale, scale = fl(fl(1 / (float)*kept) * (float)(N*H*W)) as the reference rounds numel / kept (1 when
   *kept == 0); x: [N,C,H,W] logical, physical NHWC if channels_last */
int hb_dropblock_apply(const void* x, void* out, const float* mask, const unsigned long long* kept, int N, int C, int H,
                       int W, int channels_last, int dtype, void* stream);

/* ---- losses: holocron/nn/functional.py:59-113 (focal_loss), :540-613 (poly_loss), :503-537 (dice_loss) --- */
/* logits x are [N, K, S] (S = prod of spatial dims); kind 0 focal / 1 poly-1; loss_pos: float[N*S];
 * partials: double[2 * hb_loss_max_partials()] scratch; fwd_out: float[3] = {sum, #valid, mean}. */
int hb_loss_max_partials(void);
int hb_cls_loss_hard_fwd(const void* x, const long long* target, const float* weight, float* loss_pos, double* partials,
                         float* fwd_out, int N, int K, int S, int ignore_index, int kind, float gamma, float eps,
                         int dtype, void* stream);
/* reduction: 0 none (gout[N*S]), 1 mean, 2 sum (gout[1]); dx like x */
int hb_cls_loss_hard_bwd(const void* x, const long long* target, const float* weight, const float* gout,
                         const float* fwd_out, void* dx, int N, int K, int S, int ignore_index, int kind, float gamma,
                         float eps, int reduction, int dtype, void* stream);
int hb_poly_soft_fwd(const void* x, const void* soft, const float* weight, float* loss_pos, double* partials,
                     float* fwd_out, int N, int K, int S, int ignore_index, float eps, int dtype, void* stream);
int hb_poly_soft_bwd(const void* x, const void* soft, const float* weight, const float* gout, void* dx, int N, int K,
                     int S, int ignore_index, float eps, int reduction, int dtype, void* stream);
/* scratch: double[hb_dice_scratch_doubles(K)] (per-block partial sums, folded in a fixed order: deterministic);
 * out: float[1]; coef: float[2K] (input of hb_dice_bwd) */
size_t hb_dice_scratch_doubles(int K);
int hb_dice_fwd(const void* x, const void* target, const float* weight, double* scratch, float* out, float* coef, int N,
                int K, long long S, float gamma, float eps, int dtype, void* stream);
int hb_dice_bwd(const void* target, const float* coef, const float* gout, void* dx, int N, int K, long long S, int dtype,
                void* stream);
/* multilabel_cross_entropy (holocron/nn/functional.py:150-191) is hb_poly_soft_fwd / _bwd with eps = 0. */
/* complement_cross_entropy: holocron/nn/functional.py:194-255. x [N, K, S], target int64 [N, S]; any ignore_index value
 * drops the row from the cross-entropy part, one inside [0, K) also drops that class from the complement term.
 * loss_pos: float[N*S] = w_y * ce + gamma * C; partials: double[3 * hb_loss_max_partials()] scratch;
 * fwd_out: float[3] = {sum, sum of w_y over the non-ignored rows, mean}. gamma = 0 gives the cross entropy alone. */
int hb_cce_fwd(const void* x, const long long* target, const float* weight, float* loss_pos, double* partials,
               float* fwd_out, int N, int K, int S, int ignore_index, float gamma, int dtype, void* stream);
/* reduction: 0 none (gout[N*S]), 1 mean, 2 sum (gout[1]); fwd_out from hb_cce_fwd; dx like x */
int hb_cce_bwd(const void* x, const long long* target, const float* weight, const float* gout, const float* fwd_out,
               void* dx, int N, int K, int S, int ignore_index, float gamma, int reduction, int dtype, void* stream);
/* mutual_channel_loss: holocron/nn/functional.py:258-319. x [N, cnum*xi, S], target int64 [N, S], weight float[cnum];
 * mask: uint8[cnum*xi] channel mask drawn by the caller. Outputs: row_lse float[N*cnum*xi] (spatial log-sum-exp of every
 * (sample, channel) row), loss_pos float[N*S], lse_d float[N*S] (log-sum-exp of the masked class maxima),
 * partials double[3 * hb_loss_max_partials()] scratch, fwd_out float[3] = {sum, sum of w_y over the non-ignored
 * positions, mean}. row_lse and lse_d are inputs of hb_mcl_bwd. */
int hb_mcl_fwd(const void* x, const long long* target, const float* weight, const unsigned char* mask, float* row_lse,
               float* loss_pos, float* lse_d, double* partials, float* fwd_out, int N, int cnum, int xi, int S,
               int ignore_index, float alpha, int dtype, void* stream);
/* rdot: float[N*cnum*xi] scratch. Fails with cudaErrorInvalidValue when xi > 376 (per-row sums in shared memory). */
int hb_mcl_bwd(const void* x, const long long* target, const float* weight, const unsigned char* mask,
               const float* row_lse, const float* lse_d, const float* gout, const float* fwd_out, float* rdot, void* dx,
               int N, int cnum, int xi, int S, int ignore_index, float alpha, int reduction, int dtype, void* stream);

/* ---- optimizers: holocron/optim/adabelief.py:121-167, lamb.py:79-137, tadam.py:160-212 ----------------- */
/* metas: device table of T records {p, g, m, v, vmax, aux, ext, numel} (8 x 8 bytes each, fp32 tensors);
 * chunks: device int2[num_chunks] = {tensor index, chunk index}, chunk = hb_optim_chunk_elems() elements. */
int hb_optim_chunk_elems(void);
/* ctl (may be NULL): device control block of a captured training step (see hb_train_ctl_* below): the kernels then read
 * lr (and beta1 when >= 0) from it and skip the whole update while its skip flag is set. */
int hb_adabelief_step(const void* metas, const void* chunks, int num_chunks, float lr, float beta1, float beta2,
                      float eps, float weight_decay, int amsgrad, int step, const int* step_dev, const void* ctl,
                      void* stream);
/* AdamP, holocron/optim/adamp.py:144-191 (the reference scripts' default optimizer, references/classification/train.py:340):
 * two launches per group (moments + per-tensor <p,g>, ||p||^2, ||g||^2, <p,pt>; then the projected update), 40 B/parameter.
 * scratch: double [4*T]. */
int hb_adamp_step(const void* metas, const void* chunks, int num_chunks, int T, float lr, float beta1, float beta2, float eps,
                  float weight_decay, int amsgrad, float delta, int step, const int* step_dev, const void* ctl,
                  double* scratch, void* stream);
int hb_lamb_step(const void* metas, const void* chunks, int num_chunks, int T, float lr, float beta1, float beta2,
                 float eps, float weight_decay, float clip_lo, float clip_hi, double* scratch, void* stream);
int hb_tadam_step(const void* metas, const void* chunks, int num_chunks, int T, float lr, float beta1, float beta2,
                  float eps, float weight_decay, int amsgrad, float dof, int step, const int* step_dev, double* scratch,
                  void* stream);
int hb_step_increment(int* step_dev, const void* ctl, void* stream);
/* The remaining optimizers of holocron/optim (SURVEY §8 f2), same tables:
 * Adan, adan.py:145-199 - aux = prev_grad (read, never written: reference quirk), ext = exp_avg_delta, vmax = its running max;
 *   one launch, 40 B/parameter. */
int hb_adan_step(const void* metas, const void* chunks, int num_chunks, float lr, float beta1, float beta2, float beta3,
                 float eps, float weight_decay, int amsgrad, int step, const int* step_dev, const void* ctl, void* stream);
/* AdEMAMix, ademamix.py:138-176 - ext = exp_avg_slow; one launch, 36 B/parameter. */
int hb_ademamix_step(const void* metas, const void* chunks, int num_chunks, float lr, float beta1, float beta2, float beta3,
                     float alpha, float eps, float weight_decay, int step, const int* step_dev, const void* ctl,
                     void* stream);
/* LARS, lars.py:91-135 - m = momentum_buffer (NULL without momentum); first != 0 when this step creates the buffers; with
 *   weight decay the gradients are overwritten by g + wd * p like the reference's in-place add_. scratch: double [2*T]. */
int hb_lars_step(const void* metas, const void* chunks, int num_chunks, int T, float lr, float momentum, float dampening,
                 float weight_decay, int nesterov, int first, double* scratch, void* stream);
/* RaLars, ralars.py:56-140 - mode 0 rectified update (x r_t), 1 plain Adam ratio, 2 unadapted momentum (chosen on the host
 *   from the SMA length); aux = local_lr (1 element, written). scratch: double [2*T]. */
int hb_ralars_step(const void* metas, const void* chunks, int num_chunks, int T, float lr, float beta1, float beta2, float eps,
                   float weight_decay, float clip_lo, float clip_hi, int mode, float r_t, int step, double* scratch,
                   void* stream);
/* Lookahead.sync_params, wrapper.py:122-135 - p = fast weights, m = slow weights: slow += rate * (fast - slow); fast = slow */
int hb_lookahead_sync(const void* metas, const void* chunks, int num_chunks, float sync_rate, void* stream);

/* ---- training-loop control on the device: holocron/trainer/core.py:135-227 (_fit_epoch: NaN-loss skipping :153-159,
 *      per-iteration scheduler.step() :161; _backprop_step: gradient accumulation, clip_grad_norm_, optimizer.step :184-208)
 *      and :262-269 (OneCycleLR / CosineAnnealingLR) without host synchronisation, CUDA-graph replayable -------------- */
/* ctl: device block of hb_train_ctl_bytes() bytes, zero-initialised by the caller, then [0] = lr, [1] = -1:
 *   f32 lr | f32 beta1 (<0: keep) | i32 skip | i32 bad | i32 iter | i32 nan_run | i32 opt_steps | f32 grad_norm */
int hb_train_ctl_bytes(void);
/* after a micro-batch: remember a non-finite *loss (device fp32 scalar) when skip_nan != 0 */
int hb_train_ctl_observe(void* ctl, const float* loss, int skip_nan, void* stream);
/* phase 0, before the optimizer update: lr / beta1 = table[min(iter, n-1)] (table: n x {lr, beta1} fp32 or NULL), skip =
 * bad, nan_run counts consecutive skipped updates; phase 1, after it: opt_steps += !skip, the window's bad flag is cleared */
int hb_train_ctl_step(void* ctl, const float* table, int n, int phase, void* stream);
/* once per iteration (the reference's scheduler.step()): iter += 1 */
int hb_train_ctl_tick(void* ctl, void* stream);
/* torch.nn.utils.clip_grad_norm_(params, max_norm) on a flat fp32 gradient buffer (core.py:194,205): fixed-order global L2
 * norm + in-place scaling by min(1, max_norm / (norm + 1e-6)), two launches; a NaN norm makes every gradient NaN, as in
 * torch. scratch: double [hb_grad_clip_partials_max()]; ctl (may be NULL) receives the norm. */
int hb_grad_clip_partials_max(void);
int hb_grad_clip_norm(float* grads, long long n, float max_norm, double* scratch, void* ctl, void* stream);

/* ---- transforms: holocron/transforms/interpolation.py:87-96 (Resize.forward: torchvision resize, then pad),
 *      :144-156 (RandomZoomOut.forward: resize, then constant pad) - a batch of images in one launch -------------- */
/* descs: device table of N rows of 16 int64 {src, dst, stride_c, stride_h, stride_w, C, H, W, h, w, top, left, Hc, Wc,
 * pad_mode, fill | mirror << 32}: pointers are addresses, strides count elements. Image n is read in place from the strided src [C][H][W], resampled
 * to h x w, placed with its top-left corner at the signed offset (top, left) of the contiguous canvas dst [C][Hc][Wc]
 * and the rest of the canvas filled by pad_mode (0 constant, 1 edge, 2 reflect: padding < side, 3 symmetric:
 * padding <= side); box pixels outside the canvas are dropped. The last word's low 32 bits are the constant fill as
 * fp32 bits (0: zero), cast to the image dtype as results are; a non-zero high half mirrors the canvas left-right
 * after placement (column x takes what column Wc - 1 - x takes unmirrored). filter: 0 nearest, 1 nearest-exact, 2 bilinear,
 * 3 bicubic (align_corners=False); antialias applies to 2 and 3. taps_y / taps_x: the most taps a row / column filter
 * of the batch has (1, 2 or 4 without antialias, 2*ceil(support)+1 with it). canvas_h / canvas_w: the largest canvas
 * of the batch. dtype: 0..2 as above, 3 = uint8, 4 = float64 (uint8 / fp16 / bf16 interpolate in fp32, float64 in
 * fp64; uint8 results are clamped to [0, 255] and rounded half to even). */
int hb_resample_batch(const void* descs, int N, int canvas_h, int canvas_w, int filter, int antialias, int taps_y,
                      int taps_x, int dtype, void* stream);
/* Crop boxes and horizontal flips (torchvision RandomResizedCrop, RandomHorizontalFlip) are hb_resample_batch rows: a
 * crop (i, j, h, w) points src at pixel (i, j) with H, W = h, w; a flip points src at the last column and negates
 * stride_w (resampled at its own size with the nearest filter, an exact copy). */

/* ---- random erasing: torchvision.transforms.RandomErasing (get_params: rectangle and values drawn on the host;
 *      forward: F.erase, img[..., i:i+h, j:j+w] = v on a clone or in place), as the reference's classification recipe
 *      applies it (references/classification/train.py:101-107) - a batch of images in one launch ----------------- */
/* descs: device table of N rows of 16 int64 {src, dst, stride_c, stride_h, stride_w, C, H, W, top, left, h, w, fill,
 * voff, 0, 0}: pointers are addresses, strides count elements. dst != src: dst is a contiguous [C][H][W] copy of the
 * strided src with the rectangle rows [top, top+h) x columns [left, left+w) filled; dst == src: only the rectangle is
 * written, in place through the source strides. fill: 0 none (nothing erased), 1 one value per channel at
 * values[voff + c], 2 one value per pixel at values[voff + (c*h + y)*w + x]. values: fp32, cast as torch's copy casts
 * (fp16 / bf16 round to nearest even, uint8 = (uint8_t)(int64_t)v, fp64 exact). rows: the most row segments an image
 * writes (C*H when copying, C*h in place); row_len: the longest segment (W when copying, w in place). dtype: as for
 * hb_resample_batch. */
int hb_erase_batch(const void* descs, const float* values, int N, int rows, int row_len, int dtype, void* stream);

/* ---- classification tail: torchvision's PILToTensor, ConvertImageDtype(torch.float32), Normalize and RandomErasing
 *      (rectangle and values drawn on the host), as the reference's classification recipe ends its chains
 *      (references/classification/train.py:100-107, 162-168) - a batch of images of one shape in one launch ------- */
/* descs: device table of N rows of 16 int64 {src, dst, stride_c, stride_h, stride_w, C, H, W, top, left, h, w, fill,
 * voff, 0, 0}, hb_erase_batch's rows in copy mode: image n is read from the strided src [C][H][W] (uint8 or fp32,
 * src_dtype 3 or 0) and written to the contiguous fp32 dst [C][H][W]. ops: the op program every element runs in order,
 * one op code per byte from the lowest, 0 ending it (at most 3 ops): 1 convert (v * f32(1/255), torch's uint8 to fp32
 * division by 255), 2 normalise ((v - values[noff + c]) / values[noff + C + c], rounded after each op as torch's sub_
 * and div_ round), 3 erase with the fill cast to uint8 ((uint8_t)(int64_t)v: the image is still uint8), 4 erase with
 * the fp32 fill. Erasing fills the row's rectangle as hb_erase_batch does (fill 0 none, 1 per channel at values[voff +
 * c], 2 per pixel at values[voff + (c*h + y)*w + x]). rows: C*H; row_len: W. No host synchronisation. */
int hb_image_tail_batch(const void* descs, const float* values, int N, int rows, int row_len, int src_dtype, int ops,
                        int noff, void* stream);

/* ---- TrivialAugmentWide: torchvision.transforms.TrivialAugmentWide.forward (op, magnitude and sign drawn on the
 *      host) and the torchvision.transforms.autoaugment._apply_op it calls on a uint8 tensor, as the reference's
 *      classification recipe applies it (references/classification/train.py:103) - a batch in at most two launches -- */
/* descs: device table of N rows of 16 int64 {src, dst, stride_c, stride_h, stride_w, C, H, W, op, stat, mask, fill,
 * bilinear, 0, 0, 0}: pointers are addresses, strides count elements (bytes). Image n is read in place from the
 * strided uint8 src [C][H][W] (C 1 or 3; every row of one call has the same C, H and W) and written to the contiguous
 * dst [C][H][W]. op: 0 Identity, 1 ShearX, 2 ShearY, 3 TranslateX, 4 TranslateY, 5 Rotate, 6 Brightness, 7 Color,
 * 8 Contrast, 9 Sharpness, 10 Posterize, 11 Solarize, 12 AutoContrast, 13 Equalize. stat: the image's index k in
 * stat_images for ops 8, 12 and 13, else -1. mask: the Posterize mask. fill: 1 when the affine ops fill out-of-image
 * pixels with params[n][9 + c], 0 for zeros. bilinear: 1 bilinear, 0 nearest. params: fp32 [N][16] {r, 1 - r,
 * solarize threshold, the 6 inverse affine matrix coefficients, 3 fill values, 0...}, r = 1 + magnitude formed in
 * double. stat_images: int64 [n_stat] image indices, in the order of their stat index. scratch: int32 [3 * n_stat]
 * [slices][256] histogram partials (not read when n_stat = 0). Arithmetic: torchvision's CUDA tensor path, in fp32. */
int hb_autoaugment_batch(const void* descs, const float* params, const long long* stat_images, int* scratch, int N,
                         int n_stat, int H, int W, int slices, void* stream);

/* ---- ColorJitter: torchvision.transforms.ColorJitter.forward (order and factors drawn on the host by get_params) on a
 *      uint8 or fp32 tensor, as the reference's segmentation and detection recipes apply it
 *      (references/segmentation/train.py:133-140, references/detection/train.py:116-125) - a batch in at most two
 *      launches -------------------------------------------------------------------------------------------------- */
/* descs: device table of N rows of 16 int64 {src, dst, stride_c, stride_h, stride_w, C, H, W, n_ops, op0, op1, op2,
 * op3, contrast_at, stat, 0}: pointers are addresses, strides count elements. Image n is read in place from the
 * strided src [C][H][W] (C 1 or 3; every row of one call has the same C, H and W) and written to the contiguous dst
 * [C][H][W]. op0..op(n_ops - 1): the ops in the order applied, 0 brightness, 1 contrast, 2 saturation, 3 hue (n_ops 0:
 * a copy); saturation and hue leave a one-channel image unchanged. contrast_at: the index of contrast among them (the
 * ops its mean sees come before it), or -1. stat: the image's index k in stat_images when it has a contrast op, else
 * -1. params: fp32 [N][8] {brightness r, 1 - r, contrast r, 1 - r, saturation r, 1 - r, hue factor, mean factor},
 * 1 - r formed in double; the contrast mean is the fp32 sum of the grayscale times the mean factor (torch's: f32(n) /
 * f32(n*H*W) for an image that is one of n leading indices of a tensor). stat_images: int64 [n_stat] image indices, in the order of their stat index. scratch: [n_stat][slices]
 * partial grayscale sums, int64 for uint8 and fp64 for fp32 (not read when n_stat = 0). dtype: 3 = uint8, 0 = fp32.
 * Arithmetic: torchvision's CUDA tensor path, in fp32. */
int hb_color_jitter_batch(const void* descs, const float* params, const long long* stat_images, void* scratch, int N,
                          int n_stat, int H, int W, int slices, int dtype, void* stream);

/* ---- detection transforms: the box steps of references/detection/transforms.py:58-127 (CenterCrop :58-69, Resize
 *      :72-82, RandomResizedCrop :85-105, convert_to_relative :108-116, RandomHorizontalFlip :119-127), as the
 *      reference's detection recipe chains them (references/detection/train.py:116-125) - every box of a batch in one
 *      launch ------------------------------------------------------------------------------------------------------ */
/* descs: device table of N rows of 8 int64 {boxes, labels, box_row_stride, label_stride, n, out_offset, 0, 0}: image
 * k's n boxes are read in place from the fp32 [n][4] boxes (unit column stride, rows box_row_stride elements apart)
 * and its int64 labels (label_stride elements apart). ops: int32 [n_ops], one op sequence for every image, each op
 * reading its operands from the image's row of params (fp32 [N][n_params]) in order: 0 scale (sx, sy), 1 clamp (x_lo,
 * x_hi, y_lo, y_hi), 2 subtract (dx, dy), 3 drop boxes with x1 == x2 or y1 == y2 (), 4 flip (flag, width): when flag
 * != 0, (x1, x2) = (width - x2, width - x1), 5 divide (dx, dy). Each op rounds to fp32 as a separate torch op does.
 * The survivors of image k are written in order to out_boxes fp32 [*][4] and out_labels int64 [*] (contiguous) from
 * row out_offset on, and counts[k] (int32) = their number. Nothing else is written. No atomics. */
int hb_box_transform_batch(const void* descs, const float* params, const int* ops, int n_ops, int n_params, int N,
                           float* out_boxes, long long* out_labels, int* counts, void* stream);

/* ---- detection evaluation: holocron/trainer/detection.py:17-32 (assign_iou), every image of a batch in one launch --
 * descs: device table of N rows of 16 int64 {gt, pred, gt_labels, pred_labels, n_gt, n_pred, gt_row_stride,
 * gt_col_stride, pred_row_stride, pred_col_stride, gt_label_stride, pred_label_stride, codes, out_offset, 0, 0}: image
 * k's [n_gt][4] ground-truth and [n_pred][4] predicted xyxy boxes are read in place through their strides (elements),
 * converted to fp32 as Tensor.float() converts them. codes holds one byte each, from the lowest: the gt and pred box
 * dtypes (0 fp32, 1 bf16, 2 fp16, 4 fp64), the gt and pred label types (0 int64, 1 int32). Labels (0 = not counted)
 * are read only for counts. Per image: the IoU of hb_box_pairwise mode 0, the first maximal prediction of each
 * ground-truth box (NaN wins, as in torch's max(dim=1)), kept when IoU >= iou_threshold; of the kept boxes claiming
 * one prediction, the one with the largest IoU (the lowest index on a tie) keeps it. match int64 [sum of n_gt]: from
 * out_offset on, the prediction paired with each ground-truth box, or -1. counts (int64 {assigned, correct}, or NULL)
 * is added to: the paired boxes, and those whose labels equal their prediction's. scratch: 8 bytes per ground-truth
 * box of the batch. One CTA per image; no host synchronisation. */
int hb_assign_iou_batch(const void* descs, int N, float iou_threshold, void* scratch, long long* match,
                        long long* counts, void* stream);

/* ---- YOLO inference post-processing (holocron/models/detection/yolo.py:159-233, yolov4.py:303-335) ------------------
 * One segment = one set of decoded candidates per image: boxes fp32 [B, M, 4] xyxy (16-byte aligned), objectness fp32
 * [B, M] and class scores fp32 [B, M, K], all contiguous, with its own thresholds (YOLOv1/v2: one segment; YOLOv4: one
 * per scale, suppressed independently and concatenated in segment order). Per image and segment: candidates with
 * objectness >= 0.5 and score = (first) max over classes * objectness >= score_thresh, boxes clamped to [0, 1], sorted
 * by score (descending, equal scores in candidate order), then non-maximum suppression at IoU > iou_thresh with
 * torchvision's arithmetic. Outputs, padded to cap = sum of M: out_boxes fp32 [B, cap, 4], out_scores fp32 [B, cap],
 * out_labels int64 [B, cap] (kept detections first, zeros after), counts int32 [B]. No host synchronisation, no atomics.
 * scratch: hb_detect_scratch_bytes(...) bytes, 256-byte aligned (0 = invalid table: nseg outside 1..4, B < 0, K < 1,
 * M outside 0..2^20, more than 65535 (image, segment) pairs or a cap over 2^31 - 1). */
typedef struct hb_detect_seg {
  const float* boxes;
  const float* obj;
  const float* cls;
  int M;
  float score_thresh;
  float iou_thresh;
} hb_detect_seg;
size_t hb_detect_scratch_bytes(const hb_detect_seg* segs, int nseg, int B, int K);
int hb_detect(const hb_detect_seg* segs, int nseg, int B, int K, void* scratch, float* out_boxes, float* out_scores,
              long long* out_labels, int* counts, void* stream);

/* ---- bookkeeping (not part of the reference surface) ------------------------------------------------ */
long long hb_launch_count(void);      /* kernels launched through this library since the last reset */
void hb_launch_count_reset(void);
const char* hb_version(void);

#ifdef __cplusplus
}
#endif
#endif /* HOLOCRON_B200_H */
