/* libgdrn_b200.so -- C ABI of the H100-native (sm_90a) GDR-Net hot path.
 *
 * Drop-in boundary (SURVEY.md 8b): the reference has no native code on this path -- every op below is
 * today an ATen / cuDNN / cuBLAS call issued by the `nn.Module`s cited per function.  The in-repo
 * precedent for a C-ABI extension is core/csrc/fps/src/ext.h:1-14 (raw pointers, caller-owned
 * buffers).  Conventions:
 *
 *   - every pointer is a DEVICE pointer owned by the caller (PyTorch allocates everything);
 *     kernels never allocate, no pointer is retained after return;
 *   - `stream` is a cudaStream_t passed as void* (torch.cuda.current_stream().cuda_stream);
 *   - return 0 on success, <0 on error (GDRN_ERR_ARG / GDRN_ERR_CUDA) with a thread-local message
 *     from gdrn_last_error(); nothing throws across the ABI; entry points are re-entrant;
 *   - activations are NHWC bf16 "planar pairs": a hi plane and an optional lo plane with
 *     value = hi + lo.  nsplit = 1: bf16 tensor-core math on the hi plane only (lo pointers NULL);
 *     nsplit = 3: fp32-faithful mode, three wgmma MMAs per k-step (hi*hi + hi*lo + lo*hi).
 */
#ifndef GDRN_B200_H
#define GDRN_B200_H

#ifdef __cplusplus
extern "C" {
#endif

#define GDRN_OK 0
#define GDRN_ERR_ARG (-1)
#define GDRN_ERR_CUDA (-2)

const char* gdrn_last_error(void);
long gdrn_launch_count(void); /* kernels launched by this library since load */
int gdrn_abi_version(void);
int gdrn_storage_format(void); /* 0: bf16 (hi, lo) planes; 1: fp16 planes, lo = fp16((x - hi) * gdrn_lo_scale()) */
float gdrn_lo_scale(void);
int gdrn_set_pdl(int on); /* A/B: programmatic dependent launch of the GEMM kernels (prologue under the predecessor's tail); default on, GDRN_PDL=0 disables */
int gdrn_last_gemm_variant(void); /* BLOCK_N*10 + nsplit of this thread's last conv/gemm forward launch */
int gdrn_last_gemm_block_m(void); /* tile height (128 or 256 rows) of the same launch */

/* ---- wgmma implicit-GEMM convolution, forward (and dgrad with flipped/transposed weights) ------------
 * replaces nn.Conv2d / nn.ConvTranspose2d forward: resnet_backbone.py:21-49,69-76 (torchvision BasicBlock),
 * cdpn_rot_head_region.py:82-135, conv_pnp_net.py:76-80.
 * x [N,H,W,Cin] (Cin % 64 == 0), w packed [Cout_pad][KH*KW*Cin] (gdrn_pack_weight), outputs row-major
 * [N*Ho*Wo][ldc]: bf16 planes (y_hi/y_lo) and/or fp32 (y_f32).  bias[Cout] / act (1 = LeakyReLU 0.1, 2 = ReLU) optional;
 * res_hi/res_lo: optional residual planes [N*Ho*Wo][ldc] added before the activation.  With BatchNorm folded into the
 * weights (gdrn_bn_fold_batched + row_scale of the pack jobs) and bias = the folded shift this is the eval-mode fused
 * conv + BN (+ identity) + ReLU of resnet_backbone.py:69-76 / torchvision BasicBlock / cdpn_rot_head_region.py:82-125.
 * stats (optional) [2][Cout] fp32 += per-channel sum and sum of squares of the fp32 accumulators
 * (BatchNorm batch statistics, reference get_norm("BN") layers).  With GDRN_ACT_STATS_F64 set in act, stats is double [2][Cout]
 * and each CTA's fp32 partial sums are added in double (the same applies to gdrn_gemm_fwd and gdrn_conv_dgrad_s2). */
#define GDRN_ACT_STATS_F64 16
int gdrn_conv_fwd(const void* x_hi, const void* x_lo, const void* w_hi, const void* w_lo, void* y_hi, void* y_lo,
                  float* y_f32, const float* bias, const void* res_hi, const void* res_lo, float* stats, int N, int H, int W,
                  int Cin, int Cout, int Cout_pad, int KH, int KW, int stride, int pad, int ldc, int act, int nsplit,
                  void* stream);

/* Data gradient of a stride-2 conv (k3 p1 / k1 p0 / k4 p1 / k2 p0; any other pair is GDRN_ERR_ARG) by output-parity phases over
 * the un-dilated dY: replaces the reference's cuDNN conv-backward-data for the stride-2 layers (resnet_backbone.py layerN.0.conv1 /
 * downsample, conv_pnp_net.py:76-80).  du [N][Ho][Wo][Cy], w = dgrad-packed weights (flipped taps), dx [N][2Ho][2Wo][ldc];
 * k1: dx must be pre-zeroed.  The same arithmetic is the FORWARD of the geometry head's nn.ConvTranspose2d(k, s2, p, op) --
 * k3 p1 op1, k4 p1 op0 or k2 p0 op0 (ROT_HEAD.CONV_KERNEL_SIZE, cdpn_rot_head_region.py:33-41, 81-91; its IOHW weight is the OIHW
 * weight of the transposed conv): bias / act / stats (optional) then apply to the output like gdrn_conv_fwd, in every phase. */
int gdrn_conv_dgrad_s2(const void* du_hi, const void* du_lo, const void* w_hi, const void* w_lo, void* dx_hi, void* dx_lo,
                       const float* bias, float* stats, int N, int Ho, int Wo, int Cy, int Cx, int Cx_pad, int K, int pad, int ldc,
                       int act, int nsplit, void* stream);

/* ---- plain GEMM  y[M][N] = a[M][K] * w[N_pad][K]^T (+bias, act); replaces nn.Linear (conv_pnp_net.py:89-92,
 * 152-156), the 7x7 stem over its im2col matrix (resnet_backbone.py:69) and their dgrads. */
int gdrn_gemm_fwd(const void* a_hi, const void* a_lo, const void* w_hi, const void* w_lo, void* y_hi, void* y_lo,
                  float* y_f32, const float* bias, float* stats, int M, int N, int N_pad, int K, int ldc, int act,
                  int nsplit, void* stream);

/* ---- class-aware output conv (ROT_HEAD.*_CLASS_AWARE; GDRN.py:134-151, cdpn_rot_head_region.py:114-135): grouped GEMMs.
 * gdrn_conv_fwd_grouped takes a 1x1 or a 3x3 stride-1 conv (OUT_CONV_KERNEL_SIZE; TMA zero fill supplies every crop's border).
 * w holds num_groups blocks of Cout_pad (N_pad) rows, [num_groups * Cout_pad][K]; bias num_groups blocks of bias_stride floats.
 * Output rows [g * rows_per_group, (g + 1) * rows_per_group) use block group[g] (device int array of M / rows_per_group entries,
 * clamped to [0, num_groups)); rows_per_group % 128 == 0, so no 128-row tile straddles two groups.  No residual, no statistics. */
int gdrn_conv_fwd_grouped(const void* x_hi, const void* x_lo, const void* w_hi, const void* w_lo, void* y_hi, void* y_lo,
                          float* y_f32, const float* bias, int N, int H, int W, int Cin, int Cout, int Cout_pad, int KH, int KW,
                          int stride, int pad, int ldc, int act, int nsplit, const int* group, int rows_per_group, int num_groups,
                          int bias_stride, void* stream);
int gdrn_gemm_fwd_grouped(const void* a_hi, const void* a_lo, const void* w_hi, const void* w_lo, void* y_hi, void* y_lo,
                          float* y_f32, const float* bias, int M, int N, int N_pad, int K, int ldc, int act, int nsplit,
                          const int* group, int rows_per_group, int num_groups, int bias_stride, void* stream);
/* dst[i][k] = src[idx[i]][k], 0 where idx[i] is outside [0, n_src): the per-step class-major weight / bias tables */
int gdrn_class_gather(const float* src, const int* idx, float* dst, int n_dst, int K, int n_src, void* stream);
/* out[b][c] = sum of rows [b * rows_per_crop, (b + 1) * rows_per_crop) of column c of a [B * rows_per_crop][ld] planar tensor,
 * in a fixed order (the per-crop bias partials of the class-aware output conv) */
int gdrn_crop_colsum(const void* x_hi, const void* x_lo, float* out, int B, int rows_per_crop, int ld, void* stream);
/* Weight and bias gradients of the class-aware output conv from per-crop partials: ws [B] blocks of ws_crop_stride floats holding
 * [n_slots][ws_ld] (gdrn_gemm_wgrad with ksplit = B), bias_part [B][bias_ld] (gdrn_crop_colsum).  For every reference row r < n_rows
 * grad_w[r][k] = sum over b in crop order of ws[b][slot_of[c_b][r]][k] (grad_b likewise), where c_b = classes[b] clamped to
 * [0, num_classes) and slot_of [num_classes][n_rows] is the logit slot of row r for class c or -1: rows no crop uses get 0. */
int gdrn_class_wgrad_reduce(const float* ws, long ws_crop_stride, int ws_ld, const float* bias_part, int bias_ld,
                            const int* classes, int B, const int* slot_of, int num_classes, int n_rows, int n_slots, int K,
                            float* grad_w, float* grad_b, void* stream);

/* ---- weight gradients (autograd wgrad of the layers above).  Split-K partials are written to the fp32
 * workspace ws [ksplit][ceil(Cout/128)*128][KH*KW*Cin]; reduce with gdrn_unpack_wgrad.
 * ws == NULL: size query only (*ws_need_out floats, *ksplit_out). ksplit <= 0: automatic. */
int gdrn_conv_wgrad(const void* dy_hi, const void* dy_lo, const void* x_hi, const void* x_lo, float* ws, long ws_floats,
                    long* ws_need_out, int* ksplit_out, int N, int H, int W, int Cin, int Cout, int KH, int KW,
                    int stride, int pad, int ksplit, int nsplit, void* stream);
int gdrn_gemm_wgrad(const void* dy_hi, const void* dy_lo, const void* x_hi, const void* x_lo, float* ws, long ws_floats,
                    long* ws_need_out, int* ksplit_out, long P, int M, int Ntot, int ksplit, int nsplit, void* stream);

/* ---- parameter layout conversion.  dst[o][tap*ipad + i] = src[o*so + i*si + r*sr + s*ss] (r,s flipped if flip).
 * Source layouts: Conv2d OIHW, ConvTranspose2d IOHW, Linear [out][in] (state_dict of the reference, SURVEY 8b). */
int gdrn_pack_weight(const float* src, void* dst_hi, void* dst_lo, int O, int I, int KH, int KW, int opad, int ipad,
                     int krow, long so, long si, long sr, long ss, int flip, void* stream);
/* all per-step re-packs in one launch; jobs_dev = device array of 104-byte PackJob records (csrc/pack.cu), each with an
 * optional per-output-row scale (eval-mode BatchNorm folding) */
int gdrn_pack_weight_batched(const void* jobs_dev, int njobs, long total_blocks, void* stream);
int gdrn_unpack_wgrad(const float* ws, float* grad, int O, int I, int KH, int KW, int ipad, int krow, int ksplit, long ks_stride,
                      long so, long si, long sr, long ss, int flip, int accumulate, void* stream);
/* im2col of the 7x7/2 stem: x NCHW fp32 [B,3,H,W] -> [B*H/2*W/2][192] bf16 planes, k = (r*7+s)*3 + c */
int gdrn_stem_im2col(const float* x, void* a_hi, void* a_lo, int B, int H, int W, void* stream);

/* ---- BatchNorm2d(eps, momentum) train/eval (+ReLU, + residual add) and backward -- detectron2/torch
 * BatchNorm2d via core/utils/layer_utils.py:17-39; torchvision BasicBlock residual. */
/* eval-mode folding of ALL BatchNorm layers in one launch: jobs = device array of 64-byte records {gamma, beta,
 * running_mean, running_var, scale_out, shift_out (pointers); int C; float eps; long pad} */
int gdrn_bn_fold_batched(const void* jobs_dev, int njobs, void* stream);
int gdrn_bn_finalize(const float* stats, const float* gamma, const float* beta, float* running_mean, float* running_var,
                     float* scale, float* shift, float* mean_out, float* invstd_out, int C, float count, float eps,
                     float momentum, int train, void* stream);
/* finalize + apply in one kernel (what the engine uses): batch statistics from the conv epilogue -> y, running stats.
 * relu_mask_out (optional, with relu): uint8 [rows*C/8], bit j of byte i = [pre-activation of element 8i+j > 0]; BatchNorm
 * backward (relu_mask) reads it instead of the activation to rebuild the ReLU mask (1/8 B instead of 2 B per element).
 * train = 3: stats is double [2][C] (a GEMM epilogue with GDRN_ACT_STATS_F64). */
int gdrn_bn_fwd(const void* x_hi, const void* x_lo, const void* r_hi, const void* r_lo, void* y_hi, void* y_lo,
                const float* stats, const float* gamma, const float* beta, float* running_mean, float* running_var,
                float* mean_out, float* invstd_out, void* relu_mask_out, long rows, int C, float eps, float momentum, int train,
                int relu, void* stream);
int gdrn_bn_act(const void* x_hi, const void* x_lo, const void* r_hi, const void* r_lo, void* y_hi, void* y_lo,
                const float* scale, const float* shift, long rows, int C, int relu, void* stream);
/* flags: bit 0 = the ReLU mask is recomputed from u (plain conv-BN-ReLU: pass y_hi = NULL and beta); bit 1 = `sums` is
 * already zero (the caller cleared all layers' accumulators in one memset); bit 2 = deterministic two-stage reductions */
int gdrn_bn_bwd(const void* ga_hi, const void* ga_lo, const void* gb_hi, const void* gb_lo, const void* y_hi,
                const void* u_hi, const void* u_lo, const float* mean, const float* invstd, const float* gamma,
                const float* beta, float* sums, void* du_hi, void* du_lo, void* gout_hi, void* gout_lo, float* dgamma,
                float* dbeta, const void* relu_mask, float* det_ws, long rows, int C, int train, int flags, void* stream);
/* deterministic mode (no atomics, fixed summation order; Engine.deterministic): gdrn_bn_stats computes the BatchNorm batch
 * statistics [2][C] (sum, sum of squares) from the tensor in two ordered stages instead of the GEMM epilogue's atomics;
 * gdrn_bn_bwd with flags bit 2 does the same for its reductions.  ws / det_ws: >= 2 * C * gdrn_det_parts() floats. */
int gdrn_det_parts(void);
int gdrn_bn_stats(const void* u_hi, const void* u_lo, float* ws, float* stats, long rows, int C, void* stream);

/* ---- MaxPool2d(3,2,1) resnet_backbone.py:72; UpsamplingBilinear2d(x2) cdpn_rot_head_region.py:102;
 * zero insertion (stride-2 transposed convs); GroupNorm(32)+ReLU conv_pnp_net.py:76-80 */
/* arg_out / arg_in: uint8 [B,H/2,W/2,C] window-local arg-max codes (first maximum, like ATen's saved indices) */
int gdrn_maxpool_fwd(const void* x_hi, const void* x_lo, void* y_hi, void* y_lo, void* arg_out, int B, int H, int W, int C,
                     void* stream);
int gdrn_maxpool_bwd(const void* arg_in, const void* g_hi, const void* g_lo, void* dx_hi, void* dx_lo, int B, int H, int W,
                     int C, void* stream);
int gdrn_upsample2x_fwd(const void* x_hi, const void* x_lo, void* y_hi, void* y_lo, int B, int H, int W, int C, void* stream);
int gdrn_upsample2x_bwd(const void* g_hi, const void* g_lo, void* dx_hi, void* dx_lo, int B, int H, int W, int C, void* stream);
int gdrn_zero_insert(const void* x_hi, const void* x_lo, void* y_hi, void* y_lo, int B, int H, int W, int C, int mode,
                     void* stream);
int gdrn_gn_relu_fwd(const void* u_hi, const void* u_lo, void* y_hi, void* y_lo, const float* gamma, const float* beta,
                     float* stats, int B, int HW, int C, int G, float eps, void* stream);
int gdrn_gn_relu_bwd(const void* g_hi, const void* g_lo, const void* y_hi, const void* u_hi, const void* u_lo,
                     const float* gamma, const float* stats, void* du_hi, void* du_lo, float* dgamma, float* dbeta, int B,
                     int HW, int C, int G, void* stream);
/* ---- GroupNorm(G, 256) + ReLU of the geometry head (ROT_HEAD.NORM = "GN", NUM_GN_GROUPS = G; cdpn_rot_head_region.py with
 * get_norm("GN")).  NHWC [B][HW][256] in 16-bit planes (lo = NULL: one plane), G | 256, G <= 64, HW in {256, 1024, 4096}.
 * Two-stage reductions in a fixed order, no atomics: bit-identical results run to run.
 * ws: gdrn_head_gn_workspace(B, HW) doubles (-1 for unsupported arguments).
 * fwd: stats [B][G][2] = (mean, invstd); y = relu(gamma (u - mean) invstd + beta); relu_mask_out (optional) [B*HW*32] bytes,
 *      bit j of byte i = y[8 i + j] > 0 (the gdrn_bn_fwd bitmap).
 * bwd: g is dL/dy, relu_mask the forward's bitmap; du = dL/du; dgamma / dbeta are written (not accumulated). */
long long gdrn_head_gn_workspace(int B, int HW);
int gdrn_head_gn_fwd(const void* u_hi, const void* u_lo, void* y_hi, void* y_lo, void* relu_mask_out, const float* gamma,
                     const float* beta, float* stats, double* ws, int B, int HW, int C, int G, float eps, void* stream);
int gdrn_head_gn_bwd(const void* g_hi, const void* g_lo, const void* u_hi, const void* u_lo, const void* relu_mask,
                     const float* gamma, const float* stats, void* du_hi, void* du_lo, float* dgamma, float* dbeta, double* ws,
                     int B, int HW, int C, int G, void* stream);
int gdrn_add2(const void* a_hi, const void* a_lo, const void* b_hi, const void* b_lo, void* o_hi, void* o_lo, long n,
              void* stream);
/* bias gradients (column sums of a [rows][ld] planar tensor) and LeakyReLU(0.1) backward (conv_pnp_net.py:93,152-153) */
int gdrn_colsum(const void* x_hi, const void* x_lo, float* out, long rows, int ld, void* stream);
int gdrn_leaky_bwd(const void* g_hi, const void* g_lo, const void* y_hi, void* o_hi, void* o_lo, long n, void* stream);
int gdrn_f32_to_planes(const float* x, void* y_hi, void* y_lo, long n, void* stream);
int gdrn_planes_to_f32(const void* x_hi, const void* x_lo, float* y, long n, void* stream);

/* ---- geometry glue + per-pixel losses (GDRN.py:156-169, 341-400; conv_pnp_net.py:120-125).
 * logits fp32 [B*HW][72] (0 mask | 1..3 xyz | 4 bg | 5..68 regions), Patch-PnP input bf16 [B*HW][128]:
 * with_2d = 1: xyz | coord2d | softmax64 (69 channels, PNP_NET.WITH_2D_COORD), 0: xyz | softmax64 (67 channels). */
int gdrn_head_glue_fwd(const float* logits, const float* coord2d, const float* extents, void* out_hi, void* out_lo, int B,
                       int HW, int with_2d, void* stream);
/* standalone ConvPnPNet.forward input (conv_pnp_net.py:111-125): NCHW fp32 coor_feat [B][c_feat][HW] (+ region
 * [B][c_reg][HW]) -> NHWC planes [B*HW][128]; xyz de-normalised by extents when c_feat is 3 or 5. */
int gdrn_pnp_pack_input(const float* coor_feat, int c_feat, const float* region, int c_reg, const float* extents,
                        void* out_hi, void* out_lo, int B, int HW, void* stream);
int gdrn_pixel_loss_fwd(const float* logits, const float* gt_xyz, const float* m_visib, const float* m_trunc,
                        const long long* labels, double* sums, int B, int HW, void* stream);
int gdrn_head_bwd(const float* logits, const float* gt_xyz, const float* m_visib, const float* m_trunc,
                  const long long* labels, const double* sums, const float* gw, const void* din_hi, const void* din_lo,
                  const float* extents, void* out_hi, void* out_lo, int B, int HW, int with_2d, void* stream);
/* The same with the mask head and the GT masks selectable (ROT_HEAD.MASK_LOSS_TYPE, XYZ_LOSS_MASK_GT, MASK_LOSS_GT,
 * REGION_LOSS_MASK_GT; GDRN.py:339-400).  mask_loss 0 = L1, 1 = BCE (BCEWithLogits mean), 2 = CE (2-class CrossEntropy mean,
 * label = (int) target); mask_out = mask logits per pixel, 1 for L1 / BCE and 2 for CE.  Logit row: mask [0, mask_out) | xyz |
 * bg | 64 regions, 68 + mask_out valid of 72.  m_xyz weights and normalises the xyz L1, m_mask is the mask-loss target,
 * m_region weights and normalises the region CE; they may be the same pointer.  sums double[7]: |dx|, |dy|, |dz|, mask loss,
 * region CE, sum(m_xyz), sum(m_region).  head_bwd_ex zeroes gradient columns 68 + mask_out .. 127.  The original four entry
 * points above are these with (mask_loss 0, mask_out 1, m_xyz = m_region = m_visib, m_mask = m_trunc) and six sums, slot 5
 * serving both normalisers. */
int gdrn_head_glue_fwd_ex(const float* logits, const float* coord2d, const float* extents, void* out_hi, void* out_lo, int B,
                          int HW, int with_2d, int mask_out, void* stream);
int gdrn_pixel_loss_fwd_ex(const float* logits, const float* gt_xyz, const float* m_xyz, const float* m_mask,
                           const float* m_region, const long long* labels, double* sums, int B, int HW, int mask_loss,
                           int mask_out, void* stream);
int gdrn_head_bwd_ex(const float* logits, const float* gt_xyz, const float* m_xyz, const float* m_mask, const float* m_region,
                     const long long* labels, const double* sums, const float* gw, const void* din_hi, const void* din_lo,
                     const float* extents, void* out_hi, void* out_lo, int B, int HW, int with_2d, int mask_loss, int mask_out,
                     void* stream);
/* The same for any region count (ROT_HEAD.NUM_REGIONS = num_regions, 2..64) with or without region attention
 * (PNP_NET.REGION_ATTENTION = region_att, 0 or 1).  A logit row is mask | xyz | bg | num_regions regions: N = mask_out + 4 +
 * num_regions of 72 floats valid, the rest never read.  The Patch-PnP input is xyz | coord2d (with_2d) | softmax over the
 * regions (region_att): nIn = 3 (+2) (+num_regions) channels in rows of pnp_ld = round_up(nIn, 64) = 64 or 128, the padding
 * zeroed; head_bwd_ex2 reads d(Patch-PnP input) in that layout (only xyz / coord2d without attention) and zeroes gradient
 * columns N .. 127.  The region CE runs over num_regions + 1 classes; a label above num_regions gives an unspecified loss.
 * pixel_loss_fwd_ex2 checks region_att and pnp_ld but does not depend on them; head_bwd_ex2 with 64 regions and attention is
 * head_bwd_ex.  gdrn_pnp_pack_input_ex is
 * gdrn_pnp_pack_input into rows of pnp_ld = round_up(c_feat + c_reg, 64). */
int gdrn_head_glue_fwd_ex2(const float* logits, const float* coord2d, const float* extents, void* out_hi, void* out_lo, int B,
                           int HW, int with_2d, int mask_out, int num_regions, int region_att, int pnp_ld, void* stream);
int gdrn_pixel_loss_fwd_ex2(const float* logits, const float* gt_xyz, const float* m_xyz, const float* m_mask,
                            const float* m_region, const long long* labels, double* sums, int B, int HW, int mask_loss,
                            int mask_out, int num_regions, int region_att, int pnp_ld, void* stream);
int gdrn_head_bwd_ex2(const float* logits, const float* gt_xyz, const float* m_xyz, const float* m_mask, const float* m_region,
                      const long long* labels, const double* sums, const float* gw, const void* din_hi, const void* din_lo,
                      const float* extents, void* out_hi, void* out_lo, int B, int HW, int with_2d, int mask_loss, int mask_out,
                      int num_regions, int region_att, int pnp_ld, void* stream);
int gdrn_pnp_pack_input_ex(const float* coor_feat, int c_feat, const float* region, int c_reg, const float* extents,
                           void* out_hi, void* out_lo, int B, int HW, int pnp_ld, void* stream);

/* ---- DropBlock on the Patch-PnP input (PNP_NET.PNP_HEAD_CFG.drop_prob / dropblock_size; conv_pnp_net.py:66-72,128-142,
 * core/utils/dropblock).  *step (device int64) is the LinearScheduler counter k: the step's probability is
 * np.linspace(0, drop_prob, 5000)[min(k, 4999)], computed on the device in float64, and every call adds 1 to *step.
 * train = 1 also samples the block mask of B crops of H x W pixels (H, W <= 64): seeds[B][H][W] = (uniform < float32(p /
 * block_size^2)) from Philox4x32-10 with key (seed, rank) and counter (pixel quad, crop, k); keep[B][H][W] = 1 - max_pool2d(seeds,
 * block_size, stride 1, padding block_size / 2) (even sizes crop the last row and column); counts[B] the per-crop kept
 * pixels; scale[0] = B H W / sum(counts).  train = 0 only advances *step (keep, seeds, counts, scale may be NULL).
 * drop_prob outside [0, 1], block_size outside 1..15 or H, W outside 1..64 give GDRN_ERR_ARG. */
int gdrn_dropblock_step(long long* step, long long seed, int rank, double drop_prob, int block_size, int train,
                        unsigned char* keep, unsigned char* seeds, int* counts, float* scale, int B, int H, int W, void* stream);
/* gdrn_head_glue_fwd_ex2, gdrn_head_bwd_ex2 and gdrn_pnp_pack_input_ex with DropBlock: each valid Patch-PnP input channel of
 * pixel p is multiplied by keep[p] * scale[0] in fp32 before the 16-bit split (forward), and each d(Patch-PnP input) row by
 * the same factor before its use (backward).  head_bwd_db runs its own kernels for every region setting, 64 regions with
 * attention included. */
int gdrn_head_glue_fwd_db(const float* logits, const float* coord2d, const float* extents, void* out_hi, void* out_lo, int B,
                          int HW, int with_2d, int mask_out, int num_regions, int region_att, int pnp_ld,
                          const unsigned char* keep, const float* scale, void* stream);
int gdrn_head_bwd_db(const float* logits, const float* gt_xyz, const float* m_xyz, const float* m_mask, const float* m_region,
                     const long long* labels, const double* sums, const float* gw, const void* din_hi, const void* din_lo,
                     const float* extents, void* out_hi, void* out_lo, int B, int HW, int with_2d, int mask_loss, int mask_out,
                     int num_regions, int region_att, int pnp_ld, const unsigned char* keep, const float* scale, void* stream);
int gdrn_pnp_pack_input_db(const float* coor_feat, int c_feat, const float* region, int c_reg, const float* extents,
                           void* out_hi, void* out_lo, int B, int HW, int pnp_ld, const unsigned char* keep, const float* scale,
                           void* stream);

/* ---- rot6d -> R, SITE translation, allo -> ego, PM loss (+ closest symmetric GT), centroid / z losses, re/te
 * (rot_reps.py:34-49, pose_from_pred_centroid_z.py:144-227, utils.py:208-236, pm_loss.py:82-114,
 *  pose_utils.py:430-482, GDRN.py:439-471, model_utils.py:40-52).  pred [B][ld_pred]: cols 0..5 rot6d, 6..8 t.
 * syms: device-resident table of symmetry rotations [rows][3][3] (built once per object set), sym_idx [B][2] = (first row,
 * count) per crop, count 0 = asymmetric; both NULL without PM_LOSS_SYM.  The K candidates are scanned by the whole CTA. */
int gdrn_pose_loss(const float* pred, int ld_pred, const float* cams, const float* centers, const float* whs,
                   const float* ratios, const float* extents, const float* points, const float* gt_rot,
                   const float* gt_trans, const float* gt_ratio, const float* syms, const int* sym_idx, const float* gw,
                   float* out_rot, float* out_trans, double* sums, float* vis, void* dy_hi, void* dy_lo, int B, int n_pts,
                   int do_loss, float eps, void* stream);
int gdrn_loss_finalize(const double* pix_sums, const double* pose_sums, const float* vis, float* losses, float* vis_out,
                       int B, int HW, int n_pts, void* stream);
/* pix_sums of gdrn_pixel_loss_fwd_ex (7 slots): the region loss is normalised by slot 6 */
int gdrn_loss_finalize_ex(const double* pix_sums, const double* pose_sums, const float* vis, float* losses, float* vis_out,
                          int B, int HW, int n_pts, void* stream);

/* ---- the PNP_NET pose-loss switches (GDRN.py:402-514, pm_loss.py:58-171, rot_loss.py:30-48, l2_loss.py), passed by value.
 * Loss kinds: 0 L1, 1 Smooth-L1 (PM only, fvcore: plain L1 for beta < 1e-5), 2 MSE, 3 L2 (per-crop norm, mean over B).
 * pm_mode: -1 no PM loss (PM_LW = 0), 0 R only, 1 R and t together (loss_PM_RT), 2 DISENTANGLE_T with points (PM_R, PM_T),
 * 3 DISENTANGLE_Z with points (PM_R, PM_xy, PM_z), 4 DISENTANGLE_T without points (PM_R, PM_T_noP), 5 DISENTANGLE_Z without
 * points (PM_R, PM_xy_noP, PM_z_noP).  rot_type: -1 off, 0 angular, 1 L2.  trans_type, bind_type: -1 off, else L1 / MSE / L2.
 * The default (pm_mode 0, L1, norm by extent, centroid and z L1, the rest off) is what gdrn_pose_loss computes. */
typedef struct {
    int pm_mode, pm_type;
    float pm_beta;
    int pm_norm_extent, rot_type, centroid_type, z_type, trans_type, trans_disentangle, bind_type;
} gdrn_pose_switches;
#define GDRN_POSE_SLOTS 11 /* per-crop partial sums: PM R|RT, PM T|xy, PM z, PM T_noP|xy_noP, PM z_noP, rot, centroid, z,
                              trans xy|LPnP, trans z, bind; the active ones, in this order, are the reference's loss_dict order */
/* gdrn_pose_loss with the switches: part [B][GDRN_POSE_SLOTS] per-crop partial sums (inactive slots unwritten); gw: the upstream
 * gradients of the ACTIVE pose losses in slot order; dy as gdrn_pose_loss. */
int gdrn_pose_loss_ex(const float* pred, int ld_pred, const float* cams, const float* centers, const float* whs,
                      const float* ratios, const float* extents, const float* points, const float* gt_rot,
                      const float* gt_trans, const float* gt_ratio, const float* syms, const int* sym_idx, const float* gw,
                      float* out_rot, float* out_trans, float* part, float* vis, void* dy_hi, void* dy_lo, int B, int n_pts,
                      gdrn_pose_switches sw, void* stream);
/* losses[5 + n_pose] = the five pixel losses (as gdrn_loss_finalize_ex) then the active pose losses in slot order, each the
 * crop-ordered sum of its partials (deterministic); n_pose = gdrn_pose_loss_count(sw) */
int gdrn_loss_finalize_ex2(const double* pix_sums, const float* part, const float* vis, float* losses, float* vis_out, int B,
                           int HW, int n_pts, gdrn_pose_switches sw, void* stream);
int gdrn_pose_loss_count(gdrn_pose_switches sw);

/* ---- per-instance crop / target generation of the data loader on the device (core/gdrn_modeling/data_loader.py:487-560,
 * core/utils/data_utils.py:80-137 crop_resize_by_warp_affine, :213-219 xyz_to_region), cv2.warpAffine's fixed-point sampling
 * restated.  image_u8 [B][H][W][3] (BGR uint8), centers [B][2], scales [B] (float64 like the reference's aug_bbox output) -> roi_img [B][3][R][R] = bilinear crop / pixel_std.
 * xyz [B][H][W][3] (object coordinates, 0 = background), mask_visib / mask_trunc [B][H][W] (mask_trunc may be NULL),
 * extents [B][3], fps_points [B][n_fps][3] -> roi_xyz [B][3][R][R] (normalised), roi_mask_{trunc,visib,obj} [B][R][R],
 * roi_region [B][R][R] int64 (0 = background), roi_coord_2d [B][2][R][R]. */
int gdrn_roi_crop_image(const void* image_u8, const double* centers, const double* scales, float* roi_img, int B, int H, int W,
                        int out_res, float pixel_std, void* stream);
int gdrn_roi_targets(const float* xyz, const float* mask_visib, const float* mask_trunc, const double* centers, const double* scales,
                     const float* extents, const float* fps_points, int n_fps, float* roi_xyz, float* roi_mask_trunc,
                     float* roi_mask_visib, float* roi_mask_obj, long long* roi_region, float* roi_coord_2d, int B, int H, int W,
                     int out_res, void* stream);

/* ---- evaluator metrics on the device (lib/pysixd/pose_error.py:297-337 add / adi, :400-436 re / te; the reference computes
 * them per instance in numpy with a scipy KD-tree, gdrn_evaluator.py:316-436).  R_* [B][3][3], t_* [B][3], points [B][n_pts][3]
 * (model points per instance, metres) -> out [B][4] = (ADD, ADD-S = ADI or 0 when !want_adi, re in degrees, te). */
int gdrn_pose_errors(const float* R_est, const float* t_est, const float* R_gt, const float* t_gt, const float* points, int B,
                     int n_pts, int want_adi, float* out, void* stream);

/* ---- test-time RANSAC-PnP of the evaluator on the device (core/gdrn_modeling/gdrn_evaluator.py:316-436 `process_pnp_ransac`:
 * `get_img_model_points_with_coords2d` :89-126 + lib/pysixd/misc.py:145-194 `pnp_v2` = cv2.solvePnPRansac(EPNP, reprojErr 3, 100
 * iterations) per instance on the host).  mask [B][H*W] (mask_mode 0: used as is, 1: per-ROI min-max normalised like
 * engine_utils.py:113-118 for the L1 mask head, 2: sigmoid) or [B][2][H*W] (mask_mode 3, the CE mask head: argmax over the two
 * channels, a tie giving 0, engine_utils.py:123-124), compared with mask_thr; xyz [B][3][H*W] in [0,1], coord2d [B][2][H*W] in [0,1],
 * extents [B][3], im_wh [B][2] = (im_W, im_H), K [B][3][3].  out_pose [B][3][4] = [R | t]; out_info [B][4] = (selected points,
 * inliers, RANSAC iterations run, ok); out_inliers (optional) [B][H*W] flags indexed like cv2's inlier list (position in the
 * row-major list of selected points).  Follows OpenCV's algorithm (RNG-driven 5-point subsets, EPnP minimal + final solver,
 * adaptive iteration count): same inlier sets / poses as cv2 up to round-off. */
long gdrn_pnp_ransac_workspace_bytes(int B, int HW, int iters);
int gdrn_pnp_ransac(const float* mask, const float* xyz, const float* coord2d, const float* extents, const float* im_wh,
                    const float* K, int B, int H, int W, int mask_mode, float mask_thr, double reproj_err, int iters,
                    double confidence, void* workspace, long workspace_bytes, float* out_pose, int* out_info,
                    unsigned char* out_inliers, void* stream);

/* ---- network-initialised iterative PnP of the evaluator (TEST.PNP_TYPE net_iter_pnp, gdrn_evaluator.py:187-314
 * `process_net_and_pnp`: cv2.solvePnP(SOLVEPNP_ITERATIVE, useExtrinsicGuess=True) started at the network pose, per instance on
 * the host).  Inputs as gdrn_pnp_ransac, plus R_init [B][3][3] / t_init [B][3] = the network pose.  OpenCV's Levenberg-Marquardt
 * (cvFindExtrinsicCameraParams2 + CvLevMarq, at most max_iters accepted steps, 20 in OpenCV) in fp64, one CTA per instance:
 * the same minimiser and iteration count as cv2.  The solution is rounded to float32 before R is formed, as the reference's
 * float32 guess arrays do.  out_pose [B][3][4] = [R | t]; out_info [B][4] = (selected points, iterations, ok, 0); fewer than 4
 * points: ok = 0 and out_pose = the initial pose. */
long gdrn_pnp_iterative_workspace_bytes(int B, int HW);
int gdrn_pnp_iterative(const float* mask, const float* xyz, const float* coord2d, const float* extents, const float* im_wh,
                       const float* K, const float* R_init, const float* t_init, int B, int H, int W, int mask_mode, float mask_thr,
                       int max_iters, void* workspace, long workspace_bytes, float* out_pose, int* out_info, void* stream);

/* ---- fused Ranger step (gradient centralisation + RAdam + Lookahead), lib/torch_utils/solver/ranger.py:100-200, for all
 * tensors of a param group in ONE launch.  jobs: device array of 64-byte records {float* p; const float* g; float* m; float* v;
 * float* slow; long numel; int row_len; int pad[3]} (row_len > 0: centralise rows of that length);
 * blocks: device array of {int job; int count; long begin} (rows or elements per CTA).  The scalar RAdam rectification
 * (step_lr = step_size * lr, adaptive = N_sma > threshold) is computed by the host; wd_lr = weight_decay * lr;
 * grad_scale multiplies every gradient (1/loss-scale). */
int gdrn_ranger_step(const void* jobs_dev, const void* blocks_dev, int nblocks, float step_lr, float wd_lr, float beta1,
                     float beta2, float eps, float alpha, float grad_scale, int adaptive, int lookahead, void* stream);
/* x[i] *= s over an fp32 buffer (loss-scale removal from a slice of the flat gradient buffer) */
int gdrn_scale_f32(float* x, long n, float s, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GDRN_B200_H */
