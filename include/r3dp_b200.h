/*
 * r3dp_b200.h — C ABI of libr3dp_b200.so: the H100 (sm_90a) implementation of Real3D-Portrait's per-frame
 * volumetric render + super-resolution hot path.
 *
 * The reference has no C ABI for this path: its boundary is Python `torch.nn.Module.forward` signatures
 * (SURVEY.md §8b).  The host-side mirror of those signatures lives in `real3dportrait_b200/*.py` and binds THIS
 * header through ctypes; each entry point below names the reference interface it stands behind (paths relative
 * to the reference tree).  Conventions:
 *   - every pointer is a DEVICE pointer on the current CUDA device unless the name ends in `_host`;
 *   - tensors are dense row-major fp32 unless stated; shapes are given in brackets;
 *   - `stream` is a cudaStream_t (0 = legacy default stream); all work is enqueued asynchronously on it and
 *     nothing synchronises the device;
 *   - return value 0 = success, non-zero = error; `r3dp_last_error()` returns a thread-local message
 *     (the Python mirror raises RuntimeError with it, like the reference's TORCH_CHECK in bias_act.cpp:39-55);
 *   - inputs are never written; outputs / workspaces must not alias inputs.
 * There is no CPU fallback anywhere behind this ABI.
 */
#ifndef R3DP_B200_H
#define R3DP_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define R3DP_ABI_VERSION 3

typedef void* r3dp_stream_t; /* cudaStream_t */

/* OSGDecoder parameters (modules/img2plane/triplane.py:122-146; FullyConnectedLayer networks_stylegan2.py:99-131).
 * Raw (unscaled) state_dict tensors; the 1/sqrt(fan_in) weight gains are applied by the library. */
typedef struct r3dp_mlp {
    const float* w1; /* net.0.weight [hidden, in_features]      */
    const float* b1; /* net.0.bias   [hidden]                   */
    const float* w2; /* net.2.weight [1 + out_dim, hidden]      */
    const float* b2; /* net.2.bias   [1 + out_dim]              */
    int in_features; /* 32 */
    int hidden;      /* 64 */
    int out_dim;     /* 32 (colour channels; +1 density)        */
} r3dp_mlp_t;

int         r3dp_abi_version(void);
const char* r3dp_last_error(void);
/* SM count and compute capability of the current device; fails unless it is sm_90. */
int r3dp_device_info(int* sm_count, int* cc_major, int* cc_minor);
/* Running total of CUDA kernels this library has launched in the process (bench.py's `gpu_launches`). */
unsigned long long r3dp_launch_count(void);
/* Frame exchange of a sharded clip (inference/real3d_infer.py:515-521 collects the frames of a clip on one device): copy-engine peer copy of
 * `bytes` from `src` on device `src_device` to `dst` on device `dst_device` (e.g. a CUDA-IPC mapping of rank 0's clip buffer), enqueued on
 * `stream` (a stream of the CALLING device); no SM is used and nothing is synchronised. */
int r3dp_peer_copy(void* dst, int dst_device, const void* src, int src_device, size_t bytes, r3dp_stream_t stream);

/* ---------------------------------------------------------------------------------------------------- rays ---
 * RaySampler.forward (modules/eg3ds/volumetric_rendering/ray_sampler.py:24-63).
 * cam2world [N,4,4], intrinsics [N,3,3]  ->  ray_o [N,res*res,3], ray_d [N,res*res,3]; ray m = row*res + col. */
int r3dp_gen_rays(const float* cam2world, const float* intrinsics, int N, int res, float* ray_o, float* ray_d,
                  r3dp_stream_t stream);

/* -------------------------------------------------------------------------------------------------- planes ---
 * Layout change done once per frame before sampling: reference tri-planes are [N,3,C,H,W]
 * (secc_img2plane.py:105-110); the gather kernels read channels-last [N,3,H,W,C] so one bilinear tap is one
 * 128-byte line.  C must be 32. */
int r3dp_planes_to_channels_last(const float* planes_nchw, int N, int C, int H, int W, float* planes_cl,
                                 r3dp_stream_t stream);

/* Tri-grids (`triplane_feature_type: trigrid | trigrid_v2`): grids_nchw [N,3,C*D,H,W] with channel index c*D + d (the reference views
 * it as [N*3,C,D,H,W], renderer.py:83) -> grids_cl [N,3,D,H,W,C]: every depth slice a channels-last plane.  D = 1 is the call above. */
int r3dp_grids_to_channels_last(const float* grids_nchw, int N, int C, int D, int H, int W, float* grids_cl, r3dp_stream_t stream);
/* sample_from_trigrids (renderer.py:78-89): grids_cl [N,3,D,H,W,C], coords [N,P,3] -> out [N,3,P,C]; trilinear, zero padding,
 * align_corners=False; plane p is sampled at (x,y,z), (x,z,y), (z,x,y) x 2/box_warp.  D >= 2. */
int r3dp_trigrid_sample(const float* grids_cl, int N, int C, int D, int H, int W, const float* coords, int P, float box_warp,
                        float* out, r3dp_stream_t stream);
/* r3dp_run_model for tri-grids [N,3,D,H,W,C] (D = 1: tri-planes). */
int r3dp_run_model_grid(const float* planes_cl, int N, int C, int D, int H, int W, const float* coords, int P, float box_warp,
                        const r3dp_mlp_t* mlp, float* rgb, float* sigma, r3dp_stream_t stream);

/* sample_from_planes (renderer.py:65-75): planes_cl [N,3,H,W,C], coords [N,P,3] -> out [N,3,P,C]
 * (bilinear, zero padding, align_corners=False, coords scaled by 2/box_warp; plane axes of generate_planes()). */
int r3dp_triplane_sample(const float* planes_cl, int N, int C, int H, int W, const float* coords, int P,
                         float box_warp, float* out, r3dp_stream_t stream);

/* ImportanceRenderer.run_model (renderer.py:169-188) with an OSGDecoder: gather + mean over planes + MLP.
 * -> rgb [N,P,out_dim], sigma [N,P,1]. */
int r3dp_run_model(const float* planes_cl, int N, int C, int H, int W, const float* coords, int P, float box_warp,
                   const r3dp_mlp_t* mlp, float* rgb, float* sigma, r3dp_stream_t stream);

/* OSGDecoder.forward (modules/img2plane/triplane.py:133-146) on caller-supplied features:
 * feat [N,K,P,C], K = 3 (mean over the planes) or K = 1 (already aggregated) -> rgb [N,P,out_dim], sigma [N,P,1]. */
int r3dp_decode(const float* feat, int N, int K, int P, int C, const r3dp_mlp_t* mlp, float* rgb, float* sigma,
                r3dp_stream_t stream);

/* -------------------------------------------------------------------------------------------------- render ---
 * ImportanceRenderer.forward with ray_start = ray_end = 'auto' (renderer.py:118-167), fused: box limits
 * (math_utils.py:46-98) -> stratified depths (renderer.py:209-232) -> tri-plane gather -> OSGDecoder ->
 * MipRayMarcher2 (ray_marcher.py:25-57) [-> importance resampling (renderer.py:234-297) -> second gather/MLP ->
 * depth merge (renderer.py:197-207) -> final march].
 *   ray_o, ray_d [N,M,3]          rays; if ray_o == NULL they are generated in-kernel from `camera` [N,25]
 *                                 (row-major c2w then row-major K, secc_img2plane.py:95-96) with M = res*res
 *   u_coarse [N,M,S]              the uniforms the reference draws with torch.rand_like (renderer.py:226)
 *   u_fine   [N*M,S_imp] or NULL  the uniforms of torch.rand (renderer.py:281); required when S_imp > 0
 *   res                           image side if the M rays form a res x res image (enables 2-D ray tiles), else 0
 * outputs: rgb [N,M,out_dim] (already scaled to [-1,1]), depth [N,M,1], weights_sum [N,M,1], is_ray_valid [N,M]
 * (uint8 0/1).  Batch-global quirks are reproduced per call: invalid rays inherit min/max of the valid ray starts
 * (renderer.py:123-126) and depth is clamped to the call-wide [min,max] sample depth (ray_marcher.py:50).
 * workspace: r3dp_render_workspace_bytes(N, M) bytes of scratch.
 * Kernels, chosen from the arguments alone: single-pass renders (S_imp == 0) run the warp-specialised streaming kernel (render_stream.cu:
 * gather, wgmma decoder and ray march of consecutive 128-sample tiles overlap inside one persistent CTA per SM); importance renders
 * (S_imp > 0) run the CTA-per-ray-tile kernel (render.cu), with the wgmma decoder when each pass of a tile fits two 128-sample tiles
 * and the fp32 CUDA-core decoder otherwise.  The wgmma decoder splits every fp32 operand into two fp16 halves (three partial products,
 * fp32 accumulation in registers) - fp32-grade results (rgb within 5e-6 of float64, tests/test_gpu_render_conformance.py).  The prepared
 * decoder operands live in the caller's `workspace`, so calls with different decoders may run concurrently on different streams (each
 * with its own workspace). */
size_t r3dp_render_workspace_bytes(int N, int M);

/* Channels-last plane addressing, strides in floats: the C = 32 features of texel (plane p, row y, col x) of frame n start at
 *   planes + n*frame_stride + p*plane_stride + y*row_stride + x*texel_stride      (every stride a multiple of 4 floats).
 *   [N,3,H,W,C] (r3dp_planes_to_channels_last)                      plane = H*W*C, row = W*C,   texel = C
 *   [N,H,W,3,C] = the producer's [N,3*C,H,W] conv output held in torch.channels_last memory (secc_img2plane.py:73-81,
 *                 segformer.py:704-733 emit [B,3,C,H,W] views of such a tensor): plane = C, row = W*3*C, texel = 3*C  -> no repack at all
 *   frame_stride = 0: one plane set shared by every frame of the call (the per-clip canonical planes). */
typedef struct r3dp_plane_layout {
    long long frame_stride;
    int plane_stride, row_stride, texel_stride;
    /* tri-grids (`triplane_feature_type: trigrid | trigrid_v2`, sample_from_trigrids, renderer.py:78-89; egs/os_avatar/img2plane.yaml:65-66):
     * every plane is a stack of `depth` >= 2 slices `slice_stride` floats apart, sampled trilinearly with the third projected coordinate
     * (z, y, y for planes 0, 1, 2); depth <= 1: plain tri-planes.  [N,3,D,H,W,C] (r3dp_grids_to_channels_last): slice = H*W*C. */
    int depth, slice_stride;
} r3dp_plane_layout_t;

/* The render's arguments: explicit plane layouts and an optional SECOND plane set sampled at the same points and added to the first
 * (bilinear sampling is linear): `planes = cano_planes + secc_planes` (secc_img2plane.py:73-81) without the 75 MB/frame add. */
typedef struct r3dp_render_args {
    const float* planes;  r3dp_plane_layout_t layout;
    const float* planes2; r3dp_plane_layout_t layout2;   /* NULL = none; strides (except frame_stride) must equal `layout`'s */
    int N, C, H, W;
    const float* ray_o; const float* ray_d; const float* camera; int M, res;
    int S, S_imp; float box_warp; int white_back;
    const float* u_coarse; const float* u_fine;
    const r3dp_mlp_t* mlp;
    float* rgb; float* depth; float* weights_sum; uint8_t* is_ray_valid;
    void* workspace; size_t workspace_bytes;
} r3dp_render_args_t;
int r3dp_render_ex(const r3dp_render_args_t* args, r3dp_stream_t stream);
/* The kernel r3dp_render_ex runs for `args`: 0 = streaming kernel, 1 = CTA-per-ray-tile kernel with the tensor-core decoder,
 * 2 = CTA-per-ray-tile kernel with the CUDA-core decoder; -1 if `args` or its decoder is NULL.  Launches nothing. */
int r3dp_render_path(const r3dp_render_args_t* args);

/* MipRayMarcher2.run_forward (ray_marcher.py:25-57) stand-alone: colors [N,M,S,C], sigmas [N,M,S,1],
 * depths [N,M,S,1] -> rgb [N,M,C], depth [N,M,1], weights [N,M,S-1,1].  workspace: 16 bytes. */
int r3dp_ray_march(const float* colors, const float* sigmas, const float* depths, int N, int M, int S, int C,
                   int white_back, float* rgb, float* depth, float* weights, void* workspace,
                   r3dp_stream_t stream);

/* ------------------------------------------------------------------------------------- super-resolution ---
 * Building blocks of SuperresolutionHybrid8XDC.forward (modules/eg3ds/models/superresolution.py:331-359) with
 * noise_mode='none', fp32 parameters.  Activations are NCHW fp32 at the boundary.
 *
 * r3dp_sr_styles: FullyConnectedLayer(w_dim, Cin, bias_init=1) (networks_stylegan2.py:113-127,314):
 *   styles[N,Cin] = w_lat[N,w_dim] @ (A[Cin,w_dim]/sqrt(w_dim))^T + a[Cin], then * post_scale
 *   (post_scale = 1/sqrt(Cin) for ToRGB, networks_stylegan2.py:362,366).
 * r3dp_sr_fold_weights: the per-sample weights of modulated_conv2d (networks_stylegan2.py:63-70):
 *   wf[N,O,I,k,k] = W[O,I,k,k] * styles[N,I]  (* rsqrt(sum_{I,k,k} (.)^2 + 1e-8) if demodulate). */
int r3dp_sr_styles(const float* w_lat, const float* affine_w, const float* affine_b, int N, int w_dim, int Cin,
                   float post_scale, float* styles, r3dp_stream_t stream);
int r3dp_sr_fold_weights(const float* weight, const float* styles, int N, int O, int I, int k, int demodulate,
                         float* wf, r3dp_stream_t stream);

/* F.interpolate(size, bilinear, align_corners=False, antialias=True) for UP-scaling (superresolution.py:351-355;
 * antialias is the identity when scale >= 1).  x [N,C,h,w] -> y [N,C,size,size]. */
int r3dp_sr_resize_bilinear(const float* x, int N, int C, int h, int w, int size, float* y, r3dp_stream_t stream);

/* Exact-fp32 SynthesisLayer (networks_stylegan2.py:322-342 -> conv2d_resample.py:116-138 -> bias_act lrelu):
 *   up == 1: y = lrelu(conv3x3(x, wf[n], pad 1) + bias) * sqrt(2)                       x,y [N,*,H,W]
 *   up == 2: y = lrelu(FIR4x4(conv_transpose2d(x, wf[n]^T, stride 2), pad 1, gain 4) + bias) * sqrt(2)
 *            x [N,I,H,W] -> y [N,O,2H,2W]; scratch holds the (2H+1)x(2W+1) intermediate:
 *            r3dp_sr_layer_scratch_bytes(N,O,H,W) bytes (0 needed for up == 1). */
size_t r3dp_sr_layer_scratch_bytes(int N, int O, int H, int W);
int r3dp_sr_layer_fp32(const float* x, const float* wf, const float* bias, int N, int I, int O, int H, int W, int up,
                       float* y, void* scratch, r3dp_stream_t stream);

/* ToRGB + skip (networks_stylegan2.py:365-370,463-469):
 *   img_out[N,3,H,W] = upsample2d(img_in[N,3,H/2,W/2]) + conv1x1(x[N,I,H,W], wf_rgb[N,3,I]) + bias[3]
 * upsample2d = zero-insert x2, pad (2,1,2,1), FIR [1,3,3,1]^2/64, gain 4 (upfirdn2d.py:317-354).
 * img_in may be NULL (no skip). */
int r3dp_sr_torgb_fp32(const float* x, const float* wf_rgb, const float* bias, const float* img_in, int N, int I,
                       int H, int W, float* img_out, r3dp_stream_t stream);

/* --------------------------------------------------------------- super-resolution on tensor cores (wgmma) ------
 * Same layers as above as TMA-fed wgmma implicit GEMMs: fp16 operands, fp32 accumulation in registers, fp32 epilogue.
 * Activations are NHWC fp16 with channels padded to a multiple of 64; weights are the per-sample folded weights
 * (r3dp_sr_fold_weights) packed to fp16 [Nw][9][O][Ipad] with Nw == N (per-sample styles) or 1 (shared styles).
 * Restrictions (met by SuperresolutionHybrid8XDC): W % 128 == 0, Cout % 128 == 0.
 *
 * r3dp_sr_tc_pack_weights  wf fp32 [Nw,O,I,3,3] -> packed fp16
 * r3dp_sr_tc_input         x fp32 NCHW [N,C,h,w] -> bilinear (align_corners=False) to size x size -> NHWC fp16 [N,size,size,Cpad]
 * r3dp_sr_tc_layer         SynthesisLayer (networks_stylegan2.py:322-342): up == 1 -> y [N,H,W,O]; up == 2 -> y [N,2H,2W,O]
 *                          (transposed conv as 4 parity phases + FIR, conv2d_resample.py:116-133); scratch for up == 2:
 *                          r3dp_sr_tc_scratch_bytes(N,O,H,W)
 * r3dp_sr_tc_torgb         ToRGB + upsampled skip of a non-final block -> img fp32 NCHW [N,3,H,W]
 * r3dp_sr_tc_last_layer    last conv (I -> 128) fused with ToRGB + skip: only the image is written (fp32 NCHW [N,3,H,W]);
 *                          wrgb [Nw,3,128], brgb [3], img_prev [N,3,H/2,W/2]; img_prev may be NULL (no skip: the image is
 *                          ToRGB + brgb alone, the block1(x, None, ws) of weight_fuse=False, sr_with_ref.py:161). */
int r3dp_sr_tc_pack_weights(const float* wf, int Nw, int O, int I, void* packed_f16, r3dp_stream_t stream);
int r3dp_sr_tc_input(const float* x, int N, int C, int h, int w, int size, void* y_f16, r3dp_stream_t stream);
size_t r3dp_sr_tc_scratch_bytes(int N, int O, int H, int W);
int r3dp_sr_tc_layer(const void* x_f16, const void* wp_f16, const float* bias, int N, int Nw, int I, int O, int H, int W,
                     int up, void* y_f16, void* scratch, r3dp_stream_t stream);
int r3dp_sr_tc_torgb(const void* x_f16, const float* wrgb, const float* brgb, const float* img_prev, int N, int Nw, int C,
                     int H, int W, float* img_out, r3dp_stream_t stream);
/* Up layer (up == 2) for SMALL Cin through FIR-composed weights: FIR(conv_transpose(x,w)) = four 3x3 correlations, one per output
 * parity (4x the MACs, but no (2H+1)x(2W+1) intermediate / FIR pass).  pack: wf fp32 [Nw,O,I,3,3] -> fp16 [Nw,36,O,Ipad]. */
int r3dp_sr_tc_pack_weights_up_composed(const float* wf, int Nw, int O, int I, void* packed_f16, r3dp_stream_t stream);
int r3dp_sr_tc_layer_up_composed(const void* x_f16, const void* wpc_f16, const float* bias, int N, int Nw, int I, int O, int H,
                                 int W, void* y_f16, r3dp_stream_t stream);
/* conv3x3 (up == 1) + bias/lrelu -> y fp16 NHWC, fused with the block's ToRGB + upsampled skip -> img_out fp32 NCHW
 * (block0.conv1 + block0.torgb of SynthesisBlock.forward, networks_stylegan2.py:455-469). */
int r3dp_sr_tc_layer_torgb(const void* x_f16, const void* wp_f16, const float* bias, const float* wrgb, const float* brgb,
                           const float* img_prev, int N, int Nw, int I, int O, int H, int W, void* y_f16, float* img_out,
                           r3dp_stream_t stream);
/* r3dp_sr_tc_input for a channels-last fp32 source [N,h,w,C] (the renderer's [N,M,C] output viewed as an image). */
int r3dp_sr_tc_input_nhwc(const float* x_nhwc, int N, int C, int h, int w, int size, void* y_f16, r3dp_stream_t stream);
/* ... and rgb_out [N,3,size,size] fp32 = the same resize of channels 0..2 (`rgb_image = feature_image[:, :3]`, secc_img2plane.py:126) in the same
 * launch; split != 0 writes the [hi | lo] activation layout of the r3dp_sr_tcx_* path. */
int r3dp_sr_tc_input_nhwc_rgb(const float* x_nhwc, int N, int C, int h, int w, int size, void* y_f16, float* rgb_out, int split, r3dp_stream_t stream);
int r3dp_sr_tc_last_layer(const void* x_f16, const void* wp_f16, const float* bias, const float* wrgb, const float* brgb,
                          const float* img_prev, int N, int Nw, int I, int H, int W, float* img_out, r3dp_stream_t stream);
/* The same with the caller loop's output conversion fused into the epilogue (inference/real3d_infer.py:515-519):
 *   clamp != 0       img_out clamped to [-1, 1] (imgs.clamp(-1,1))
 *   img_out_u8       non-NULL: write uint8 HWC video frames [N,H,W,3] = uint8(int((clamp(x) + 1) / 2 * 255)) INSTEAD of the fp32 image
 *                    (4x fewer bytes to gather / copy to the host); img_out may then be NULL.
 * img_prev may be NULL (no skip), as for r3dp_sr_tc_last_layer; so may it for r3dp_sr_tcx_last_layer. */
int r3dp_sr_tc_last_layer_ex(const void* x_f16, const void* wp_f16, const float* bias, const float* wrgb, const float* brgb,
                             const float* img_prev, int N, int Nw, int I, int H, int W, float* img_out, uint8_t* img_out_u8, int clamp,
                             r3dp_stream_t stream);

/* ---- fp32-grade tensor-core SR (`sr_mode='tc_exact'`): the same layers with SPLIT fp16 operands ------------------------------------------
 * The reference SR computes in fp32 (networks_stylegan2.py:37-94, conv2d_resample.py:48-145).  These entry points keep that accuracy on
 * wgmma: every fp32 operand is stored as two fp16 halves v = hi + lo (activations NHWC [N,H,W, 2*Cpad] = [hi | lo]; packed weights
 * [Nw,taps,O, 2*Ipad] = [hi | lo] of w * 2^10) and every convolution accumulates hi*hi + lo*hi + hi*lo in fp32 (three times the MMAs; the
 * dropped lo*lo term is ~2^-22).  Same arguments and meaning as the r3dp_sr_tc_* functions of the same name; tensors are twice as wide. */
int r3dp_sr_tcx_pack_weights(const float* wf, int Nw, int O, int I, void* packed_f16, r3dp_stream_t stream);
int r3dp_sr_tcx_pack_weights_up_composed(const float* wf, int Nw, int O, int I, void* packed_f16, r3dp_stream_t stream);
int r3dp_sr_tcx_input(const float* x, int N, int C, int h, int w, int size, void* y_f16, r3dp_stream_t stream);
int r3dp_sr_tcx_input_nhwc(const float* x_nhwc, int N, int C, int h, int w, int size, void* y_f16, r3dp_stream_t stream);
size_t r3dp_sr_tcx_scratch_bytes(int N, int O, int H, int W);
int r3dp_sr_tcx_layer(const void* x_f16, const void* wp_f16, const float* bias, int N, int Nw, int I, int O, int H, int W,
                      int up, void* y_f16, void* scratch, r3dp_stream_t stream);
int r3dp_sr_tcx_layer_up_composed(const void* x_f16, const void* wpc_f16, const float* bias, int N, int Nw, int I, int O, int H,
                                  int W, void* y_f16, r3dp_stream_t stream);
int r3dp_sr_tcx_layer_torgb(const void* x_f16, const void* wp_f16, const float* bias, const float* wrgb, const float* brgb,
                            const float* img_prev, int N, int Nw, int I, int O, int H, int W, void* y_f16, float* img_out,
                            r3dp_stream_t stream);
int r3dp_sr_tcx_last_layer(const void* x_f16, const void* wp_f16, const float* bias, const float* wrgb, const float* brgb,
                           const float* img_prev, int N, int Nw, int I, int H, int W, float* img_out, uint8_t* img_out_u8, int clamp,
                           r3dp_stream_t stream);

/* r3dp_sr_tc_conv with split fp16 operands (x [N,H,W,2*Ipad], weights from r3dp_sr_tcx_pack_weights, y [N,H,W,2*O] = [hi | lo]); used for the small
 * head_torso_alpha_predictor of fuse mode v3, whose output is thresholded (sr_with_ref.py:129-143) and therefore wants fp32-grade arithmetic. */
int r3dp_sr_tcx_conv(const void* x_f16, const void* wp_f16, const float* bias, int N, int Nw, int I, int O, int H, int W, int ksize,
                     int act, void* y_f16, r3dp_stream_t stream);
/* The torso head (SuperresolutionHybrid8XDC_Warp) and large_sr in split form.  Same arguments as the r3dp_sr_tc_* / r3dp_sr_* twin; every fp16 tensor is
 * [hi | lo] (twice as wide, lo half at half the pixel stride) and every output is written as hi = fp16(v), lo = fp16(v - hi) of the full fp32 value v.
 * r3dp_sr_tcx_conv_res            residual [N,H,W,2*O] summed to fp32 and added to the activated value BEFORE the hi/lo split (ResBlock2d)
 * r3dp_sr_tcx_layer_torgb_noup    SynthesisBlockNoUp tail; ToRGB over the fp32 activation
 * r3dp_sr_tcx_alpha_cat_ex        out [N,H,W,2*(Ca+Cb)] = split of cat[xa*alpha, xb*(1-alpha)]; stride_a / stride_b are the physical pixel strides
 * r3dp_sr_tcx_alpha_mix           out [N,H,W,2*C] = split of xa*alpha + xb*(1-alpha); strides as above
 * r3dp_sr_tcx_torgb_ex            x [N,H,W,2*C]: the dot product runs over hi + lo in fp32
 * r3dp_sr_tcx_cat3                out [N,H,W,2*(Ca+Cb+Cc)] = [hi | lo] layout of cat[xa, xb, xc]: each operand's hi and lo halves are copied unchanged */
int r3dp_sr_tcx_conv_res(const void* x_f16, const void* wp_f16, const float* bias, int N, int Nw, int I, int O, int H, int W, int ksize,
                         int act, const void* residual_f16, void* y_f16, r3dp_stream_t stream);
int r3dp_sr_tcx_layer_torgb_noup(const void* x_f16, const void* wp_f16, const float* bias, const float* wrgb, const float* brgb,
                                 const float* img_prev, int N, int Nw, int I, int O, int H, int W, void* y_f16, float* img_out,
                                 r3dp_stream_t stream);
int r3dp_sr_tcx_alpha_cat_ex(const void* xa_f16, int Ca, int stride_a, const void* xb_f16, int Cb, int stride_b, int xb_shared, const float* alpha,
                             int N, int H, int W, void* out_f16, r3dp_stream_t stream);
int r3dp_sr_tcx_alpha_mix(const void* xa_f16, int stride_a, const void* xb_f16, int stride_b, const float* alpha, int C, int N, int H, int W,
                          void* out_f16, r3dp_stream_t stream);
int r3dp_sr_tcx_torgb_ex(const void* x_f16, const float* wrgb, const float* brgb, const float* img_prev, int same_res, int N, int Nw, int C,
                         int H, int W, float* img_out, r3dp_stream_t stream);
int r3dp_sr_tcx_cat3(const void* xa_f16, int Ca, int stride_a, const void* xb_f16, int Cb, int stride_b, const void* xc_f16, int Cc, int stride_c,
                     int xc_shared, int N, int H, int W, void* out_f16, r3dp_stream_t stream);

/* Measurement hooks (bench.py): time every tensor-core conv launch with a CUDA-event pair on its launching stream. */
int r3dp_sr_tc_prof(int enable);
int r3dp_sr_tc_prof_read(float* total_ms, int* launches);
/* Debug builds only (-DR3DP_TC_DEBUG_TIMING=1): 32 x 24 uint64 device buffer; row i receives the MMA / epilogue warps' clock sums of the i-th conv launch (NULL = off). */
int r3dp_sr_tc_debug_buffer(void* buf);

/* ------------------------------------------------------- torso head: SuperresolutionHybrid8XDC_Warp building blocks ---
 * (modules/real3d/super_resolution/sr_with_ref.py:16-162; the torso warper itself stays the caller's PyTorch module)
 * r3dp_sr_tc_conv              nn.Conv2d k=1|3, stride 1, same padding (+bias) [+ act: 0 linear, 1 lrelu(0.2)*sqrt2, 2 nn.LeakyReLU 0.01]
 *                              x [N,H,W,Ipad] fp16, weights packed with r3dp_sr_tc_pack_weights (k=1: value in tap 4), y [N,H,W,O] fp16
 * r3dp_sr_tc_layer_torgb_noup  SynthesisBlockNoUp tail: conv3x3 + act -> y, img_out = img_prev (same resolution) + ToRGB(y) + brgb
 * r3dp_sr_alpha_cat            out = cat[xa*alpha, xb*(1-alpha)] on fp16 NHWC (pixel strides stride_a/stride_b in elements), alpha fp32 [N,H,W]
 * r3dp_sr_blend                out = a*alpha + b*(1-alpha), fp32 NCHW, alpha [N,1,H,W]
 * r3dp_sr_person_occlusion     out = clamp(torso_occlusion + (head_alpha > threshold ? 1 : head_alpha), 0, 1)
 * r3dp_sr_resize_aa_down2      F.interpolate(scale 1/2, bilinear, antialias=True): x [N,C,2h,2w] -> y [N,C,h,w] fp32 */
int r3dp_sr_tc_conv(const void* x_f16, const void* wp_f16, const float* bias, int N, int Nw, int I, int O, int H, int W, int ksize,
                    int act, void* y_f16, r3dp_stream_t stream);
/* large_sr (LargeSynthesisBlock0/1 + ResBlock2d, modules/eg3ds/models/superresolution.py:263-329):
 * r3dp_sr_tc_conv_res  r3dp_sr_tc_conv with act 3 = ReLU and an optional residual (NHWC fp16, the output's shape) added AFTER the activation:
 *                      ResBlock2d's `out = act(conv2(act(conv1(x)))) + x`
 * r3dp_sr_tc_torgb_ex  plain 1x1 conv to RGB; same_res != 0: img_out = img_prev[N,3,H,W] + conv1x1(x) + b  (`rgb = rgb + self.to_rgb(x)`) */
int r3dp_sr_tc_conv_res(const void* x_f16, const void* wp_f16, const float* bias, int N, int Nw, int I, int O, int H, int W, int ksize,
                        int act, const void* residual_f16, void* y_f16, r3dp_stream_t stream);
int r3dp_sr_tc_torgb_ex(const void* x_f16, const float* wrgb, const float* brgb, const float* img_prev, int same_res, int N, int Nw, int C,
                        int H, int W, float* img_out, r3dp_stream_t stream);
/* htbsr_head_weight_fuse_mode v1 / v3 (sr_with_ref.py:96-104,126-152):
 * r3dp_sr_alpha_mix   out[...,0:C] = xa * alpha + xb * (1 - alpha), fp16 NHWC with pixel strides stride_a / stride_b (v1's feature blend)
 * r3dp_sr_alpha_gate  out [N,1,H,W] fp32 = min(sigmoid(logit), cap): logit = channel 0 of an NHWC fp16 tensor (+ channel lo_off when lo_off > 0: split
 *                     output of r3dp_sr_tcx_conv) = tail of head_torso_alpha_predictor + the cap by the head weights (v3) */
int r3dp_sr_alpha_mix(const void* xa_f16, int stride_a, const void* xb_f16, int stride_b, const float* alpha, int C, int N, int H, int W,
                      void* out_f16, r3dp_stream_t stream);
int r3dp_sr_alpha_gate(const void* logits_f16, int stride, int lo_off, const float* cap, int N, int H, int W, float* out, r3dp_stream_t stream);
int r3dp_sr_tc_layer_torgb_noup(const void* x_f16, const void* wp_f16, const float* bias, const float* wrgb, const float* brgb,
                                const float* img_prev, int N, int Nw, int I, int O, int H, int W, void* y_f16, float* img_out,
                                r3dp_stream_t stream);
int r3dp_sr_alpha_cat(const void* xa_f16, int Ca, int stride_a, const void* xb_f16, int Cb, int stride_b, const float* alpha, int N,
                      int H, int W, void* out_f16, r3dp_stream_t stream);
/* xb_shared != 0: xb holds ONE frame [1,H,W,Cb] read by every frame of the batch (per-clip constant features, e.g. bg_encoder(ref_bg)). */
int r3dp_sr_alpha_cat_ex(const void* xa_f16, int Ca, int stride_a, const void* xb_f16, int Cb, int stride_b, int xb_shared, const float* alpha,
                         int N, int H, int W, void* out_f16, r3dp_stream_t stream);
/* weight_fuse=False (sr_with_ref.py:159): out [N,H,W,Ca+Cb+Cc] = cat[xa, xb, xc] on fp16 NHWC, unweighted (a bit-exact copy); pixel strides
 * stride_a/b/c in elements; xc_shared != 0: xc holds ONE frame [1,H,W,Cc] read by every frame of the batch (the per-clip bg_encoder(ref_bg)). */
int r3dp_sr_cat3(const void* xa_f16, int Ca, int stride_a, const void* xb_f16, int Cb, int stride_b, const void* xc_f16, int Cc, int stride_c,
                 int xc_shared, int N, int H, int W, void* out_f16, r3dp_stream_t stream);
int r3dp_sr_blend(const float* a, const float* b, const float* alpha, int N, int C, int H, int W, float* out, r3dp_stream_t stream);
int r3dp_sr_person_occlusion(const float* head_alpha, const float* torso_occlusion, float threshold, int N, int H, int W, float* out,
                             r3dp_stream_t stream);
int r3dp_sr_resize_aa_down2(const float* x, int N, int C, int h_out, int w_out, float* y, r3dp_stream_t stream);
/* The torso head's inputs straight from the renderer's channels-last output, in one launch (modules/real3d/super_resolution/sr_with_ref.py:70-78):
 *   x_nhwc [N,h,w,C] fp32 (C % 8 == 0), wsum [N,h*w,1] fp32 (the layout of the weight image [N,1,h,w]), h, w <= size <= 256
 *   y_f16   [N,size,size,Cpad] fp16 = r3dp_sr_tc_input_nhwc's output ([hi | lo] when split != 0)
 *   rgb0    [N,3,size,size] fp32   = the resize of channels 0..2 (rgb_out of r3dp_sr_tc_input_nhwc_rgb)
 *   rgb_256 [N,3,256,256] fp32     = r3dp_sr_resize_bilinear(rgb0, 256)            (sr_with_ref.py:77)
 *   w_256   [N,1,256,256] fp32     = r3dp_sr_resize_bilinear(weight image, 256)    (sr_with_ref.py:78)
 * Every output is bit-identical to that three-launch sequence. */
int r3dp_sr_warp_input(const float* x_nhwc, const float* wsum, int N, int C, int h, int w, int size, void* y_f16, float* rgb0, float* rgb_256,
                       float* w_256, int split, r3dp_stream_t stream);

/* Stage 2 of the torso warper: Generator (modules/real3d/facev2v_warp/network2.py:248-301) + occlusion_2_predictor (model2.py:212-219,
 * 260-263).  Activations NHWC fp16 ([hi | lo] halves when split != 0, as in the r3dp_sr_tcx_* family), weights folded on the host.
 * r3dp_tw_gather3d          Generator.get_deformed_feature (network2.py:298-301): F.grid_sample(fs, grid, trilinear, padding_mode='border',
 *                           align_corners=True).view(N, C*D, H, W).  fs NDHWC fp32 [N,D,H,W,C] ([1,D,H,W,C] read by every image when fs_shared != 0), grid [N,D,H,W,3] -> y [N,H,W,C*D] fp16,
 *                           channel c*D + d
 * r3dp_tw_conv              nn.Conv2d k=1|3 (+ folded SpectralNorm / BatchNorm) with act max(v, slope*v) and an optional residual added after
 *                           it (ResBlock2D, layers.py:104-105): in_conv, mid_conv, res.*; W % 64 == 0, O = 128 | 256, weights as r3dp_sr_tc_conv
 * r3dp_tw_conv_up_nearest   UpBlock2D (layers.py:77-88): nn.Upsample(x2, nearest) + 3x3 conv (+ folded BatchNorm) + act, x [N,H,W,Ipad] ->
 *                           y [N,2H,2W,O]; weights = 4 output-parity sets of composed 2x2 taps packed by r3dp_sr_tc_pack_weights with Nw = 4
 * r3dp_tw_affine_relu       relu(scale[c] * x + shift[c]): eval BatchNorm + ReLU at the head of a pre-activation ResBlock2D (layers.py:100)
 * r3dp_tw_narrow_conv       KxK conv to CO = 1 | 3 | 32 channels on CUDA cores in fp32 (Generator.out_conv, the occlusion_2_predictor convs):
 *                           input xa (NHWC fp16, pixel stride sa, ca channels, split remainder at lo_a > 0) or xf (NHWC fp32), plus optionally the
 *                           bilinear (align_corners=False) resize of ex [N,1,eh,ew] to HxW as the last channel (model2.py:262's concat);
 *                           wk [K*K][cin][CO] fp32, act 0 linear / 1 ReLU / 2 sigmoid, out fp32 NCHW (nchw != 0) or NHWC
 * r3dp_tw_hid_to_nchw       NHWC fp16 (pixel stride cs, split remainder at lo > 0) -> [N,C,H,W] fp32: ret['deformed_torso_hid'] (model2.py:261) */
int r3dp_tw_gather3d(const float* fs_ndhwc, int fs_shared, const float* grid, int N, int C, int D, int H, int W, void* y_f16, int split,
                     r3dp_stream_t stream);
int r3dp_tw_conv(const void* x_f16, const void* wp_f16, const float* bias, int N, int I, int O, int H, int W, int ksize, float slope,
                 const void* residual_f16, void* y_f16, int split, r3dp_stream_t stream);
int r3dp_tw_conv_up_nearest(const void* x_f16, const void* wp_f16, const float* bias, int N, int I, int O, int H, int W, float slope, void* y_f16,
                            int split, r3dp_stream_t stream);
int r3dp_tw_affine_relu(const void* x_f16, const float* scale, const float* shift, int N, int H, int W, int C, int split, void* y_f16,
                        r3dp_stream_t stream);
int r3dp_tw_narrow_conv(const void* xa_f16, int sa, int ca, int lo_a, const float* xf, int sf, int cf, const float* ex, int eh, int ew,
                        const float* wk, const float* bias, int N, int H, int W, int K, int CO, int act, int nchw, float* out, r3dp_stream_t stream);
int r3dp_tw_hid_to_nchw(const void* x_f16, int N, int C, int H, int W, int cs, int lo, float* y, r3dp_stream_t stream);

/* The torso warper's motion-field estimator (modules/real3d/facev2v_warp/network2.py:162-244, MotionFieldEstimator('standard')).
 * Activations NDHWC fp16 with voxel stride xs / ys halves; split != 0: the fp16 remainder of each value sits `lo` halves after it in the same
 * voxel ([hi | lo]) and the weights are [hi | lo] of w * 2^10, as in the r3dp_sr_tcx_* family.
 * r3dp_mf_conv3d       3-D conv on wgmma (stride 1, zero padding): box taps kd x kh x kw (odd) centred, or with up != 0 the 4 output-parity
 *                      phases of nn.Upsample((1,2,2), nearest) + 3x3x3 conv as kd x 2 x 2 taps on the low-resolution input (layers.py:77-93).
 *                      M space = the input grid N x D x H x W; x channels [0, cin) (cin % 32 == 0); wp [nph][taps][cop][cin (x2 split)] fp16,
 *                      bias [cop]; y = act(conv + bias) (+ res, same layout as y) stored at channels [yc0, yc0 + cout) of voxels of ys
 *                      halves (up: output grid D x 2H x 2W), fp16 or fp32 (out_f32, no residual); act (the `relu` argument): 0 none,
 *                      1 ReLU, 2 exact GELU (nn.GELU(), erf form)
 * r3dp_mf_input        create_heatmap_representations + create_sparse_motions + create_deformed_source_image (func_utils.py:130-191, Rs = Rd = I):
 *                      fc [N or 1,D,H,W,4] fp32 (the compressed source), kp_s / kp_d [N,K,3] -> channel k*5 + j of y, zeros up to cpad
 * r3dp_mf_pool         AvgPool3d((1,2,2)) (layers.py:58-74); H, W: the pooled size
 * r3dp_mf_head_input   interpolate(cat[rgb, weights], 1/2, bilinear) = the 2x2 mean, [N,3|1,2H,2W] fp32 -> NHWC channels 0..3, zeros up to cpad
 * r3dp_mf_head_bcast   interpolate(head features, 1/2, bilinear) repeated over depth (network2.py:221-224) into channels [yc0, yc0 + C) of y
 * r3dp_mf_deform       softmax over the K+1 fp32 logits (voxel stride ls) and deformation [N,D,H,W,3] = sum_k mask_k * sparse_motion_k
 * r3dp_mf_occlusion    occlusion_conv / occlusion_conv2 (7x7, C*D -> 1, sigmoid) on x.view(N, C*D, H, W): wk [D][49][C][2] fp32, bias [2] */
int r3dp_mf_conv3d(const void* x_f16, int xs, int xlo, int cin, const void* wp_f16, const float* bias, const void* res_f16, int N, int D, int H,
                   int W, int kd, int kh, int kw, int up, int cout, int cop, int relu, void* y, int ys, int yc0, int ylo, int out_f32, int split,
                   r3dp_stream_t stream);
int r3dp_mf_input(const float* fc, int fc_shared, const float* kp_s, const float* kp_d, int N, int K, int D, int H, int W, int cpad, void* y_f16,
                  int ys, int ylo, int split, r3dp_stream_t stream);
int r3dp_mf_pool(const void* x_f16, int N, int D, int H, int W, int C, int xs, int xlo, void* y_f16, int ys, int ylo, int split, r3dp_stream_t stream);
int r3dp_mf_head_input(const float* rgb, const float* wts, int N, int H, int W, int cpad, void* y_f16, int ys, int ylo, int split, r3dp_stream_t stream);
int r3dp_mf_head_bcast(const void* x_f16, int N, int D, int H, int W, int C, int xs, int xlo, void* y_f16, int ys, int yc0, int ylo, int split,
                       r3dp_stream_t stream);
int r3dp_mf_deform(const float* logits, int ls, const float* kp_s, const float* kp_d, int N, int K, int D, int H, int W, float* deformation,
                   r3dp_stream_t stream);
int r3dp_mf_occlusion(const void* x_f16, int N, int D, int H, int W, int C, int xs, int xlo, int split, const float* wk, const float* bias, float* occ,
                      float* occ2, r3dp_stream_t stream);

/* ------------------------------------------------ SECC -> plane backbone: SegFormerSECC2PlaneBackbone('b0') ---
 * (modules/real3d/segformer.py:673-733; called per frame by cal_secc_plane, modules/real3d/secc_img2plane.py:64-81).  Token tensors are
 * row-major [N, h*w, C] (row = the NHWC pixel h*W + w).  The GEMMs (q, kv, proj, fc1, fc2, patch embeds 2-4, the spatial reduction, the folded
 * head maps and the last conv) run on r3dp_mf_conv3d with 1x1x1 or 1x3x3 taps; to_plane_cnn.0/2/4 on r3dp_sr_tc_conv (act 2) where W % 128 == 0.
 * r3dp_sp_prenet          prenet 1x1 (Conv2dLayer, networks_stylegan2.py:139-183, weight gain folded into w [3,cin]): x [N,cin,H,W] -> y [N,3,H,W];
 *                         used once per clip on the cano/src channels to make the constant image
 * r3dp_sp_embed           prenet + patch_embed1.proj (7x7 stride 4 pad 3, segformer.py:206-232) -> y fp32 [N, ceil(H/4)*ceil(W/4), 32], before its
 *                         LayerNorm.  Prenet output = (base ? base[1,3,H,W] : bpre[3]) + w [3,cin] . x[N,cin,H,W]; wpe [32,3,7,7], bpe [32]
 * r3dp_sp_layernorm       v = x + t (t may be NULL); xo = v if non-NULL (xo may be x: the in-place residual add of Block.forward, segformer.py:236-239);
 *                         u = LayerNorm(v)(g, b, eps) (segformer.py:118,216,411) -> yf fp32 [R,C] and/or yh fp16 with row stride yhs; C % 32 == 0, <= 1024
 * r3dp_sp_patches         y fp16 [N*Ho*Wo, k*k*C], column (ky*k + kx)*C + c = x[n, oy*s - p + ky, ox*s - p + kx, c] (zero outside): GEMM rows of
 *                         the 3x3/2 patch embeds (segformer.py:286-291) and of Attention.sr (k = s = sr_ratio, segformer.py:126-128); C % 8 == 0
 * r3dp_sp_patches_dil     the same rows for a conv of dilation d (x[n, oy*s - p + ky*d, ox*s - p + kx*d, c]), each row ldy halves long (ldy % 8 == 0,
 *                         >= k*k*C) with columns from k*k*C on zero, so that the GEMM's K can be a multiple of 32; r3dp_sp_patches is d = 1,
 *                         ldy = k*k*C
 * r3dp_sp_attention       Attention.forward's core (segformer.py:130-150) for head_dim 32: q fp16 [N,Tq, >= heads*32] (row stride qs), kv fp16
 *                         [N,Tk, >= 2*heads*32] (k in channels [0, 32 heads), v after it), Tk <= 256 -> o fp16 (row stride os), channel head*32 + d;
 *                         fp32 scores and an exact full-row softmax
 * r3dp_sp_dwconv_gelu     Mlp's DWConv 3x3 + bias then nn.GELU (erf) (segformer.py:82-84,459-468): x, y fp16 NHWC [N,H,W,C], w [C,9], b [C]
 * r3dp_sp_head_fuse       SegFormerHead.forward (segformer.py:525-537) after the fold: y fp16 NHWC [N,h1,h1,256] = ReLU(sum_i resize_i(g_i) + bias),
 *                         g_i fp32 NHWC [N,h_i,h_i,256] = G_i c_i, resize = bilinear align_corners=False to h1 x h1
 * r3dp_sp_leaky           nn.LeakyReLU(slope) in place on n fp16 values (to_plane_cnn.1/3/5 where the conv ran on r3dp_mf_conv3d)
 * r3dp_sp_upsample2_flip  nn.UpsamplingBilinear2d(x2) (align_corners=True) of x fp16 NHWC [N,h,w,C] written twice, mirrored: yr [N,2h,2w,C] rows
 *                         mirrored, yrc rows and columns mirrored.  A 3x3 zero-padded conv of a mirrored image with mirrored taps is the mirrored
 *                         conv, so the last conv run on these writes the flipped planes of segformer.py:722-730 directly. */
int r3dp_sp_prenet(const float* x, int N, int cin, int H, int W, const float* w, const float* b, float* y, r3dp_stream_t stream);
int r3dp_sp_embed(const float* x, int N, int cin, int H, int W, const float* wpre, const float* base, const float* bpre, const float* wpe,
                  const float* bpe, float* y, r3dp_stream_t stream);
int r3dp_sp_layernorm(const float* x, const float* t, int R, int C, const float* g, const float* b, float eps, float* xo, float* yf, void* yh_f16,
                      int yhs, r3dp_stream_t stream);
int r3dp_sp_patches(const void* x_f16, int N, int H, int W, int C, int k, int s, int p, void* y_f16, r3dp_stream_t stream);
int r3dp_sp_patches_dil(const void* x_f16, int N, int H, int W, int C, int k, int s, int p, int d, void* y_f16, int ldy, r3dp_stream_t stream);
int r3dp_sp_attention(const void* q_f16, int qs, const void* kv_f16, int kvs, int N, int Tq, int Tk, int heads, float scale, void* o_f16, int os,
                      r3dp_stream_t stream);
int r3dp_sp_dwconv_gelu(const void* x_f16, int N, int H, int W, int C, const float* w, const float* b, void* y_f16, r3dp_stream_t stream);
int r3dp_sp_head_fuse(const float* g1, int h1, const float* g2, int h2, const float* g3, int h3, const float* g4, int h4, int N, const float* bias,
                      void* y_f16, r3dp_stream_t stream);
int r3dp_sp_leaky(void* x_f16, long long n, float slope, r3dp_stream_t stream);
int r3dp_sp_upsample2_flip(const void* x_f16, int N, int h, int w, int C, void* yr_f16, void* yrc_f16, r3dp_stream_t stream);
/* The backbone in precision='tc_exact': every GEMM and conv operand split fp16 (r3dp_mf_conv3d split, r3dp_sr_tcx_conv), every activation that
 * the `tc` path passes between launches as fp16 passed as fp32 or as split rows [hi C | lo C] (hi = fp16(v), lo = fp16(v - hi), C halves
 * apart).  LayerNorm without a residual runs on r3dp_hb_layernorm, the embed and fp32-output LayerNorms on r3dp_sp_embed / r3dp_sp_layernorm.
 * r3dp_sp_layernorm_split      r3dp_sp_layernorm's residual form (t required, xo may be NULL or x) with u written as split rows yh (yhs halves,
 *                              lo at yhlo >= C)
 * r3dp_sp_patches_split        r3dp_sp_patches of split pixels x [N,H,W][hi C | lo C] -> rows [N*Ho*Wo][hi k*k*C | lo k*k*C], the operand of
 *                              r3dp_mf_conv3d with xs = 2K, xlo = K (K = k*k*C)
 * r3dp_sp_attention_split      r3dp_sp_attention on fp32 q / kv (row strides qs, kvs floats) -> o split rows (os halves, lo at olo >= C)
 * r3dp_sp_dwconv_gelu_split    r3dp_sp_dwconv_gelu on fp32 x [N,H,W,C] -> y split rows [N*H*W][hi C | lo C]
 * r3dp_sp_head_fuse_split      r3dp_sp_head_fuse -> y split rows [N*h1*h1][hi 256 | lo 256]
 * r3dp_sp_leaky_split          nn.LeakyReLU(slope) in place on P split rows [hi C | lo C] of the full value hi + lo
 * r3dp_sp_upsample2_flip_split r3dp_sp_upsample2_flip on split pixels: x [N,h,w][hi C | lo C] -> yr, yrc [N,2h,2w][hi C | lo C]; C % 4 == 0 */
int r3dp_sp_layernorm_split(const float* x, const float* t, int R, int C, const float* g, const float* b, float eps, float* xo, void* yh_f16,
                            int yhs, int yhlo, r3dp_stream_t stream);
int r3dp_sp_patches_split(const void* x_f16, int N, int H, int W, int C, int k, int s, int p, void* y_f16, r3dp_stream_t stream);
int r3dp_sp_attention_split(const float* q, int qs, const float* kv, int kvs, int N, int Tq, int Tk, int heads, float scale, void* o_f16, int os,
                            int olo, r3dp_stream_t stream);
int r3dp_sp_dwconv_gelu_split(const float* x, int N, int H, int W, int C, const float* w, const float* b, void* y_f16, r3dp_stream_t stream);
int r3dp_sp_head_fuse_split(const float* g1, int h1, const float* g2, int h2, const float* g3, int h3, const float* g4, int h4, int N,
                            const float* bias, void* y_f16, r3dp_stream_t stream);
int r3dp_sp_leaky_split(void* x_f16, long long P, int C, float slope, r3dp_stream_t stream);
int r3dp_sp_upsample2_flip_split(const void* x_f16, int N, int h, int w, int C, void* yr_f16, void* yrc_f16, r3dp_stream_t stream);

/* ------------------------------------------------ canonical plane backbone: Img2PlaneModel ---
 * (modules/img2plane/img2plane_model.py:12-81; run once per clip on the source image by cal_cano_plane, modules/real3d/secc_img2plane.py:50-62).
 * Activations NHWC fp16; token tensors row-major [N, h*w, C].  Convolutions and token GEMMs run on r3dp_mf_conv3d (strided and dilated convs on
 * r3dp_sp_patches_dil rows), LayerNorm on r3dp_sp_layernorm, the Mlp's DWConv + GELU on r3dp_sp_dwconv_gelu.
 * r3dp_ip_attention      Attention.forward's core (segformer/base.py:101-122) for head_dim 256 on wgmma: q fp16 [N,Tq, >= heads*256] (row stride
 *                        qs), kv fp16 [N,Tk, >= 2*heads*256] (k in channels [0, 256 heads), v after it) -> o fp16 (row stride os), channel
 *                        head*256 + d.  Any Tq, Tk >= 1; qs, kvs multiples of 8; q, kv 16-byte aligned.  Online softmax in fp32, P rounded to
 *                        fp16 for P.V; no Tq x Tk buffer
 * r3dp_ip_input          x fp32 [N,3,H,W] -> y fp16 [N,H,W,8] = (rgb, i/H, j/H, 0, 0, 0): the coordinate channels of img2plane_model.py:59-64
 * r3dp_ip_maxpool        nn.MaxPool2d(3, 2, 1): x fp16 NHWC [N,H,W,C] -> y [N, (H-1)/2+1, (W-1)/2+1, C]; C % 8 == 0
 * r3dp_ip_channel_mean   AdaptiveAvgPool2d(1): x fp16 [N,HW,C] -> y fp16 [N,C]; C % 32 == 0
 * r3dp_ip_broadcast      y[n, p, yc0 + c] = v[n, c] for every pixel p < HW (pixel stride ys): ASPPPooling's upsampling of a 1x1 map
 * r3dp_ip_pixel_shuffle  nn.PixelShuffle(2) of tokens x (+ t, may be NULL) fp32 [N, h*w, 4C] -> y fp16 [N,2h,2w] pixels of ys halves, channels
 *                        [yc0, yc0 + C): y[n, 2a+i, 2b+j, c] = x[n, a*w + b, 4c + 2i + j]
 * r3dp_ip_upsample2      nn.UpsamplingBilinear2d(x2) (align_corners=True): x fp16 NHWC [N,h,w,C] -> y [N,2h,2w,C]; C % 8 == 0
 * r3dp_ip_flip_hwpc      the last conv's x fp32 [N,H,W,96] -> planes fp32 [N,H,W,3,32] (the render's hwpc layout) with the flips of
 *                        img2plane_model.py:72-81: out[n,Y,X,p,c] = x[n, H-1-Y, p < 2 ? X : W-1-X, 32p + c] */
int r3dp_ip_attention(const void* q_f16, int qs, const void* kv_f16, int kvs, int N, int Tq, int Tk, int heads, float scale, void* o_f16, int os,
                      r3dp_stream_t stream);
int r3dp_ip_input(const float* x, int N, int H, int W, void* y_f16, r3dp_stream_t stream);
int r3dp_ip_maxpool(const void* x_f16, int N, int H, int W, int C, void* y_f16, r3dp_stream_t stream);
int r3dp_ip_channel_mean(const void* x_f16, int N, int HW, int C, void* y_f16, r3dp_stream_t stream);
int r3dp_ip_broadcast(const void* v_f16, int N, int HW, int C, void* y_f16, int ys, int yc0, r3dp_stream_t stream);
int r3dp_ip_pixel_shuffle(const float* x, const float* t, int N, int h, int w, int C, void* y_f16, int ys, int yc0, r3dp_stream_t stream);
int r3dp_ip_upsample2(const void* x_f16, int N, int h, int w, int C, void* y_f16, r3dp_stream_t stream);
int r3dp_ip_flip_hwpc(const float* x, int N, int H, int W, float* out, r3dp_stream_t stream);

/* ------------------------------------------------ SECC renderer: SECC_Renderer (deep_3drecon/secc_renderer.py) ---
 * The 3DMM face mesh rasterised at S x S with pytorch3d's rules (blur 0, one face per pixel, perspective-correct barycentrics, no culling
 * or clipping; DESIGN.md) and shaded with the per-vertex NCC code.  All fp32.
 * r3dp_secc_vertices  basis [3N, n_id + n_exp] (row 3v + axis, id columns then exp columns, 16-byte aligned), mean [3N] (recentred),
 *                     id [B, >= n_id] (row stride ids), exp [B, >= n_exp] (row stride exps; a stride of 0 reads row 0 for every frame),
 *                     euler, trans [B,3] (NULL = zero)
 *                     -> verts [B,N,4] = (x_ndc, y_ndc, z_view, 0): s = basis . [id|exp] + mean, v = Rz Ry Rx s + t (bfm.py:204-238,260-270),
 *                     z = cam_dist - v_z, x_ndc = -v_x / (z tan_half), y_ndc = v_y / (z tan_half).  n_id + n_exp <= 256, a multiple of 4.
 *                     Each basis row is read once per chunk of frames: one chunk when N fills the GPU, more for small N.
 * r3dp_secc_raster    verts [B,N,4], faces int32 [F,3] (0-based) -> keys [B,S,S] uint64: atomicMin of (bits of pz) << 32 | face over every
 *                     covered pixel centre (nearest pz, ties to the lower face).  keys must hold ~0 (empty) on entry.
 * r3dp_secc_resolve   keys -> secc [B,3,S,S] = 2 mask sum_i w_i ncc[v_i] - 1 (-1 where empty) and mask [B,1,S,S] (may be NULL); ncc [N,4]
 *                     (x, y, z, pad).  drop_face0: face 0 counts as background in image 0 (pix_to_face > 0 on the packed index,
 *                     mesh_renderer.py:116).  Resets every key to empty. */
int r3dp_secc_vertices(const float* basis, const float* mean, int N, int n_id, int n_exp, const float* id, int ids, const float* exp, int exps,
                       const float* euler, const float* trans, int B, float cam_dist, float tan_half, float* verts, r3dp_stream_t stream);
int r3dp_secc_raster(const float* verts, int N, const int* faces, int F, int B, int S, void* keys, r3dp_stream_t stream);
int r3dp_secc_resolve(const float* verts, int N, const int* faces, const float* ncc, int B, int S, int drop_face0, void* keys, float* secc,
                      float* mask, r3dp_stream_t stream);

/* ------------------------------------------------ SECC blink: blink_eye_for_secc (inference/edit_secc.py) ---
 * r3dp_secc_blink     edits secc [B,3,S,S] fp32 (r3dp_secc_resolve's layout) in place, 64 <= S <= 1024: closes the eye holes of each image to
 *                     the fraction p (DESIGN.md, "SECC blink") and quantises the image to the reference's 8-bit codes (q / 127.5 - 1).
 *                     Control per image, exactly one of: p [B] double (outside [0, 1] or NaN = untouched), or rows (fp32, row stride
 *                     row_stride) whose first two values are (t, T): p = -4/T^2 t^2 + 4/T t in double; T <= 0, t < 0 or t >= T = untouched.
 *                     Untouched images are not written; p == 0 only quantises.  Images on which the reference raises (no non-face pixel
 *                     in either prior eye region, or no face pixel left around the eyes after the erosion) are left as they are and
 *                     add one to *faults (int32, device).  scratch: r3dp_secc_blink_scratch_bytes(B, S) bytes, 256-byte aligned, any
 *                     content (each call initialises what it reads).  Four launches, no host synchronisation. */
size_t r3dp_secc_blink_scratch_bytes(int B, int S);
int r3dp_secc_blink(float* secc, int B, int S, const double* p, const float* rows, int row_stride, void* scratch, int* faults,
                    r3dp_stream_t stream);

/* ------------------------------------------------ clip motion: cameras and torso key points (real3d_infer.py:271-321, 428-452) ---
 * r3dp_motion_camera     per frame i < T: the pose (fp32, as the reference): driving row mirror_index(i, P) of drv_euler / drv_trans [P,3]
 *                        (pass the source pose with P = 1 for the 'static' pose), z translation of frame 0, + (src - pose[0]) when
 *                        map_to_init_pose -> euler, trans [T,3]; and cameras [T,25] = row-major c2w (16) and intrinsics (9) of
 *                        get_eg3d_convention_camera_pose_intrinsic, smoothed by smooth_camera_sequence over the truncated 7-frame window
 *                        (translation mean; rotation mean = top eigenvector of sum q q^T, in double).
 * r3dp_motion_keypoints  verts_s [K,4] / verts_d [T,K,4] (r3dp_secc_vertices at the key points, 16-byte aligned) -> kp_s [K,3] =
 *                        (clamp(-x_ndc), clamp(-y_ndc), 0) (clamp to [-1, 1]), kp_d [T,K,3] = the same smoothed by smooth_features_xd
 *                        (7-tap box filter over frames, the first and last three mirrored); T >= 3.
 * r3dp_motion_lm2d       verts [n,4] -> lm2d [n,2] = (1 - x_ndc, 1 - y_ndc) / 2 (Face3DHelper.reconstruct_lm2d's coordinates).
 * No host synchronisation and no allocation: capturable in a CUDA graph. */
int r3dp_motion_camera(const float* src_euler, const float* src_trans, const float* drv_euler, const float* drv_trans, int P, int T,
                       int map_to_init_pose, float* euler, float* trans, float* cameras, r3dp_stream_t stream);
int r3dp_motion_keypoints(const float* verts_s, const float* verts_d, int T, int K, float* kp_s, float* kp_d, r3dp_stream_t stream);
int r3dp_motion_lm2d(const float* verts, long long n, float* lm2d, r3dp_stream_t stream);

/* ------------------------------------------------ 3DMM fit: coefficients from mediapipe landmarks (data_gen/utils/process_{image,video}/fit_3dmm_landmark.py) ---
 * The parameters x [80 + 70 T] fp64: id [80], then per frame exp [64], euler [3], trans [3]; Adam's m and v share that layout.  The 468 key
 * points are 8 chunks of 64 (the last 44 padded): basis [8][192][144] fp32 (chunk rows x | y | z blocks of 64 points, columns id | exp),
 * mean [8][192], weight [512] (the landmark loss's per-point weights, 0 on the padding).
 * r3dp_fit_grad  one iteration's landmark-loss gradient (mean over T 468 2 of w (proj - lms)^2) at x; lms [T, L, 2] mediapipe pixels (y down,
 *                L >= 468 points per frame, 8-byte aligned), img_size the image side.  stage 1: the mean shape (id and exp unused, basis may be
 *                NULL), writes part_frame only.  stage 2: the shape mean + [id | exp] basis^T.  Writes (never accumulates):
 *                  part_frame [8][T][12]  fp64, per chunk and frame dL/dR (R = Rz Ry Rx, row-major) and dL/dtrans
 *                  part_exp   [8][T][64]  per chunk and frame dL/dexp
 *                  part_id    [8][16][80] fp64, per chunk and frame-tile CTA dL/did (min(ceil(T / 64), 16) CTAs per chunk)
 * r3dp_fit_adam  sums the partials in a fixed order, adds lam_id mean(id^2) + lam_exp mean(exp^2) + lam_lap (lap(exp) + 0.3 lap(euler) +
 *                0.3 lap(trans)) (cal_lap_loss over frames) when step_idexp > 0, and takes torch's Adam step (lr, betas 0.9 / 0.999, eps
 *                1e-8) from x into x_next (not x): euler / trans at step step_frame, id / exp at step_idexp (0: copied unchanged, no
 *                regulariser).  grad (NULL or [80 + 70 T]) receives the gradient.
 * No host synchronisation and no allocation: a whole fit is capturable in a CUDA graph. */
int r3dp_fit_grad(const float* basis, const float* mean, const float* weight, const float* lms, int T, int L, int img_size, const double* x,
                  int stage, double* part_frame, float* part_exp, double* part_id, r3dp_stream_t stream);
int r3dp_fit_adam(const double* part_frame, const float* part_exp, const double* part_id, int T, int step_frame, int step_idexp, double lr,
                  double lam_id, double lam_exp, double lam_lap, const double* x, double* x_next, double* m, double* v, double* grad,
                  r3dp_stream_t stream);

/* ------------------------------------------------ audio2motion: the audio2secc VAE (modules/audio2motion/vae.py, inference path) ---
 * PitchContourVAEModel / VAEModel: audio features and f0 -> expression coefficients.  Activations are channels-last rows per frame; split fp16
 * rows hold [hi | lo] of each value, weights [hi | lo] of w * 2^10 (as r3dp_mf_conv3d with split).  The convolutions and GEMMs around the
 * WaveNets run on r3dp_mf_conv3d (1-D as D = H = 1, W = T).
 * r3dp_a2m_wn_layer  one WaveNet layer (flow_base.py:70-96) fused, (hidden, k) = (64, 3) or (256, 5), dilation 1, x_mask = 1: x [B,T,hidden]
 *                    fp32 -> x_out = x + res_skip[:hidden] (not last; a buffer other than x), skip [B,T,hidden] fp32 (+)= res_skip[hidden:]
 *                    (first: =), last: out [B,T, hi hidden | lo hidden] split fp16 = skip + res_skip.  cond: per-frame rows of cs floats,
 *                    this layer's cond_layer output with the in_layer bias added, rows interleaved (2c: tanh half, 2c + 1: sigmoid half of
 *                    channel c).  w: the packed steps of the in_layer and res_skip weights (audio2motion.py, pack_wn_layer); bias: res_skip's.
 * r3dp_a2m_input     audio [B,Tx,A] fp32 downsampled x0.5 (mean = 0: frame 2i, nearest; 1: the mean of frames 2i, 2i+1, linear) into split
 *                    rows of y (ys halves, lo at ylo): channels [0, A) the features, [A, Ap) zero; with pitch_table [300,128] fp32 also
 *                    [Ap, Ap+128) pitch_table[f0_to_coarse(f0[2i])] (mel_min, mel_span: pitch_utils' f0_mel_min, f0_mel_max - f0_mel_min)
 *                    and the 32 split channels of yb (ybs halves, lo at yblo): blink[2i] == 0, blink[2i] == 1 (int64 [B,Tx], NULL = 0),
 *                    mouth_amp[b], eye_amp[b] (NULL = 0), zeros
 * r3dp_a2m_split     x [R,C] fp32 -> y1 split rows [R, hi C | lo C] and / or y4 split rows per group of four [R/4, hi 4C | lo 4C]
 * r3dp_a2m_latent    z [B,16,T4] fp32 x temperature -> split rows [B*T4, hi 32 | lo 32] (channels 16..31 zero)
 * r3dp_a2m_store     x [N,C] fp32 x mask[n] (NULL = 1) -> out[n * ld + c] */
int r3dp_a2m_wn_layer(const float* x, float* x_out, const float* cond, int cs, const void* w_f16, const float* bias, float* skip, void* out_f16,
                      int B, int T, int hidden, int k, int first, int last, r3dp_stream_t stream);
int r3dp_a2m_input(const float* audio, int B, int Tx, int A, int Ap, int mean, const float* f0, const long long* blink, const float* mouth_amp,
                   const float* eye_amp, const float* pitch_table, float mel_min, float mel_span, void* y_f16, int ys, int ylo, void* yb_f16, int ybs,
                   int yblo, r3dp_stream_t stream);
int r3dp_a2m_split(const float* x, long long R, int C, void* y1_f16, void* y4_f16, r3dp_stream_t stream);
int r3dp_a2m_latent(const float* z, int B, int T4, float temperature, void* y_f16, r3dp_stream_t stream);
int r3dp_a2m_store(const float* x, const float* mask, long long N, int C, float* out, long long ld, r3dp_stream_t stream);

/* ------------------------------------------------ audio features: HuBERT (transformers' HubertModel, hubert-large architecture) ---
 * Split fp16 rows hold [hi | lo] of each value; weights are [N][hi Kp | lo Kp] of w * 2^10.  Every GEMM operand is split (three MMAs, fp32
 * accumulation).
 * r3dp_hb_gemm       y = A W^T + bias on wgmma (TMA producer warp, two consumer warpgroups, n128 tiles, 64-channel K steps).  A: M rows of
 *                    a_width halves, a_stride halves apart (a_stride < a_width reads overlapping windows: a strided conv's A row t is the k
 *                    frames from frame s t, a_stride = s * 2 seg); K channel kk sits at column (kk / seg) * 2 seg + kk % seg (hi), + seg (lo).
 *                    w [N][hi Kp | lo Kp].  epi 0: split rows into y (fp16, ldy halves, lo at ylo); 1: GELU, then as 0; 2: y fp32 (ldy floats)
 *                    += result; 3: y fp32 = result.  bias may be NULL.  Any M >= 1, N even; Kp and seg multiples of 64
 * r3dp_hb_pos_conv   the positional conv (k128, pad 64, last frame dropped, groups of 64 channels) on each of nseg segments of Lseg frames
 *                    with its own zero padding: y fp32 [M][H] += GELU(conv(x) + bias).  x: split rows [nseg * Lseg][hi H | lo H], rows >= M
 *                    zero; w [H][hi 8192 | lo 8192], K channel 64 j + i = tap j, input channel i of the output's group
 * r3dp_hb_attention  softmax(q k^T) v per head (head_dim 64; scale folded into q) within each of nseg consecutive segments of seg_len[i]
 *                    rows (<= 64 segments, lengths >= 1): qkv split rows [rows][ld], q / k / v of head h at columns 64 h, H + 64 h,
 *                    2H + 64 h (hi) and lo + those (lo), H = 64 heads.  o: split rows (os halves), hi at 64 h, lo at olo + 64 h
 * r3dp_hb_stats      stats = (mean, 1 / sqrt(var + 1e-7)) of x[0, L) in fp64 (Wav2Vec2FeatureExtractor's normalisation), deterministic
 * r3dp_hb_conv0      feature extractor layer 0 on F frames: ((x - mean) * rstd) conv w [C][10] (stride 5) + bias (may be NULL), LayerNorm
 *                    (g, b, eps), GELU -> split rows y (ys halves, lo at ylo); C a multiple of 32, at most 512
 * r3dp_hb_layernorm  LayerNorm of x [R][C] fp32 (C <= 1024), * g + b if given, GELU if gelu; yf fp32 rows (yfs floats) and / or split rows
 *                    yh (yhs halves, lo at yhlo) */
int r3dp_hb_gemm(const void* a_f16, int M, int a_width, int a_stride, int seg, const void* w_f16, int N, int Kp, const float* bias, int epi,
                 void* y, int ldy, int ylo, r3dp_stream_t stream);
int r3dp_hb_pos_conv(const void* x_f16, int nseg, int Lseg, int M, int H, const void* w_f16, const float* bias, float* y, r3dp_stream_t stream);
int r3dp_hb_attention(const void* qkv_f16, int rows, int ld, int lo, int heads, const int* seg_len, int nseg, void* o_f16, int os, int olo,
                      r3dp_stream_t stream);
int r3dp_hb_stats(const float* x, long long L, double* stats, r3dp_stream_t stream);
int r3dp_hb_conv0(const float* x, const double* stats, int F, int C, const float* w, const float* bias, const float* g, const float* b,
                  float eps, void* y_f16, int ys, int ylo, r3dp_stream_t stream);
int r3dp_hb_layernorm(const float* x, int R, int C, const float* g, const float* b, float eps, int gelu, float* yf, int yfs, void* yh_f16,
                      int yhs, int yhlo, r3dp_stream_t stream);

/* ------------------------------------------------ source images: ref_head_img, ref_torso_img and bg_img (real3d_infer.py:243-260) ---
 * img uint8 [H,W,3] RGB; seg [6,H,W] float32 (seg_u8 = 0) or uint8 (seg_u8 = 1) in _cal_seg_map's channel order (0 bg, 1 hair, 2 body skin,
 * 3 face skin, 4 clothes, 5 others).  64 <= H, W <= 1024.  Float outputs are [3,H,W] planes of (u - 127.5) / 127.5 in float32.
 * r3dp_src_inpaint      inpaint_torso_job up to the blur: img2 uint8 [H,W,3] = img with head pixels ((s1 + s3 + s5) != 0) zeroed, the torso
 *                       (9 rows) and neck (53 rows, after the torso) darkened copies written, numpy's negative-row wrap; flags uint8 [H,W]:
 *                       bit 0 kept in torso_img, bit 1 neck-inpainted.  tab_torso [9] / tab_neck [53]: numpy's 0.98 ** np.arange(L), float64
 * r3dp_src_compose      cv2.GaussianBlur(img2, (5,5), 4) at the neck-inpainted pixels, zero outside the torso mask -> torso_f32 and / or
 *                       torso_u8 [H,W,3]; head_f32 = img where s1 + s3 + s5 > 0.5, else 0 (each output may be NULL, not all)
 * r3dp_src_bg_distance  extract_background's first pass over F selected frames (segs + f seg_stride elements): each pixel's max over frames of
 *                       the squared distance to the frame's nearest non-bg (s0 == 0) pixel, maxd2 int32 [H,W], and the first frame
 *                       attaining it, argmax int32 [H,W]; has_fg int32 [F] = 1 where the frame has a non-bg pixel.  g: int16 scratch
 *                       [chunk,H,W] (frames are processed chunk at a time)
 * r3dp_src_bg_fill      the second pass: every pixel takes the colour of frame argmax[q] at q = its nearest pixel with maxd2 > 100 (itself
 *                       when maxd2 > 100; ties: smallest column, then smallest row) -> bg_u8 [H,W,3] and / or bg_f32.  frames: the selected
 *                       frames, uint8 [H,W,3] each, frame_stride bytes apart; g: int16 scratch [H,W]; has_bc int32 = 1 + the raster index of
 *                       the last pixel with maxd2 > 100 (0: none).  Pixel 0, when maxd2 > 100 there, takes the frame argmax has of that last
 *                       pixel, as the reference's fancy-index assignment leaves it
 * No host synchronisation and no allocation: capturable in a CUDA graph. */
int r3dp_src_inpaint(const unsigned char* img, const void* seg, int seg_u8, int H, int W, const double* tab_torso, const double* tab_neck,
                     unsigned char* img2, unsigned char* flags, r3dp_stream_t stream);
int r3dp_src_compose(const unsigned char* img, const void* seg, int seg_u8, const unsigned char* img2, const unsigned char* flags, int H, int W,
                     float* head_f32, float* torso_f32, unsigned char* torso_u8, r3dp_stream_t stream);
int r3dp_src_bg_distance(const void* segs, int seg_u8, long long seg_stride, int F, int H, int W, short* g, int chunk, int* maxd2, int* argmax,
                         int* has_fg, r3dp_stream_t stream);
int r3dp_src_bg_fill(const unsigned char* frames, long long frame_stride, const int* maxd2, const int* argmax, int H, int W, short* g,
                     int* has_bc, unsigned char* bg_u8, float* bg_f32, r3dp_stream_t stream);

/* ------------------------------------------------ the 'concat_debug' video frames (real3d_infer.py:494-521) --------------------------------
 * A frame is a uint8 RGB strip [512][2560][3]: panels source | driving SECC | image_raw | depth | image, 512 x 512 each.  dst is byte 0 of
 * frame 0's strip; frames are frame_stride bytes apart, rows row_pitch (>= 7680) bytes apart, so a strip may be a slice of a wider buffer.
 * Every panel is converted as the reference's float64 torch.cat makes it: clamp(-1, 1), then ((x + 1) / 2 * 255).int() in float64.
 * r3dp_debug_panels       panels 0, 1, 2 and 4 of B frames.  ref_gt [3,512,512] fp32 (the source image, every frame); secc [B,3,512,512]
 *                         fp32 (as ((secc + 1) * 127.5).int() / 127.5 - 1); feat [B,4096,feat_c] fp32, the render's channels-last features
 *                         with rgb in channels 0-2 (x8 nearest); image [B,3,512,512] fp32, the final frame.  Writes nothing else
 * r3dp_debug_depth_panel  panel 3 of F frames: depth [F,64,64] fp32, normalised by its min and max over all F frames in float32, x8
 *                         nearest, the one channel three times (a constant clip gives 0 / 0 = NaN, i.e. byte 0).  minmax: 2 unsigned of
 *                         device scratch.  Two launches; the min and max never leave the device
 * No host synchronisation and no allocation: capturable in a CUDA graph. */
int r3dp_debug_panels(const float* ref_gt, const float* secc, const float* feat, int feat_c, const float* image, int B, unsigned char* dst,
                      long long frame_stride, long long row_pitch, r3dp_stream_t stream);
int r3dp_debug_depth_panel(const float* depth, int F, unsigned* minmax, unsigned char* dst, long long frame_stride, long long row_pitch,
                           r3dp_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* R3DP_B200_H */
