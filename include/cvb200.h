/*
 * cvb200.h -- C ABI of libcvb200.so: the H100 (sm_90a) detector forward hot path.
 *
 * The reference (shanglianlm0525/CvPytorch) is pure Python on PyTorch and has no FFI; every entry
 * point below replaces a run of PyTorch/torchvision library calls on the reference's inference
 * path.  The "replaces" notes cite the reference file:line (paths relative to the reference checkout).
 *
 * Conventions
 *   - plain pointers + sizes only; no torch / C++ types cross this boundary.
 *   - every device buffer (activations, weights, workspaces, outputs) is OWNED BY THE CALLER; the
 *     library never allocates or frees device memory and keeps no reference after a call returns,
 *     except for the raw pointers baked into a CvbConvPlan (valid while the caller keeps them alive).
 *   - all work is enqueued on the cudaStream_t passed in (as void*); no call synchronises the
 *     device or reads device memory from the host, so every *_run entry point is CUDA-graph
 *     capturable.  Plan creation only encodes TMA descriptors on the host.
 *   - return value: 0 = CVB_OK, negative = error; cvb_last_error_string() gives the thread-local text.
 *
 * Activation layout ("split-NHWC"): two fp16 planes [2][B][H][W][C]; plane 0 = hi = fp16(x),
 * plane 1 = lo = fp16(x - hi).  hi+lo carries ~22 mantissa bits, so three fp16 tensor-core
 * products (hi*hi + hi*lo + lo*hi, fp32 accumulate) reproduce fp32 convolution to ~1e-5.
 */
#ifndef CVB200_H_
#define CVB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CVB_OK 0
#define CVB_ERR_INVALID (-1)   /* bad argument / unsupported shape            */
#define CVB_ERR_CUDA (-2)      /* CUDA runtime / driver error                 */
#define CVB_ERR_NO_DEVICE (-3) /* no sm_90 device / driver entry point found  */

#define CVB_ACT_NONE 0
#define CVB_ACT_SILU 1 /* x*sigmoid(x)   src/models/bricks/swish.py:9-25, nn.SiLU */
#define CVB_ACT_RELU 2

#define CVB_OUT_SPLIT16 0 /* two fp16 planes (hi, lo)          */
#define CVB_OUT_F32 1     /* plain fp32 NHWC (partials / heads) */
#define CVB_OUT_YOLO 2    /* fused YOLOv5 decode: the conv writes z rows + NMS histogram / per-row best scores (CvbConvDesc.yolo) */

/* A channel-slice view of an NHWC tensor. */
typedef struct CvbView {
  void* base;           /* device pointer to element (b=0,h=0,w=0,c=first channel of the view), plane 0 */
  int32_t B, H, W, C;   /* logical extent of the view                                                */
  int32_t c_pitch;      /* channels per pixel of the underlying buffer (>= C)                         */
  int64_t plane_stride; /* bytes from plane 0 (hi) to plane 1 (lo); ignored for fp32 tensors          */
} CvbView;

/*
 * Fused conv2d + folded-BN bias + activation (+ residual) (+ nearest-upsampled fp32 partial).
 *   out = act( conv(in, W) + up2x(partial) + bias ) + residual          (residual_before_act = 0, Darknet bottleneck)
 *   out = act( conv(in, W) + up2x(partial) + bias + residual )          (residual_before_act = 1, ResNet bottleneck:
 *                                                                        torchvision Bottleneck.forward `out += identity; relu`)
 * replaces: ConvModule.forward  src/models/bricks/conv_module.py:201-214 (conv -> BN -> act),
 *           Conv.forward        src/models/modules/yolo11_modules.py:27-39,
 *           the shortcut add of DarknetBottleneck.forward src/models/modules/yolo_modules.py:95-104,
 *           nn.UpsamplingNearest2d + torch.cat of UpsamplingModule.forward
 *           src/models/modules/yolo11_modules.py:388-397 (via conv1x1(up(x)) == up(conv1x1(x))),
 *           BN folding algebra src/utils/fuse.py:33-54 (done by the caller when packing weights).
 * Weights: device fp16 [2 planes][cout_pad][kh*kw*cin] with k = (ky*kw + kx)*cin + c  (K-major).
 */
/*
 * Fused head: 1x1 detect conv + sigmoid + box decode + NMS pre-pass in ONE kernel (out_kind = CVB_OUT_YOLO).  The conv's epilogue turns
 * the accumulator of (anchor a, pixel) into the z row the reference builds with permute + sigmoid + two slice writes + cat
 * (src/models/detects/yolov5_detect.py:42-55) and, when nms_workspace is given, accumulates what cvb_yolo_decode would have (score
 * histogram, per-row best score) -- the fp32 raw tensor [B,ny,nx,na*no] is never written or re-read.  Same arithmetic as
 * CVB_OUT_F32 conv + cvb_yolo_decode: bit-identical z.
 *   weights / bias: packed with ONE ANCHOR PER 128-WIDE N-TILE: row a*128 + o = output channel a*no + o of nn.Conv2d (o < no <= 96, the
 *   rest zero), i.e. cout_pad = na * 128; `out` only carries B/H/W (C = na * 128); base may be the z pointer.
 */
typedef struct CvbYoloDecode {
  int32_t na, no;          /* anchors per level (<= 4), outputs per anchor (5 + classes, <= 96) */
  float anchors_px[8];     /* anchor (w, h) in pixels = anchors * stride                        */
  float stride;
  float* z;                /* [B, z_rows, no] fp32; this level's rows start at z_off (a * ny * nx + y * nx + x inside the level) */
  int64_t z_rows, z_off;
  void* nms_workspace;     /* prepared with cvb_nms_workspace_reset (sized for A = z_rows), or NULL */
  float conf_thres;
  int32_t multi_label;
} CvbYoloDecode;

typedef struct CvbConvDesc {
  CvbView in;           /* split16 input view, C = cin (multiple of 16)              */
  CvbView out;          /* output view, C = cout                                     */
  const void* weights;  /* packed fp16 hi/lo weights, see above                      */
  int32_t cout_pad;     /* rows of the packed weight matrix (>= cout, multiple of 8) */
  const float* bias;    /* fp32 [cout_pad] folded bias (never NULL)                  */
  int32_t kh, kw, stride, pad, dilation;
  int32_t act;          /* CVB_ACT_*  */
  int32_t out_kind;     /* CVB_OUT_*  */
  CvbView residual;     /* base == NULL -> none; split16, same B/H/W/C as out        */
  CvbView up_partial;   /* base == NULL -> none; fp32 [B, ceil(H/2), ceil(W/2), C]   */
  int32_t block_n;      /* 0 = auto, else 32/64/128/256                              */
  int32_t sm_limit;     /* 0 = all SMs; else cap on the persistent grid              */
  int32_t no_resident;  /* 1 = never pin the weights in shared memory (tuning / testing)  */
  int32_t residual_before_act; /* see formula above */
  int32_t w_window;     /* 0 = off.  n > 0 ("row window" mode for tiny cin, used by the stem): `in` describes a
                           tensor that is physically zero-padded along W (1 column left, n-2 right: in.W =
                           out.W + n - 1, c_pitch == C) and the GEMM K chunk of filter row ky is the n adjacent
                           pixels starting at the output column, i.e. the packed weights are
                           [2][cout_pad][kh * n*C] with k = ky*n*C + kx*C + c and zeros for kx >= kw.
                           n*C must be 32 or 64.  Filter row ky reads input row h + ky - pad (rows outside the tensor are zero);
                           out.H is taken from the output view (allows the asymmetric 2-above/1-below padding of the
                           7x7/s2/p3 ResNet stem expressed as 4 rows over the space-to-depth input). */
  int32_t halo;         /* activation loading of multi-tap layers.  0 = auto (cost model), -1 = classic: one TMA box per filter tap,
                           1 / 2 = force "halo" mode where the layer allows it: the 8x16-pixel tile is loaded once per K chunk including
                           the filter halo (2: one box per input map; 1: one box per horizontal tap offset) and every tap is a
                           row-shifted shared-memory descriptor view of it -- up to 6x less L2->SM fill traffic for 3x3 layers. */
  const CvbYoloDecode* yolo; /* required iff out_kind == CVB_OUT_YOLO */
  float residual_scale; /* out = act(...) + residual_scale * residual (0 is read as 1): the learnable shortcut weight `alpha` of the YOLOv6
                           BottleRep block (src/models/modules/yolo_modules.py:474-492) */
  int32_t schedule;     /* CVB_SCHED_*: how the two MMA warpgroups share the work.  0 = auto (cost model), 1 = cooperative: both
                           warpgroups compute each 128-pixel tile and run its epilogue together, 2 = ping-pong: 64-pixel tiles alternate
                           between the warpgroups and one's epilogue overlaps the other's MMAs (plans that run one CTA per SM, without
                           the halo loader or the fused decode, with block_n = 128, or block_n <= 64 on a layer of at most 128 channels;
                           a plan that fits two CTAs per SM already overlaps one CTA's epilogue with the other's MMAs; anything else is
                           rejected).  Both give bit-identical outputs. */
} CvbConvDesc;

#define CVB_SCHED_AUTO 0
#define CVB_SCHED_COOPERATIVE 1
#define CVB_SCHED_PINGPONG 2

typedef struct CvbConvPlan CvbConvPlan;

int cvb_conv_plan_create(const CvbConvDesc* desc, CvbConvPlan** plan);
int cvb_conv_plan_run(const CvbConvPlan* plan, void* stream);
void cvb_conv_plan_destroy(CvbConvPlan* plan);
/* Diagnostics: attach a device buffer of rows * 16 int64 cycle counters (NULL detaches); every CTA then records how long its TMA
 * producer, MMA issuer and epilogue spent in total and waiting on each pipeline barrier
 * ([0..2] producer: total, wait free A slot, wait free weight slot; [4..7] MMA: total, wait accumulator, wait activations, wait
 * weights; [8..9] epilogue: total, wait accumulator).  *grid receives the number of counter rows: one per CTA, or with the ping-pong
 * schedule one per warpgroup (row r + grid * w for warpgroup w of CTA r; both rows carry the CTA's producer counters).
 * Used by tools/conv_pipeline_profile.py. */
int cvb_conv_plan_set_profile(CvbConvPlan* plan, long long* counters, int32_t* grid);
/* Run n plans back to back on one stream (one C call per forward instead of one per layer). */
int cvb_conv_plan_run_many(CvbConvPlan* const* plans, int32_t n, void* stream);

/*
 * Layout / precision conversion at the drop-in boundary (reference tensors are NCHW fp32).
 * replaces: nothing in the reference (it stays NCHW); this is the module-boundary adapter.
 */
int cvb_nchw_to_split(const float* src, int32_t B, int32_t C, int32_t H, int32_t W, const CvbView* dst,
                      void* stream);
int cvb_split_to_nchw(const CvbView* src, float* dst, void* stream);
/* fp32 NHWC view (e.g. head output) -> NCHW fp32 */
int cvb_f32nhwc_to_nchw(const CvbView* src, float* dst, void* stream);
/*
 * Stem input adapter: NCHW fp32 [B,3,H,W] -> space-to-depth split16 [B,H/2,W/2,16] (12 used,
 * channel = (dy*2+dx)*3 + c, 4 zero pad) so that the 6x6/s2/p2 stem conv
 * (src/models/backbones/det/yolov5_csp_darknet.py:36-45) becomes a 3x3/s1/p1 tensor-core conv.
 * dst may also be a zero-padded row-window layout [B,H/2,W/2+3,16] (data in columns pad_left..pad_left+W/2-1; the pad
 * columns must already be zero) consumed by a CvbConvDesc with w_window = 4: pad_left = 1 for the YOLOv5 6x6 stem,
 * pad_left = 2 for the ResNet 7x7/s2/p3 stem (== 4x4 taps over the space-to-depth input, torchvision resnet conv1).
 */
int cvb_stem_s2d(const float* src, int32_t B, int32_t H, int32_t W, const CvbView* dst, int32_t pad_left, void* stream);

/*
 * Same output from the camera-side format (SURVEY.md 8(f) rank 1): uint8 HWC frames [B,H,W,3].  Fuses the reference's input
 * transforms into the stem loader: ToTensor (src/data/transforms/det_transforms.py:85-99: HWC->CHW, channel reversal BGR->RGB when
 * reverse_channels != 0, float32 / 255) and Normalize (:102-109 = torchvision F.normalize, (x - mean[c]) / std[c] in fp32, mean/std
 * indexed by the OUTPUT channel; conf/coco_yolov5_s.yml:59 mean [0.406,0.456,0.485] std [0.225,0.224,0.229]).  Same operation order
 * and IEEE division as the reference, so dst is bit-identical to cvb_stem_s2d on the tensor those transforms would have produced;
 * the fp32 NCHW image never exists and the host->device copy shrinks 4x.  mean/std: host pointers to 3 floats.
 */
int cvb_stem_s2d_u8(const uint8_t* src, int32_t B, int32_t H, int32_t W, const float* mean, const float* std, int32_t reverse_channels,
                    const CvbView* dst, int32_t pad_left, void* stream);

/*
 * ResNet stem max pool 3x3 / stride 2 / pad 1 on a split16 tensor.
 * replaces: nn.MaxPool2d(3, 2, 1) of torchvision.models.resnet (src/models/backbones/seg/resnet.py:80-83).
 */
int cvb_maxpool3x3s2(const CvbView* x, const CvbView* y, void* stream);

/* split16 -> fp32 NHWC copy (an FPN level that is both a conv input and an upsampled partial of the next level) */
int cvb_split_to_f32nhwc(const CvbView* x, const CvbView* y, void* stream);

/*
 * GroupNorm with 8 channels per group (+ optional ReLU), per-sample statistics, split16 in/out.
 * replaces: nn.GroupNorm(32, 256) + nn.ReLU of the FCOS head towers (src/models/heads/fcos_head.py:39-50).
 * workspace: cvb_groupnorm_workspace_bytes(B, groups) bytes (fp64 sums), caller-owned.
 */
size_t cvb_groupnorm_workspace_bytes(int32_t B, int32_t groups);
int cvb_groupnorm_relu(const CvbView* x, int32_t groups, const float* gamma, const float* beta, float eps, int32_t relu,
                       const CvbView* y, void* workspace, size_t workspace_bytes, void* stream);

/*
 * Depthwise 3x3 convolution (stride 1, padding = dilation) + folded-BN bias + optional ReLU, split16 in/out.
 * weights: fp32 [9][C] tap-major (BN scale folded by the caller), bias fp32 [C].
 * replaces: the depthwise ConvModule of DepthwiseSeparableConvModule (src/models/bricks/depthwise_separable_conv_module.py:73-99)
 *           used by DepthwiseSeparableASPPModule / Deeplabv3PlusHead.fuse (src/models/heads/seg/deeplabv3plus_head.py:14-54).
 */
int cvb_dwconv3x3(const CvbView* x, const float* weights, const float* bias, int32_t dilation, int32_t relu, const CvbView* y,
                  void* stream);

/* nn.AdaptiveAvgPool2d(1) of the ASPP image-pool branch (src/models/heads/seg/deeplabv3_head.py:59-62): [B,H,W,C] -> [B,1,1,C] */
int cvb_global_avgpool(const CvbView* x, const CvbView* y, void* stream);

/* F.interpolate(mode='bilinear', align_corners=False) on split16 tensors, any size (deeplabv3plus_head.py:57,63) */
int cvb_bilinear_resize(const CvbView* x, const CvbView* y, void* stream);

/*
 * Fused bilinear upsample (align_corners=False) + argmax over classes: fp32 NHWC logits [B,h,w,>=nc] -> int64 labels [B,Ho,Wo].
 * replaces: F.interpolate(preds, size=targets.shape[-2:]) + torch.argmax(dim=1) (src/models/segmentors/encoder_decoder.py:132-133).
 */
int cvb_upsample_argmax(const CvbView* logits, int32_t nc, int64_t* labels, int32_t Ho, int32_t Wo, void* stream);

/*
 * SPPF pooling: y1=maxpool5(x), y2=maxpool5(y1), y3=maxpool5(y2) (stride 1, pad 2), written to
 * three channel slices.  replaces: SPPF.forward src/models/modules/yolo_modules.py:185-194 /
 * src/models/modules/yolo11_modules.py:282-288 (3 x nn.MaxPool2d + torch.cat).
 */
int cvb_sppf_pool(const CvbView* x, const CvbView* y1, const CvbView* y2, const CvbView* y3, void* stream);

/*
 * YOLOv5 decode of one level.  raw: fp32 NHWC [B,ny,nx,c_pitch>=na*no] conv output (+bias).
 *   z[b, z_off + (a*ny+y)*nx + x, :] = decode(sigmoid(raw))   (z row pitch = no floats, z_rows rows/img)
 *   xperm (optional) = raw permuted to [B,na,ny,nx,no]
 *   nms_workspace (optional): a workspace prepared with cvb_nms_workspace_reset(); the decode then also accumulates the
 *   NMS score histogram and the per-row best score (conf_thres / multi_label as later passed to cvb_yolo_nms with
 *   hist_ready = 1; z_rows must then be the A of that call, the workspace must have been sized for it), which saves one full
 *   pass over the prediction tensor and lets the NMS emit passes skip rows below their threshold.
 * replaces: YOLOv5Detect.forward src/models/detects/yolov5_detect.py:42-55, _make_grid :60-65.
 */
int cvb_yolo_decode(const CvbView* raw, int32_t na, int32_t no, const float* anchors_px /*[na*2]*/, float stride,
                    float* z, int64_t z_rows, int64_t z_off, float* xperm, void* nms_workspace, float conf_thres,
                    int32_t multi_label, void* stream);

/*
 * Batched YOLOv5 NMS.  prediction: fp32 [B, A, 5+nc].  Outputs (fixed capacity, device):
 *   det [B, max_det, 6] = (x1,y1,x2,y2,conf,cls), det_idx [B, max_det] = anchor*nc+cls of each kept
 *   row (the "NMS-surviving box index"), det_count [B].
 * replaces: non_max_suppression src/models/yolov5.py:62-153 (multi_label / best-class, class-offset
 *           4096, max_nms 30000, max_det 300; the 10 s wall-clock break :149-151 is NOT reproduced),
 *           xywh2xyxy :52-59, torchvision.ops.nms (third party) called at :137.
 * workspace: cvb_nms_workspace_bytes(B, A, nc) bytes, caller-owned, 256-byte aligned (histogram, counters, 64-bit candidate keys,
 *            per-row best scores).  The phase-B sort is one cooperative launch (grid = number of SMs).
 * status (device int32[4], optional): [0] overflow flag (candidate capacity exceeded), rest reserved.
 */
typedef struct CvbNmsParams {
  int32_t B, A, nc;
  float conf_thres;    /* compared in fp32: x > float(conf_thres) like the reference's tensor > scalar */
  double iou_thres;    /* compared in double: torchvision's CPU kernel tests float IoU > double threshold */
  int32_t multi_label; /* 1: one candidate per (box,class) pair; 0: best class only */
  int32_t max_nms;     /* 30000 */
  int32_t max_det;     /* 300   */
  float max_wh;        /* 4096 class offset; 0 = agnostic */
  int32_t hist_ready;  /* 1: histogram + per-row best scores were already produced by cvb_yolo_decode (all levels) */
} CvbNmsParams;

size_t cvb_nms_workspace_bytes(int32_t B, int32_t A, int32_t nc);
/* zero the per-image histogram / counters (only needed before cvb_yolo_decode(..., nms_workspace, ...)) */
int cvb_nms_workspace_reset(void* workspace, size_t workspace_bytes, int32_t B, void* stream);
int cvb_yolo_nms(const float* prediction, const CvbNmsParams* p, float* det, int32_t* det_idx, int32_t* det_count,
                 void* workspace, size_t workspace_bytes, int32_t* status, void* stream);

/*
 * FCOS decode of one pyramid level.  cls: fp32 NHWC [B,h,w,>=nc] logits; regcnt: fp32 NHWC [B,h,w,>=5] = (l,t,r,b raw
 * regression, centerness logit).  Writes at location offset loc_off (of n_total locations per image):
 *   scores[B,n_total] = sqrt(max_c sigmoid(cls) * sigmoid(cnt)), classes[B,n_total] = argmax + 1 (first maximum),
 *   boxes[B,n_total,4] = (cx - exp(l*scale), cy - exp(t*scale), cx + exp(r*scale), cy + exp(b*scale)),
 *   (cx, cy) = (x*stride + stride/2, y*stride + stride/2).
 * replaces: FCOSDetect.forward / _reshape_cat_out / _coords2boxes / coords_fmap2orig
 *           (src/models/detects/fcos_detect.py:42-62,14-31,155-186) and ScaleExp (src/models/heads/fcos_head.py:13-19).
 */
int cvb_fcos_decode(const CvbView* cls, const CvbView* regcnt, int32_t nc, float stride, float scale, float* scores,
                    int32_t* classes, float* boxes, int64_t n_total, int64_t loc_off, void* stream);

/*
 * FCOS post-processing, one image per CTA, no host sync: top-k by score (ties: lower location index), score >= thres,
 * class offset = cls * (max candidate coordinate + 1), greedy NMS with '+1' areas keeping boxes with iou <= thres (fp32).
 * Outputs are fixed capacity [B,topk] (+ out_count[B]); out_loc = kept location indices ("NMS-surviving box index").
 * replaces: torch.topk + FCOSDetect._post_process / batched_nms / box_nms (src/models/detects/fcos_detect.py:64-153; the
 *           reference's python while-loop with .item() per kept box, and its torch.stack that needs equal counts).
 */
int cvb_fcos_nms(const float* scores, const int32_t* classes, const float* boxes, int32_t B, int32_t N, float score_thres,
                 float iou_thres, int32_t topk, float* out_scores, int32_t* out_classes, float* out_boxes, int32_t* out_loc,
                 int32_t* out_count, int32_t* status, void* stream);

/*
 * YOLOX post-processing (SURVEY.md 8 row a16), replaces yolox_post_process (src/models/yolox.py:18-68) incl. the third-party
 * torchvision.ops.batched_nms call at :64.
 *
 * cvb_yolox_decode: one head level.  reg_obj / cls: fp32 NHWC views [B,h,w,>=5] (reg 4, obj 1) and [B,h,w,>=nc] (class logits),
 * i.e. the three predictors of heads/yolox_head.py:74-86 before their torch.cat.  Writes one 8-float record per location into
 * cand[B, A, 8] at rows off .. off + h*w:  (x1, y1, x2, y2, obj, class_conf, class_pred, obj * class_conf) with
 * xy = (p + grid) * stride, wh = exp(p) * stride (:33-35), sigmoids (:37-39), corner form (:46-51), best class (:57).
 *
 * cvb_yolox_nms: per image keeps locations with obj * class_conf >= conf_thres (:58), then batched_nms(boxes, scores, class, iou_thres):
 * stable descending score order; more than `vanilla_above` boxes (torchvision: numel > 4000 on CPU tensors, i.e. 1000 boxes;
 * 5000 on CUDA tensors) -> class-wise NMS on the raw boxes, else one NMS on boxes + class * (max_coordinate + 1); fp32 IoU
 * compared in double, areas without +1.  det[B, A, 7] receives the kept rows (x1, y1, x2, y2, obj, class_conf, class_pred) in
 * score order, det_count[B] their number (the reference returns None for 0).  A <= 16384.  workspace: cvb_yolox_workspace_bytes.
 */
size_t cvb_yolox_workspace_bytes(int32_t B, int32_t A);
int cvb_yolox_decode(const CvbView* reg_obj, const CvbView* cls, int32_t nc, float stride, float* cand, int64_t A, int64_t off, void* stream);
int cvb_yolox_nms(const float* cand, int32_t B, int32_t A, float conf_thres, double iou_thres, int32_t vanilla_above, float* det,
                  int32_t* det_count, void* workspace, size_t workspace_bytes, void* stream);

/*
 * Output side of the path (SURVEY.md 8(f) rank 2), on the device instead of a per-image `.cpu().numpy()` loop.
 *
 * cvb_rescale_clip_boxes: rows [B, M, row_stride] fp32 (x1, y1, x2, y2 first), in place for the first count[b] rows:
 *   x -= pad[1]; y -= pad[0]; x /= scale[1]; y /= scale[0]; clip to [0, width] / [0, height]
 *   (src/models/yolov5.py:274-281, src/models/yolox.py:171-178, src/models/fcos.py:150-161); pads / scales / wh = device [B,2] fp32
 *   (wh = width, height).  Same fp32 operations as the numpy lines: bit-identical results.
 * cvb_confusion_matrix: cm[num_classes, num_classes] (int64, accumulated) += bincount(num_classes * gt[mask] + pred[mask]) with
 *   mask = 0 <= gt < num_classes (src/evaluator/eval_segmentation.py:52-57); gt / pred = int64 label maps of n pixels; num_classes <= 64.
 */
int cvb_rescale_clip_boxes(float* rows, int32_t B, int32_t M, int32_t row_stride, const int32_t* count, const float* pads, const float* scales,
                           const float* wh, void* stream);
int cvb_confusion_matrix(const int64_t* gt, const int64_t* pred, int64_t n, int32_t num_classes, int64_t* cm, void* stream);

/*
 * Input side of the path (SURVEY.md 8(f) rank 1): the reference's Resize(size=[640,640], keep_ratio=True, fill=[114,114,114]) transform
 * (src/data/transforms/det_transforms.py:162-198, conf/coco_yolov5_s.yml:56) on the device: cv2.resize(INTER_LINEAR) of each uint8 HWC
 * frame to (oh, ow) -- OpenCV's 11-bit fixed-point 8-bit bilinear kernel restated, bit-identical to cv2 4.x -- and the constant border of
 * cv2.copyMakeBorder, for a batch of frames of DIFFERENT sizes.  The output [B,out_h,out_w,3] uint8 is what cvb_stem_s2d_u8 consumes.
 *   src_ptrs: device array of B device pointers (frame b = uint8 [h_b, w_b, 3]); geom: device int32 [B,6] = (h, w, oh, ow, top, left) as
 *   det_transforms.py:177-189 computes them (host side: python round(), see cvpytorch_b200.ops.letterbox_geometry); fill: host int32[3].
 */
int cvb_letterbox_u8(const uint8_t* const* src_ptrs, const int32_t* geom, int32_t B, int32_t out_h, int32_t out_w, const int32_t* fill,
                     uint8_t* dst, void* stream);

/*
 * Output side, COCO records on the device (SURVEY.md 8(f) rank 2): replaces CocoEvaluator.prepare_for_coco_detection + convert_to_xywh
 * (src/evaluator/eval_coco.py:87-111, 200-202) for the fixed-capacity detections of a batch.  rows [B, M, row_stride] fp32 =
 * (x1, y1, x2, y2, score, class, ...) after cvb_rescale_clip_boxes, count [B]; image_ids device int64 [B]; id2category device int32
 * [num_classes] or NULL (dataset.id2category).  Writes, compacted in image order, rec_ids [n,2] int64 = (image_id, category_id) and
 * rec_box [n,5] fp32 = (x, y, x2 - x1, y2 - y1, score) (the fp32 subtraction of the torch lines), and *total = n (device int32).
 */
int cvb_coco_pack(const float* rows, int32_t B, int32_t M, int32_t row_stride, const int32_t* count, const int64_t* image_ids,
                  const int32_t* id2category, int32_t num_classes, int64_t* rec_ids, float* rec_box, int32_t* total, void* stream);

/*
 * Training step of the YOLOX C3 block (SURVEY.md 8(f) rank 3; BASELINE.json configs[3]): one  BaseConv = nn.Conv2d(bias=False) ->
 * nn.BatchNorm2d (batch statistics) -> SiLU  (src/models/modules/yolox_modules.py:35-55) forward and backward, i.e. what
 * trainer.py:177-207 gets from cuDNN / ATen autograd, as bf16 wgmma implicit GEMMs + element-wise passes (csrc/train_kernels.cu).
 * All activations / gradients: device bf16 NHWC, dense ([B,H,W,C]); convolutions k = 1 or 3, stride 1, pad k/2.  Every channel count of the
 * convolutions (cin, cout) is 16, 32 or a multiple of 64: a 16- or 32-channel tensor is one partial 64-channel K chunk / N tile.
 *
 * cvb_train_pack_weights: fp32 master weights [cout,cin,k,k] -> w_fwd bf16 [cout][k*k][kpad(cin)] and w_bwd bf16 [cin][k*k][kpad(cout)]
 *   (taps rotated by 180 degrees: the operand of the backward-data convolution); kpad(c) = c rounded up to a multiple of 64, the padding
 *   zero (16 and 32 channels only; kpad(c) = c otherwise).
 * cvb_train_conv: out[B,H,W,cout] = conv(x[B,H,W,cin], w_packed [cout][k*k][cin]).  Forward: (x, w_fwd).  Backward-data: (dy, w_bwd) with
 *   cin/cout swapped.  y_prev / bn_stat_prev != NULL: SiLU' epilogue -- the result is multiplied by silu'(y_prev * scale + shift) of the
 *   layer that produced this conv's input (bn_stat layout below), giving dz of that layer directly.
 *   stride = 2 (k = 3, pad 1; the downsampling BaseConv in front of every CSPLayer, src/models/backbones/det/csp_darknet.py): the forward
 *   reads the input through four parity tensor maps, out is [B,(H-1)/2+1,(W-1)/2+1,cout].
 * cvb_train_conv_dgrad_s2: backward-data of that stride-2 convolution, dx[B,H,W,cin] from dy[B,Ho,Wo,cout] and w_bwd: four dense
 *   sub-convolutions, one per parity class of dx (1 + 2 + 2 + 4 taps), same optional SiLU' epilogue.
 * cvb_train_conv_wgrad: dw[cout][k*k][cin] (fp32, ZEROED BY THE CALLER, accumulated with atomics) += sum over pixels of dy x (shifted x);
 *   x is [B,H,W,cin], dy the conv output's gradient (stride 1: same H, W; stride 2: (H-1)/2+1 etc.); output channels in blocks of 256,
 *   128 or 64, the widest that divides cout (cout = 16 or 32: one block).
 * cvb_train_bn_stats: batch mean / biased variance of y over npix = B*H*W -> stat [4][C] fp32 = (mean, rstd, scale = gamma*rstd,
 *   shift = beta - mean*scale); running_mean / running_var (may be NULL) updated like nn.BatchNorm2d (momentum, unbiased variance).
 *   sums_scratch: [2][C] fp32 (sums of y - y[pixel 0] and of its square: the variance keeps its precision when |mean| >> std).
 * cvb_train_bn_silu_fwd: out = silu(y * scale + shift).
 * cvb_train_bn_silu_bwd: g = d(loss)/d(out) (or, g_is_dz != 0, already multiplied by silu'): sums [2][C] = (dbeta, dgamma) and
 *   dy = gamma * rstd * (dz - dbeta / N - xhat * dgamma / N)   (the batch-norm backward of torch.autograd).
 *
 * Whole-backbone training (CSPDarknet, src/models/backbones/det/csp_darknet.py:25-129) adds the Focus stem and the SPPF pools:
 * cvb_train_focus_s2d: img fp32 NCHW [B,3,H,W] (H, W even) -> out bf16 NHWC [B,H/2,W/2,16], channel 3 * patch + c in the reference's patch
 *   order (top-left, bottom-left, top-right, bottom-right; src/models/modules/yolo_modules.py:19-37), channels 12..15 zero.  The stem conv
 *   then runs as a 16 -> cout cvb_train_conv with the reference weight zero-padded to 16 input channels.  No input gradient.
 * cvb_train_spp_pool_fwd: a bf16 NHWC [B,H,W,C] (C % 8 == 0) -> cat [B,H,W,4C] = [a | maxpool5(a) | maxpool9(a) | maxpool13(a)] (stride 1,
 *   padding k/2, the pools in parallel: yolo_modules.py:165-194) and idx uint8 [3][B*H*W][C], the winner's row-major offset in its window
 *   (ties: the first maximal element, as torch's max_pool2d).
 * cvb_train_spp_pool_bwd: g = d(loss)/d(cat) [B,H,W,4C], idx of the forward -> da [B,H,W,C] = g[..., :C] + the pooled gradients routed to
 *   their winners; a gather summed in fp32 in a fixed order (bitwise reproducible).
 * cvb_train_sppf_chain_fwd: the chained SPPF of YOLOv5 (kernel_sizes = 5: y1 = maxpool5(a), y2 = maxpool5(y1), y3 = maxpool5(y2)) ->
 *   cat [B,H,W,4C] = [a | y1 | y2 | y3] (the values of the parallel pools) and idx uint8 [3][B*H*W][C]: per stage, the row-major offset
 *   (0..24) of the first maximum of the 5 x 5 window of that stage's input (NaN propagates, as torch's max_pool2d).
 * cvb_train_sppf_chain_bwd: g = d(loss)/d(cat), idx of the forward -> da [B,H,W,C], autograd through the chain (y3 -> y2 -> y1 -> a, each
 *   stage adding its slice of g); deterministic fp32 gathers, scratch: 2 * B*H*W*C floats owned by the caller.
 *
 * YOLOX neck and head training (src/models/necks/yolox_neck.py:13-74, src/models/heads/yolox_head.py:14-88) adds:
 * cvb_train_upsample_cat_fwd: cat [B,2h,2w,Ca+Cb] = [nearest_up2(a [B,h,w,Ca]) | b [B,2h,2w,Cb]] (the neck's top-down upsample + concat,
 *   the upsampled map first).  Ca, Cb multiples of 8; a plain copy, bit-exact.
 * cvb_train_upsample_cat_bwd: g = d(loss)/d(cat) -> da [B,h,w,Ca] = 2x2 sum of g[..., :Ca] (fp32 in a fixed order, rounded to bf16 once)
 *   and db = g[..., Ca:]; no atomics, bitwise reproducible.
 * cvb_train_conv_pad / cvb_train_conv_wgrad_pad: cvb_train_conv / cvb_train_conv_wgrad at stride 1 with padding `pad`: the output is
 *   (H + 2 pad - k + 1) x (W + 2 pad - k + 1), tap t reads (h + t / k - pad, w + t % k - pad).  k = 1 with pad -1, 0 or 1; k = 3 with pad 1.
 *   The head stems are 1x1 convs with pad 1 (every head map is 2 pixels larger than its feature map); their backward-data is the pad
 *   k - 1 - 1 = -1 conv of dy with w_bwd (the border is cropped).  cvb_train_conv / cvb_train_conv_wgrad are these with pad = k / 2.
 * cvb_train_pred_conv: the head's prediction convs (1x1, bias, no BatchNorm or activation).  A cout_pad-wide GEMM over x [B,H,W,cin] with
 *   w_packed = cvb_train_pack_weights of the weight zero-padded to cout_pad rows; out fp32 NCHW [B,c_tot,H,W] channels
 *   [c_off, c_off + cout) = GEMM columns [0, cout) + bias (the other channels are not written).  cout_pad = cout rounded up to 16, 32 or a
 *   multiple of 64.
 * cvb_train_pred_grad: g fp32 NCHW [B,c_tot,h,w] (the loss's gradient of the head output) -> dy bf16 NHWC [B,h,w,cout_pad] = channels
 *   [c_off, c_off + cout) of g, zero past cout (the operand of backward-data / backward-weight), and dbias [cout] = the sum of those
 *   channels over images and pixels (fp32, fixed order).
 */
int cvb_train_pack_weights(const float* w, int32_t cout, int32_t cin, int32_t k, void* w_fwd, void* w_bwd, void* stream);
int cvb_train_conv(const void* x, int32_t B, int32_t H, int32_t W, int32_t cin, const void* w_packed, int32_t cout, int32_t k, int32_t stride, void* out,
                   const void* y_prev, const float* bn_stat_prev, void* stream);
int cvb_train_conv_dgrad_s2(const void* dy, int32_t B, int32_t Ho, int32_t Wo, int32_t cout, const void* w_bwd, int32_t cin, int32_t H, int32_t W, void* dx,
                            const void* y_prev, const float* bn_stat_prev, void* stream);
int cvb_train_conv_wgrad(const void* x, const void* dy, int32_t B, int32_t H, int32_t W, int32_t cin, int32_t cout, int32_t k, int32_t stride, float* dw,
                         void* stream);
int cvb_train_bn_stats(const void* y, int64_t npix, int32_t C, const float* gamma, const float* beta, float eps, float momentum, float* running_mean,
                       float* running_var, float* sums_scratch, float* stat, void* stream);
int cvb_train_bn_silu_fwd(const void* y, int64_t npix, int32_t C, const float* stat, void* out, void* stream);
int cvb_train_bn_silu_bwd(const void* g, int32_t g_is_dz, const void* y, int64_t npix, int32_t C, const float* stat, const float* gamma, float* sums,
                          void* dy, void* stream);
int cvb_train_focus_s2d(const float* img, int32_t B, int32_t H, int32_t W, void* out, void* stream);
int cvb_train_spp_pool_fwd(const void* a, int32_t B, int32_t H, int32_t W, int32_t C, void* cat, void* idx, void* stream);
int cvb_train_spp_pool_bwd(const void* g, const void* idx, int32_t B, int32_t H, int32_t W, int32_t C, void* da, void* stream);
int cvb_train_sppf_chain_fwd(const void* a, int32_t B, int32_t H, int32_t W, int32_t C, void* cat, void* idx, void* stream);
int cvb_train_sppf_chain_bwd(const void* g, const void* idx, int32_t B, int32_t H, int32_t W, int32_t C, float* scratch, void* da, void* stream);
int cvb_train_upsample_cat_fwd(const void* a, int32_t B, int32_t h, int32_t w, int32_t Ca, const void* b, int32_t Cb, void* cat, void* stream);
int cvb_train_upsample_cat_bwd(const void* g, int32_t B, int32_t h, int32_t w, int32_t Ca, int32_t Cb, void* da, void* db, void* stream);
int cvb_train_conv_pad(const void* x, int32_t B, int32_t H, int32_t W, int32_t cin, const void* w_packed, int32_t cout, int32_t k, int32_t pad, void* out,
                       const void* y_prev, const float* bn_stat_prev, void* stream);
int cvb_train_conv_wgrad_pad(const void* x, const void* dy, int32_t B, int32_t H, int32_t W, int32_t cin, int32_t cout, int32_t k, int32_t pad, float* dw,
                             void* stream);
int cvb_train_pred_conv(const void* x, int32_t B, int32_t H, int32_t W, int32_t cin, const void* w_packed, int32_t cout, int32_t cout_pad, const float* bias,
                        float* out, int32_t c_tot, int32_t c_off, void* stream);
int cvb_train_pred_grad(const float* g, int32_t B, int32_t c_tot, int32_t h, int32_t w, int32_t c_off, int32_t cout, int32_t cout_pad, void* dy, float* dbias,
                        void* stream);

/* SyncBatchNorm (nn.SyncBatchNorm in training mode: batch statistics over every rank's pixels).  The caller runs the collectives between
 * the calls; nothing here synchronises the host, so the whole sequence can be captured in a CUDA graph.
 * cvb_train_bn_partial: y [npix][C] bf16 (16-byte aligned, C % 8 == 0, C <= 2048) -> record fp64 [2C + 1] = (mean [C], M2 [C] = sum of
 *   squared deviations from that mean, npix).  sums_scratch: [2][C] fp32, as cvb_train_bn_stats.  Records merge; the pivoted sums of
 *   cvb_train_bn_stats do not (every rank's pivot is a different pixel).  npix = 0 is refused: unlike nn.SyncBatchNorm, a rank with an
 *   empty shard cannot take part (the training convolutions refuse B = 0 before the BatchNorm is reached).
 * cvb_train_bn_merge: records fp64 [world][2C + 1] (every rank's record, in rank order, as all_gather lays them out) -> Chan's pairwise merge
 *   in rank order in fp64 (every rank computes the same bits) -> stat [4][C] and the running statistics exactly as cvb_train_bn_stats computes
 *   them from a mean, a biased variance and a count; count fp64 [1] = the global pixel count, left on the device for the backward.
 *   Every record's count must be positive (as cvb_train_bn_partial writes them); a zero count would divide 0 by 0 in the merge.
 * cvb_train_bn_silu_bwd_reduce: the first half of cvb_train_bn_silu_bwd: sums [2][C] = this rank's (dbeta, dgamma).
 * cvb_train_bn_silu_bwd_apply: the second half, from the sums summed over every rank and N = *count (device fp64, e.g. cvb_train_bn_merge's):
 *   dy = gamma * rstd * (dz - sums[0] / N - xhat * sums[1] / N).
 */
int cvb_train_bn_partial(const void* y, int64_t npix, int32_t C, float* sums_scratch, double* record, void* stream);
int cvb_train_bn_merge(const double* records, int32_t world, int32_t C, const float* gamma, const float* beta, float eps, float momentum,
                       float* running_mean, float* running_var, float* stat, double* count, void* stream);
int cvb_train_bn_silu_bwd_reduce(const void* g, int32_t g_is_dz, const void* y, int64_t npix, int32_t C, const float* stat, float* sums, void* stream);
int cvb_train_bn_silu_bwd_apply(const void* g, int32_t g_is_dz, const void* y, int64_t npix, int32_t C, const float* stat, const float* gamma,
                                const float* sums, const double* count, void* dy, void* stream);

/* YOLOX training loss (src/losses/det/yolox_loss.py:73-436; csrc/yolox_loss.cu): SimOTA assignment, the IoU / objectness / class losses
 * and their gradient with respect to the head outputs.  preds[l]: fp32 NCHW [B, 5 + nc, h_l, w_l] (read in place), shapes[4 l ..] =
 * (B, 5 + nc, h_l, w_l), strides[l] > 0, 1 <= nlev <= 4; anchors in level order, row-major within a level (A = sum h_l w_l).
 * targets: fp32 [B, max_gt, 5] rows (class, cx, cy, w, h) in pixels, 1 <= max_gt <= 1024; an image uses its first nlabel rows, nlabel =
 * the number of rows with a positive sum.
 * cvb_train_yolox_loss_fwd: out fp32 [6] = (loss, iou_loss, conf_loss, cls_loss, num_fg / max(num_gt, 1), num_fg) with num_fg = max(foreground
 *   anchors, 1); matched_gt int32 [B, A] (the matched GT row, -1 = background) and matched_iou fp32 [B, A] (0 for background).  Ties: the lower
 *   anchor index in a GT's top-k, the lower GT index in the conflict argmin; a GT in an image without candidate anchors matches nothing.
 *   workspace: cvb_train_yolox_loss_workspace_bytes(B, A) bytes, 256-byte aligned, owned by the caller.  No host sync; bitwise reproducible.
 * cvb_train_yolox_loss_bwd: grads[l] fp32 NCHW, shapes of preds[l] (every element written) = d(sum_i grad_out[i] out[i]) / d(preds[l]) for
 *   i < 4, under the forward's assignment (matched_gt, matched_iou, fwd_out = its out).  grad_out: fp32 [4] on the device.
 */
/* YOLOv5 training loss (src/losses/yolov5_loss.py:135-278; csrc/yolov5_loss.cu): build_targets' candidate list, the CIoU box,
 * objectness and class BCE losses and their gradient with respect to the detect convs' outputs.  preds[l]: fp32 NCHW [B, na (5 + nc), ny_l,
 * nx_l] (read in place as [B, na, 5 + nc, ny, nx]), shapes[4 l ..] = (B, na (5 + nc), ny_l, nx_l), 1 <= nlev <= 4, 1 <= na <= 8.
 * anchors: host fp32 [nlev][na][2] in grid units; balance: host fp32 [nlev]; hyp: host fp32 [5] = (anchor_t, box, obj, cls, gr).
 * targets: fp32 [nt, 6] rows (image, class, cx, cy, w, h) normalised to [0, 1] on the device, nt >= 0.  A class outside [0, nc) gets no
 * one-hot entry; an image index outside [0, B) matches nothing.  cap = 5 na nt candidates per level.
 * cvb_train_yolov5_loss_fwd: out fp32 [4] = (loss, lbox, lobj, lcls) of the reference ((lbox + lobj + lcls) B with the hyper-parameter
 *   weights applied); per level l the candidate list in the reference's order: ncand[l], cand_idx int32 [nlev][cap][5] = (image, anchor,
 *   gj, gi, class) and cand_box fp32 [nlev][cap][6] = (tbox x, y, w, h, anchor w, h).  workspace: cvb_train_yolov5_loss_workspace_bytes(nlev,
 *   na, nt) bytes, 256-byte aligned, kept for the backward.  No host sync; bitwise reproducible.
 * cvb_train_yolov5_loss_bwd: grads[l] fp32, shapes of preds[l] (every element written) = grad_out[0] d(loss)/d(preds[l]) under the
 *   forward's candidates and workspace.  grad_out: fp32 [1] on the device.
 */
size_t cvb_train_yolov5_loss_workspace_bytes(int32_t nlev, int32_t na, int32_t nt);
int cvb_train_yolov5_loss_fwd(const float* const* preds, const int32_t* shapes, const float* anchors, const float* balance, int32_t nlev, int32_t na,
                              int32_t nc, const float* targets, int32_t nt, const float* hyp, int32_t* cand_idx, float* cand_box, int32_t* ncand,
                              float* out, void* workspace, size_t ws_bytes, void* stream);
int cvb_train_yolov5_loss_bwd(const float* const* preds, const int32_t* shapes, const float* anchors, const float* balance, int32_t nlev, int32_t na,
                              int32_t nc, const float* targets, int32_t nt, const float* hyp, const int32_t* cand_idx, const float* cand_box,
                              const int32_t* ncand, const void* workspace, size_t ws_bytes, const float* grad_out, float* const* grads, void* stream);

/* FCOS training loss (src/losses/fcos_loss.py; csrc/fcos_loss.cu): GenTargets' point assignment, the sigmoid focal, centerness BCE and
 * 1 - GIoU losses and their gradient with respect to the head outputs.  Per level l (1 <= nlev <= 8): cls[l] fp32 NCHW [B, nc, h_l, w_l],
 * cnt[l] [B, 1, h_l, w_l], reg[l] [B, 4, h_l, w_l] (ltrb), all read in place; shapes[12 l ..] = the three shapes in that order.
 * strides[l]: positive integers (as fp32); limit_range fp32 [nlev][2] = (lo, hi), lo < hi.  Points in level order, row-major within a level
 * (A = sum h_l w_l), at (column stride + stride / 2, row stride + stride / 2).  boxes: fp32 [B, m, 4] (x1, y1, x2, y2 in pixels, 16-byte
 * aligned), labels: int32 [B, m], 0 <= m <= 1024 (both may be NULL when m = 0); padded rows are -1.  A (point, GT) pair is positive when the
 * point is strictly inside the box, max(l, t, r, b) is in (lo, hi] and the centre offset is below 1.5 stride; a point's GT is the first
 * minimum of the area over the m rows (99999999 for a pair that is not positive), and a point without a positive pair is background.  A
 * label outside 1..nc gives an all-zero one-hot row.  m = 0 gives an all-background batch (the reference raises).
 * cvb_train_fcos_loss_fwd: out fp32 [4] = (cls_loss, cnt_loss, reg_loss, total), each term the batch mean of the image's sum over
 *   max(num_pos_b, 1); matched_gt int32 [B, A] (-1 = background) and num_pos int32 [B], both kept for the backward; targets (optional,
 *   NULL to skip) fp32 [B, A, 5] = the point's centerness and (l, t, r, b) regression targets, -1 for background.  workspace:
 *   cvb_train_fcos_loss_workspace_bytes(B, A, nc) bytes, 256-byte aligned, owned by the caller.  No host sync; bitwise reproducible.
 * cvb_train_fcos_loss_bwd: gcls / gcnt / greg[l] fp32 NCHW, shapes of cls / cnt / reg[l] (every element written) = d(sum_i grad_out[i]
 *   out[i]) / d(outputs) under the forward's matched_gt and num_pos.  grad_out: fp32 [4] on the device.  A logit whose sigmoid saturates
 *   against its target gives an inf loss and a NaN gradient, as the reference does.
 */
size_t cvb_train_fcos_loss_workspace_bytes(int32_t B, int32_t A, int32_t nc);
int cvb_train_fcos_loss_fwd(const float* const* cls, const float* const* cnt, const float* const* reg, const int32_t* shapes, const float* strides,
                            const float* limit_range, int32_t nlev, const float* boxes, const int32_t* labels, int32_t B, int32_t m,
                            int32_t* matched_gt, int32_t* num_pos, float* targets, float* out, void* workspace, size_t ws_bytes, void* stream);
int cvb_train_fcos_loss_bwd(const float* const* cls, const float* const* cnt, const float* const* reg, const int32_t* shapes, const float* strides,
                            const float* limit_range, int32_t nlev, const float* boxes, const int32_t* labels, int32_t B, int32_t m,
                            const int32_t* matched_gt, const int32_t* num_pos, const float* grad_out, float* const* gcls, float* const* gcnt,
                            float* const* greg, void* stream);

size_t cvb_train_yolox_loss_workspace_bytes(int32_t B, int32_t A);
int cvb_train_yolox_loss_fwd(const float* const* preds, const int32_t* shapes, const float* strides, int32_t nlev, int32_t nc, const float* targets,
                             int32_t B, int32_t max_gt, int32_t* matched_gt, float* matched_iou, float* out, void* workspace, size_t ws_bytes,
                             void* stream);
int cvb_train_yolox_loss_bwd(const float* const* preds, const int32_t* shapes, const float* strides, int32_t nlev, int32_t nc, const float* targets,
                             int32_t B, int32_t max_gt, const int32_t* matched_gt, const float* matched_iou, const float* fwd_out,
                             const float* grad_out, float* const* grads, void* stream);

/* Model EMA (src/utils/ema.py ModelEMA.update; csrc/ema.cu): one EMA step over every entry of a table in ONE launch,
 * ema[j] = fl(fl(ema[j] * decay) + fl(src[j] * one_minus_decay)) for j < numel, fp32, no FMA contraction: bitwise the reference's
 * `item *= decay; item += (1 - decay) * src` with decay = (float)d and one_minus_decay = (float)(1.0 - d) rounded from the host's double d.
 * cvb_ema_table_upload: checks the host table entries [n] (n >= 1; numel >= 0; ema and src non-null when numel > 0) and enqueues its copy
 *   on `stream` into `table`, caller-owned device memory of n * CVB_EMA_TABLE_ENTRY_BYTES bytes, 16-byte aligned.  The entries' ema ranges
 *   must not overlap each other or any src range.  Not capturable (host-to-device copy from pageable memory).
 * cvb_ema_update: the step over an uploaded table of n entries; any pointer alignment (float4 where ema and src are both 16-byte aligned).
 *   No host sync, CUDA-graph capturable.
 */
#define CVB_EMA_TABLE_ENTRY_BYTES 32
typedef struct {
  float* ema;       /* fp32, contiguous, updated in place */
  const float* src; /* fp32, contiguous, the model's tensor */
  int64_t numel;
} CvbEmaEntry;
int cvb_ema_table_upload(const CvbEmaEntry* entries, int32_t n, void* table, void* stream);
int cvb_ema_update(const void* table, int32_t n, float decay, float one_minus_decay, void* stream);

/* SGD step (torch.optim.SGD under torch.amp.GradScaler; csrc/sgd.cu): every parameter of every group in ONE launch, fp32, bitwise the
 * reference's GradScaler.unscale_ + _multi_tensor_sgd on the same GPU (the per-element formula is in sgd.cu).  Momentum buffer validity
 * lives on the device: `valid` holds one int32 per CVB_SGD_CHUNK elements of the parameter (one for an empty parameter), 0 while the
 * buffer has never been written (the next applied step copies d into it, as the reference's first step clones it), 1 after.
 * cvb_sgd_table_upload: checks the host table entries [n] (n >= 1; 1 <= n_groups <= CVB_SGD_MAX_GROUPS; numel >= 0; 0 <= group < n_groups;
 *   param and grad non-null when numel > 0; valid non-null with a momentum_buffer, and a momentum_buffer with valid when numel > 0) and
 *   enqueues its copy on `stream` into `table`, caller-owned device memory of n * CVB_SGD_TABLE_ENTRY_BYTES bytes, 16-byte aligned.  Every
 *   entry of a group with CVB_SGD_MOMENTUM needs valid (and a momentum_buffer when numel > 0); the params must not overlap each other.
 *   Not capturable (host-to-device copy from pageable memory).
 * cvb_sgd_step: the step over an uploaded table of n entries with the groups [n_groups] passed by value (no copy of their own).
 *   grad_scale (optional, device fp32 scalar): the gradients are multiplied by (float)(1.0 / (double)*grad_scale) first.  found_inf
 *   (optional, device fp32 scalar): when non-zero, nothing is written.  Any pointer alignment (float4 where param, grad and buffer are
 *   16-byte aligned).  No host sync, CUDA-graph capturable.
 */
#define CVB_SGD_TABLE_ENTRY_BYTES 64
#define CVB_SGD_CHUNK 4096
#define CVB_SGD_MAX_GROUPS 1024 /* 16 KB of kernel arguments */
#define CVB_SGD_NESTEROV 1      /* CvbSgdGroup.flags: nesterov=True */
#define CVB_SGD_WEIGHT_DECAY 2  /* weight_decay != 0 (in the Python double) */
#define CVB_SGD_MOMENTUM 4      /* momentum != 0 (in the Python double) */
typedef struct {
  float lr;
  float weight_decay;
  float momentum;
  int32_t flags;
} CvbSgdGroup;
typedef struct {
  float* param;           /* fp32, contiguous, updated in place */
  const float* grad;      /* fp32, contiguous, shaped as param; read only */
  float* momentum_buffer; /* fp32, contiguous, shaped as param; NULL in a group without momentum */
  int32_t* valid;         /* max(1, ceil(numel / CVB_SGD_CHUNK)) flags; NULL in a group without momentum */
  int64_t numel;
  int32_t group;
} CvbSgdEntry;
int cvb_sgd_table_upload(const CvbSgdEntry* entries, int32_t n, int32_t n_groups, void* table, void* stream);
int cvb_sgd_step(const void* table, int32_t n, const CvbSgdGroup* groups, int32_t n_groups, const float* grad_scale, const float* found_inf,
                 void* stream);

/* COCO box mAP (pycocotools COCOeval, iouType 'bbox', default parameters; csrc/coco_eval.cu): matching, precision / recall accumulation and
 * the 12 summary statistics on the device, stream-ordered, no host sync.  Area ranges all / small / medium / large are [0, 1e10] /
 * [0, 1024] / [1024, 9216] / [9216, 1e10] (inclusive bounds), maxDets 1 / 10 / 100, every detection segment cut to its best 100.
 * Ground truths: gt_key [n_gt] = category index * n_images + image index, ascending, annotation order within a key; gt_box [n_gt][4] xywh
 *   float64; gt_area [n_gt] (the annotation's area field); gt_crowd [n_gt] (1 = iscrowd: ignored, matched by any number of detections).
 * Images are indexed in ascending image id order; img_evaluated [n_images] is 1 for the images the evaluation covers.
 * Detections [n_det]: det_img (image index, evaluated), det_cat (category index, or -1 for a category the ground truth does not list: not
 *   evaluated), det_score (fp32, no NaN), det_box [n_det][4] xywh float64.
 * Outputs (device): det_masks [n_det][4] per area range (bits 0..9 matched at IoU threshold t, bits 16..25 ignored; 0 for detections past
 *   rank 100 or of no category); precision [T=10][R=101][n_cats][4][3] and recall [10][n_cats][4][3] float64 laid out as COCOeval's
 *   eval['precision'] / eval['recall'] (-1 where a category has no non-ignored ground truth); stats [12] float64 in summarize() order.
 * workspace: cvb_coco_eval_workspace_bytes(n_det, n_gt, n_cats) bytes of device memory, 256-byte aligned (0 = sizes outside the limits).
 * Limits: n_images <= CVB_COCO_MAX_IMAGES, 1 <= n_cats <= CVB_COCO_MAX_CATS, n_gt <= CVB_COCO_MAX_GT, n_det <= CVB_COCO_MAX_DETS (LVIS
 *   val has 1 203 categories and 20 k images).  Index ranges and the key order are the caller's contract; the sizes and pointers are checked.
 */
#define CVB_COCO_IOU_THRS 10
#define CVB_COCO_REC_THRS 101
#define CVB_COCO_MAX_IMAGES (1 << 20)
#define CVB_COCO_MAX_CATS 4000
#define CVB_COCO_MAX_GT (1 << 26)
#define CVB_COCO_MAX_DETS (1 << 28)
typedef struct {
  int32_t n_images;
  int32_t n_cats;
  int32_t n_gt;
  int32_t n_det;
  double iou_thrs[CVB_COCO_IOU_THRS]; /* np.linspace(.5, .95, 10) */
  double rec_thrs[CVB_COCO_REC_THRS]; /* np.linspace(0, 1, 101) */
} CvbCocoEvalParams;
size_t cvb_coco_eval_workspace_bytes(int32_t n_det, int32_t n_gt, int32_t n_cats);
int cvb_coco_eval_bbox(const CvbCocoEvalParams* params, const uint32_t* gt_key, const double* gt_box, const double* gt_area, const uint8_t* gt_crowd,
                       const uint8_t* img_evaluated, const int32_t* det_img, const int32_t* det_cat, const float* det_score, const double* det_box,
                       uint32_t* det_masks, double* precision, double* recall, double* stats, void* workspace, size_t ws_bytes, void* stream);

/* Segmentation confusion matrix (src/evaluator/eval_segmentation.py SegmentationEvaluator._generate_matrix + update; csrc/seg_eval.cu):
 * one stream-ordered pass, no host sync.  gt / pred are contiguous label arrays of n elements, each CVB_SEG_U8, _I32 or _I64 (chosen
 * independently) and aligned to its element size.  For every pixel with 0 <= gt < nc, flat = nc * gt + pred in int64 (wrapping as numpy's
 * int64 does):
 *   0 <= flat < nc²  ->  matrix[flat] += 1, so an out-of-range prediction aliases into a neighbouring row as np.bincount + reshape do
 *                         (nc = 3: gt 0 / pred 3 counts at (1, 0), gt 2 / pred -1 at (1, 2));
 *   flat < 0          ->  *err |= CVB_SEG_ERR_NEGATIVE (np.bincount raises "no negative elements");
 *   flat >= nc²       ->  *err |= CVB_SEG_ERR_OVERFLOW (reshape raises).
 * matrix: uint64 [nc][nc] on the device, accumulated in place with integer atomics (exact, the same on every run); err: int32 device word.
 * Limits, checked before any launch: 1 <= nc <= cvb_seg_confusion_nc_max() (the largest nc whose nc² uint32 bins fit one CTA's opt-in
 *   shared memory: 241 on sm_90; ADE20K's 150 and COCO-Stuff's 182 fit), 0 <= n <= 2^31 - 1, known dtype codes, and non-null, aligned
 *   pointers when n > 0.  Larger nc are refused: there is no global-memory fallback.
 */
#define CVB_SEG_U8 0
#define CVB_SEG_I32 1
#define CVB_SEG_I64 2
#define CVB_SEG_ERR_NEGATIVE 1
#define CVB_SEG_ERR_OVERFLOW 2
int32_t cvb_seg_confusion_nc_max(void);
int cvb_seg_confusion_update(const void* gt, int32_t gt_dtype, const void* pred, int32_t pred_dtype, int64_t n, int32_t nc, uint64_t* matrix,
                             int32_t* err, void* stream);

/* Library info / errors */
const char* cvb_last_error_string(void);
int cvb_version(void);
/* number of kernels this library has launched in this process (for bench.py's gpu_launches) */
int64_t cvb_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* CVB200_H_ */
