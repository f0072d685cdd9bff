/*
 * focoos_b200 — C ABI of the H100-native (sm_90a) kernels behind the Focoos detection hot path.
 *
 * The reference (FocoosAI/focoos v0.25.0) is pure Python: it has NO FFI boundary for this path; every
 * operator below replaces a chain of torch library calls at the cited reference call site
 * (paths relative to the reference's `focoos/` package).  The Python side of the boundary is
 * `focoos_b200/ops.py` (ctypes + torch.library registration `focoos_b200::*`); the binding a
 * reference maintainer would add is shown in INTEGRATION.md.
 *
 * Conventions
 *   - Every pointer is a DEVICE pointer unless the name ends in `_host`.  The caller owns all
 *     buffers (activations, weights, outputs); the library allocates nothing persistent.
 *   - Activations are NHWC ("channels-last"): element (b,h,w,c) at ((b*H+h)*W+w)*pitch + c,
 *     `pitch >= C` in ELEMENTS, which lets a kernel read/write a channel slice of a wider tensor
 *     (concat-free CSP/FPN blocks).  Token tensors [B,L,C] are the same thing with H=1.
 *   - `dtype`: FB200_F32 (fp32 SIMT kernels; the near-bit-exact parity mode) or FB200_F16
 *     (fp16 storage, fp32 accumulate; wgmma tensor cores for conv / linear).
 *   - Work is enqueued on `stream` (a cudaStream_t passed as void*); nothing synchronises.
 *     Stateless and re-entrant; one process per GPU.
 *   - Return value: 0 on success, negative fb200_status on error; message via fb200_last_error()
 *     (thread-local).  Python wrappers raise RuntimeError.
 */
#ifndef FOCOOS_B200_H_
#define FOCOOS_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum { FB200_OK = 0, FB200_ERR_INVALID = -1, FB200_ERR_UNSUPPORTED = -2, FB200_ERR_CUDA = -3 } fb200_status;
typedef enum { FB200_F32 = 0, FB200_F16 = 1,
               /* an fp32 value stored as TWO fp16 planes: hi = fp16(v), lo = fp16(v - hi) (exact to ~2^-22): the operand format of fb200_conv2d_pair, also accepted
                * as its output / residual so that activations stay in it between two convs */
               FB200_F16PAIR = 2 } fb200_dtype;
typedef enum { FB200_ACT_NONE = 0, FB200_ACT_RELU = 1, FB200_ACT_SILU = 2, FB200_ACT_GELU = 3, FB200_ACT_SIGMOID = 4 /* SIMT path only */,
               FB200_ACT_RESIDUAL_AFTER = 16 /* OR-ed flag: out = act(conv) + residual instead of act(conv + residual) */ } fb200_act;
/* the kernel of fb200_conv2d; the fp32-accurate split-precision products are fb200_conv2d_pair */
typedef enum { FB200_ALGO_AUTO = 0, FB200_ALGO_SIMT = 1, FB200_ALGO_TCGEN05 = 2 } fb200_algo;

const char* fb200_last_error(void);
int fb200_version(void);

/* ---- a2: ResNet-vd stem, first conv fused with the input normalisation ------------------------
 * Replaces `(images - pixel_mean) / pixel_std` (models/fai_detr/modelling.py:1349) followed by
 * ConvNormLayer conv1_1 (3x3, stride 2, pad 1, BN, ReLU; nn/backbone/resnet.py:181-186,
 * nn/layers/conv.py:93-97).  Zero padding applies to the NORMALISED image (SURVEY A.1).
 * img: [B,3,H,W] fp32 NCHW, 0..255.  mean3_host/std3_host: 3 floats each in HOST memory.  w: [Cout][3][3][3] fp32 as (kh,kw,ci).  out: NHWC [B,H/2,W/2,Cout]. */
int fb200_stem_conv3x3s2(const float* img, int B, int H, int W, const float* w, const float* scale, const float* bias,
                         const float* mean3_host, const float* std3_host, int act, void* out, int out_dtype, int Cout, void* stream);

/* Same, reading the decoded image directly: img_nhwc [B,H,W,3] uint8 RGB (fuses the uint8->float, HWC->CHW conversion of
 * Processor.get_torch_batch, processor/base_processor.py:262-287, into the first conv; SURVEY §8f.1). */
int fb200_stem_conv3x3s2_u8(const uint8_t* img_nhwc, int B, int H, int W, const float* w, const float* scale, const float* bias,
                            const float* mean3_host, const float* std3_host, int act, void* out, int out_dtype, int Cout, void* stream);

/* ---- a2,a3,a5,a7: conv (+ folded BN scale/bias, + residual, + activation), implicit GEMM -------
 * Replaces ConvNormLayer.forward (nn/layers/conv.py:78-98), BottleNeck residual add + ReLU
 * (nn/backbone/resnet.py:106-121), RepVggBlock (models/fai_detr/modelling.py:39-45, re-parameterised
 * on the host), CSPRepLayer add (:103-107), and every nn.Linear on the path (as a 1x1 conv over
 * H=1,W=M tokens: modelling.py:848-882,1204-1207; nn/layers/base.py:51-62).
 *   out[m, n] = act( (sum_k A[m,k] * w[n,k]) * scale[n] + bias[n] + residual[m,n] )
 * x: [B,H,W,Cin] (pitch x_pitch), w: [Cout][KH][KW][Cin] same dtype as x.
 * w_batch_stride: 0 = one weight set for the batch; otherwise w is [B][Cout][KH][KW][Cin] with w_batch_stride elements between images (at least one
 * weight set; no residual).  This is the per-query mask product einsum("bqc,bchw->bqhw") of PredictionHeads.forward (models/fai_mf/modelling.py:86,
 * bisenetformer/modelling.py:364): x = mask features [B,h,w,C], "weights" = the B x Q mask embeddings; one tensor-core launch for the batch.
 * scale/bias: fp32 [Cout] or NULL (=1 / 0).  residual: NULL or same dtype as out, [B,Ho,Wo,Cout]
 * (pitch res_pitch).  out dtype may differ from x dtype (fp32 heads on fp16 features).
 * out_batch_stride: elements between consecutive images of `out` (0 = dense Ho*Wo*out_pitch); lets a level's
 * projection be written straight into its rows of the concatenated [B, sum(HW), C] memory (modelling.py:1165).
 * algo: FB200_ALGO_AUTO picks the tensor-core kernel when dtype==F16 and the shape qualifies; any value outside fb200_algo is FB200_ERR_INVALID. */
int fb200_conv2d(const void* x, int x_dtype, int B, int H, int W, int Cin, int x_pitch, const void* w, int64_t w_batch_stride, int KH, int KW,
                 int stride, int pad, const float* scale, const float* bias, const void* residual, int res_pitch,
                 int act, void* out, int out_dtype, int out_pitch, int64_t out_batch_stride, int Cout, int algo, void* stream);

/* fp32-accurate conv on pair-format activations (precision "fp32_tc"): x is the HI plane of a [hi | lo] pair tensor with C logical channels, its lo plane
 * `x_lo_off` elements further (pitch x_pitch covers both); w3 = [Cout][KH][KW][W_hi | W_lo | W_hi] (3C), or per image as in fb200_conv2d (w_batch_stride);
 * hi*W_hi + hi*W_lo + lo*W_hi as three fp16 tensor-core products per chunk, fp32 accumulation (error ~2^-21).
 * out_dtype FB200_F32: fp32 output / residual as in fb200_conv2d.  out_dtype FB200_F16PAIR: the epilogue writes the result AS a pair (hi plane at `out`, lo plane
 * `out_lo_off` elements further, pitch out_pitch) and reads the residual as a pair (`res_lo_off`), so consecutive convs exchange activations without a split pass
 * (replaces the fb200_split_f32_pair launch in front of every conv: nn/layers/conv.py:78-98 chains such as resnet.py:106-121). */
int fb200_conv2d_pair(const void* x, int B, int H, int W, int C, int x_pitch, int64_t x_lo_off, const void* w3, int64_t w_batch_stride, int KH, int KW, int stride, int pad,
                      const float* scale, const float* bias, const void* residual, int res_pitch, int64_t res_lo_off, int act, void* out, int out_dtype,
                      int out_pitch, int64_t out_lo_off, int64_t out_batch_stride, int Cout, void* stream);

/* The HBM-bound spatial operators between convs, on pair-format activations (hi plane at the pointer, lo plane `*_lo_off` elements further, C % 8 == 0):
 * mode 0 = F.max_pool2d(3,2,1) (resnet.py:254), 1 = AvgPool2d(2,2,ceil_mode) of the vd shortcut (resnet.py:91-102), 2 = F.interpolate(bilinear,
 * align_corners=False) of the FPN / PAN (fai_detr/modelling.py:334,342).  Arithmetic in fp32 on hi + lo, result re-split. */
int fb200_pair_pool(int mode, const void* x, int64_t x_lo_off, int x_pitch, int B, int H, int W, int C, void* out, int64_t out_lo_off, int out_pitch, int Ho, int Wo,
                    void* stream);

/* rowmax[m] = max_n (x[m,:] . w[n,:] + bias[n]) for fp16 x [M,K] / w [Cout,K] on the tensor cores, WITHOUT writing the [M,Cout] product:
 * the query-selection score enc_outputs_class.max(-1) of _get_decoder_input (models/fai_detr/modelling.py:1204-1214; 268 800 x 365 fp32 logits = 395 MB at
 * bs=32 that are otherwise written and read back).  rowmax must be pre-filled with -inf (combined with integer atomics across N tiles). */
int fb200_linear_rowmax(const void* x, int64_t M, int K, int x_pitch, const void* w, const float* bias, int Cout, float* rowmax, void* stream);
/* Same on pair-format rows (fp32-accurate mode): x = hi plane of [M, K] rows, lo plane x_lo_off elements further, w3 = [Cout][W_hi | W_lo | W_hi]. */
int fb200_linear_rowmax_pair(const void* x, int64_t M, int K, int x_pitch, int64_t x_lo_off, const void* w3, const float* bias, int Cout, float* rowmax, void* stream);

/* x fp32 [rows, C] (row pitch x_pitch) -> out fp16 [rows, 2C]: out[:, :C] = hi = fp16(x), out[:, C:] = lo = fp16(x - hi).
 * Operand preparation of the split-precision conv/linear mode (precision="fp32_tc"). */
int fb200_split_f32_pair(const float* x, int64_t rows, int C, int x_pitch, void* out, void* stream);

/* ---- a2: pools.  F.max_pool2d(3,2,1) (nn/backbone/resnet.py:254); AvgPool2d(2,2,0,ceil_mode=True)
 * of the vd shortcut (nn/backbone/resnet.py:95). */
int fb200_maxpool3x3s2(const void* x, int dtype, int B, int H, int W, int C, void* out, void* stream);
int fb200_avgpool2x2_ceil(const void* x, int dtype, int B, int H, int W, int C, void* out, void* stream);

/* ---- a5: F.interpolate(mode="bilinear", align_corners=False) (models/fai_detr/modelling.py:334,342),
 * writing straight into a channel slice of the concat buffer. */
int fb200_resize_bilinear(const void* x, int dtype, int B, int H, int W, int C, int x_pitch, void* out, int Ho, int Wo,
                          int out_pitch, void* stream);

/* ---- a13 / f1: the resize of the pre-processing step (processor/base_processor.py:284-294, F.interpolate(..., mode="bilinear", align_corners=False) on the float
 * image) for a whole batch in one launch: images = uint8 NHWC [B,H,W,3] (u8_nhwc = 1) or float NCHW [B,3,H,W] (0) -> out_nchw float [B,3,Ho,Wo]. */
int fb200_image_resize(const void* images, int u8_nhwc, int B, int H, int W, float* out_nchw, int Ho, int Wo, void* stream);

/* ---- elementwise: out = a + b (b broadcast over the leading `rows/brows` blocks when brows < rows).
 * with_pos_embed (nn/layers/transformer.py:579-581, modelling.py:918-919). */
int fb200_add(const void* a, const void* b, void* out, int dtype, int64_t rows, int64_t brows, int C, void* stream);

/* ---- a4,a9: out = LayerNorm(x (+ res)) * gamma + beta, eps 1e-5, biased variance (nn.LayerNorm;
 * nn/layers/transformer.py:590-600, modelling.py:939-956).  x,res,out: [M,C] contiguous. */
int fb200_layernorm(const void* x, const void* res, const float* gamma, const float* beta, void* out, int dtype,
                    int64_t M, int C, float eps, void* stream);

/* ---- a8,a9,a4 in the fp32-accurate mode: the row-wise glue between two tensor-core linears, fused so that each linear finds its operand already in the pair
 * format (csrc/head_fused.cu).  Arithmetic identical to the separate launches they replace.
 * fb200_layernorm_ex: y = LayerNorm(sel(x)[src(m)] (+ res[m])) * gamma + beta for output rows m < M, where src(m) = m, or (m / gather_k) * S + gather_idx[m] with a
 * top-k index tensor [B, gather_k] (torch.gather of the selected queries, modelling.py:1216-1229), and sel() replaces a source row r with !valid[r % S] by fill[C]
 * (memory * valid_mask folded behind enc_output.0, modelling.py:1202-1207).  Outputs (each optional): out_f32 [M, C]; out_pair [M, 2C] = [hi | lo] fp16;
 * out_pair_pos = pair of (y + pos[m % pos_rows]) - with_pos_embed in front of the q/k and sampling-offset projections (modelling.py:918-919, 934-947). */
int fb200_layernorm_ex(const float* x, int x_pitch, const float* res, const int* gather_idx, int gather_k, const uint8_t* valid, int S, const float* fill,
                       const float* gamma, const float* beta, float eps, int64_t M, int C, float* out_f32, void* out_pair, const float* pos, int64_t pos_rows,
                       void* out_pair_pos, void* stream);
/* out_pair = pair(act(x)) and / or out_pair_pos = pair(x + pos[r % pos_rows]) of fp32 rows x [rows, C] (pitch x_pitch); act as fb200_act (exact-erf GELU of the AIFI FFN,
 * nn/layers/transformer.py:600) */
int fb200_split_pair_ex(const float* x, int64_t rows, int C, int x_pitch, int act, const float* pos, int64_t pos_rows, void* out_pair, void* out_pair_pos, void* stream);
/* decoder box refinement + first query_pos_head layer in one pass (modelling.py:990-1008): ref_out = sigmoid(delta + inverse_sigmoid(ref_in)) when delta != NULL (else the
 * boxes are ref_in), qpos_pair [M, 2N] = pair(relu(box . w0[N,4]^T + b0)) when qpos_pair != NULL (N % 64 == 0). */
int fb200_box_refine_qpos(const float* delta, const float* ref_in, float* ref_out, const float* w0, const float* b0, int N, void* qpos_pair, int64_t M, void* stream);
/* out[M, C] dense = sigmoid(x[M, C] with row pitch x_pitch): class scores from the 16-byte-padded logits of the tensor-core score head (modelling.py:378) */
int fb200_sigmoid_rows(const float* x, int x_pitch, int64_t M, int C, float* out, void* stream);

/* ---- a4,a9: softmax(Q K^T * scale) V per (batch, head); nn.MultiheadAttention core
 * (SURVEY A.6).  q/k/v/out rows are tokens; head h uses columns [h*hd, (h+1)*hd). hd must be 32.
 * B, Lq, Lk, heads > 0 and every pitch >= heads*32, else FB200_ERR_INVALID without a launch.  Any Lk: the kernels that keep a head's K and V in shared memory
 * take Lk <= 792 (fp32, or fp16 rows that are not 16-byte aligned) and Lk <= 1408 (fp16 tensor cores); longer keys are streamed by the kernels of
 * fb200_attention_masked without a mask. */
int fb200_attention(const void* q, int q_pitch, const void* k, int k_pitch, const void* v, int v_pitch, void* out,
                    int out_pitch, int dtype, int B, int Lq, int Lk, int heads, int head_dim, float scale, void* stream);
/* fp32 tensors on the fp16 tensor cores (precision="fp32_tc"): Q, K, V are split into [hi|lo] halves on the way into shared memory and every product
 * is formed as hi*hi + hi*lo + lo*hi with fp32 accumulation (mma.sync m16n8k16), softmax in fp32.  Same semantics as fb200_attention(FB200_F32).
 * out_dtype FB200_F32: fp32 rows.  FB200_F16PAIR: rows written as [hi(heads*32) | lo(heads*32)] fp16 (out_pitch in halves) - the operand of the out_proj linear.
 * The resident kernel takes self-attention up to L = 640 (Lk = 704 for Lq <= 32); above that fp32 rows are streamed by the kernel of fb200_attention_masked_split
 * without a mask, and pair rows are refused with FB200_ERR_UNSUPPORTED (no caller writes pair rows at such lengths). */
int fb200_attention_split(const float* q, int q_pitch, const float* k, int k_pitch, const float* v, int v_pitch, void* out, int out_dtype, int out_pitch, int B,
                          int Lq, int Lk, int heads, int head_dim, float scale, void* stream);

/* ---- a10: multi-scale deformable attention core, softmax over levels*points fused.
 * Replaces MSDeformableAttention.forward lines 854-880 (models/fai_detr/modelling.py) +
 * ms_deform_attn_core_pytorch (nn/layers/deformable.py:10-35).
 * value: [B,S,heads*32] (pitch v_pitch).  oa: [B*Q, heads*L*P*3] fp32 or fp16 = sampling offsets
 * [heads][L][P][2] followed by attention logits [heads][L*P] (one fused linear).  ref: [B*Q,4] fp32
 * (cx,cy,w,h in sigmoid space).  shapes_host: L pairs (H_l, W_l) in HOST memory.  out: [B*Q, heads*32]
 * (out_dtype FB200_F16PAIR with fp32 value / oa: rows [hi(heads*32) | lo(heads*32)] fp16, out_pitch in halves). */
int fb200_msda(const void* value, int v_dtype, int v_pitch, const void* oa, int oa_dtype, int oa_pitch, const float* ref,
               const int* shapes_host, int L, int P, int B, int S, int Q, int heads, void* out, int out_dtype,
               int out_pitch, void* stream);

/* ---- a8: query selection helpers (models/fai_detr/modelling.py:1202-1229) ---------------------- */
/* out[r,:] = valid[r % S] ? x[r,:] : fill[:]   (memory * valid_mask folded behind enc_output.0) */
int fb200_row_select(const void* x, const uint8_t* valid, const float* fill, void* out, int dtype, int64_t rows, int S,
                     int C, void* stream);
/* out[r] = max_n x[r,n] (fp32 out).  enc_outputs_class.max(-1) (:1210) */
int fb200_rowmax(const void* x, int dtype, int64_t rows, int N, int pitch, float* out, void* stream);
/* per row: K largest, sorted descending, ties by ascending index.  torch.topk (:1214; processor.py:147) */
int fb200_topk(const float* x, int B, int N, int K, int* out_idx, float* out_val, void* stream);
/* out[b,k,:] = src[b, idx[b,k], :]   (gather :1216-1229) */
int fb200_gather_rows(const void* src, int dtype, int B, int S, int C, int pitch, const int* idx, int K, void* out,
                      void* stream);

/* ---- a8,a9,a11: box arithmetic in fp32 ---------------------------------------------------------
 * mode 0: out = sigmoid(x)                                    (modelling.py:985, :397)
 * mode 1: out = sigmoid(x + inverse_sigmoid(ref)), eps 1e-5   (modelling.py:1003; nn/layers/functional.py:4-6)
 * mode 2: out = x + anchors[idx]  (x,[n,4]; anchors [S,4]; idx [n] with per-batch rows)  (:1207 after gather)
 * mode 3: out = cxcywh -> xyxy                                (utils/box.py:14-17) */
int fb200_box_op(int mode, const float* x, const float* ref, const int* idx, float* out, int64_t n, void* stream);

/* ---- a12: DETRProcessor.postprocess (models/fai_detr/processor.py:146-217), whole batch, one launch.
 * scores [B,Q,C] fp32 probabilities, boxes [B,Q,4] xyxy in [0,1], sizes [B,2] int32 (H,W) of the ORIGINAL
 * images.  Outputs are padded to K per image, sorted by descending score (ties: ascending flat index);
 * count[b] = number with score > threshold (strict); boxes scaled, rintf (half-to-even) -> int32. */
int fb200_detr_postprocess(const float* scores, const float* boxes, const int* sizes, int B, int Q, int C, int K,
                           float threshold, float* out_scores, int* out_labels, int* out_boxes, int* out_query,
                           int* out_count, void* stream);

/* ---- f3: evaluator post-process -----------------------------------------------------------------
 * Replaces DETRProcessor.eval_postprocess + detector_postprocess (models/fai_detr/processor.py:19-57,121-144; called per batch from
 * trainer/evaluation/evaluator.py:179-190): per image top-K over the flattened [Q*C] scores WITHOUT threshold, label = i % C, query = i / C,
 * xyxy boxes scaled to sizes[b] = (height, width) of the dataset entry as floats, clipped to the image, empty boxes dropped.
 * Outputs are compacted per image in descending-score order: out_scores/out_labels [B,K], out_boxes [B,K,4] fp32, out_count [B]. */
int fb200_detr_eval_postprocess(const float* scores, const float* boxes, const int* sizes, int B, int Q, int C, int K, float* out_scores,
                                int* out_labels, float* out_boxes, int* out_count, void* stream);

/* ======== MaskFormer family (SURVEY §8 a14-a17; focoos/models/fai_mf/{modelling,processor}.py) ======================== */

/* out = cur + F.interpolate(y, size=(H,W), mode="nearest")   TransformerFPN top-down path (fai_mf/modelling.py:364).
 * y [B,h,w,C], cur/out [B,H,W,C], NHWC contiguous. */
int fb200_upsample_nearest_add(const void* y, const void* cur, void* out, int dtype, int B, int h, int w, int H, int W, int C, void* stream);

/* Attention mask of the masked decoder (fai_mf/modelling.py:96-105,510-513): x [B,Lk,Qp] mask logits already resized to the
 * level, mask[b,q,k] (uint8, row pitch LkP) = x[b,k,q] < 0 ("not allowed"); allowed[b,q] (int32, ZERO-INITIALISED by the caller)
 * += number of allowed keys — a row with 0 allowed keys attends everywhere. */
int fb200_attn_mask_build(const void* x, int dtype, int B, int Lk, int Qp, int Q, uint8_t* mask, int LkP, int* allowed, void* stream);

/* softmax(q k^T * scale + mask) v per (batch, head), keys streamed (Lk up to H/8*W/8), head_dim 32; mask/allowed as above and shared
 * by all heads (the reference replicates a [B*heads,Q,Lk] bool tensor, :513); mask == NULL -> unmasked.
 * nn.MultiheadAttention inside CrossAttentionLayer (nn/layers/transformer.py:206-238).
 * B, Lq, Lk, heads > 0, every pitch >= heads*32 and (with a mask) LkP >= Lk, else FB200_ERR_INVALID without a launch. */
int fb200_attention_masked(const void* q, int q_pitch, const void* k, int k_pitch, const void* v, int v_pitch, const uint8_t* mask, int LkP,
                           const int* allowed, void* out, int out_pitch, int dtype, int B, int Lq, int Lk, int heads, int head_dim, float scale,
                           void* stream);

/* The same masked attention with fp32-accurate tensor-core products (precision "fp32_tc"): Q (fp32), K, V and the softmax numerators as fp16 hi / lo halves,
 * S = Qh Kh^T + Qh Kl^T + Ql Kh^T and O += Ph Vh + Ph Vl + Pl Vh with fp32 accumulation (error ~2^-21), keys streamed in chunks.  kv_dtype FB200_F32: k / v are fp32 tensors,
 * split while they are staged; FB200_F16PAIR: k / v are the [hi | lo] pairs their projection already wrote (fb200_conv2d_pair with a pair output): hi plane at the pointer, lo
 * plane kv_lo_off halves further, pitches in halves - staged by 16-byte asynchronous copies, double buffered. */
int fb200_attention_masked_split(const float* q, int q_pitch, const void* k, int k_pitch, const void* v, int v_pitch, int kv_dtype, int64_t kv_lo_off, const uint8_t* mask,
                                 int LkP, const int* allowed, float* out, int out_pitch, int B, int Lq, int Lk, int heads, int head_dim, float scale, void* stream);

/* out[r, 0..N-2] = softmax(x[r, 0..N-1])[..., :-1]  (drop the no-object class; fai_mf/modelling.py:618). fp32. */
int fb200_softmax_drop_last(const float* x, int64_t rows, int N, int pitch, float* out, void* stream);

/* MaskFormerHead sigmoid (fai_mf/modelling.py:619) + final F.interpolate(bilinear) to the input size (:722-723), fused:
 * x [B,h,w,Qp] mask logits NHWC -> out [B,Q,H,W] fp32 probabilities. */
int fb200_mask_sigmoid_upsample(const void* x, int dtype, int B, int h, int w, int Qp, int Q, float* out, int H, int W, void* stream);
/* The same upsampling with the SEMANTIC post-process fused in (models/fai_mf/processor.py:208-220 on top of :722-723): per output pixel
 * argmax_q(scores[b,q] * prob[b,q,y,x]) -> labels [B,H,W] uint8 and counts [B,Q] (pixels per query); the [B,Q,H,W] probabilities are never
 * written.  Bit-identical to fb200_mask_argmax(fb200_mask_sigmoid_upsample(x)). */
int fb200_mask_sigmoid_upsample_argmax(const void* x, int dtype, int B, int h, int w, int Qp, int Q, const float* scores, int H, int W, uint8_t* labels,
                                       int* counts, void* stream);
/* The INSTANCE post-process fused in the same way (processor.py:222-257): count[b,q] = #pixels with prob >= thr, psum[b,q] = their probability mass,
 * straight from the low-resolution logits; and the upsampled probabilities of only the n kept (b,q) pairs (bq [n,2] i32 -> out [n,H,W] f32). */
int fb200_mask_sigmoid_upsample_stats(const void* x, int dtype, int B, int h, int w, int Qp, int Q, int H, int W, float thr, int* count, float* psum, void* stream);
int fb200_mask_sigmoid_upsample_select(const void* x, int dtype, int h, int w, int Qp, const int* bq, int n, float* out, int H, int W, void* stream);
/* The probabilities of fb200_mask_sigmoid_upsample (same values) in NHWC, as the operand of the class x mask product of semantic evaluation
 * (fai_mf/processor.py:99-105,142-166): out [B,H,W,Qo] with channels Q..Qo-1 zero, Qo % 4 == 0.  out_dtype FB200_F32 / FB200_F16: one plane;
 * FB200_F16PAIR: per pixel [hi(Qo) | lo(Qo)] fp16, the operand of fb200_conv2d_pair. */
int fb200_mask_sigmoid_upsample_nhwc(const void* x, int dtype, int B, int h, int w, int Qp, int Q, void* out, int out_dtype, int Qo, int H, int W, void* stream);

/* SemSegEvaluator.process (trainer/evaluation/sem_seg_evaluation.py:86-107): conf[(C+1) * pred + gt] += 1 for every pixel of scores [B,H,W,*] fp32 NHWC
 * (pixel pitch `pitch`, `batch_stride` elements between images; only channels 0..C-1 count), pred = argmax over c < C with the FIRST maximum winning
 * and a NaN counting as the maximum (the first NaN wins), as torch.argmax on the CPU; gt = labels[b,y,x] (uint8 or int32: label_bytes 1 / 4), mapped
 * to C when it equals ignore_label.  conf: (C+1) x (C+1) int64 on the device, added into (row = prediction, column = ground truth).  A label outside
 * [0, C] that is not ignore_label is not counted; `invalid` (one int64) is incremented instead (the reference's bincount raises on it). */
int fb200_sem_seg_confusion(const float* scores, int B, int H, int W, int C, int pitch, int64_t batch_stride, const void* labels, int label_bytes,
                            int ignore_label, int64_t* conf, int64_t* invalid, void* stream);

/* The greedy matching of box AP (trainer.BoxAPEvaluator.evaluate) for a batch of B images, bit for bit: per image, its detections of one class are
 * visited in (score descending, detection index ascending) order; at threshold t a detection takes the FIRST unmatched same-class ground truth of
 * maximum IoU and is a true positive iff that IoU >= thresholds_host[t] (compared as double; used ground truths count as IoU -1, a NaN IoU as the
 * maximum).  The IoU is numpy's arithmetic of trainer._iou_matrix, without contraction: fp32 when gt_fp64 == 0, fp64 (detections widened) otherwise.
 * Detections as DETRProcessor.eval_postprocess leaves them: scores [B,K] fp32, classes [B,K] int32, boxes [B,K,4] fp32 absolute xyxy, the first
 * counts[b] of row b valid.  Ground truth: boxes [G,4] fp32 / fp64, classes [G] int32, image b owns rows gt_offsets[b] .. gt_offsets[b+1]-1
 * (gt_offsets [B+1] on the device, gt_offsets_host the same values on the host: checked to be monotonic, to start at 0 and end at G).
 * Out: tp [B,K] (bit t of tp[b,k]: true positive at threshold t; 0 past counts[b]); gt_count [C] int64 += the ground truths of each class in [0, C).
 * Limits: K <= 1024, at most 1024 ground truths per image, 1 <= T <= 16 thresholds. */
int fb200_box_ap_match(const float* scores, const int* classes, const float* boxes, const int* counts, int B, int K, const void* gt_boxes, int gt_fp64,
                       const int* gt_classes, const int* gt_offsets, const int* gt_offsets_host, int G, const double* thresholds_host, int T, int C,
                       uint16_t* tp, int64_t* gt_count, void* stream);

/* MaskFormerProcessor.postprocess reductions (fai_mf/processor.py:222-257): per plane of masks [planes, hw] fp32:
 * count = #(p >= thr), psum = sum of those p. */
int fb200_mask_stats(const float* masks, int64_t planes, int64_t hw, float thr, int* count, float* psum, void* stream);

/* Kept masks -> original image size (fai_mf/processor.py:275-283): for pair i = (b,q) in bq [n,2]: (masks[b,q] >= thr) as float,
 * bilinear resize to (Ho,Wo), != 0 -> out [n,Ho,Wo] uint8; bbox [n,4] = (xmin,ymin,xmax,ymax) of the set pixels, zeros if empty
 * (masks_to_xyxy, utils/vision.py:344-370). */
int fb200_mask_resize_bbox(const float* masks, int Q, int H, int W, const int* bq, int n, float thr, uint8_t* out, int Ho, int Wo, int* bbox,
                           void* stream);

/* ======== BiSeNetFormer family (SURVEY §8 a18-a19; focoos/nn/backbone/stdc.py, focoos/models/bisenetformer/modelling.py) ===== */

/* CatBottleneck.avd_layer: depthwise 3x3 stride-2 pad-1 conv + BatchNorm (nn/backbone/stdc.py:117-130). x [B,H,W,C] NHWC,
 * w9c fp32 [9][C] (tap-major), scale/bias = folded BN. out [B,ceil(H/2),ceil(W/2),C]. */
int fb200_dwconv3x3s2_bn(const void* x, int dtype, int B, int H, int W, int C, const float* w9c, const float* scale, const float* bias, void* out, void* stream);
/* CatBottleneck.skip: AvgPool2d(3, 2, 1), count_include_pad=True (nn/backbone/stdc.py:131); out may be a channel slice. */
int fb200_avgpool3x3s2(const void* x, int dtype, int B, int H, int W, int C, void* out, int out_pitch, void* stream);
/* feat.mean(dim=(2,3)) / adaptive_avg_pool2d(1) (bisenetformer/modelling.py:162,187,228): [B,HW,C] -> [B,C]. */
int fb200_global_avgpool(const void* x, int dtype, int B, int HW, int C, void* out, void* stream);
/* ARM / FFM gating: out = x * gate[b,c] (+ addvec[b,c]) (+ addt[b,hw,c]) (+ x if self_add) (bisenetformer/modelling.py:166,190,196,232-234). */
int fb200_channel_scale(const void* x, const void* gate, const void* addvec, const void* addt, int self_add, void* out, int dtype, int B, int64_t HW, int C,
                        void* stream);
/* Semantic post-process (processor.py:208-220, predict_all_pixels): labels[b,p] = argmax_q(scores[b,q] * masks[b,q,p]) (first maximum),
 * counts[b,q] (ZERO-INITIALISED by the caller) += pixels labelled q. masks [B,Q,HW] fp32, Q <= 255. */
int fb200_mask_argmax(const float* masks, const float* scores, int B, int Q, int64_t HW, uint8_t* labels, int* counts, void* stream);
/* kept one-hot masks -> original image size + boxes: pair i = (b,q): (labels[b] == q) -> bilinear resize -> != 0 (processor.py:275-283). */
int fb200_label_resize_bbox(const uint8_t* labels, int H, int W, const int* bq, int n, uint8_t* out, int Ho, int Wo, int* bbox, void* stream);

/* PNG files of the kept mask crops (trim_mask + binary_mask_to_base64, utils/vision.py:264-293; fai_mf/processor.py:275-304): for mask i of
 * masks [n,H,W] uint8 (non-zero = set) and bbox[i] = (x1,y1,x2,y2) from fb200_mask_resize_bbox / fb200_label_resize_bbox, the crop
 * masks[i][y1:min(y2,H), x1:min(x2,W)] encoded byte for byte as cv2.imencode(".png", crop * 255) encodes it (SUB-filtered rows, zlib
 * Z_RLE deflate, 8192-byte IDAT chunks).  out receives the files back to back (mask i at the sum of the lengths before it) and must hold
 * n * fb200_mask_png_bound(H, W) bytes; lengths [n] i32: bytes of each file, 0 for a crop with no rows or no columns, -1 for a crop zlib
 * would store uncompressed (not produced by any 0/255 mask seen) or a negative x1 / y1.  workspace: fb200_mask_png_workspace_bytes. */
int fb200_mask_png_bound(int H, int W);
int64_t fb200_mask_png_workspace_bytes(int n, int H, int W);
int fb200_mask_png(const uint8_t* masks, int n, int H, int W, const int* bbox, uint8_t* out, int* lengths, void* workspace, void* stream);

/* ---- training criterion (SURVEY 8 a20) ---------------------------------------------------------------------
 * Replaces BoxHungarianMatcher.forward (focoos/models/fai_detr/modelling.py:693-758) and SetCriterion.forward with
 * loss_labels_vfl / loss_boxes (:464-531, :553-612) for all L supervised layers at once.
 * logits [L,B,Q,C] f32 raw, boxes [L,B,Q,4] f32 cxcywh; targets concatenated over the batch: tgt_labels [T] i32,
 * tgt_boxes [T,4] f32 cxcywh, tgt_offsets [B+1] i32 (prefix sums of per-image target counts). */

/* cost[l][t][q] = w_bbox*L1 + w_class*(focal pos - neg) + w_giou*(-GIoU) for every target t against the Q queries of
 * its own image (the diagonal blocks the reference keeps after C.split, :744-747).  cost: [L,T,Q] f32. */
int fb200_detr_match_cost(const float* logits, const float* boxes, const int* tgt_labels, const float* tgt_boxes, const int* tgt_offsets,
                          int L, int B, int Q, int C, int T, float w_class, float w_bbox, float w_giou, float alpha, float gamma,
                          float* cost, void* stream);
/* Linear-sum assignment per (layer, image) on the device (replaces scipy.optimize.linear_sum_assignment, :747).
 * match_q [L,T] i32: the query assigned to each target (-1 only if the costs were not finite).  Needs n_b <= Q. */
int fb200_hungarian(const float* cost, const int* tgt_offsets, int L, int B, int Q, int T, int max_targets, int* match_q, void* stream);
int64_t fb200_detr_loss_workspace_bytes(int L, int B, int Q);
/* losses [L,3] = {w_vfl*loss_vfl, w_bbox*loss_bbox, w_giou*loss_giou}; gradients of those weighted losses:
 * grad_logits [L,B,Q,C] (d loss_vfl), grad_boxes_l1 / grad_boxes_giou [L,B,Q,4] (d loss_bbox, d loss_giou w.r.t. cxcywh). */
int fb200_detr_loss(const float* logits, const float* boxes, const int* tgt_labels, const float* tgt_boxes, const int* tgt_offsets,
                    const int* match_q, int L, int B, int Q, int C, int T, float num_boxes, float w_vfl, float w_bbox, float w_giou,
                    float alpha, float gamma, float* losses, float* grad_logits, float* grad_boxes_l1, float* grad_boxes_giou,
                    void* workspace, void* stream);

/* ---- optimiser step of the fine-tune loop (SURVEY 8 a21) -------------------------------------------------------
 * Replaces, on one flat fp32 buffer of all trainable parameters (each tensor padded to a multiple of 4 elements):
 * GradScaler.unscale_/step/update + clip_grad_norm_ x2 + AdamW.step with per-tensor lr / weight decay
 * (focoos/trainer/trainer.py:757-773,782-794; focoos/trainer/solver/build.py:29-37,40-138).
 * Control block `ctrl`: 16 x 4-byte words in device memory, never read by the host on the step path: */
#define FB200_CTRL_SCALE 0          /* f32 loss scale (GradScaler init 2^10, trainer.py:645) */
#define FB200_CTRL_GROWTH_TRACKER 1 /* i32 consecutive finite steps */
#define FB200_CTRL_FOUND_INF 2      /* i32 1 = this step's gradients were not finite -> adamw_step is a no-op */
#define FB200_CTRL_GRAD_NORM 3      /* f32 global L2 norm of the unscaled, world-averaged gradient (before clipping) */
#define FB200_CTRL_GMUL 4           /* f32 multiplier adamw_step applies to the raw gradient buffer: clip / (scale * world) */
#define FB200_CTRL_STEP 5           /* i32 number of optimiser steps taken (skipped steps do not count) */
#define FB200_CTRL_BC1 6            /* f32 1 - beta1^step */
#define FB200_CTRL_BC2_SQRT 7       /* f32 sqrt(1 - beta2^step) */
#define FB200_CTRL_CLIP_COEF 8      /* f32 product of the clip coefficients */
int64_t fb200_optim_workspace_bytes(void);
/* sum of squares + non-finite flag of the flat gradient buffer (per-block partials, reduced in a fixed order) */
int fb200_grad_stats(const float* grads, int64_t n, void* workspace, void* stream);
/* one thread: norm, `clip_passes` successive clip_grad_norm_(max_norm) coefficients, loss-scale update, bias corrections 1 - beta^step with
 * beta = 1 - one_minus_beta in double (fp32(0.001) puts 1 - beta2 within 5e-8 relative of torch's) */
int fb200_optim_finalize(const void* workspace, float* ctrl, float max_norm, int clip_passes, float inv_world, int use_scaler, float growth,
                         float backoff, int growth_interval, float one_minus_beta1, float one_minus_beta2, void* stream);
/* AdamW over chunks (chunk c covers [chunk_start[c], +chunk_len[c]) of tensor chunk_seg[c]; lr = seg_lr[seg]*lr_factor).
 * seg_active: NULL, or one int per tensor, 0 = the tensor received no gradient this step and is skipped (torch: p.grad is None).
 * The Adam betas arrive as 1 - beta, formed by the caller before the rounding to fp32 as torch forms its scalars: 1 - fp32(0.999) would be
 * 1.3e-5 smaller than fp32(1 - 0.999).  fp32(1 - fp32(1 - beta)) rounds back to fp32(beta) for the betas in use (0.9, 0.999). */
int fb200_adamw_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, const int64_t* chunk_start, const int* chunk_len,
                     const int* chunk_seg, int nchunks, const float* seg_lr, const float* seg_wd, const int* seg_active, float lr_factor,
                     float one_minus_beta1, float one_minus_beta2, float eps, const float* ctrl, void* stream);
/* Model EMA update (focoos/trainer/solver/ema.py:112-140), one launch: ema[i] = fma(one_minus_decay, params[i], ema[i] * decay) over the
 * n-element arena laid out like the flat parameter buffer (n a multiple of 4, both 16-byte aligned), the bit-exact result of
 * torch._foreach_mul_ + torch._foreach_add_(alpha) on the device; plus `nchunks` rows of `chunks` (int64 [nchunks][4]: source address,
 * EMA address, element count, kind) for the entries outside that buffer: kind 0 = fp32 as above, kind 1 = int64 as
 * trunc(fp32(ema) * decay + fp32(src) * one_minus_decay) with fp32 products and sum.  decay and 1 - decay are formed in double by the caller
 * and rounded to fp32.  The loss scaler's found-inf flag is not read: the EMA follows the weights on skipped steps too. */
int fb200_ema_update(float* ema, const float* params, int64_t n, const int64_t* chunks, int nchunks, float decay, float one_minus_decay,
                     void* stream);

/* ---- backward / training-mode kernels (SURVEY 8 a21: what autograd executes under TrainerLoop.run_step, trainer/trainer.py:757) ----
 * fp32, NHWC, caller-owned workspaces.  Each replaces the aten backward of the torch call the reference makes at the cited site. */

/* weight gradient of nn.Conv2d (nn/layers/conv.py:84-92): dw[Cout][KH][KW][Cin] (+)= sum_p dy[p,co] * x[pix(p,kh,kw),ci] */
int64_t fb200_conv_wgrad_workspace_bytes(int B, int Ho, int Wo, int Cin, int Cout, int KH, int KW);
int fb200_conv_wgrad(const float* x, int B, int H, int W, int Cin, int x_pitch, const float* dy, int Ho, int Wo, int Cout, int dy_pitch, int KH,
                     int KW, int stride, int pad, float* dw, int accumulate, void* workspace, void* stream);
/* Same weight gradient on the tensor cores (k=1/3 stride-1 convs and linears, 3x3 stride-2 convs through TMA element strides; fb200_conv_wgrad_tc_supported says when): x_pair / dy_pair are
 * the dense [hi|lo] fp16 pairs (fb200_split_f32_pair) of x [B,H,W,Cin] and dy [B,H,W,Cout]; three wgmma products per 64-pixel chunk
 * (hi*hi + hi*lo + lo*hi, fp32 accumulation in registers) reproduce the fp32 result to ~2^-21. */
int fb200_conv_wgrad_tc_supported(int B, int H, int W, int Cin, int Ho, int Wo, int Cout, int KH, int KW, int stride, int pad);
int64_t fb200_conv_wgrad_tc_workspace_bytes(int B, int Ho, int Wo, int Cin, int Cout, int KH, int KW);
int fb200_conv_wgrad_tc(const void* x_pair, int B, int H, int W, int Cin, const void* dy_pair, int Cout, int KH, int KW, int stride, int pad, float* dw,
                        int accumulate, void* workspace, void* stream);
/* The same tensor-core weight gradient on PLAIN fp16 operands x [B,H,W,Cin], dy [B,Ho,Wo,Cout] (dense), one product per chunk, fp32 accumulation and fp32 dw: the arithmetic of
 * the reference's fine-tuning under torch.autocast(fp16) + GradScaler (trainer/trainer.py:645,735-771); used by the "amp" training precision. */
int fb200_conv_wgrad_tc_f16(const void* x, int B, int H, int W, int Cin, const void* dy, int Cout, int KH, int KW, int stride, int pad, float* dw,
                            int accumulate, void* workspace, void* stream);
/* zero-dilation of dy for the stride-2 data gradient (dx = conv(dilate(dy), flipped transposed weights) through fb200_conv2d) */
int fb200_dilate2(const float* dy, int B, int Ho, int Wo, int C, int Hd, int Wd, float* out, void* stream);
/* column sums of [R,C] (bias gradients); workspace of fb200_col_workspace_bytes(C) also serves the BN / LayerNorm calls below */
int64_t fb200_col_workspace_bytes(int C);
int fb200_colsum(const float* x, int64_t R, int C, int pitch, float* out, int accumulate, void* workspace, void* stream);
/* nn.BatchNorm2d in training mode (+ residual add + ReLU/SiLU): batch mean / biased variance over R = B*H*W rows, running stats
 * updated with `momentum` (unbiased variance), y = act((x-mean)*rstd*gamma + beta + res)   (conv.py:93-97, resnet.py:106-121) */
int fb200_bn_train_fwd(const float* x, int x_pitch, int64_t R, int C, const float* gamma, const float* beta, const float* res, int res_pitch, int act,
                       float eps, float momentum, float* running_mean, float* running_var, float* save_mean, float* save_rstd, float* y, int y_pitch,
                       void* workspace, void* stream);
int fb200_bn_train_bwd(const float* x, int x_pitch, const float* dy, int dy_pitch, const float* y, int y_pitch, int64_t R, int C, const float* gamma,
                       const float* beta, const float* save_mean, const float* save_rstd, int act, float* dx, int dx_pitch, float* dres, int dres_pitch,
                       float* dgamma, float* dbeta, int accumulate, void* workspace, void* stream);
/* The same BatchNorm in phases, for the two variants the reference's trainer switches to:
 *   torch.nn.SyncBatchNorm.convert_sync_batchnorm when world_size > 1 (trainer/trainer.py:334): fb200_bn_stats gives the LOCAL mean / biased variance per channel,
 *     the host all-gathers them with the row counts and combines (what aten's batch_norm_gather_stats_with_counts does), fb200_bn_apply normalises with the GLOBAL
 *     statistics; backward: fb200_bn_bwd_reduce gives the local sum(g), sum(g*xhat) (g = dy through the fused activation), the host all-reduces them,
 *     fb200_bn_bwd_apply forms dx with the global sums and inv_count = 1 / total rows;
 *   FrozenBatchNorm2d (nn/backbone/resnet.py:226-250, TrainerArgs.freeze_bn): fb200_bn_apply with the RUNNING statistics, fb200_bn_bwd_apply with zero sums. */
int fb200_bn_stats(const float* x, int x_pitch, int64_t R, int C, float* mean, float* var_biased, void* workspace, void* stream);
/* SyncBatchNorm, between the all_gather of the per-rank statistics and fb200_bn_apply: all_stats [world][2C+1] = rows [mean (C) | biased variance (C) | row count] ->
 * global mean / rstd, running statistics updated with the unbiased variance over the global count (aten batch_norm_gather_stats_with_counts), and inv_total[0] = 1 / (sum of
 * the row counts) left on the device for the backward pass (no host read-back between two layers). */
int fb200_bn_sync_combine(const float* all_stats, int world, int C, float eps, float momentum, float* running_mean, float* running_var, float* mean, float* rstd,
                          float* inv_total, void* stream);
int fb200_bn_apply(const float* x, int x_pitch, int64_t R, int C, const float* mean, const float* rstd, const float* gamma, const float* beta,
                   const float* res, int res_pitch, int act, float* y, int y_pitch, void* stream);
int fb200_bn_bwd_reduce(const float* x, int x_pitch, const float* dy, int dy_pitch, const float* y, int y_pitch, int64_t R, int C, const float* gamma,
                        const float* beta, const float* mean, const float* rstd, int act, float* sum_dy, float* sum_dy_xhat, void* workspace, void* stream);
int fb200_bn_bwd_apply(const float* x, int x_pitch, const float* dy, int dy_pitch, const float* y, int y_pitch, int64_t R, int C, const float* gamma,
                       const float* beta, const float* mean, const float* rstd, const float* sum_dy, const float* sum_dy_xhat, float inv_count, int act,
                       float* dx, int dx_pitch, float* dres, int dres_pitch, void* stream);
/* out = act(a + b) when dy == NULL, else out = dy * act'(a + b)   (RepVggBlock :45, GELU of the AIFI FFN) */
int fb200_add_act(const float* a, const float* b, const float* dy, int act, int64_t n, float* out, void* stream);
int fb200_maxpool3x3s2_bwd(const float* x, const float* dy, int B, int H, int W, int C, float* dx, void* stream);
int fb200_avgpool2x2_ceil_bwd(const float* dy, int B, int H, int W, int C, float* dx, void* stream);
int fb200_resize_bilinear_bwd(const float* dy, int dy_pitch, int B, int H, int W, int C, int Ho, int Wo, float* dx, void* stream);
/* nn.LayerNorm backward over s = x (+ res): dx is the gradient w.r.t. s */
int fb200_layernorm_bwd(const float* x, const float* res, const float* gamma, const float* dy, int64_t M, int C, float eps, float* dx, float* dgamma,
                        float* dbeta, int accumulate, void* workspace, void* stream);
/* nn.MultiheadAttention core backward (o = forward output).  Q, K, V and dO of a (batch, head) stay in shared memory: Lq = Lk up to 433.
 * B, Lq, Lk, heads > 0 and every pitch >= heads*32, else FB200_ERR_INVALID without a launch. */
int fb200_attention_bwd(const float* q, int q_pitch, const float* k, int k_pitch, const float* v, int v_pitch, const float* o, int o_pitch,
                        const float* dout, int do_pitch, int B, int Lq, int Lk, int heads, int head_dim, float scale, float* dq, int dq_pitch,
                        float* dk, int dk_pitch, float* dv, int dv_pitch, void* stream);
/* adjoint of fb200_msda (fp32): the gradient is ADDED to dvalue [B,S,heads*32] with atomics (zero it for a plain gradient); doa like oa, overwritten.
 * Pitches: v_pitch, do_pitch, dv_pitch >= heads*32 and oa_pitch, doa_pitch >= heads*L*P*3, else FB200_ERR_INVALID without a launch. */
int fb200_msda_bwd(const float* value, int v_pitch, const float* oa, int oa_pitch, const float* ref, const float* dout, int do_pitch,
                   const int* shapes_host, int L, int P, int B, int S, int Q, int heads, float* dvalue, int dv_pitch, float* doa, int doa_pitch,
                   void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FOCOOS_B200_H_ */
