// talkshow_b200 — incremental gated-PixelCNN sampler: execution plan shared by the packer
// (host), the CUDA executor (pixelcnn.cu) and the CPU plan interpreter used by the tests.
#pragma once
#include "kernels.h"

namespace ts {

constexpr int PIX_D = 256;      // hidden width (config/body_pixel.json: convert_to_6d=false)
constexpr int PIX_MB = 64;      // batch tile: every activation row is [channel][64 samples]
constexpr int PIX_SEG = PIX_D * PIX_MB;  // floats in one [256][64] activation segment
constexpr int PIX_THREADS = 256;
constexpr int PIX_MAXROWS = 16; // weight rows one CTA handles per stage
constexpr int PIX_WBUF = 18560; // floats per weight staging buffer (74.2 KB), two buffers
constexpr int PIX_NCODE = 2048;

enum PixEpi {
  EPI_IDLE = 0,
  EPI_VERT0 = 1,   // layer-0 vertical stack (mask A), one output column
  EPI_VERT = 2,    // layers >= 1 vertical stack, one output column
  EPI_V2H = 3,     // vert_to_horiz of one layer, both columns (2 passes)
  EPI_FUSEV = 4,   // fusion_v (x_v half), both columns (2 passes)
  EPI_HGATE = 5,   // horizontal stack + gate, one column
  EPI_HRES = 6,    // horiz_resid (+ residual)
  EPI_FUSEH = 7,   // fusion_h (x_h half)
  EPI_OUT1 = 8,    // output_conv.0 + ReLU
  EPI_OUT2 = 9,    // output_conv.2 -> logits
  EPI_SAMPLE = 10, // softmax + categorical draw + embedding gather (K = 1: also emits layer-0 G of column 1)
  // fused plan (52 stages): linear stages folded into the gate matmul that consumes them
  EPI_HRESF = 11,  // (fusion_h . horiz_resid_0) G_0 + audio term -> x_h[1]
  EPI_HGATE2 = 12, // gate of layer l on (horiz_stack_l . horiz_resid_{l-1}) G_{l-1} + horiz_stack_l x_h[l-1] (+ column-0 tap)
  EPI_OUT1F = 13,  // output_conv.0 on (W horiz_resid_{L-1}) G_{L-1} + W x_h[L-1], ReLU
  // schedule 2: vert_to_horiz leaves the vertical stages and runs one column at a time beside the horizontal stage
  // that precedes its consumer
  EPI_V2H1 = 14    // vert_to_horiz of one layer, column t.col only
};

struct PixTask {  // one CTA's work in one stage (8 ints)
  int epi, layer, col, row0, nrows, wofs, K, rpad;
};

struct PixLayout {  // arena offsets in floats
  int E, XV1P, XV, HV, V2H, G, XHP, XH, Y, LOG, CLS, total;
};

struct PixelPlan {
  int L = 0, ncta = 0, nstages = 0, nclasses = 4;
  int D = PIX_D;               // hidden width of the checkpoint (the grid-wide executor is built for 256 only)
  bool has_v1 = false;         // stage table / blob of the grid-wide executor built (D == 256)
  int cl = 1;                  // CTAs per work unit
  bool fused = false;          // 52-stage plan (EPI_HRESF / EPI_HGATE2 / EPI_OUT1F), else the plain 84-stage plan
  int sched = 1;               // 0 plain, 1 fused, 2 fused + vert_to_horiz moved into the horizontal pass (EPI_V2H1)
  PixLayout lay;
  std::vector<PixTask> table;  // [nstages][ncta]
  std::vector<float> blob;     // packed per-task weights: [K][rpad] then bias [rpad]
  int64_t row_bytes = 0;       // algorithmic weight bytes per latent row (dense fp32 weights, once)
  int64_t staged_row_bytes = 0;  // bytes the kernel actually stages per row (blob incl. padding/duplication)
  // device copies
  PixTask* d_table = nullptr;
  float* d_blob = nullptr;
  float* d_emb = nullptr;      // [2048][256]
  float* d_cls = nullptr;      // [L][4][512]
  float* d_arena = nullptr;
  unsigned* d_barrier = nullptr;
  Layer emb_aud, fuse_v_a, fuse_h_a;  // audio terms (precomputed per call for all rows)
  void* p3 = nullptr;          // Plan3 of the cluster-resident executor (pixelcnn3.inc)
  void* tf = nullptr;          // TfPlan of the time-parallel teacher-forced scorer (pixelcnn_tf.cu)
  unsigned long long* d_trace = nullptr;  // stage trace buffer (ts_pixelcnn_trace)
  int trace_row = -1;
  bool timing = false, pending = false;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int64_t timed_rows = 0, timed_launches = 0;
};

// Sampling controls of ts_pixelcnn_sample_ctl / ts_body_sample_ctl (include/talkshow_b200.h).  A call without them runs the
// default sampler kernels; a call with them runs the WARP instantiations, whose only difference is the draw.
struct SampleCtl {
  float temperature = 1.f;   // > 0: softmax(l / temperature); 0: greedy (first-index argmax of l, noise unread)
  int top_k = 0;             // 0 or 2048: off; else keep codes with l >= the k-th largest logit
  float* logp_out = nullptr; // [B,T,2] log_softmax(l)[code] of the untempered, untruncated model, or null
  float top_p = 1.f;         // < 1: nucleus sampling on integer masses (nucleus_key, pixelcnn.cu); 1: off
  float min_p = 0.f;         // > 0: keep codes with exp(l / t - max l / t) >= min_p; 0: off
  int* kept_out = nullptr;   // [B,T,2] size of each draw's final keep set, or null
};
// Validates the controls (TS_ERR_INVALID): temperature finite and >= 0, top_k in [0, 2048], top_p in (0, 1], min_p in
// [0, 1], noise (or seeds) given when sampling.
void check_sample_ctl(const SampleCtl& c, const float* noise, const int64_t* seeds = nullptr);
// The public struct as the internal one (TS_ERR_INVALID when null).
SampleCtl sample_ctl_of(const ts_sample_ctl* c);

// aud: AudioEncoder output, channel-last [B, T0+T, 256].  ctl = nullptr: the default sampler.  seeds [B] (device): the
// draws' noise is computed from the per-clip seeds (ts_pixelcnn_sample_seeded) and `noise` is not read.  anchors
// [B,T,2] (device): the pinned draws of ts_pixelcnn_sample_anchored; the call then runs the WARP kernels, at the default
// controls when ctl is null.  style [B,T0+T,ncls] (device): the speaker schedule of ts_pixelcnn_sample_styled (label
// unread), likewise on the WARP kernels.  clip_ctl [B] (HOST, validated with check_clip_ctl): the per-clip controls of
// ts_pixelcnn_sample_clips, copied to the workspace on s; each clip draws with its entry in place of ctl's four controls.
// clip_shape [B] (HOST, validated with check_clip_shape) and code_bias [B,2,2048] (device): the logit shaping of
// ts_pixelcnn_sample_shaped, likewise on the WARP kernels (clip_shape copied to the workspace on s).
// guide [B / 2] (HOST, validated with check_guidance): the scales of ts_pixelcnn_sample_guided, copied to the workspace on
// s.  B is then the branch count 2P: aud, label, style, idx_out and logits_out are per branch; noise [2T][P][2048], seeds,
// anchors, pre, clip_ctl, clip_shape and code_bias are per pair (pre is copied once per branch into the workspace).
void pixelcnn_generate_act(ts_engine* e, const Act3& aud, const int64_t* label, const float* noise, int64_t* idx_out,
                           float* logits_out, int B, int T, const int64_t* pre, int T0, cudaStream_t s,
                           bool logits_all = false, const SampleCtl* ctl = nullptr, const int64_t* seeds = nullptr,
                           const int64_t* anchors = nullptr, const float* style = nullptr,
                           const ts_clip_ctl* clip_ctl = nullptr, const ts_clip_shape* clip_shape = nullptr,
                           const float* code_bias = nullptr, const float* guide = nullptr);
// The class terms of gate channel q (tanh half) and D + q (sigmoid half) under one row's speaker weights w[0..ncls)
// (ts_pixelcnn_sample_styled): acc = w0 E[0][ch], then acc + w_s E[s][ch] for s = 1 .. ncls-1, every product and sum
// rounded to fp32 without contraction.  tab: one layer's class_cond_embedding [ncls][2D]; w null (a padding sample of the
// tile): zero, as in the CLS arena.
__device__ __forceinline__ void style_pair(const float* __restrict__ tab, const float* __restrict__ w, int ncls, int D, int q,
                                           float& ct, float& cs) {
  if (!w) { ct = 0.f; cs = 0.f; return; }
  const float w0 = __ldg(w);
  ct = __fmul_rn(w0, __ldg(tab + q));
  cs = __fmul_rn(w0, __ldg(tab + D + q));
  for (int s = 1; s < ncls; ++s) {
    const float ws = __ldg(w + s);
    const float* e = tab + (size_t)s * 2 * D;
    ct = __fadd_rn(ct, __fmul_rn(ws, __ldg(e + q)));
    cs = __fadd_rn(cs, __fmul_rn(ws, __ldg(e + D + q)));
  }
}
// Styled calls blend at most this many classes (ts_pixelcnn_sample_styled).
constexpr int PIX_MAXCLS = 16;
// The class input of a styled entry point (TS_ERR_INVALID): without style a label is required; with style, ncls in
// [1, PIX_MAXCLS] and equal to the loaded prior's class count.
void check_style(const ts_engine* e, const int64_t* label, const float* style, int ncls, const char* who);
// The noise source of an anchored call (TS_ERR_INVALID): exactly one of noise and seeds unless ctl is greedy.
void check_anchored_source(const SampleCtl* ctl, const float* noise, const int64_t* seeds, const char* who);
// The per-clip controls of ts_pixelcnn_sample_clips (TS_ERR_INVALID, naming the clip): every entry by the rules of
// check_sample_ctl, and exactly one of noise and seeds when any clip samples (temperature > 0).  clip_ctl: B host entries.
void check_clip_ctl(const ts_clip_ctl* clip_ctl, int B, const float* noise, const int64_t* seeds, const char* who);
// The per-clip shaping of ts_pixelcnn_sample_shaped (TS_ERR_INVALID, naming the clip): a finite repetition_penalty >= 1
// and a repetition_window >= 1.  clip_shape: B host entries.
void check_clip_shape(const ts_clip_shape* clip_shape, int B, const char* who);
// The scales of ts_pixelcnn_sample_guided (TS_ERR_INVALID, naming the pair): P host values, each finite and in
// [0, TS_GUIDANCE_MAX]; NULL is refused.
void check_guidance(const float* guidance, int P, const char* who);
// The controls of a shaped call: with clip_ctl, check_clip_ctl and ctl's logp_out / kept_out; else ctl's controls (the
// default draw when ctl is NULL), checked with check_sample_ctl and check_anchored_source.
SampleCtl shaped_ctl(const ts_sample_ctl* ctl, const ts_clip_ctl* clip_ctl, int B, const float* noise, const int64_t* seeds,
                     const char* who);
// idx [B,T,2] -> idx_c [2][B][T]; optionally copies idx to codes_out
void split_codes(ts_engine* e, const int64_t* idx, int64_t* idx_c, int B, int T, int64_t* codes_out, cudaStream_t s);
// A guided call's idx [2P,T,2] -> idx_c [2][P][T] of the conditional branches (rows 2p); optionally copies idx to codes_out
void split_guided_codes(ts_engine* e, const int64_t* idx, int64_t* idx_c, int P, int T, int64_t* codes_out, cudaStream_t s);
void pixel_destroy(ts_engine* e);
// weights of ts_pixelcnn_score packed for its GEMMs (pixelcnn_tf.cu); nullptr on a host-only engine
void* tf_build(ts_engine* e, const Ckpt& ck, int L, int D, int ncls);
void tf_free(void* p);
void face_destroy(ts_engine* e);
// face.cu: s2g_face.Generator.forward into out [B,frame,ts_face_dim] (workspace from e->ws, sizing-pass aware), and
// whether the loaded net is the identity net (reads id)
void face_run(ts_engine* e, const float* wave, const float* idv, float* out, int B, int N, int frame, cudaStream_t s);
bool face_has_identity(const ts_engine* e);
void mfcc_destroy(ts_engine* e);
void smplx_destroy(ts_engine* e);
void nccl_destroy(ts_engine* e);

}  // namespace ts
