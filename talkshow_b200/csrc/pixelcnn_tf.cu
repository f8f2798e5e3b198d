// talkshow_b200 — time-parallel teacher-forced GatedPixelCNN.forward (nets/spg/gated_pixelcnn_v2.py:61-87,130-150,
// bh_model=True) with a per-position cross-entropy: ts_pixelcnn_score.
//
// With every code known, no position waits for another, so the whole forward is a fixed sequence of large GEMMs over all
// B x T x 2 grid positions ("cells") instead of the sampler's serial chain of stages per row.
//
// Layout: an activation is channel-last over cells, cell (t, j) of sample b at row 2t + j of an Act3 with T' = 2T rows
// (the reference grid [B, C, T, 2] read row-major).  The inputs of the masked convs carry 6 zero rows (= 3 grid rows)
// in front of every sample.  Then
//  * vert_stack of output row t reads the grid rows t-R..t-1+r0 (R = 3 and the masked row t dropped for layer 0 /
//    mask A, R = 1 and rows t-1, t later), both columns: that is the contiguous cell window [2(t-R), 2t + 2r0) for BOTH
//    output columns, so the conv is one stride-2 implicit GEMM (k = 6 or 4 cells) with N = 2 x 2D: the weights of output
//    column j sit in rows [2Dj, 2Dj + 2D) and the kw taps that fall on the width padding are zero;
//  * horiz_stack reads columns j-1, j of row t: the window [2t, 2t+2) (layer 0, mask A: only cell 2t), stride 2, N = 4D;
//  * vert_to_horiz, horiz_resid, fusion_v / fusion_h, embedding_aud and output_conv are 1x1 convs over cells.
// The GEMMs run on conv_auto (wgmma fp16-split kernel by default, the FFMA kernel after ts_set_tensor_cores(e, 0)), except
// output_conv, which always runs on the FFMA kernel (see tf_forward); the
// stride-2 output rows [B][T][4D] are the cells [B][2T][2D] of the same memory.  vert_to_horiz takes horiz_stack's
// output as its residual, so the horizontal gate reads one tensor.
#include <memory>

#include "convstack.h"
#include "pixelcnn.h"

namespace ts {

constexpr int TF_PAD = 6;   // zero cells in front of every sample: 3 grid rows, layer 0's vertical reach

struct TfLayer {
  Layer vs, hs, v2h, hres;
};
struct TfPlan {
  int D = 0, L = 0, ncls = 0;
  std::vector<TfLayer> layers;
  Layer emb_aud, fuse_v_a, fuse_v_x, fuse_h_a, fuse_h_x, out0, out2;
  float* emb = nullptr;  // [2048][D]
  float* cls = nullptr;  // [L][ncls][2D]
};

// ---- packing ---------------------------------------------------------------------------------
// split: also the operand copies of the tensor-core kernel (fp16 planes, 3xTF32 pair), else fp32 for the FFMA kernel only
static Layer tf_upload(ts_engine* e, const std::vector<float>& W, const float* bias, int N, int taps, int cin, bool split = true) {
  Layer L;
  L.N = N; L.K = taps * cin; L.taps = taps; L.cin = cin;
  if (split) upload_weights(e, W, &L);
  else L.W = e->upload(W);
  if (bias) L.bias = e->upload(std::vector<float>(bias, bias + N));
  return L;
}

// vert_stack [2D, D, kh, 3] as the stride-2 cell conv: tap = 2 r + c (grid row r of the window, input column c), output
// column j uses kw = c - j + 1
static Layer pack_vert(ts_engine* e, const Ckpt& ck, int l, int D) {
  const std::string p = "layers." + std::to_string(l) + ".vert_stack.";
  const int kh = l == 0 ? 4 : 2, rows = l == 0 ? 3 : 2, taps = 2 * rows, N = 4 * D;
  const float* w = ck.f32(p + "weight", {2 * D, D, kh, 3});
  const float* b = ck.f32(p + "bias", {2 * D});
  std::vector<float> W((size_t)N * taps * D, 0.f), bias(N);
  for (int j = 0; j < 2; ++j)
    for (int o = 0; o < 2 * D; ++o) {
      const int n = j * 2 * D + o;
      bias[n] = b[o];
      for (int tap = 0; tap < taps; ++tap) {
        const int r = tap / 2, kw = tap % 2 - j + 1;
        if (kw < 0 || kw > 2) continue;
        for (int c = 0; c < D; ++c) W[((size_t)n * taps + tap) * D + c] = w[(((size_t)o * D + c) * kh + r) * 3 + kw];
      }
    }
  return tf_upload(e, W, bias.data(), N, taps, D);
}

// horiz_stack [2D, D, 1, 2]: tap = input column c, output column j uses kw = c - j + 1 (kw 1 masked in layer 0)
static Layer pack_horiz(ts_engine* e, const Ckpt& ck, int l, int D) {
  const std::string p = "layers." + std::to_string(l) + ".horiz_stack.";
  const int taps = l == 0 ? 1 : 2, N = 4 * D;
  const float* w = ck.f32(p + "weight", {2 * D, D, 1, 2});
  const float* b = ck.f32(p + "bias", {2 * D});
  std::vector<float> W((size_t)N * taps * D, 0.f), bias(N);
  for (int j = 0; j < 2; ++j)
    for (int o = 0; o < 2 * D; ++o) {
      const int n = j * 2 * D + o;
      bias[n] = b[o];
      for (int tap = 0; tap < taps; ++tap) {
        const int kw = tap - j + 1;
        if (kw < 0 || kw > 1 || (l == 0 && kw == 1)) continue;
        for (int c = 0; c < D; ++c) W[((size_t)n * taps + tap) * D + c] = w[((size_t)o * D + c) * 2 + kw];
      }
    }
  return tf_upload(e, W, bias.data(), N, taps, D);
}

// 1x1 conv weight [N, ldw, 1, 1], input channels [koff, koff + K)
static Layer pack_dense(ts_engine* e, const float* w, int ldw, int koff, const float* b, int N, int K, bool split = true) {
  std::vector<float> W((size_t)N * K);
  for (int n = 0; n < N; ++n)
    for (int k = 0; k < K; ++k) W[(size_t)n * K + k] = w[(size_t)n * ldw + koff + k];
  return tf_upload(e, W, b, N, 1, K, split);
}

void* tf_build(ts_engine* e, const Ckpt& ck, int L, int D, int ncls) {
  if (e->host_only) return nullptr;
  std::unique_ptr<TfPlan> P(new TfPlan());
  P->D = D; P->L = L; P->ncls = ncls;
  for (int l = 0; l < L; ++l) {
    const std::string p = "layers." + std::to_string(l) + ".";
    TfLayer t;
    t.vs = pack_vert(e, ck, l, D);
    t.hs = pack_horiz(e, ck, l, D);
    t.v2h = pack_dense(e, ck.f32(p + "vert_to_horiz.weight", {2 * D, 2 * D, 1, 1}), 2 * D, 0,
                       ck.f32(p + "vert_to_horiz.bias", {2 * D}), 2 * D, 2 * D);
    t.hres = pack_dense(e, ck.f32(p + "horiz_resid.weight", {D, D, 1, 1}), D, 0, ck.f32(p + "horiz_resid.bias", {D}), D, D);
    P->layers.push_back(t);
  }
  P->emb_aud = pack_dense(e, ck.f32("embedding_aud.weight", {D, 256, 1, 1}), 256, 0, ck.f32("embedding_aud.bias", {D}), D, 256);
  // fusion(cat[x, a]) = W[:, :D] x + (W[:, D:] a + b): the audio half (with the bias) is the residual of the x half
  const float* fv = ck.f32("fusion_v.weight", {D, 2 * D, 1, 1});
  const float* fh = ck.f32("fusion_h.weight", {D, 2 * D, 1, 1});
  P->fuse_v_a = pack_dense(e, fv, 2 * D, D, ck.f32("fusion_v.bias", {D}), D, D);
  P->fuse_v_x = pack_dense(e, fv, 2 * D, 0, nullptr, D, D);
  P->fuse_h_a = pack_dense(e, fh, 2 * D, D, ck.f32("fusion_h.bias", {D}), D, D);
  P->fuse_h_x = pack_dense(e, fh, 2 * D, 0, nullptr, D, D);
  P->out0 = pack_dense(e, ck.f32("output_conv.0.weight", {512, D, 1, 1}), D, 0, ck.f32("output_conv.0.bias", {512}), 512, D, false);
  P->out2 = pack_dense(e, ck.f32("output_conv.2.weight", {PIX_NCODE, 512, 1, 1}), 512, 0,
                       ck.f32("output_conv.2.bias", {PIX_NCODE}), PIX_NCODE, 512, false);
  const float* ew = ck.f32("embedding.weight", {PIX_NCODE, D});
  P->emb = e->upload(std::vector<float>(ew, ew + (size_t)PIX_NCODE * D));
  std::vector<float> cls((size_t)L * ncls * 2 * D);
  for (int l = 0; l < L; ++l) {
    const float* c = ck.f32("layers." + std::to_string(l) + ".class_cond_embedding.weight", {ncls, 2 * D});
    std::copy(c, c + (size_t)ncls * 2 * D, cls.begin() + (size_t)l * ncls * 2 * D);
  }
  P->cls = e->upload(cls);
  return P.release();
}

void tf_free(void* p) { delete (TfPlan*)p; }

// ---- kernels ----------------------------------------------------------------------------------
// element (b, t, c) of an activation whatever its storage: plain fp32, 3xTF32 (hi, lo) pair or fp32 + fp16-split planes
__device__ __forceinline__ float tf_load(const Act3& a, int b, int t, int c) {
  float v = a.row(b, t)[c];
  if (a.lo) v += a.row_lo(b, t)[c];
  return v;
}
__device__ __forceinline__ void tf_store(const Act3& a, int b, int t, int c, float v) {
  if (a.lo) {
    const float h = __uint_as_float(__float_as_uint(v) & 0xffffe000u);
    a.row(b, t)[c] = h;
    a.row_lo(b, t)[c] = v - h;
    return;
  }
  a.row(b, t)[c] = v;
  if (a.h16) split16(v, a.row_h16(b, t)[c], a.row_l16(b, t)[c]);
}

// aud [B, 256, T] -> cells [B][2T][256] (the reference repeats the audio over the two columns)
__global__ void tf_aud_cells_kernel(const float* __restrict__ aud, Act3 out, int T) {
  const long n = (long)out.B * 256 * out.T;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const int cell = i % out.T;
    const long bc = i / out.T;
    const int c = bc % 256, b = bc / 256;
    tf_store(out, b, cell, c, aud[((long)b * 256 + c) * T + (cell >> 1)]);
  }
}

// nn.Embedding of the codes [B, T, 2] into the cells
__global__ void tf_embed_kernel(const int64_t* __restrict__ codes, const float* __restrict__ emb, Act3 out) {
  const int D = out.C;
  const long n = (long)out.B * out.T * D;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const int c = i % D;
    const long cell = i / D;
    tf_store(out, (int)(cell / out.T), (int)(cell % out.T), c, emb[codes[cell] * D + c]);
  }
}

// GatedActivation (:16-22) of x + class_cond_embedding[label]: y = tanh(x[:D] + h[:D]) * sigmoid(x[D:] + h[D:]).
// style [B][T][ncls] (ts_pixelcnn_score_styled): h of cell (t, j) is the blend of row t's speaker weights (style_pair, the
// sampler's fp32 order) and label is not read; null: the label's row.
__global__ void tf_gate_kernel(Act3 x, const float* __restrict__ cls, const int64_t* __restrict__ label, int ncls, Act3 y,
                               const float* __restrict__ style) {
  const int D = y.C;
  const long n = (long)y.B * y.T * D;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const int o = i % D;
    const long cell = i / D;
    const int b = (int)(cell / y.T), t = (int)(cell % y.T);
    float ht, hs;
    if (style) {
      style_pair(cls, style + ((size_t)b * (y.T >> 1) + (t >> 1)) * ncls, ncls, D, o, ht, hs);
    } else {
      const long lab = min(max(label[b], (int64_t)0), (int64_t)ncls - 1);
      const float* h = cls + lab * 2 * D;
      ht = h[o];
      hs = h[D + o];
    }
    const float a = tf_load(x, b, t, o) + ht, g = tf_load(x, b, t, D + o) + hs;
    tf_store(y, b, t, o, tanhf(a) * (1.f / (1.f + expf(-g))));
  }
}

// one warp per cell: nll = logsumexp(logits) - logits[code] over the 2048 logits (F.cross_entropy, reduction='none');
// optionally the logits in the reference's [B, 2048, T, 2] layout
constexpr int TF_NLL_WARPS = 8;
__global__ void __launch_bounds__(TF_NLL_WARPS * 32) tf_nll_kernel(Act3 lg, const int64_t* __restrict__ codes,
                                                                   float* __restrict__ nll, float* __restrict__ logits_out) {
  const int cell = blockIdx.x * TF_NLL_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (cell >= lg.B * lg.T) return;
  const int b = cell / lg.T, tc = cell % lg.T;
  const float4* x = reinterpret_cast<const float4*>(lg.row(b, tc));
  float4 v[PIX_NCODE / 128];
  float m = -INFINITY;
#pragma unroll
  for (int i = 0; i < PIX_NCODE / 128; ++i) {
    v[i] = x[lane + 32 * i];
    m = fmaxf(m, fmaxf(fmaxf(v[i].x, v[i].y), fmaxf(v[i].z, v[i].w)));
  }
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < PIX_NCODE / 128; ++i) s += expf(v[i].x - m) + expf(v[i].y - m) + expf(v[i].z - m) + expf(v[i].w - m);
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) nll[cell] = (m + logf(s)) - lg.row(b, tc)[codes[cell]];
  if (logits_out) {
    const int T = lg.T >> 1, t = tc >> 1, j = tc & 1;
    float* out = logits_out + ((long)b * PIX_NCODE * T + t) * 2 + j;
#pragma unroll
    for (int i = 0; i < PIX_NCODE / 128; ++i) {
      const long k = 4L * (lane + 32 * i);
      out[(k + 0) * T * 2] = v[i].x;
      out[(k + 1) * T * 2] = v[i].y;
      out[(k + 2) * T * 2] = v[i].z;
      out[(k + 3) * T * 2] = v[i].w;
    }
  }
}

static int tf_blocks(ts_engine* e, long n) { return (int)std::min<long>((n + 255) / 256, (long)e->sm_count * 16); }

// ---- forward ----------------------------------------------------------------------------------
static void tf_forward(ts_engine* e, const TfPlan* P, const float* aud, const int64_t* label, const float* style,
                       const int64_t* codes, float* nll, float* logits_out, int B, int T, cudaStream_t s) {
  const int D = P->D, R = 2 * T;
  const bool sp = e->use_tc;   // GEMM operands stored in the split format the tensor-core kernel reads
  auto cells = [&](int C, int pad, bool split) { return new_act(e, B, R, C, pad, s, split); };
  auto as_cells = [&](Act3 a) { a.T *= 2; a.C /= 2; return a; };   // stride-2 conv output rows [T][4D] -> cells [2T][2D]
  const bool run = !e->ws.sizing;

  Act3 ac = cells(256, 0, sp);
  if (run) {
    tf_aud_cells_kernel<<<tf_blocks(e, (long)B * 256 * R), 256, 0, s>>>(aud, ac, T);
    e->launches++;
    TS_CUDA(cudaGetLastError());
  }
  Act3 ae = cells(D, 0, sp), av = cells(D, 0, false), ah = cells(D, 0, false);
  conv_auto(e, P->emb_aud, ac, 1, 1, 0, ae, R, ACT_NONE, nullptr, s);
  conv_auto(e, P->fuse_v_a, ae, 1, 1, 0, av, R, ACT_NONE, nullptr, s);
  conv_auto(e, P->fuse_h_a, ae, 1, 1, 0, ah, R, ACT_NONE, nullptr, s);

  Act3 x0 = cells(D, TF_PAD, sp);
  if (run) {
    tf_embed_kernel<<<tf_blocks(e, (long)B * R * D), 256, 0, s>>>(codes, P->emb, x0);
    e->launches++;
    TS_CUDA(cudaGetLastError());
  }
  Act3 hv = new_act(e, B, T, 4 * D, 0, s, sp), hh = new_act(e, B, T, 4 * D, 0, s, false);
  Act3 sum = cells(2 * D, 0, false), g = cells(D, 0, sp), tv = cells(D, 0, sp), th = cells(D, 0, sp);
  Act3 xv[2] = {cells(D, TF_PAD, sp), cells(D, TF_PAD, sp)}, xh[2] = {cells(D, TF_PAD, sp), cells(D, TF_PAD, sp)};
  auto gate = [&](const Act3& x, int l, const Act3& y) {
    if (!run) return;
    tf_gate_kernel<<<tf_blocks(e, (long)B * R * D), 256, 0, s>>>(x, P->cls + (size_t)l * P->ncls * 2 * D, label, P->ncls, y, style);
    e->launches++;
    TS_CUDA(cudaGetLastError());
  };
  int cur = 0;
  for (int l = 0; l < P->L; ++l) {
    const TfLayer& w = P->layers[l];
    const Act3& in_v = l == 0 ? x0 : xv[cur];
    const Act3& in_h = l == 0 ? x0 : xh[cur];
    const int nxt = cur ^ 1;
    conv_auto(e, w.vs, in_v, l == 0 ? 6 : 4, 2, l == 0 ? 6 : 2, hv, T, ACT_NONE, nullptr, s);
    conv_auto(e, w.hs, in_h, l == 0 ? 1 : 2, 2, 0, hh, T, ACT_NONE, nullptr, s);
    const Act3 hv_c = as_cells(hv), hh_c = as_cells(hh);
    conv_auto(e, w.v2h, hv_c, 1, 1, 0, sum, R, ACT_NONE, &hh_c, s);            // v2h + h_horiz
    gate(hv_c, l, l == 0 ? tv : xv[nxt]);                                        // out_v
    gate(sum, l, g);                                                             // out
    conv_auto(e, w.hres, g, 1, 1, 0, l == 0 ? th : xh[nxt], R, ACT_NONE, l == 0 ? nullptr : &in_h, s);   // out_h
    if (l == 0) {   // audio fusion before layer 1 (:134-144)
      conv_auto(e, P->fuse_v_x, tv, 1, 1, 0, xv[nxt], R, ACT_NONE, &av, s);
      conv_auto(e, P->fuse_h_x, th, 1, 1, 0, xh[nxt], R, ACT_NONE, &ah, s);
    }
    cur = nxt;
  }
  Act3 y1 = cells(512, 0, false), lg = cells(PIX_NCODE, 0, false);
  // output_conv on the FFMA kernel (round-to-nearest fp32): the tensor core's fp32 accumulation truncates toward zero, which
  // shrinks the logits' scale, and -log softmax(logits)[code] moves with that scale by about (max logit - logit[code])
  conv1d(e, P->out0, xh[cur], 1, 1, 0, y1, R, ACT_RELU, nullptr, s);
  conv1d(e, P->out2, y1, 1, 1, 0, lg, R, ACT_NONE, nullptr, s);
  if (run) {
    tf_nll_kernel<<<cdiv(B * R, TF_NLL_WARPS), TF_NLL_WARPS * 32, 0, s>>>(lg, codes, nll, logits_out);
    e->launches++;
    TS_CUDA(cudaGetLastError());
  }
}

}  // namespace ts

using namespace ts;

static void score_call(ts_engine* e, const float* aud, const int64_t* label, const float* style, const int64_t* codes,
                       float* nll_out, float* logits_out, int B, int T, void* stream) {
  const TfPlan* P = (const TfPlan*)e->pix->tf;
  if (!P) fail(TS_ERR_NOT_LOADED, "pixelcnn scoring weights not loaded");
  cudaStream_t s = (cudaStream_t)stream;
  e->ws.begin_sizing();
  tf_forward(e, P, aud, label, style, codes, nll_out, logits_out, B, T, s);
  const size_t need = e->ws.need;
  e->ws.buf.ensure(need + 256);
  e->ws.begin(need);
  tf_forward(e, P, aud, label, style, codes, nll_out, logits_out, B, T, s);
}

extern "C" int ts_pixelcnn_score(ts_engine* e, const float* aud, const int64_t* label, const int64_t* codes, float* nll_out,
                                 float* logits_out, int B, int T, void* stream) {
  TS_API_BEGIN(e)
  if (!e->pix) fail(TS_ERR_NOT_LOADED, "pixelcnn weights not loaded");
  ts::require_device(e);
  if (B <= 0 || T <= 0) fail(TS_ERR_INVALID, "pixelcnn_score: B=%d T=%d", B, T);
  if (!aud || !label || !codes || !nll_out) fail(TS_ERR_INVALID, "pixelcnn_score: aud, label, codes and nll_out are required");
  score_call(e, aud, label, nullptr, codes, nll_out, logits_out, B, T, stream);
  TS_API_END(e)
}

// style [B,T,ncls] (device): per-row speaker weights in place of label (which may then be NULL); NULL: ts_pixelcnn_score.
extern "C" int ts_pixelcnn_score_styled(ts_engine* e, const float* aud, const int64_t* label, const float* style, int ncls,
                                        const int64_t* codes, float* nll_out, float* logits_out, int B, int T, void* stream) {
  TS_API_BEGIN(e)
  if (!e->pix) fail(TS_ERR_NOT_LOADED, "pixelcnn weights not loaded");
  ts::require_device(e);
  if (B <= 0 || T <= 0) fail(TS_ERR_INVALID, "pixelcnn_score_styled: B=%d T=%d", B, T);
  check_style(e, label, style, ncls, "ts_pixelcnn_score_styled");
  if (!aud || !codes || !nll_out) fail(TS_ERR_INVALID, "pixelcnn_score_styled: aud, codes and nll_out are required");
  score_call(e, aud, label, style, codes, nll_out, logits_out, B, T, stream);
  TS_API_END(e)
}
