// talkshow_b200 — gated PixelCNN prior sampled step by step, as an exact O(T) incremental
// evaluation (reference: GatedPixelCNN.generate / forward / GatedMaskedConv2d.forward,
// nets/spg/gated_pixelcnn_v2.py:61-87,130-177 — which re-runs the whole network over the whole
// [T,2] grid for each of the 2T sampled positions).
//
// Design (DESIGN.md §3): one PERSISTENT cooperative kernel, one CTA per SM.  A latent row is a
// fixed sequence of 84 dependent "stages" (16 vertical-stack, 2 x 34 horizontal-stack + output +
// sample); in each stage every CTA owns a slice of the stage's OUTPUT CHANNELS for all samples of
// the batch tile, so every weight byte is read exactly once per row per GPU.  The CTA's weight slice
// for stage s+1 is pulled into shared memory by a 1-D TMA bulk copy (cp.async.bulk + mbarrier) while
// stage s computes; activations live in an L2-resident arena laid out [channel][64 samples] and are
// exchanged between CTAs through a release/acquire grid barrier.  All arithmetic is fp32 FFMA with a
// fixed summation order (bit-reproducible run to run, independent of batch position).
#include "pixelcnn.h"
#include "convstack.h"

#include <algorithm>
#include <climits>
#include <memory>
#include <cmath>

namespace ts {

// =============================================================================================
// host: plan construction
// =============================================================================================

struct Job {
  int epi, layer, col, nrows, K, ncol;
  bool pairs;
  int rofs = 0;   // first output row of this job inside the layer's row space (output_conv.2 split over two stages)
};

constexpr double PIX_ROWCOST = 0.0;   // default per-row fixed cost of the CTA split, in units of K (TS_PIX_ROWCOST overrides)

// weight rows one CTA can take in a matmul task of depth K: 16 (the accumulator tile), fewer when (K + 1) x rows would not fit
// one staging buffer — K = 1536 (layer-0 vertical stack): 12
static int rows_cap(int K) { return std::min(PIX_MAXROWS, (PIX_WBUF / (K + 1)) & ~3); }

// layer-0 vertical stack of both columns: one stage, or one stage per column when the plan has too few CTAs for both
// (2 x ceil(512 / 12) = 86)
static void push_vert0(std::vector<std::vector<Job>>& st, int D, bool split) {
  if (split) {
    st.push_back({{EPI_VERT0, 0, 0, 2 * D, 6 * D, 1, true}});
    st.push_back({{EPI_VERT0, 0, 1, 2 * D, 6 * D, 1, true}});
  } else {
    st.push_back({{EPI_VERT0, 0, 0, 2 * D, 6 * D, 1, true}, {EPI_VERT0, 0, 1, 2 * D, 6 * D, 1, true}});
  }
}

// Fused plan: every linear stage of the horizontal stack is folded into the gate matmul that consumes it
// (W_next (W_res g + b + x) = (W_next W_res) g + W_next b + W_next x), the layer-0 gate of column 0 (no
// matmul) rides in the last vertical stage, and the layer-0 gate of column 1 is a table lookup done by the
// sampler itself: 16 + 2 x 18 = 52 dependent stages per row instead of 84.
static std::vector<std::vector<Job>> build_stages_fused(int L, int D = PIX_D, int out2_split = 1, bool v0_split = false) {
  std::vector<std::vector<Job>> st;
  push_vert0(st, D, v0_split);
  st.push_back({{EPI_FUSEV, 0, 0, D, D, 2, false}, {EPI_V2H, 0, 0, 2 * D, 2 * D, 2, false}});
  for (int l = 1; l < L; ++l) {
    std::vector<Job> j = {{EPI_VERT, l, 0, 2 * D, 4 * D, 1, true}, {EPI_VERT, l, 1, 2 * D, 4 * D, 1, true}};
    if (l >= 2) j.push_back({EPI_V2H, l - 1, 0, 2 * D, 2 * D, 2, false});
    if (l == 1) j.push_back({EPI_HGATE, 0, 0, 2 * D, 0, 1, true});   // G_0 of column 0: v2h_0 (previous stage) + class term only
    st.push_back(j);
  }
  for (int c = 0; c < 2; ++c) {
    std::vector<Job> j = {{EPI_HRESF, 0, c, D, D, 1, false}};
    if (c == 0) j.push_back({EPI_V2H, L - 1, 0, 2 * D, 2 * D, 2, false});
    st.push_back(j);
    st.push_back({{EPI_HGATE, 1, c, 2 * D, c ? 2 * D : D, 1, true}});
    for (int l = 2; l < L; ++l)
      st.push_back({{EPI_HGATE2, l, c, 2 * D, c ? 3 * D : 2 * D, 1, true}, {EPI_HRES, l - 1, c, D, D, 1, false}});
    st.push_back({{EPI_OUT1F, 0, c, 512, 2 * D, 1, false}});
    // output_conv.2 (2048 rows): one stage, or `out2_split` stages when the plan has fewer than 128 CTAs (16 rows per CTA)
    for (int q = 0; q < out2_split; ++q) st.push_back({{EPI_OUT2, 0, c, PIX_NCODE / out2_split, 512, 1, false, q * (PIX_NCODE / out2_split)}});
    st.push_back({{EPI_SAMPLE, 0, c, 0, c == 0 ? 1 : 0, 1, false}});     // K = 1: also emit G_0 of column 1
  }
  return st;
}

// Schedule 2 (experimental): the fused plan with vert_to_horiz out of the vertical stages, which otherwise take rows
// per CTA away from the vertical jobs (vert_to_horiz of the previous layer occupies part of the grid).  Its output is consumed only by the
// horizontal pass of the same row, so here it runs per column (EPI_V2H1) beside the horizontal stage that precedes
// its consumer; the pre-gate vertical outputs (HV) get one slot per layer instead of a 2-deep ring.
static std::vector<std::vector<Job>> build_stages_fused2(int L, int D = PIX_D, int out2_split = 1, bool v0_split = false) {
  std::vector<std::vector<Job>> st;
  push_vert0(st, D, v0_split);
  st.push_back({{EPI_FUSEV, 0, 0, D, D, 2, false}, {EPI_V2H, 0, 0, 2 * D, 2 * D, 2, false}});   // layer 0: needed by both layer-0 gates
  for (int l = 1; l < L; ++l) {
    std::vector<Job> j = {{EPI_VERT, l, 0, 2 * D, 4 * D, 1, true}, {EPI_VERT, l, 1, 2 * D, 4 * D, 1, true}};
    if (l == 1) j.push_back({EPI_HGATE, 0, 0, 2 * D, 0, 1, true});
    st.push_back(j);
  }
  for (int c = 0; c < 2; ++c) {
    st.push_back({{EPI_HRESF, 0, c, D, D, 1, false}, {EPI_V2H1, 1, c, 2 * D, 2 * D, 1, false}});
    {
      std::vector<Job> j = {{EPI_HGATE, 1, c, 2 * D, c ? 2 * D : D, 1, true}};
      if (L > 2) j.push_back({EPI_V2H1, 2, c, 2 * D, 2 * D, 1, false});
      st.push_back(j);
    }
    for (int l = 2; l < L; ++l) {
      std::vector<Job> j = {{EPI_HGATE2, l, c, 2 * D, c ? 3 * D : 2 * D, 1, true}, {EPI_HRES, l - 1, c, D, D, 1, false}};
      if (l + 1 < L) j.push_back({EPI_V2H1, l + 1, c, 2 * D, 2 * D, 1, false});
      st.push_back(j);
    }
    st.push_back({{EPI_OUT1F, 0, c, 512, 2 * D, 1, false}});
    for (int q = 0; q < out2_split; ++q) st.push_back({{EPI_OUT2, 0, c, PIX_NCODE / out2_split, 512, 1, false, q * (PIX_NCODE / out2_split)}});
    st.push_back({{EPI_SAMPLE, 0, c, 0, c == 0 ? 1 : 0, 1, false}});
  }
  return st;
}

static std::vector<std::vector<Job>> build_stages(int L, int D = PIX_D) {
  std::vector<std::vector<Job>> st;
  // ---- vertical pass -----------------------------------------------------------------------
  st.push_back({{EPI_VERT0, 0, 0, 2 * D, 6 * D, 1, true}, {EPI_VERT0, 0, 1, 2 * D, 6 * D, 1, true}});
  st.push_back({{EPI_FUSEV, 0, 0, D, D, 2, false}, {EPI_V2H, 0, 0, 2 * D, 2 * D, 2, false}});
  for (int l = 1; l < L; ++l) {
    std::vector<Job> j = {{EPI_VERT, l, 0, 2 * D, 4 * D, 1, true}, {EPI_VERT, l, 1, 2 * D, 4 * D, 1, true}};
    if (l >= 2) j.push_back({EPI_V2H, l - 1, 0, 2 * D, 2 * D, 2, false});
    st.push_back(j);
  }
  // ---- horizontal pass, column 0 then column 1 ------------------------------------------------
  for (int c = 0; c < 2; ++c) {
    std::vector<Job> j = {{EPI_HGATE, 0, c, 2 * D, c ? D : 0, 1, true}};
    if (c == 0) j.push_back({EPI_V2H, L - 1, 0, 2 * D, 2 * D, 2, false});
    st.push_back(j);
    st.push_back({{EPI_HRES, 0, c, D, D, 1, false}});
    st.push_back({{EPI_FUSEH, 0, c, D, D, 1, false}});
    for (int l = 1; l < L; ++l) {
      st.push_back({{EPI_HGATE, l, c, 2 * D, c ? 2 * D : D, 1, true}});
      st.push_back({{EPI_HRES, l, c, D, D, 1, false}});
    }
    st.push_back({{EPI_OUT1, 0, c, 512, D, 1, false}});
    st.push_back({{EPI_OUT2, 0, c, PIX_NCODE, 512, 1, false}});
    st.push_back({{EPI_SAMPLE, 0, c, 0, 0, 1, false}});
  }
  return st;
}

static PixLayout make_layout(int L, int hvslots, int MB = PIX_MB) {
  PixLayout a;
  int o = 0;
  auto take = [&](int nseg) { int r = o; o += nseg * PIX_D * MB; return r; };
  a.E = take(4 * 2);
  a.XV1P = take(2);
  a.XV = take(L * 2 * 2);
  a.HV = take(hvslots * 2 * 2);   // pre-gate vertical outputs: [slot][column][tanh half, sigmoid half]
  a.V2H = take(L * 2 * 2);
  a.G = take(2);     // gate output of layer l lives in slot l & 1
  a.XHP = take(1);
  a.XH = take(2 * (L + 1));
  a.Y = take(2);
  a.LOG = take(PIX_NCODE / PIX_D);
  a.CLS = take(L * 2);
  a.total = o;
  return a;
}

// weight of output row `jr` (job row space) at reduction index k, and its bias
struct WeightSrc {
  const Ckpt& ck;
  int L;
  int D;   // hidden width (256; 512 for the convert_to_6d geometry)
  std::vector<const float*> vs, vsb, v2h, v2hb, hs, hsb, hr, hrb;
  const float *fv, *fh, *o1, *o1b, *o2, *o2b;
  // fused plan: products of adjacent linear maps, accumulated in fp64 and rounded once
  std::vector<std::vector<float>> Mh, bh;   // [l]: horiz_stack_l(tap 1) . horiz_resid_{l-1}  [2D][D], and . bias  [2D]
  std::vector<float> Mf, bf, Mo, bo;        // fusion_h(x half) . horiz_resid_0 [D][D];  output_conv.0 . horiz_resid_{L-1} [512][D]
  static void compose(const float* A, int lda, int astride, int N, const float* Bm, const float* bb, int D,
                      std::vector<float>& M, std::vector<float>& mb) {
    // M[n][j] = sum_i A[n*lda + i*astride] * Bm[i*D + j];  mb[n] = sum_i A[..] * bb[i]
    M.assign((size_t)N * D, 0.f); mb.assign(N, 0.f);
    std::vector<double> acc(D);
    for (int n = 0; n < N; ++n) {
      std::fill(acc.begin(), acc.end(), 0.0);
      double ab = 0.0;
      for (int i = 0; i < D; ++i) {
        const double a = A[(size_t)n * lda + (size_t)i * astride];
        const float* brow = Bm + (size_t)i * D;
        for (int j = 0; j < D; ++j) acc[j] += a * (double)brow[j];
        ab += a * (double)bb[i];
      }
      for (int j = 0; j < D; ++j) M[(size_t)n * D + j] = (float)acc[j];
      mb[n] = (float)ab;
    }
  }
  void build_fused() {
    Mh.resize(L); bh.resize(L);
    for (int l = 2; l < L; ++l) compose(hs[l] + 1, 2 * D, 2, 2 * D, hr[l - 1], hrb[l - 1], D, Mh[l], bh[l]);
    compose(fh, 2 * D, 1, D, hr[0], hrb[0], D, Mf, bf);
    compose(o1, D, 1, 512, hr[L - 1], hrb[L - 1], D, Mo, bo);
  }
  WeightSrc(const Ckpt& c, int L_, int D_ = PIX_D) : ck(c), L(L_), D(D_) {
    for (int l = 0; l < L; ++l) {
      std::string p = "layers." + std::to_string(l) + ".";
      vs.push_back(ck.f32(p + "vert_stack.weight", {2 * D, D, l == 0 ? 4 : 2, 3}));
      vsb.push_back(ck.f32(p + "vert_stack.bias", {2 * D}));
      v2h.push_back(ck.f32(p + "vert_to_horiz.weight", {2 * D, 2 * D, 1, 1}));
      v2hb.push_back(ck.f32(p + "vert_to_horiz.bias", {2 * D}));
      hs.push_back(ck.f32(p + "horiz_stack.weight", {2 * D, D, 1, 2}));
      hsb.push_back(ck.f32(p + "horiz_stack.bias", {2 * D}));
      hr.push_back(ck.f32(p + "horiz_resid.weight", {D, D, 1, 1}));
      hrb.push_back(ck.f32(p + "horiz_resid.bias", {D}));
    }
    fv = ck.f32("fusion_v.weight", {D, 2 * D, 1, 1});
    fh = ck.f32("fusion_h.weight", {D, 2 * D, 1, 1});
    o1 = ck.f32("output_conv.0.weight", {512, D, 1, 1});
    o1b = ck.f32("output_conv.0.bias", {512});
    o2 = ck.f32("output_conv.2.weight", {PIX_NCODE, 512, 1, 1});
    o2b = ck.f32("output_conv.2.bias", {PIX_NCODE});
  }
  int chan(const Job& j, int jr) const { return j.pairs ? (jr & 1) * D + (jr >> 1) : jr; }
  float w(const Job& j, int jr, int k) const {
    int ch = chan(j, jr), sidx = k / D, ci = k % D, l = j.layer;
    switch (j.epi) {
      case EPI_VERT0: {  // seg = kh*2 + input col; kw = input col - out col + 1   (Appendix C of SURVEY.md)
        int kh = sidx >> 1, icol = sidx & 1, kw = icol - j.col + 1;
        return vs[0][(((size_t)ch * D + ci) * 4 + kh) * 3 + kw];
      }
      case EPI_VERT: {
        int kh = sidx >> 1, icol = sidx & 1, kw = icol - j.col + 1;
        return vs[l][(((size_t)ch * D + ci) * 2 + kh) * 3 + kw];
      }
      case EPI_V2H: case EPI_V2H1: return v2h[l][(size_t)ch * 2 * D + k];
      case EPI_FUSEV: return fv[(size_t)ch * 2 * D + k];
      case EPI_FUSEH: return fh[(size_t)ch * 2 * D + k];
      case EPI_HGATE: {
        int tap;
        if (l == 0) tap = 0;                 // col 1 reads emb(code(r,0)) through tap 0 (tap 1 is masked)
        else if (j.col == 0) tap = 1;        // col 0: only its own (tap 1) term, col -1 is padding
        else tap = sidx;                     // col 1: seg 0 = x_h[r,0] (tap 0), seg 1 = x_h[r,1] (tap 1)
        return hs[l][((size_t)ch * D + ci) * 2 + tap];
      }
      case EPI_HRES: return hr[l][(size_t)ch * D + k];
      case EPI_HRESF: return Mf[(size_t)ch * D + k];
      case EPI_HGATE2:   // seg 0 = G_{l-1} (composed), seg 1 = x_h[l-1] of this column (tap 1), seg 2 = x_h[l] of column 0 (tap 0)
        if (sidx == 0) return Mh[l][(size_t)ch * D + ci];
        return hs[l][((size_t)ch * D + ci) * 2 + (sidx == 1 ? 1 : 0)];
      case EPI_OUT1F: return sidx == 0 ? Mo[(size_t)ch * D + ci] : o1[(size_t)ch * D + ci];
      case EPI_OUT1: return o1[(size_t)ch * D + k];
      case EPI_OUT2: return o2[(size_t)(ch + j.rofs) * 512 + k];
    }
    return 0.f;
  }
  float bias(const Job& j, int jr) const {
    int ch = chan(j, jr), l = j.layer;
    switch (j.epi) {
      case EPI_VERT0: case EPI_VERT: return vsb[l][ch];
      case EPI_V2H: case EPI_V2H1: return v2hb[l][ch];
      case EPI_HGATE: return hsb[l][ch];
      case EPI_HRES: return hrb[l][ch];
      case EPI_HRESF: return bf[ch];
      case EPI_HGATE2: return hsb[l][ch] + bh[l][ch];
      case EPI_OUT1F: return o1b[ch] + bo[ch];
      case EPI_OUT1: return o1b[ch];
      case EPI_OUT2: return o2b[ch + j.rofs];
    }
    return 0.f;  // FUSEV / FUSEH: bias lives in the precomputed audio term
  }
};

static Layer pack_1x1(ts_engine* e, const float* w, int ldw, int koff, const float* b, int N, int K) {
  std::vector<float> W((size_t)N * K), B(b, b + N);
  for (int n = 0; n < N; ++n)
    for (int k = 0; k < K; ++k) W[(size_t)n * K + k] = w[(size_t)n * ldw + koff + k];
  Layer L;
  L.N = N; L.K = K; L.taps = 1; L.cin = K;
  L.W = e->upload(W);
  L.bias = e->upload(B);
  return L;
}

// parts of the plan shared by the executors: algorithmic bytes per row and the audio-term layers
static void plan_common(ts_engine* e, const Ckpt& ck, PixelPlan* P, int L, int D) {
  // algorithmic bytes per row (SURVEY.md §8d): every dense PixelCNN weight + bias once — unique
  // weights, i.e. without the duplication of the shared kw=1 vertical tap across the two output
  // columns and without the row padding of the staged blob; mask-A-zeroed taps and the gathered
  // tables (code embedding, class embedding) excluded.
  int64_t w = 0;
  for (int l = 0; l < L; ++l) {
    w += (int64_t)2 * D * D * (l == 0 ? 3 : 2) * 3 + 2 * D;   // vert_stack (layer 0: masked row dropped)
    w += (int64_t)2 * D * 2 * D + 2 * D;                      // vert_to_horiz
    w += (int64_t)2 * D * D * (l == 0 ? 1 : 2) + 2 * D;       // horiz_stack (layer 0: masked tap dropped)
    w += (int64_t)D * D + D;                                  // horiz_resid
  }
  w += 2 * ((int64_t)D * 2 * D + D) + ((int64_t)D * 256 + D);  // fusion_v, fusion_h, embedding_aud
  w += (int64_t)512 * D + 512 + (int64_t)PIX_NCODE * 512 + PIX_NCODE;
  P->row_bytes = 4 * w;
  // audio terms: a = embedding_aud(aud); AUDV = fusion_v[:, D:]*a + b_v; AUDH = fusion_h[:, D:]*a + b_h
  P->emb_aud = pack_1x1(e, ck.f32("embedding_aud.weight", {D, 256, 1, 1}), 256, 0, ck.f32("embedding_aud.bias", {D}), D, 256);
  P->fuse_v_a = pack_1x1(e, ck.f32("fusion_v.weight", {D, 2 * D, 1, 1}), 2 * D, D, ck.f32("fusion_v.bias", {D}), D, D);
  P->fuse_h_a = pack_1x1(e, ck.f32("fusion_h.weight", {D, 2 * D, 1, 1}), 2 * D, D, ck.f32("fusion_h.bias", {D}), D, D);
}

static PixelPlan* build_plan(ts_engine* e, const Ckpt& ck, int level) {
  const int cl = 1;   // CTAs per work unit
  const int D = PIX_D;
  const ts_tensor* emb = ck.get("embedding.weight");
  if (emb->ndim != 2 || emb->shape[1] != D || emb->shape[0] != PIX_NCODE)
    fail(TS_ERR_UNSUPPORTED, "pixelcnn: only input_dim=2048, dim=256 (convert_to_6d=false) is built; got [%lld,%lld]",
         (long long)emb->shape[0], (long long)emb->shape[1]);
  int L = 0;
  while (ck.has("layers." + std::to_string(L) + ".vert_stack.weight")) ++L;
  if (L < 2 || L > 30) fail(TS_ERR_MISSING, "pixelcnn: %d layers found", L);
  const ts_tensor* cls0 = ck.get("layers.0.class_cond_embedding.weight");
  const int ncls = (int)cls0->shape[0];

  std::unique_ptr<PixelPlan> owner(new PixelPlan());   // released to the caller at the end; a failed build frees it
  PixelPlan* P = owner.get();
  P->L = L;
  P->ncta = e->sm_count;
  // ts_set_pixelcnn_ctas: a plan for FEWER persistent CTAs than SMs leaves whole TPCs free for kernels of another
  // stream (the face regressor runs beside the latency-bound sampler when the per-GPU batch is small)
  if (e->pixel_ctas > 0) {
    if (e->pixel_ctas < PIX_MB || e->pixel_ctas > e->sm_count) {
      const int n = e->pixel_ctas, sms = e->sm_count;
      fail(TS_ERR_UNSUPPORTED, "pixelcnn plan: ts_set_pixelcnn_ctas(%d) outside [%d, %d] (one CTA per sample of a 64-sample tile; SM count)", n, PIX_MB, sms);
    }
    P->ncta = e->pixel_ctas & ~1;
  }
  if (const char* v = getenv("TS_PIX_CTAS")) {   // experiment switch: persistent CTAs (every CTA re-reads the stage's activations from L2)
    const int n = atoi(v);
    if (n >= PIX_MB && n <= e->sm_count) P->ncta = n;
  }
  P->cl = cl;
  P->nclasses = ncls;
  bool fused = level >= 1 && L >= 3;
  P->sched = fused ? level : 0;
  P->lay = make_layout(L, P->sched == 2 ? L : 2);
  if (P->ncta < PIX_MB) fail(TS_ERR_UNSUPPORTED, "pixelcnn plan needs >= %d SMs (have %d)", PIX_MB, P->ncta);
  P->fused = fused;
  const int out2_split = (PIX_NCODE + PIX_MAXROWS * P->ncta - 1) / (PIX_MAXROWS * P->ncta);   // 1 for >= 128 CTAs
  if (out2_split > 1 && !fused) fail(TS_ERR_UNSUPPORTED, "pixelcnn plan: %d CTAs need the fused plan", P->ncta);
  const bool v0_split = fused && 2 * cdiv(2 * D, rows_cap(6 * D)) > P->ncta / cl;   // fewer than 86 CTAs
  auto stages = P->sched == 2 ? build_stages_fused2(L, PIX_D, out2_split, v0_split)
                : fused       ? build_stages_fused(L, PIX_D, out2_split, v0_split)
                              : build_stages(L);
  P->nstages = (int)stages.size();
  if (P->nstages > 160) fail(TS_ERR_UNSUPPORTED, "pixelcnn plan: %d stages per row (> 160)", P->nstages);
  P->table.assign((size_t)P->nstages * P->ncta, PixTask{0, 0, 0, 0, 0, 0, 0, 0});
  WeightSrc ws(ck, L);
  if (fused) ws.build_fused();
  int64_t dense = 0;
  int t0_ofs = 0;
  if (fused) {
    // T0[code][jr] = bias + horiz_stack_0(tap 0) . embedding[code]: the layer-0 gate pre-activation of column 1
    // depends on the sampled column-0 code only -> a 2048 x 512 table the sampler gathers from (kept in the blob
    // so that the exported plan is self-contained)
    const float* ew = ck.f32("embedding.weight", {PIX_NCODE, D});
    const Job j0{EPI_HGATE, 0, 1, 2 * D, D, 1, true};
    P->blob.resize((size_t)PIX_NCODE * 2 * D);
    std::vector<float> wrow((size_t)2 * D * D), brow(2 * D);
    for (int jr = 0; jr < 2 * D; ++jr) {
      brow[jr] = ws.bias(j0, jr);
      for (int k = 0; k < D; ++k) wrow[(size_t)jr * D + k] = ws.w(j0, jr, k);
    }
    for (int code = 0; code < PIX_NCODE; ++code)
      for (int jr = 0; jr < 2 * D; ++jr) {
        double a = 0.0;
        for (int k = 0; k < D; ++k) a += (double)wrow[(size_t)jr * D + k] * (double)ew[(size_t)code * D + k];
        P->blob[(size_t)code * 2 * D + jr] = (float)(a + (double)brow[jr]);
      }
  }
  const size_t table_floats = P->blob.size();
  for (int s = 0; s < P->nstages; ++s) {
    auto& jobs = stages[s];
    if (jobs[0].epi == EPI_SAMPLE) {
      for (int c = 0; c < P->ncta; ++c)
        P->table[(size_t)s * P->ncta + c] = PixTask{EPI_SAMPLE, 0, jobs[0].col, 0, 0, jobs[0].K ? t0_ofs : 0, jobs[0].K, 0};
      continue;
    }
    // CTAs per job proportional to FMA cost
    std::vector<double> cost;
    double tot = 0;
    // cost of a job ~ rows x (K + alpha): alpha (TS_PIX_ROWCOST, default 0 = FMA count) is the per-row fixed cost in units of
    // K — the stage trace shows K = 256 tasks with 12-13 rows finishing last, i.e. rows cost more than their FMAs
    const double alpha = getenv("TS_PIX_ROWCOST") ? atof(getenv("TS_PIX_ROWCOST")) : PIX_ROWCOST;   // read per plan build
    for (auto& j : jobs) { double c = (double)j.nrows * (j.K ? std::max(j.K, 256) + alpha : 16) * j.ncol; cost.push_back(c); tot += c; }
    std::vector<int> nc(jobs.size()), lo(jobs.size());
    int used = 0;
    const int nunit = P->ncta / cl;                    // work units of a stage: CTAs, or clusters of the cluster plan
    const int rowcap = PIX_MAXROWS;
    for (size_t i = 0; i < jobs.size(); ++i) {
      const int cap = jobs[i].K ? rows_cap(jobs[i].K / cl) : 4 * PIX_MAXROWS;  // matmul rows per unit; epilogue-only tasks: 64
      lo[i] = (jobs[i].nrows + cap - 1) / cap;
      nc[i] = std::max(lo[i], (int)std::floor(nunit * cost[i] / tot));
      used += nc[i];
    }
    for (size_t i = 0; used < nunit; i = (i + 1) % jobs.size()) { nc[i]++; used++; }
    while (used > nunit) {
      size_t big = 0; int slack = -1;
      for (size_t i = 0; i < jobs.size(); ++i) if (nc[i] - lo[i] > slack) { slack = nc[i] - lo[i]; big = i; }
      if (slack <= 0) fail(TS_ERR_UNSUPPORTED, "pixelcnn plan: %d SMs are too few for stage %d", P->ncta, s);
      nc[big]--; used--;
    }
    int cta = 0;
    for (size_t i = 0; i < jobs.size(); ++i) {
      const Job& j = jobs[i];
      const int unit = j.pairs ? 2 : 1, units = j.nrows / unit;
      const int base = units / nc[i], rem = units % nc[i];
      int u0 = 0;
      for (int q = 0; q < nc[i]; ++q) {
        int nu = base + (q < rem ? 1 : 0);
        for (int rank = 0; rank < cl; ++rank, ++cta) {   // the CTAs of a unit: same rows, K slice `rank` of `cl`
          PixTask t{0, 0, 0, 0, 0, 0, 0, 0};
          if (nu > 0) {
            t.epi = j.epi; t.layer = j.layer; t.col = j.col;
            t.row0 = j.rofs + u0 * unit; t.nrows = nu * unit; t.K = j.K; t.rpad = (t.nrows + 3) & ~3;
            if (t.K > 0 && t.nrows > rowcap) fail(TS_ERR_UNSUPPORTED, "pixelcnn plan: %d rows per unit (> %d) with %d SMs", t.nrows, rowcap, P->ncta);
            const int Ks = t.K / cl, k0 = rank * Ks;       // K is a multiple of 256
            size_t sz = (size_t)(Ks + 1) * t.rpad;
            if (sz > (size_t)PIX_WBUF) fail(TS_ERR_UNSUPPORTED, "pixelcnn plan: task blob %zu floats > staging buffer", sz);
            t.wofs = (int)P->blob.size();
            P->blob.resize(P->blob.size() + sz, 0.f);
            float* dst = P->blob.data() + t.wofs;
            for (int r = 0; r < t.nrows; ++r) {
              for (int k = 0; k < Ks; ++k) dst[(size_t)k * t.rpad + r] = ws.w(j, t.row0 - j.rofs + r, k0 + k);
              dst[(size_t)Ks * t.rpad + r] = ws.bias(j, t.row0 - j.rofs + r);
            }
            dense += (int64_t)t.nrows * Ks;
          }
          P->table[(size_t)s * P->ncta + cta] = t;
        }
        u0 += nu;
      }
    }
  }
  P->staged_row_bytes = 4 * ((int64_t)(P->blob.size() - table_floats) + 3LL * D * D);
  (void)dense;
  P->has_v1 = true;

  if (!e->host_only) {
    P->d_table = (PixTask*)e->dmalloc(P->table.size() * sizeof(PixTask));
    TS_CUDA(cudaMemcpy(P->d_table, P->table.data(), P->table.size() * sizeof(PixTask), cudaMemcpyHostToDevice));
    P->d_blob = e->upload(P->blob);
    const float* ew = ck.f32("embedding.weight", {PIX_NCODE, D});
    P->d_emb = e->upload(std::vector<float>(ew, ew + (size_t)PIX_NCODE * D));
    std::vector<float> cls((size_t)L * ncls * 2 * D);
    for (int l = 0; l < L; ++l) {
      const float* c = ck.f32("layers." + std::to_string(l) + ".class_cond_embedding.weight", {ncls, 2 * D});
      std::copy(c, c + (size_t)ncls * 2 * D, cls.begin() + (size_t)l * ncls * 2 * D);
    }
    P->d_cls = e->upload(cls);
    P->d_arena = (float*)e->dmalloc((size_t)P->lay.total * sizeof(float) + 256);
    P->d_barrier = (unsigned*)e->dmalloc(4096);   // one flag word per CTA
  }
  return owner.release();
}

// =============================================================================================
// device
// =============================================================================================
struct PixArgs {
  const PixTask* table;
  const float* blob;
  float* arena;
  const float* emb;
  const float* audv;   // [B*Ttot][256]
  const float* audh;
  const float* noise;  // [2T][B][2048]
  const int64_t* pre;  // [B][T0][2] forced codes for rows < T0 (may be null when T0 == 0)
  int64_t* idx_out;    // [B][Ttot-T0][2]
  float* logits_out;   // [2*(Ttot-log_r0)][B][2048] or null
  unsigned* barrier;
  PixLayout lay;
  int B, T0, Ttot, log_r0, L, nstages, ncta, fused;
  unsigned long long* trace;   // [nstages][ncta][4] globaltimer stamps of row trace_row (debug builds of the kernel only)
  int trace_row;
  // the draw inputs (device copies).  The default kernels read seeds only; every other field is read by the WARP
  // instantiations.  Indexed by the global clip index, or in a guided call by the pair (draw_index).
  SampleCtl draw;
  // styled sampling, read by the WARP instantiations only: the class embeddings [L][ncls][2D] that draw.style blends at
  // every gate in place of the CLS arena (style_pair).  After `draw`, so that draw.seeds keeps its offset.
  const float* cls_w;
  int ncls;
};

// The draw-input index of sample m (WARP instantiations only): in a guided call samples 2p and 2p + 1 are the two branches
// of pair p and read pair p's noise or seed, controls, anchors, shaping and scale; otherwise sample m's own.
template <class Args>
__device__ __forceinline__ int draw_index(const Args& A, int m) {
  return A.draw.guide ? m >> 1 : m;
}

// The sampling controls of clip m (global index): its entry of A.draw.clip_ctl, else the call's scalar controls.  Every draw
// of one clip runs in one CTA, so the value is uniform over the threads that call draw_controlled together.
static_assert(sizeof(ts_clip_ctl) == 16, "ts_clip_ctl is read as one 16-byte load");
struct DrawCtl {
  float temperature;
  int top_k;
  float top_p, min_p;
};
template <class Args>
__device__ __forceinline__ DrawCtl draw_ctl(const Args& A, int m) {
  if (A.draw.clip_ctl) {
    const int4 v = __ldg(reinterpret_cast<const int4*>(A.draw.clip_ctl) + m);
    return {__int_as_float(v.x), v.y, __int_as_float(v.z), __int_as_float(v.w)};
  }
  return {A.draw.temperature, A.draw.top_k, A.draw.top_p, A.draw.min_p};
}
// The temperature of clip m alone (the noise prefetch before the barrier wait: a greedy clip reads no noise).
template <class Args>
__device__ __forceinline__ float draw_temperature(const Args& A, int m) {
  return A.draw.clip_ctl ? __ldg(&A.draw.clip_ctl[m].temperature) : A.draw.temperature;
}

// ---- logit shaping: the rule of ts_pixelcnn_sample_shaped (include/talkshow_b200.h) --------------------------------
// The sample stage's scratch words (red) past draw_controlled's 578 that the shaping stages into: the history bitmap of
// the draw (64 words, one bit per code) and the clip's bias row of the draw's column (2048 floats, each read back by the
// thread that wrote it).
constexpr int SHAPE_BITS = 1024, SHAPE_BIAS = 2048, SHAPE_END = SHAPE_BIAS + PIX_NCODE;
static_assert(sizeof(ts_clip_shape) == 8, "ts_clip_shape is read as one 8-byte load");
struct ShapeCtl {
  float theta;
  int window;
};
template <class Args>
__device__ __forceinline__ ShapeCtl shape_ctl(const Args& A, int m) {
  if (!A.draw.clip_shape) return {1.f, 0};
  const int2 v = __ldg(reinterpret_cast<const int2*>(A.draw.clip_shape) + m);
  return {__int_as_float(v.x), v.y};
}

// Stages what the shaping of draw (r, c) of clip m reads: the bitmap of the codes at column c in rows max(0, r - W) ..
// r - 1 (rows < T0 from pre, later rows from this call's idx_out, written earlier in the launch by the CTA that samples
// clip m: coherent L2 loads, never the read-only path) and the bias row.  Everything it reads is final before the sample
// stage starts, so both persistent executors stage it before their barrier wait, where it overlaps the wait; the bitmap is
// published by the caller's next barrier.  Out-of-range history codes are skipped.  Uniform over the CTA (one clip).
// Guided: theta, W and the bias row are the pair's (draw_index); the history is the branch's own, which holds the pair's
// codes (both branches write every guided code, and the host gives each branch a copy of the pair's pre rows).
template <class Args, class Bar>
__device__ __forceinline__ void shape_stage(const Args& A, int m, int r, int c, float* red, Bar bar) {
  const int tid = threadIdx.x;
  const ShapeCtl sc = shape_ctl(A, draw_index(A, m));
  if (sc.theta != 1.f) {
    unsigned* bits = reinterpret_cast<unsigned*>(red + SHAPE_BITS);
    if (tid < PIX_NCODE / 32) bits[tid] = 0u;
    bar();
    const int lo = sc.window >= r ? 0 : r - max(sc.window, 0);
    for (int i = lo + tid; i < r; i += 256) {
      const int64_t* src = i < A.T0 ? A.pre + ((size_t)m * A.T0 + i) * 2 + c
                                    : A.idx_out + ((size_t)m * (A.Ttot - A.T0) + (i - A.T0)) * 2 + c;
      const long long code = __ldcg(reinterpret_cast<const long long*>(src));
      if (code >= 0 && code < PIX_NCODE) atomicOr(&bits[code >> 5], 1u << (code & 31));
    }
  }
  if (A.draw.code_bias) {
    const float* b = A.draw.code_bias + ((size_t)draw_index(A, m) * 2 + c) * PIX_NCODE;
#pragma unroll
    for (int j = 0; j < 8; ++j) red[SHAPE_BIAS + tid + 256 * j] = __ldg(b + tid + 256 * j);
  }
}

// Shapes the raw logits l of clip m's draw in place from what shape_stage staged: the penalty on the history's codes,
// then the bias.  Returns whether the draw is shaped (theta != 1 or a bias), the same in every thread.  Guided: the pair's
// theta (draw_index).
template <class Args>
__device__ __forceinline__ bool shape_logits(const Args& A, int m, const float* red, float (&l)[8]) {
  const int tid = threadIdx.x;
  const ShapeCtl sc = shape_ctl(A, draw_index(A, m));
  if (sc.theta != 1.f) {
    const unsigned* bits = reinterpret_cast<const unsigned*>(red + SHAPE_BITS);
#pragma unroll
    for (int j = 0; j < 8; ++j)   // code tid + 256 j: word (tid >> 5) + 8 j, bit tid & 31
      if ((bits[(tid >> 5) + 8 * j] >> (tid & 31)) & 1u)
        l[j] = l[j] > 0.f ? __fdiv_rn(l[j], sc.theta) : __fmul_rn(l[j], sc.theta);
  }
  if (A.draw.code_bias) {
#pragma unroll
    for (int j = 0; j < 8; ++j) l[j] = __fadd_rn(l[j], red[SHAPE_BIAS + tid + 256 * j]);
  }
  return sc.theta != 1.f || A.draw.code_bias != nullptr;
}

// The speaker weights of row r of clip m (global index) under A.draw.style, or null for a padding sample (m >= B).
template <class Args>
__device__ __forceinline__ const float* style_row(const Args& A, int m, int r) {
  return m < A.B ? A.draw.style + ((size_t)m * A.Ttot + r) * A.ncls : nullptr;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE;\n"
      "bra WAIT_LOOP;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// 1-D TMA bulk copy global -> shared, completion on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void tma_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_add(unsigned* p, unsigned v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// CTA arrives at the grid barrier: all of this CTA's global writes become visible before the count moves
// (bar.sync orders the CTA's writes before thread 0's release; red.release.gpu / ld.acquire.gpu carry the
// inter-CTA ordering, so no separate fences are needed.  A flag-per-CTA barrier polled by a whole warp was
// measured slower: a full grid of CTAs polling 5 lines is a worse L2 hot spot than one counter.)
__device__ __forceinline__ void grid_arrive(unsigned* ctr) {
  __syncthreads();
  if (threadIdx.x == 0) red_release_add(ctr, 1u);
}
__device__ __forceinline__ void grid_wait(const unsigned* ctr, unsigned target) {
  if (threadIdx.x == 0) {
    while (ld_acquire(ctr) < target) { /* spin */ }
  }
  __syncthreads();
}

__device__ __forceinline__ bool task_active(const PixTask& t, int r, int log_r0) {
  if (t.epi == EPI_IDLE) return false;
  if (t.epi == EPI_OUT1 || t.epi == EPI_OUT2 || t.epi == EPI_OUT1F) return r >= log_r0;
  return true;
}
__device__ __forceinline__ uint32_t task_bytes(const PixTask& t) { return (uint32_t)((t.K + 1) * t.rpad) * 4u; }

// arena offsets (floats) of the K segments of a matmul task; returns the segment count
template <int MB, bool S2 = false>
__device__ __forceinline__ int resolve_segments(const PixTask& t, int pass, int r, const PixLayout& a, int L, int* seg) {
  constexpr int SEG = PIX_D * MB;
  if constexpr (S2) {   // schedule 2: one HV slot per layer, single-column vert_to_horiz
    if (t.epi == EPI_V2H || t.epi == EPI_V2H1) {
      const int col = t.epi == EPI_V2H1 ? t.col : pass;
      seg[0] = a.HV + ((t.layer * 2 + col) * 2) * SEG;
      seg[1] = seg[0] + SEG;
      return 2;
    }
  }
  switch (t.epi) {
    case EPI_VERT0:
      for (int kh = 0; kh < 3; ++kh)
        for (int ci = 0; ci < 2; ++ci) seg[kh * 2 + ci] = a.E + ((((r - 3 + kh) & 3) * 2) + ci) * SEG;
      return 6;
    case EPI_VERT:
      for (int kh = 0; kh < 2; ++kh)
        for (int ci = 0; ci < 2; ++ci) seg[kh * 2 + ci] = a.XV + ((t.layer * 2 + ((r - 1 + kh) & 1)) * 2 + ci) * SEG;
      return 4;
    case EPI_V2H:
      seg[0] = a.HV + (((t.layer & 1) * 2 + pass) * 2) * SEG;
      seg[1] = seg[0] + SEG;
      return 2;
    case EPI_FUSEV: seg[0] = a.XV1P + pass * SEG; return 1;
    case EPI_HGATE:
      if (t.layer == 0) {
        if (t.col == 0) return 0;
        seg[0] = a.E + ((r & 3) * 2 + 0) * SEG;
        return 1;
      }
      seg[0] = a.XH + (0 * (L + 1) + t.layer) * SEG;
      if (t.col == 0) return 1;
      seg[1] = a.XH + (1 * (L + 1) + t.layer) * SEG;
      return 2;
    case EPI_HRES: seg[0] = a.G + (t.layer & 1) * SEG; return 1;
    case EPI_HRESF: seg[0] = a.G; return 1;
    case EPI_HGATE2:
      seg[0] = a.G + ((t.layer - 1) & 1) * SEG;
      seg[1] = a.XH + (t.col * (L + 1) + t.layer - 1) * SEG;
      if (t.col == 0) return 2;
      seg[2] = a.XH + (0 * (L + 1) + t.layer) * SEG;
      return 3;
    case EPI_OUT1F:
      seg[0] = a.G + ((L - 1) & 1) * SEG;
      seg[1] = a.XH + (t.col * (L + 1) + L - 1) * SEG;
      return 2;
    case EPI_FUSEH: seg[0] = a.XHP; return 1;
    case EPI_OUT1: seg[0] = a.XH + (t.col * (L + 1) + L) * SEG; return 1;
    case EPI_OUT2: seg[0] = a.Y; seg[1] = a.Y + SEG; return 2;
  }
  return 0;
}

// Two IEEE fp32 FMAs on a register pair: the accumulator pair is the lane's two samples, the weight is the broadcast
// operand.  The pair layout keeps 64-bit loads of the activations; the pack / unpack moves compile to nothing.
__device__ __forceinline__ void fma2(unsigned long long& acc, float w, unsigned long long x) {
  float a0, a1, x0, x1;
  asm("mov.b64 {%0, %1}, %2;" : "=f"(a0), "=f"(a1) : "l"(acc));
  asm("mov.b64 {%0, %1}, %2;" : "=f"(x0), "=f"(x1) : "l"(x));
  a0 = fmaf(w, x0, a0);
  a1 = fmaf(w, x1, a1);
  asm("mov.b64 %0, {%1, %2};" : "=l"(acc) : "f"(a0), "f"(a1));
}

// Partial products of this CTA's rows over the warp's K slice (64-sample tile): lane owns samples 2*lane, 2*lane+1, every
// accumulator sums its K slice in k order with one fmaf per term.  The activation loads form a ring of G groups x 8 rows;
// a group is re-issued for k+32 as soon as its FMAs are done, so every warp keeps 24-32 L2 loads in flight while it
// computes instead of alternating a load burst and an FMA burst (which also synchronises the L2 traffic of all CTAs into
// bursts).
template <int RC, int G>
__device__ __forceinline__ void mm_rows_pipe2(const float* __restrict__ Wsm, int K, const int* seg, const float* arena,
                                              float* red, int warp, int lane) {
  constexpr int MB = 64;
  unsigned long long acc[4 * RC];
#pragma unroll
  for (int j = 0; j < 4 * RC; ++j) acc[j] = 0ull;
  const int kper = K >> 3;  // multiple of 32
  // K slices are rotated by CTA so that the CTAs do not all pull the same L2 lines at the same time;
  // partials are stored by slice index, so the reduction order does not depend on the rotation
  const int slice = (warp + blockIdx.x) & 7;
  const int kbeg = slice * kper, kend = kbeg + kper;
  constexpr int GS = 8;
  unsigned long long x[G][GS];
#pragma unroll
  for (int g = 0; g < G; ++g) {   // kper is a multiple of G * GS = 32
    const int k = kbeg + g * GS;
    const float* base = arena + seg[k >> 8] + ((k & 255) * MB) + lane * 2;
#pragma unroll
    for (int u = 0; u < GS; ++u) x[g][u] = __ldcg(reinterpret_cast<const unsigned long long*>(base + u * MB));
  }
  for (int k0 = kbeg; k0 < kend; k0 += G * GS) {
    const bool more = k0 + G * GS < kend;
#pragma unroll
    for (int g = 0; g < G; ++g) {
#pragma unroll
      for (int u = 0; u < GS; ++u) {
        const float4* w4 = reinterpret_cast<const float4*>(Wsm + (size_t)(k0 + g * GS + u) * (4 * RC));
        const unsigned long long xv = x[g][u];
#pragma unroll
        for (int rc = 0; rc < RC; ++rc) {
          const float4 w = w4[rc];
          fma2(acc[rc * 4 + 0], w.x, xv);
          fma2(acc[rc * 4 + 1], w.y, xv);
          fma2(acc[rc * 4 + 2], w.z, xv);
          fma2(acc[rc * 4 + 3], w.w, xv);
        }
      }
      if (more) {
        const int k = k0 + G * GS + g * GS;
        const float* base = arena + seg[k >> 8] + ((k & 255) * MB) + lane * 2;
#pragma unroll
        for (int u = 0; u < GS; ++u) x[g][u] = __ldcg(reinterpret_cast<const unsigned long long*>(base + u * MB));
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 4 * RC; ++j)
    *reinterpret_cast<unsigned long long*>(&red[(slice * PIX_MAXROWS + j) * MB + lane * 2]) = acc[j];
}

__device__ __forceinline__ void fma2p(unsigned long long& acc, unsigned long long wp, float x) {
  float a0, a1, w0, w1;
  asm("mov.b64 {%0, %1}, %2;" : "=f"(a0), "=f"(a1) : "l"(acc));
  asm("mov.b64 {%0, %1}, %2;" : "=f"(w0), "=f"(w1) : "l"(wp));
  a0 = fmaf(w0, x, a0);
  a1 = fmaf(w1, x, a1);
  asm("mov.b64 %0, {%1, %2};" : "=l"(acc) : "f"(a0), "f"(a1));
}

// arena index of (channel, sample) inside a tensor: [channel][MB samples] (channels beyond 256 continue into the next segment)
template <int MB>
__device__ __forceinline__ int ax(int ch, int m) { return ch * MB + m; }

// Batch tiles below 64 samples (MB = 8 / 16 / 32): lane = (sample m, row group rq) with 32 / MB row groups, each lane
// owns RPL = rpad * MB / 32 consecutive weight rows of the task for ONE sample.  Same K slicing (8 contiguous slices, one
// per warp, summed in k order) and the same slice-ordered reduction as the 64-sample kernels, so every output is
// bit-identical whatever tile a sample runs in.  Packed fp32 FMAs over ROW pairs when RPL is even.
template <int RC, int MB, int G>
__device__ __forceinline__ void mm_rows_small(const float* __restrict__ Wsm, int K, const int* seg, const float* arena,
                                              float* red, int warp, int lane) {
  constexpr int RPL = RC * MB / 8, RPAD = 4 * RC;
  constexpr bool PACK = (RPL % 2) == 0;
  const int m = lane % MB, rq = lane / MB;
  float acc[PACK ? 1 : RPL];
  unsigned long long acc2[PACK ? RPL / 2 : 1];
#pragma unroll
  for (int j = 0; j < (PACK ? 1 : RPL); ++j) acc[j] = 0.f;
#pragma unroll
  for (int j = 0; j < (PACK ? RPL / 2 : 1); ++j) acc2[j] = 0ull;
  const int kper = K >> 3;  // multiple of 32
  const int slice = (warp + blockIdx.x) & 7;
  const int kbeg = slice * kper, kend = kbeg + kper;
  constexpr int GS = 8;   // ring of G groups x 8 activation loads, re-issued as soon as a group's FMAs are done
  float x[G][GS];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const int k = kbeg + g * GS;
    const float* base = arena + seg[k >> 8] + (k & 255) * MB + m;
#pragma unroll
    for (int u = 0; u < GS; ++u) x[g][u] = __ldcg(base + u * MB);
  }
  const float* wl = Wsm + rq * RPL;
  for (int k0 = kbeg; k0 < kend; k0 += G * GS) {
    const bool more = k0 + G * GS < kend;
#pragma unroll
    for (int g = 0; g < G; ++g) {
#pragma unroll
      for (int u = 0; u < GS; ++u) {
        const float* wr = wl + (size_t)(k0 + g * GS + u) * RPAD;
        const float xv = x[g][u];
        if constexpr (RPL % 4 == 0) {
#pragma unroll
          for (int q = 0; q < RPL / 4; ++q) {
            const ulonglong2 w = *reinterpret_cast<const ulonglong2*>(wr + 4 * q);
            fma2p(acc2[2 * q], w.x, xv);
            fma2p(acc2[2 * q + 1], w.y, xv);
          }
        } else if constexpr (PACK) {
#pragma unroll
          for (int q = 0; q < RPL / 2; ++q) fma2p(acc2[q], *reinterpret_cast<const unsigned long long*>(wr + 2 * q), xv);
        } else {
#pragma unroll
          for (int j = 0; j < RPL; ++j) acc[j] = fmaf(wr[j], xv, acc[j]);
        }
      }
      if (more) {
        const int k = k0 + G * GS + g * GS;
        const float* base = arena + seg[k >> 8] + (k & 255) * MB + m;
#pragma unroll
        for (int u = 0; u < GS; ++u) x[g][u] = __ldcg(base + u * MB);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < RPL; ++j) {
    float v;
    if constexpr (PACK) {
      const unsigned long long a2 = acc2[j >> 1];
      v = __uint_as_float((j & 1) ? (unsigned)(a2 >> 32) : (unsigned)(a2 & 0xffffffffu));
    } else {
      v = acc[j];
    }
    red[(slice * PIX_MAXROWS + rq * RPL + j) * MB + m] = v;
  }
}

template <int MB>
__device__ __forceinline__ float red_sum(const float* red, int j, int m) {
  float s = red[(0 * PIX_MAXROWS + j) * MB + m];
#pragma unroll
  for (int w = 1; w < 8; ++w) s += red[(w * PIX_MAXROWS + j) * MB + m];
  return s;
}
__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

// one matmul task (all passes): weights already in Wsm
struct EpiPre {  // epilogue operands fetched before the grid-barrier wait (they do not depend on the previous stage)
  float a, b;
  bool valid;
};

// operands of thread-item `tid` of an H-pass task whose epilogue has at most one item per thread
template <int MB, bool S2 = false>
__device__ __forceinline__ EpiPre prefetch_epilogue(const PixTask& t, const PixArgs& A, int r) {
  constexpr int SEG = PIX_D * MB;
  EpiPre p;
  p.a = 0.f; p.b = 0.f; p.valid = false;
  if constexpr (S2) {   // schedule 2: the vert_to_horiz operand of a gate is written by the PREVIOUS stage
    if (t.epi == EPI_HGATE || t.epi == EPI_HGATE2) return p;
  }
  const int tid = threadIdx.x, m = tid & (MB - 1), j = tid / MB;
  const PixLayout& a = A.lay;
  if (t.epi == EPI_HGATE || t.epi == EPI_HGATE2) {
    if (j < (t.nrows >> 1) && (t.nrows >> 1) * MB <= PIX_THREADS) {
      const int q = (t.row0 >> 1) + j;
      const float* v2h = A.arena + a.V2H + ((t.layer * 2 + t.col) * 2) * SEG;
      p.a = __ldcg(v2h + ax<MB>(q, m));
      p.b = __ldcg(v2h + ax<MB>(PIX_D + q, m));
      p.valid = true;
    }
  } else if (t.epi == EPI_HRES && t.layer > 0 && !A.fused) {   // fused plan: x_h[l] is written by the previous stage
    if (j < t.nrows && t.nrows * MB <= PIX_THREADS) {
      p.a = __ldcg(A.arena + a.XH + (t.col * (A.L + 1) + t.layer) * SEG + ax<MB>(t.row0 + j, m));
      p.valid = true;
    }
  } else if (t.epi == EPI_FUSEH || t.epi == EPI_HRESF) {
    if (j < t.nrows && t.nrows * MB <= PIX_THREADS) {
      p.a = m < A.B ? A.audh[((size_t)m * A.Ttot + r) * PIX_D + t.row0 + j] : 0.f;
      p.valid = true;
    }
  }
  return p;
}

// WARP: a styled call (A.draw.style) blends each gate's class term from row r's speaker weights; every gate a stage computes
// at latent row r belongs to a position of row r (the vertical stack of row r reads rows < r only, the horizontal pass and
// the forced prefix rows run at their own row), so row r of the schedule is the row of every gate here.
template <int MB, bool S2 = false, bool WARP = false>
__device__ void run_matmul_task(const PixTask& t, const PixArgs& A, int r, const float* Wsm, float* red, const EpiPre& pre) {
  constexpr int SEG = PIX_D * MB;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const PixLayout& a = A.lay;
  const int npass = (t.epi == EPI_V2H || t.epi == EPI_FUSEV) ? 2 : 1;
  const float* bias = Wsm + (size_t)t.K * t.rpad;
  float* arena = A.arena;
  for (int pass = 0; pass < npass; ++pass) {
    int s_seg[6];  // at most 6 segments (EPI_VERT0)
    resolve_segments<MB, S2>(t, pass, r, a, A.L, s_seg);
    if (pass > 0) __syncthreads();  // previous pass's epilogue finished reading red
    if (t.K > 0) {
      if constexpr (MB < 64) {   // small batch tiles: lane = (sample, row group), paired FMAs over row pairs
        // K slices that are a multiple of 64 (K = 512, 1024, 1536) keep 64 loads in flight per lane at the 16-sample tile
        // (a K = 512 stage is then ONE round trip to L2), the others 32
        if (MB == 16 && (t.K & 511) == 0) {
          switch (t.rpad >> 2) {
            case 1: mm_rows_small<1, MB, MB == 16 ? 8 : 4>(Wsm, t.K, s_seg, arena, red, warp, lane); break;
            case 2: mm_rows_small<2, MB, MB == 16 ? 8 : 4>(Wsm, t.K, s_seg, arena, red, warp, lane); break;
            case 3: mm_rows_small<3, MB, MB == 16 ? 8 : 4>(Wsm, t.K, s_seg, arena, red, warp, lane); break;
            default: mm_rows_small<4, MB, MB == 16 ? 8 : 4>(Wsm, t.K, s_seg, arena, red, warp, lane); break;
          }
        } else {
          switch (t.rpad >> 2) {
            case 1: mm_rows_small<1, MB, 4>(Wsm, t.K, s_seg, arena, red, warp, lane); break;
            case 2: mm_rows_small<2, MB, 4>(Wsm, t.K, s_seg, arena, red, warp, lane); break;
            case 3: mm_rows_small<3, MB, 4>(Wsm, t.K, s_seg, arena, red, warp, lane); break;
            default: mm_rows_small<4, MB, 4>(Wsm, t.K, s_seg, arena, red, warp, lane); break;
          }
        }
      } else {
        switch (t.rpad >> 2) {
          case 1: mm_rows_pipe2<1, 4>(Wsm, t.K, s_seg, arena, red, warp, lane); break;
          case 2: mm_rows_pipe2<2, 4>(Wsm, t.K, s_seg, arena, red, warp, lane); break;
          case 3: mm_rows_pipe2<3, 4>(Wsm, t.K, s_seg, arena, red, warp, lane); break;
          default: mm_rows_pipe2<4, 4>(Wsm, t.K, s_seg, arena, red, warp, lane); break;
        }
      }
    }
    __syncthreads();
    const bool pairs = (t.epi == EPI_VERT0 || t.epi == EPI_VERT || t.epi == EPI_HGATE || t.epi == EPI_HGATE2);
    const int items = (pairs ? t.nrows >> 1 : t.nrows) * MB;
    for (int it = tid; it < items; it += PIX_THREADS) {
      const int m = it & (MB - 1), j = it / MB;
      if (pairs) {
        const int q = (t.row0 >> 1) + j;  // gate channel
        float at = (t.K > 0 ? red_sum<MB>(red, 2 * j, m) : 0.f) + bias[2 * j];
        float as = (t.K > 0 ? red_sum<MB>(red, 2 * j + 1, m) : 0.f) + bias[2 * j + 1];
        const float* cls = arena + a.CLS + (t.layer * 2) * SEG;
        float ct = cls[ax<MB>(q, m)], cs = cls[ax<MB>(PIX_D + q, m)];
        if constexpr (WARP) {
          if (A.draw.style) style_pair(A.cls_w + (size_t)t.layer * A.ncls * 2 * PIX_D, style_row(A, m, r), A.ncls, PIX_D, q, ct, cs);
        }
        if (t.epi == EPI_HGATE || t.epi == EPI_HGATE2) {
          const float* v2h = arena + a.V2H + ((t.layer * 2 + t.col) * 2) * SEG;
          float vt = pre.valid ? pre.a : __ldcg(v2h + ax<MB>(q, m));
          float vs = pre.valid ? pre.b : __ldcg(v2h + ax<MB>(PIX_D + q, m));
          float zt = (vt + at) + ct;
          float zs = (vs + as) + cs;
          arena[a.G + (t.layer & 1) * SEG + ax<MB>(q, m)] = tanhf(zt) * sigmoidf_(zs);
        } else {
          float* hv = arena + a.HV + (((S2 ? t.layer : (t.layer & 1)) * 2 + t.col) * 2) * SEG;
          hv[ax<MB>(q, m)] = at;
          hv[ax<MB>(PIX_D + q, m)] = as;
          float g = tanhf(at + ct) * sigmoidf_(as + cs);
          if (t.epi == EPI_VERT0) arena[a.XV1P + t.col * SEG + ax<MB>(q, m)] = g;
          else if (t.layer + 1 < A.L)
            arena[a.XV + (((t.layer + 1) * 2 + (r & 1)) * 2 + t.col) * SEG + ax<MB>(q, m)] = g;
        }
      } else {
        const int ch = t.row0 + j;
        float v = red_sum<MB>(red, j, m) + bias[j];
        switch (t.epi) {
          case EPI_V2H: arena[a.V2H + ((t.layer * 2 + pass) * 2) * SEG + ax<MB>(ch, m)] = v; break;
          case EPI_V2H1:
            if constexpr (S2) arena[a.V2H + ((t.layer * 2 + t.col) * 2) * SEG + ax<MB>(ch, m)] = v;
            break;
          case EPI_FUSEV: {
            float au = m < A.B ? A.audv[((size_t)m * A.Ttot + r) * PIX_D + ch] : 0.f;
            arena[a.XV + ((1 * 2 + (r & 1)) * 2 + pass) * SEG + ax<MB>(ch, m)] = v + au;
          } break;
          case EPI_HRES:
            if (t.layer == 0) arena[a.XHP + ax<MB>(ch, m)] = v;
            else {
              float xh = pre.valid ? pre.a : __ldcg(arena + a.XH + (t.col * (A.L + 1) + t.layer) * SEG + ax<MB>(ch, m));
              arena[a.XH + (t.col * (A.L + 1) + t.layer + 1) * SEG + ax<MB>(ch, m)] = v + xh;
            }
            break;
          case EPI_FUSEH: case EPI_HRESF: {
            float au = pre.valid ? pre.a : (m < A.B ? A.audh[((size_t)m * A.Ttot + r) * PIX_D + ch] : 0.f);
            arena[a.XH + (t.col * (A.L + 1) + 1) * SEG + ax<MB>(ch, m)] = v + au;
          } break;
          case EPI_OUT1: case EPI_OUT1F: arena[a.Y + ax<MB>(ch, m)] = v > 0.f ? v : 0.f; break;
          case EPI_OUT2: arena[a.LOG + ax<MB>(ch, m)] = v; break;
        }
      }
    }
  }
}

// ---- sampling controls (WARP instantiations): temperature, top-k, greedy, log-likelihood of the draw -----------------
// 256 threads own the 2048 logits of one draw, thread tid codes tid + 256 j; `Bar` synchronises those threads.
struct CtaBar { __device__ __forceinline__ void operator()() const { __syncthreads(); } };

// order-preserving uint32 key of a logit; -0 is folded onto +0 so that keys compare like the floats
__device__ __forceinline__ uint32_t logit_key(float x) {
  const uint32_t u = __float_as_uint(x == 0.f ? 0.f : x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

template <class Bar>
__device__ __forceinline__ float cta_max8(float v, float* sf, Bar bar) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  if (lane == 0) sf[warp] = v;
  bar();
  v = sf[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) v = fmaxf(v, sf[w]);
  bar();
  return v;
}
// same summation order as the default sampler's softmax denominator
template <class Bar>
__device__ __forceinline__ float cta_sum8(float v, float* sf, Bar bar) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane == 0) sf[warp] = v;
  bar();
  v = sf[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) v += sf[w];
  bar();
  return v;
}

// Key of the k-th largest of the 2048 logits, multiplicity counted (1 <= k <= 2048): a 4-pass radix select over 8-bit
// digits, most significant first, on integer shared-memory histograms (deterministic: no float atomics, the result
// does not depend on the order of the increments).  hist: 256 words, sel: 2 words.
template <class Bar>
__device__ __forceinline__ uint32_t kth_largest_key(const uint32_t (&key)[8], int k, unsigned* hist, unsigned* sel, Bar bar) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  uint32_t prefix = 0u, pmask = 0u;
  unsigned krem = (unsigned)k;   // rank still to find among the keys that match `prefix` (always <= their count)
  for (int shift = 24; shift >= 0; shift -= 8) {
    hist[tid] = 0u;
    bar();
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if ((key[j] & pmask) == prefix) atomicAdd(&hist[(key[j] >> shift) & 255u], 1u);
    bar();
    if (warp == 0) {
      // lane owns digits 255 - 8 lane - i, i = 0..7 (descending): the digit where the count from the top reaches krem
      unsigned c[8], s = 0u;
#pragma unroll
      for (int i = 0; i < 8; ++i) { c[i] = hist[255 - 8 * lane - i]; s += c[i]; }
      unsigned incl = s;
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      unsigned before = incl - s;
      if (before < krem && krem <= incl) {
        bool found = false;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          if (!found && before + c[i] >= krem) { sel[0] = 255u - 8u * lane - i; sel[1] = krem - before; found = true; }
          before += c[i];
        }
      }
    }
    bar();
    prefix |= sel[0] << shift;
    pmask |= 255u << shift;
    krem = sel[1];
  }
  return prefix;
}

// Boundary key of nucleus (top-p) sampling over integer masses w (w = 0 for a code that is already dropped; w is
// non-decreasing in the key): the largest key whose mass strictly above it, A, satisfies (double)A < p * (double)W, W the
// total mass.  Keeping key >= the result keeps the smallest set of most likely codes whose mass reaches p W, with the
// ties at the boundary.  The same 4-pass radix select as kth_largest_key, on a histogram of mass instead of counts:
// integer addition is associative, so neither the histogram nor the result depends on the order of the increments, and
// every partial sum (<= 2^43) is exact both in uint64 and in a double.  hist: 256 uint64, sel: 1 word.
template <class Bar>
__device__ __forceinline__ uint32_t nucleus_key(const uint32_t (&key)[8], const unsigned long long (&w)[8], float p,
                                                unsigned long long* hist, unsigned* sel, Bar bar) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  uint32_t prefix = 0u, pmask = 0u;
  unsigned long long above = 0ull;   // mass of the keys above every key that matches `prefix` (warp 0 only)
  double P = 0.0;                    // p W, known once the first pass has the total (warp 0 only)
  for (int shift = 24; shift >= 0; shift -= 8) {
    hist[tid] = 0ull;
    bar();
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (w[j] != 0ull && (key[j] & pmask) == prefix) atomicAdd(&hist[(key[j] >> shift) & 255u], w[j]);
    bar();
    if (warp == 0) {
      // lane owns digits 255 - 8 lane - i, i = 0..7 (descending): the first digit where the mass from the top reaches P
      unsigned long long c[8], s = 0ull;
#pragma unroll
      for (int i = 0; i < 8; ++i) { c[i] = hist[255 - 8 * lane - i]; s += c[i]; }
      unsigned long long incl = s;
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      if (shift == 24) P = (double)p * (double)__shfl_sync(0xffffffffu, incl, 31);
      unsigned long long before = above + (incl - s);
      const bool mine = (double)before < P && (double)(above + incl) >= P;
      unsigned digit = 0u;
      if (mine) {
        bool found = false;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          if (!found && (double)(before + c[i]) >= P) { digit = 255u - 8u * lane - i; found = true; }
          if (!found) before += c[i];
        }
        sel[0] = digit;
      }
      // the owning lane is unique: P <= W, and the mass from the top only grows
      const unsigned owner = __ballot_sync(0xffffffffu, mine);
      above = __shfl_sync(0xffffffffu, before, owner ? __ffs(owner) - 1 : 0);
    }
    bar();
    prefix |= sel[0] << shift;
    pmask |= 255u << shift;
  }
  return prefix;
}

// number of set flags over the 256 threads (integer, so independent of the combine order)
template <class Bar>
__device__ __forceinline__ int cta_count8(int v, int* si, Bar bar) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  v = __reduce_add_sync(0xffffffffu, v);
  if (lane == 0) si[warp] = v;
  bar();
  v = si[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) v += si[w];
  bar();
  return v;
}

// Block-wide (value, index) maximum with first-index ties, same combine order as the default draw; every thread gets the
// index (0x7fffffff when no thread had a candidate).
template <class Bar>
__device__ __forceinline__ long long cta_argmax(float bv, int bi, float* sf, int* si, long long* scode, Bar bar) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
  }
  if (lane == 0) { sf[warp] = bv; si[warp] = bi; }
  bar();
  if (tid == 0) {
    for (int w = 1; w < 8; ++w)
      if (sf[w] > bv || (sf[w] == bv && si[w] < bi)) { bv = sf[w]; bi = si[w]; }
    *scode = bi;
  }
  bar();
  return *scode;
}

// first index of the maximum of the 2048 logits (0x7fffffff when every logit is NaN)
template <class Bar>
__device__ __forceinline__ long long cta_first_argmax(const float (&l)[8], float* sf, int* si, long long* scode, Bar bar) {
  float bv = -INFINITY;
  int bi = 0x7fffffff;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int n = threadIdx.x + 256 * j;
    if (l[j] > bv || (l[j] == bv && n < bi)) { bv = l[j]; bi = n; }
  }
  return cta_argmax(bv, bi, sf, si, scode, bar);
}

// log p of code under the untempered, untruncated logits l with maximum mx: *logp_dst = (l[code] - mx) - logf(sum_raw),
// sum_raw = sum exp(l - mx) summed in the default sampler's order (taken as given when have_sum).  Written by the thread
// that owns the code.
template <class Bar>
__device__ __forceinline__ void draw_logp(const float (&l)[8], float mx, long long code, bool have_sum, float sum_raw, float* sf,
                                          float* logp_dst, Bar bar) {
  if (!have_sum) {
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) s += expf(l[j] - mx);
    sum_raw = cta_sum8(s, sf, bar);
  }
  if (threadIdx.x == (int)(code & 255)) {
    // l[code >> 8] as a sum of selected terms: a plain select chain is turned into an indexed load of a local copy of l
    const int jc = (int)(code >> 8);
    float lc = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) lc += j == jc ? l[j] : 0.f;
    *logp_dst = (lc - mx) - logf(sum_raw);
  }
}

// One controlled draw over the raw logits l (include/talkshow_b200.h, ts_pixelcnn_sample):
//   temperature 0: first-index argmax of l (q is not read);
//   else s = l / temperature (IEEE division), codes below the k-th largest logit -> -inf, then the default draw
//   argmax((exp(s - max s) / sum) / q) with first-index ties, over the kept codes only.
//   top_p < 1 / min_p > 0 (ts_pixelcnn_sample_ctl) drop further codes before the sum: with e = exp(s - max s) of the
//   codes top-k kept and the integer mass w = rint(e 2^32), top-p keeps the codes at or above nucleus_key, min-p those
//   with e >= min_p.  kept_dst (may be null) receives the size of the final keep set (1 for a greedy draw).  A code whose
//   logit is -inf (a shaped draw's ban, ts_pixelcnn_sample_shaped) is never in the keep set.
// At temperature 1 without truncation this is the default sampler's arithmetic step for step (s == l).
// A temperature so small that max(l) / temperature overflows makes every p / q NaN, so no code wins the draw: the code is
// then the greedy one, the limit of the tempered draw as the temperature goes to 0.  The returned code always lies in
// [0, 2048): logits that are all NaN give code 0.
// logp_dst (may be null) receives (l[code] - max l) - log(sum exp(l - max l)).  scratch: the first 578 words of red (64 of
// reductions, then one histogram region that the count and the mass select use in turn, then 2 words of selection).
template <class Bar>
__device__ __forceinline__ long long draw_controlled(const float (&l)[8], const float (&q)[8], float temperature, int top_k, float top_p,
                                     float min_p, float* red, float* logp_dst, int* kept_dst, Bar bar) {
  const int tid = threadIdx.x;
  float* sf = red;
  int* si = reinterpret_cast<int*>(red + 16);
  long long* scode = reinterpret_cast<long long*>(red + 32);
  unsigned* hist = reinterpret_cast<unsigned*>(red + 64);
  unsigned long long* hist64 = reinterpret_cast<unsigned long long*>(red + 64);
  unsigned* sel = reinterpret_cast<unsigned*>(red + 576);
  float mx = l[0];
#pragma unroll
  for (int j = 1; j < 8; ++j) mx = fmaxf(mx, l[j]);
  mx = cta_max8(mx, sf, bar);
  const bool greedy = temperature == 0.f;
  const bool nucleus = !greedy && top_p < 1.f, floor_p = !greedy && min_p > 0.f;
  const bool truncate = !greedy && ((top_k > 0 && top_k < PIX_NCODE) || nucleus || floor_p);
  bool keep[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) keep[j] = l[j] != -INFINITY;
  uint32_t key[8];
  if (!greedy && ((top_k > 0 && top_k < PIX_NCODE) || nucleus)) {
#pragma unroll
    for (int j = 0; j < 8; ++j) key[j] = logit_key(l[j]);
  }
  if (!greedy && top_k > 0 && top_k < PIX_NCODE) {
    const uint32_t kth = kth_largest_key(key, top_k, hist, sel, bar);
#pragma unroll
    for (int j = 0; j < 8; ++j) keep[j] = keep[j] && key[j] >= kth;
  }
  float sum_raw = 0.f;
  long long code;
  if (greedy) {
    code = cta_first_argmax(l, sf, si, scode, bar);
  } else {
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    // max_i (l_i / t) = (max_i l_i) / t: a correctly rounded division by t > 0 is monotone, and the maximum is always kept
    const float mxs = mx / temperature;
    float ex[8], sum = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) ex[j] = keep[j] ? expf(l[j] / temperature - mxs) : 0.f;
    if (nucleus) {
      unsigned long long w[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) w[j] = __float2ull_rn(ex[j] * 0x1p32f);   // exact scaling, round to nearest even
      const uint32_t theta = nucleus_key(key, w, top_p, hist64, sel, bar);
#pragma unroll
      for (int j = 0; j < 8; ++j) keep[j] = keep[j] && key[j] >= theta;
    }
    if (floor_p) {
#pragma unroll
      for (int j = 0; j < 8; ++j) keep[j] = keep[j] && ex[j] >= min_p;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) { ex[j] = keep[j] ? ex[j] : 0.f; sum += ex[j]; }
    sum = cta_sum8(sum, sf, bar);
    if (temperature == 1.f && !truncate) sum_raw = sum;   // s == l: the softmax denominator is the untempered one
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int n = tid + 256 * j;
      const float v = (ex[j] / sum) / q[j];
      if (keep[j] && (v > bv || (v == bv && n < bi))) { bv = v; bi = n; }
    }
    code = cta_argmax(bv, bi, sf, si, scode, bar);
    // every p / q NaN (s = l / temperature overflowed): the greedy code.  `code` is the same in every thread, so the
    // barriers inside the branch are reached by the whole CTA.
    if (code == 0x7fffffff) code = cta_first_argmax(l, sf, si, scode, bar);
  }
  if (code >= PIX_NCODE) code = 0;   // all logits NaN: keep the embedding gather inside the table
  if (kept_dst) {
    int n = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) n += keep[j] ? 1 : 0;
    n = cta_count8(n, si, bar);
    if (tid == 0) *kept_dst = greedy ? 1 : n;
  }
  if (logp_dst) draw_logp(l, mx, code, !(greedy || temperature != 1.f || truncate), sum_raw, sf, logp_dst, bar);
  return code;
}

// A draw pinned to `code` (ts_pixelcnn_sample_anchored): no noise, no draw.  logp_dst gets the log p of draw_controlled's
// tail on the same logits (the same max, sum and reduction order), kept_dst gets 0.  scratch: the first 16 words of red.
template <class Bar>
__device__ __forceinline__ void draw_pinned(const float (&l)[8], long long code, float* red, float* logp_dst, int* kept_dst,
                                            Bar bar) {
  if (kept_dst && threadIdx.x == 0) *kept_dst = 0;
  if (logp_dst) {
    float mx = l[0];
#pragma unroll
    for (int j = 1; j < 8; ++j) mx = fmaxf(mx, l[j]);
    mx = cta_max8(mx, red, bar);
    draw_logp(l, mx, code, false, 0.f, red, logp_dst, bar);
  }
}

// The pin of draw `at` ([B][T][2] index) of an anchored call: the anchor when it lies in [0, 2048), else -1 (sampled).
// Any other value samples, so malformed device data never reaches the embedding gather.
template <class Args>
__device__ __forceinline__ long long anchor_of(const Args& A, size_t at) {
  if (!A.draw.anchors) return -1;
  const long long a = __ldg(A.draw.anchors + at);
  return (a >= 0 && a < PIX_NCODE) ? a : -1;
}

// ---- seeded noise: the RNG contract of ts_pixelcnn_sample_seeded (include/talkshow_b200.h) --------------------------
// Philox4x32-10 (Salmon et al., SC'11; the Random123 / cuRAND generator), the ten rounds written out.
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c;
}

// Exp(1) value of one 32-bit output: u = ((x >> 8) | 1) 2^-24 is an odd multiple of 2^-24 (exact in fp32, never 0 or 1),
// so q = -log(u) lies in (0, 16.7] and is never inf
__device__ __forceinline__ float philox_exp1(uint32_t x) { return -logf((float)((x >> 8) | 1u) * 0x1p-24f); }

// The q of codes tid + 256 j (j = 0..7) of draw (absolute latent row r, column c) of the clip seeded `seed`: code n is
// output n >> 9 of counter (n & 511, r, c, 0) under key (seed lo, seed hi), so the thread evaluates counters tid and
// tid + 256 and uses all four outputs of each.  One definition for both executors and ts_sampler_noise.
__device__ __forceinline__ void seeded_q(int64_t seed, int r, int c, int tid, float (&q)[8]) {
  const uint32_t k0 = (uint32_t)(uint64_t)seed, k1 = (uint32_t)((uint64_t)seed >> 32);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const uint4 x = philox4x32_10(make_uint4((uint32_t)(tid + 256 * h), (uint32_t)r, (uint32_t)c, 0u), k0, k1);
    q[h] = philox_exp1(x.x);
    q[2 + h] = philox_exp1(x.y);
    q[4 + h] = philox_exp1(x.z);
    q[6 + h] = philox_exp1(x.w);
  }
}

// The noise of draw (r, c) of sample m (global clip index): computed from A.draw.seeds, else read from A.noise.  The WARP
// kernels read by draw_index: a guided call's pair p = m >> 1 reads seeds[p], or column p of noise [2T][B / 2][2048].
// The guided read is its own branch: a select on the index changes the code of the WARP kernels.
template <bool WARP, class Args>
__device__ __forceinline__ void draw_noise(const Args& A, int r, int c, int m, float (&q)[8]) {
  const int tid = threadIdx.x;
  auto read = [&](int d, bool pair) {
    if (A.draw.seeds) {
      seeded_q(A.draw.seeds[d], r, c, tid, q);
    } else {
      const float* src = A.noise + ((size_t)(2 * (r - A.T0) + c) * (pair ? A.B >> 1 : A.B) + d) * PIX_NCODE;
#pragma unroll
      for (int j = 0; j < 8; ++j) q[j] = __ldcs(src + tid + 256 * j);
    }
  };
  if constexpr (WARP) {
    if (A.draw.guide) { read(draw_index(A, m), true); return; }
  }
  read(m, false);
}

// The guided logits of branch m's draw (ts_pixelcnn_sample_guided), in place of its raw logits l: with l_c the raw logits
// of branch 2p (the conditional one, p = m >> 1), l_u those of branch 2p + 1 and s = w_p - 1, g = l_c + s (l_c - l_u) in
// three separately rounded fp32 operations.  l holds branch m's raw logits; `partner` points at code 0 of branch m ^ 1's
// LOG slot, `stride` floats between codes.  Both branches of a pair compute the same g from the same two slots, so they
// draw the same code with no exchange.  Every slot is final: the sample stage follows the barrier after the logits stage.
template <class Args>
__device__ __forceinline__ void guide_logits(const Args& A, int m, const float* partner, int stride, float (&l)[8]) {
  const int tid = threadIdx.x;
  const float s = __fsub_rn(__ldg(A.draw.guide + (m >> 1)), 1.f);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float o = __ldcg(partner + (size_t)(tid + 256 * j) * stride);
    const float lc = (m & 1) ? o : l[j], lu = (m & 1) ? l[j] : o;
    l[j] = __fadd_rn(lc, __fmul_rn(s, __fsub_rn(lc, lu)));
  }
}

// The draw of one sample stage, shared by both executors: softmax over the 2048 logits + categorical draw = argmax(p / q)
// (ATen multinomial, num_samples = 1) with first-index ties.  One CTA per sample; its 256 threads, synchronised by `bar`,
// own codes tid + 256 j.  logit(j): the address of code tid + 256 j in the sample's LOG slot (each executor keeps its own
// address arithmetic, which the register allocation of its kernels depends on); partner: code 0 of branch m ^ 1's slot,
// `stride` floats between codes (read by a guided draw only); m: the global clip index; q: the draw's noise, loaded (or,
// seeded, computed) before the stage barrier (unread by forced rows and by pinned and greedy draws).  Rows r < T0 take
// pre's code.  Writes logits_out and idx_out, and (WARP) logp_out and kept_out; returns the code.
// WARP: the draw applies the anchors, controls, shaping and guidance of A.draw (draw_controlled); otherwise the default
// draw below.
template <bool WARP, class Args, class Bar, class Logit>
__device__ __forceinline__ long long sample_draw(const Args& A, Bar bar, Logit logit, const float* partner, int stride, int m,
                                                 int r, int c, float* red, const float (&q)[8]) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  float* sf = red;                                  // [8] scratch
  int* si = reinterpret_cast<int*>(red + 16);       // [8] scratch
  long long* scode = reinterpret_cast<long long*>(red + 32);
  const bool forced = r < A.T0;
  const bool have_logits = r >= A.log_r0;
  float l[8];
  if (have_logits) {
#pragma unroll
    for (int j = 0; j < 8; ++j) l[j] = __ldcg(logit(j));
    if (A.logits_out) {
      float* dst = A.logits_out + ((size_t)(2 * (r - A.log_r0) + c) * A.B + m) * PIX_NCODE;
#pragma unroll
      for (int j = 0; j < 8; ++j) dst[tid + 256 * j] = l[j];
    }
  }
  long long code;
  if constexpr (WARP) {
    if (!forced) {
      const size_t at = ((size_t)m * (A.Ttot - A.T0) + (r - A.T0)) * 2 + c;
      // m, or a guided call's pair (its branches 2d, 2d + 1 share the tile or cluster: the cluster's MB is even)
      const int d = draw_index(A, m);
      const long long pin = anchor_of(A, ((size_t)d * (A.Ttot - A.T0) + (r - A.T0)) * 2 + c);   // uniform branch
      if (pin >= 0) {
        code = pin;
        draw_pinned(l, code, red, A.draw.logp_out ? A.draw.logp_out + at : nullptr,
                    A.draw.kept_out ? A.draw.kept_out + at : nullptr, bar);
      } else {
        const DrawCtl dc = draw_ctl(A, d);   // clip m's (pair d's) controls: the whole CTA serves clip m
        if (A.draw.guide) guide_logits(A, m, partner, stride, l);
        const bool shaped = shape_logits(A, m, red, l) || A.draw.guide;   // staged before the stage barrier
        float* logp = A.draw.logp_out ? A.draw.logp_out + at : nullptr;
        code = draw_controlled(l, q, dc.temperature, dc.top_k, dc.top_p, dc.min_p, red, shaped ? nullptr : logp,
                               A.draw.kept_out ? A.draw.kept_out + at : nullptr, bar);
        if (shaped && logp) {   // log p under the branch's raw prior: the LOG slot still holds its unshaped logits
#pragma unroll
          for (int j = 0; j < 8; ++j) l[j] = __ldcg(logit(j));
          draw_pinned(l, code, red, logp, nullptr, bar);
        }
      }
    } else {
      code = A.pre[((size_t)m * A.T0 + r) * 2 + c];
    }
  } else if (!forced) {
    float mx = l[0];
#pragma unroll
    for (int j = 1; j < 8; ++j) mx = fmaxf(mx, l[j]);
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) sf[warp] = mx;
    bar();
    mx = sf[0];
#pragma unroll
    for (int w = 1; w < 8; ++w) mx = fmaxf(mx, sf[w]);
    bar();
    float ex[8], sum = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) { ex[j] = expf(l[j] - mx); sum += ex[j]; }
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (lane == 0) sf[warp] = sum;
    bar();
    sum = sf[0];
#pragma unroll
    for (int w = 1; w < 8; ++w) sum += sf[w];
    bar();
    float bv = -INFINITY;
    int bi = 0x7fffffff;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int n = tid + 256 * j;
      const float v = (ex[j] / sum) / q[j];
      if (v > bv || (v == bv && n < bi)) { bv = v; bi = n; }
    }
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    if (lane == 0) { sf[warp] = bv; si[warp] = bi; }
    bar();
    if (tid == 0) {
      for (int w = 1; w < 8; ++w)
        if (sf[w] > bv || (sf[w] == bv && si[w] < bi)) { bv = sf[w]; bi = si[w]; }
      *scode = bi;
    }
    bar();
    code = *scode;
  } else {
    code = A.pre[((size_t)m * A.T0 + r) * 2 + c];
  }
  if (r >= A.T0 && tid == 0) A.idx_out[((size_t)m * (A.Ttot - A.T0) + (r - A.T0)) * 2 + c] = code;
  return code;
}

// The sample stage of the grid-wide executor: sample_draw, then the embedding gather of the code into the E ring and, in
// the fused plan, the layer-0 gate of column 1.  m: the CTA's sample (global clip index); q as in sample_draw.
template <int MB, bool WARP = false>
__device__ void run_sample_task(const PixTask& t, const PixArgs& A, int r, int m, float* red, const float (&q)[8]) {
  constexpr int SEG = PIX_D * MB;
  const int tid = threadIdx.x;
  const int c = t.col;
  const long long code = sample_draw<WARP>(A, CtaBar(), [&](int j) { return A.arena + A.lay.LOG + ax<MB>(tid + 256 * j, m); },
                                           A.arena + A.lay.LOG + (m ^ 1), MB, m, r, c, red, q);
  // embedding gather into the ring slot of this row (x_v = x_h = embedding(code) at layer 0)
  A.arena[A.lay.E + ((r & 3) * 2 + c) * SEG + ax<MB>(tid, m)] = A.emb[(size_t)code * PIX_D + tid];
  if (t.K) {
    // fused plan: layer-0 gate of column 1 (its matmul input is embedding[code] only -> gathered from T0)
    const float2 tw = *reinterpret_cast<const float2*>(A.blob + t.wofs + (size_t)code * (2 * PIX_D) + 2 * tid);
    const float* v2h = A.arena + A.lay.V2H + ((0 * 2 + 1) * 2) * SEG;
    if constexpr (WARP) {
      if (A.draw.style) {   // position (r, 1): row r of the schedule
        float ct, cs;
        style_pair(A.cls_w, style_row(A, m, r), A.ncls, PIX_D, tid, ct, cs);
        const float zt = (__ldcg(v2h + ax<MB>(tid, m)) + tw.x) + ct;
        const float zs = (__ldcg(v2h + ax<MB>(PIX_D + tid, m)) + tw.y) + cs;
        A.arena[A.lay.G + ax<MB>(tid, m)] = tanhf(zt) * sigmoidf_(zs);
        return;
      }
    }
    const float* cls = A.arena + A.lay.CLS;
    const float zt = (__ldcg(v2h + ax<MB>(tid, m)) + tw.x) + cls[ax<MB>(tid, m)];
    const float zs = (__ldcg(v2h + ax<MB>(PIX_D + tid, m)) + tw.y) + cls[ax<MB>(PIX_D + tid, m)];
    A.arena[A.lay.G + ax<MB>(tid, m)] = tanhf(zt) * sigmoidf_(zs);
  }
}

constexpr int PIX_MAXSTAGES = 160;  // this CTA's column of the stage table is kept in shared memory
static_assert(SHAPE_END <= 8 * PIX_MAXROWS * 64, "the shaping inputs are staged in the sampler's scratch");
constexpr size_t PIX_SMEM = (size_t)(2 * PIX_WBUF + 8 * PIX_MAXROWS * 64) * sizeof(float) + 64 + PIX_MAXSTAGES * sizeof(PixTask);

__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// TRACE: a second instantiation of the persistent kernel that stamps, for one latent row, when each CTA's thread 0
// has its weights, leaves the grid barrier, finishes its task and has arrived again (ts_pixelcnn_trace): the
// measurement the stage cost model and the CTA split should be fitted to.  The default kernel is TRACE = false.
// WARP: the sample stage applies the sampling controls of A (ts_pixelcnn_sample); every other stage is unchanged.
template <bool PERSISTENT, bool TRACE = false, bool S2 = false, int MB = 64, bool WARP = false>
__global__ void __launch_bounds__(PIX_THREADS, 1) pixelcnn_kernel(PixArgs A, int r_single, int s_single) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* wbuf = reinterpret_cast<float*>(smem_raw);
  float* red = wbuf + 2 * PIX_WBUF;
  uint64_t* bars = reinterpret_cast<uint64_t*>(red + 8 * PIX_MAXROWS * 64);
  PixTask* tasks = reinterpret_cast<PixTask*>(bars + 8);
  const int tid = threadIdx.x, cta = blockIdx.x;

  if (!PERSISTENT) {
    // debug cross-check mode: one launch per stage, weights copied synchronously
    const PixTask t = A.table[(size_t)s_single * A.ncta + cta];
    if (!task_active(t, r_single, A.log_r0)) return;
    if (t.epi == EPI_SAMPLE) {
      if (cta < A.B) {
        float q[8];
        if (r_single >= A.T0 && (!WARP || draw_temperature(A, draw_index(A, cta)) > 0.f))
          draw_noise<WARP>(A, r_single, t.col, cta, q);   // greedy: no noise
        if constexpr (WARP) {   // the shaping inputs of the draw (ts_pixelcnn_sample_shaped)
          if (r_single >= A.T0 && (A.draw.clip_shape || A.draw.code_bias)) {
            shape_stage(A, cta, r_single, t.col, red, CtaBar());
            __syncthreads();
          }
        }
        run_sample_task<MB, WARP>(t, A, r_single, cta, red, q);
      }
      return;
    }
    const int nf = (t.K + 1) * t.rpad;
    for (int i = tid; i < nf; i += PIX_THREADS) wbuf[i] = A.blob[t.wofs + i];
    __syncthreads();
    EpiPre pre; pre.a = pre.b = 0.f; pre.valid = false;
    run_matmul_task<MB, S2, WARP>(t, A, r_single, wbuf, red, pre);
    return;
  }

  if (tid == 0) {
    mbar_init(&bars[0], 1);
    mbar_init(&bars[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = tid; i < A.nstages * 8; i += PIX_THREADS)
    reinterpret_cast<int*>(tasks)[i] = reinterpret_cast<const int*>(A.table + (size_t)(i >> 3) * A.ncta + cta)[i & 7];
  __syncthreads();
  uint32_t uses[2] = {0u, 0u};
  const int total = A.Ttot * A.nstages;
  // prefetch the first task's weights
  if (tid == 0) {
    const PixTask t0 = tasks[0];
    if (task_active(t0, 0, A.log_r0) && t0.epi != EPI_SAMPLE) {
      mbar_expect_tx(&bars[0], task_bytes(t0));
      tma_load_1d(wbuf, A.blob + t0.wofs, task_bytes(t0), &bars[0]);
    }
  }
  int r = 0, s = 0;
  for (int g = 0; g < total; ++g) {
    const PixTask t = tasks[s];
    const int buf = g & 1;
    // prefetch next stage's weight slice into the other buffer (its last reader finished before the
    // __syncthreads of the previous grid_arrive)
    if (tid == 0 && g + 1 < total) {
      int s1 = s + 1, r1 = r;
      if (s1 == A.nstages) { s1 = 0; r1 = r + 1; }
      const PixTask tn = tasks[s1];
      if (task_active(tn, r1, A.log_r0) && tn.epi != EPI_SAMPLE) {
        fence_proxy_async();
        mbar_expect_tx(&bars[buf ^ 1], task_bytes(tn));
        tma_load_1d(wbuf + (buf ^ 1) * PIX_WBUF, A.blob + tn.wofs, task_bytes(tn), &bars[buf ^ 1]);
      }
    }
    const bool active = task_active(t, r, A.log_r0);
    const bool has_w = active && t.epi != EPI_SAMPLE;  // K == 0 tasks still stage their bias row
    EpiPre pre;
    pre.a = pre.b = 0.f; pre.valid = false;
    if (active && t.epi != EPI_SAMPLE) pre = prefetch_epilogue<MB, S2>(t, A, r);   // in flight while we wait below
    // the sampler noise of this position is an input of the call (or, seeded, a function of the seed and the position):
    // loaded / computed before the barrier wait, so it overlaps the wait
    float qpre[8];
    if (active && t.epi == EPI_SAMPLE && cta < A.B && r >= A.T0 && (!WARP || draw_temperature(A, draw_index(A, cta)) > 0.f))
      draw_noise<WARP>(A, r, t.col, cta, qpre);   // greedy: no noise
    if constexpr (WARP) {   // the shaping inputs of this draw (ts_pixelcnn_sample_shaped), likewise before the wait
      if (active && t.epi == EPI_SAMPLE && cta < A.B && r >= A.T0 && (A.draw.clip_shape || A.draw.code_bias))
        shape_stage(A, cta, r, t.col, red, CtaBar());
    }
    if (has_w) { mbar_wait(&bars[buf], uses[buf] & 1u); uses[buf]++; }
    unsigned long long* tr = nullptr;
    if constexpr (TRACE) {
      if (tid == 0 && r == A.trace_row && A.trace) { tr = A.trace + ((size_t)s * A.ncta + cta) * 4; tr[0] = globaltimer_ns(); }
    }
    if (g > 0) grid_wait(A.barrier, (unsigned)g * (unsigned)A.ncta);  // every CTA finished stage g-1
    if constexpr (TRACE) { if (tr) tr[1] = globaltimer_ns(); }
    if (active) {
      if (t.epi == EPI_SAMPLE) {
        if (cta < A.B) run_sample_task<MB, WARP>(t, A, r, cta, red, qpre);
      }
      else run_matmul_task<MB, S2, WARP>(t, A, r, wbuf + buf * PIX_WBUF, red, pre);
    }
    if constexpr (TRACE) { __syncthreads(); if (tr) tr[2] = globaltimer_ns(); }
    grid_arrive(A.barrier);
    if constexpr (TRACE) { if (tr) tr[3] = globaltimer_ns(); }
    if (++s == A.nstages) { s = 0; ++r; }
  }
}

#include "pixelcnn3.inc"

__global__ void build_cls_kernel(const float* __restrict__ cls_w, const int64_t* __restrict__ label, float* arena, int cls_off,
                                 int L, int ncls, int B, int MB) {
  // CLS[l][ch][m] = class_cond_embedding_l[label[m]][ch]; zero without a label (a styled call, which does not read CLS)
  int n = L * 2 * PIX_D * MB;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    int m = i % MB, ch = (i / MB) % (2 * PIX_D), l = i / (2 * PIX_D * MB);
    float v = 0.f;
    if (m < B && label) {
      long long lb = label[m];
      lb = lb < 0 ? 0 : (lb >= ncls ? ncls - 1 : lb);
      v = cls_w[((size_t)l * ncls + lb) * 2 * PIX_D + ch];
    }
    arena[cls_off + i] = v;
  }
}

__global__ void split_codes_kernel(const int64_t* __restrict__ idx, int64_t* __restrict__ idx_c, int64_t* codes_out, int BT) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < BT; i += gridDim.x * blockDim.x) {
    int64_t a = idx[2 * i], b = idx[2 * i + 1];
    idx_c[i] = a;
    idx_c[BT + i] = b;
    if (codes_out) { codes_out[2 * i] = a; codes_out[2 * i + 1] = b; }
  }
}
void split_codes(ts_engine* e, const int64_t* idx, int64_t* idx_c, int B, int T, int64_t* codes_out, cudaStream_t s) {
  if (e->ws.sizing) return;
  split_codes_kernel<<<cdiv(B * T, 256), 256, 0, s>>>(idx, idx_c, codes_out, B * T);
  e->launches++;
  TS_CUDA(cudaGetLastError());
}

// one thread per (branch, row): every branch's codes to codes_out, the conditional branches' (2p) to idx_c [2][P][T]
__global__ void split_guided_codes_kernel(const int64_t* __restrict__ idx, int64_t* __restrict__ idx_c, int64_t* codes_out,
                                          int P, int T) {
  const int n = 2 * P * T;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int64_t a = idx[2 * i], b = idx[2 * i + 1];
    const int br = i / T, t = i - br * T;
    if ((br & 1) == 0) {
      const int j = (br >> 1) * T + t;
      idx_c[j] = a;
      idx_c[(size_t)P * T + j] = b;
    }
    if (codes_out) { codes_out[2 * i] = a; codes_out[2 * i + 1] = b; }
  }
}
void split_guided_codes(ts_engine* e, const int64_t* idx, int64_t* idx_c, int P, int T, int64_t* codes_out, cudaStream_t s) {
  if (e->ws.sizing) return;
  split_guided_codes_kernel<<<cdiv(2 * P * T, 256), 256, 0, s>>>(idx, idx_c, codes_out, P, T);
  e->launches++;
  TS_CUDA(cudaGetLastError());
}

// logits [2T][B][2048] (step-major) -> [B][2048][T][2]
__global__ void logits_to_ref_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int T) {
  long n = (long)2 * T * B * PIX_NCODE;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    int code = i % PIX_NCODE;
    long sb = i / PIX_NCODE;
    int b = sb % B, step = sb / B;
    int t = step >> 1, c = step & 1;
    out[(((long)b * PIX_NCODE + code) * T + t) * 2 + c] = in[i];
  }
}

static void generate_chunk(ts_engine* e, const Act3& aud, int b0, const int64_t* label, const float* noise, int noise_B,
                           int64_t* idx_out, float* logits_out, int B, int T, const int64_t* pre, int T0, cudaStream_t s,
                           bool logits_all, const SampleCtl& d) {
  PixelPlan* P = e->pix;
  Plan3* Q = (Plan3*)P->p3;
  const int Ttot = T0 + T, D = P->D;
  const bool v3 = (e->pixel_mode == 2 && Q) || !P->has_v1;
  // audio terms for all rows of this chunk: three GEMMs over B*Ttot rows
  float* a_emb = e->ws.alloc<float>((size_t)B * Ttot * D);
  float* audv = e->ws.alloc<float>((size_t)B * Ttot * D);
  float* audh = e->ws.alloc<float>((size_t)B * Ttot * D);
  const int MB3 = v3 ? c3_pick_mb(Q, B) : 0;
  float* arena3 = v3 ? e->ws.alloc<float>((size_t)((B + MB3 - 1) / MB3) * make_layout3(Q->L, Q->D, MB3).total) : nullptr;
  if (e->ws.sizing) return;
  GemmP g;
  g.A = aud.row(b0, 0); g.W = P->emb_aud.W; g.bias = P->emb_aud.bias; g.C = a_emb;
  g.M = B * Ttot; g.N = D; g.K = 256; g.mper = Ttot; g.a_bs = aud.bstride(); g.a_rs = aud.C; g.kc = 256; g.a_ts = 256;
  g.c_bs = (long)Ttot * D; g.c_rs = D; g.ldw = 256;
  launch_gemm(e, g, s);
  GemmP h;
  h.A = a_emb; h.W = P->fuse_v_a.W; h.bias = P->fuse_v_a.bias; h.C = audv;
  h.M = B * Ttot; h.N = D; h.K = D; h.mper = Ttot; h.a_bs = (long)Ttot * D; h.a_rs = D; h.kc = D; h.a_ts = D;
  h.c_bs = (long)Ttot * D; h.c_rs = D; h.ldw = D;
  launch_gemm(e, h, s);
  h.W = P->fuse_h_a.W; h.bias = P->fuse_h_a.bias; h.C = audh;
  launch_gemm(e, h, s);
  (void)noise_B;

  if (v3) {   // cluster-resident executor (pixelcnn3.inc): any batch size, clusters of 16 CTAs per 4 / 8 samples
    launch_pixelcnn3(e, P, Q, audv, audh, label, noise, idx_out, logits_out, B, T0, Ttot, pre, logits_all, arena3, MB3, s, d);
    return;
  }
  if (B > PIX_MB)
    fail(TS_ERR_UNSUPPORTED, "pixelcnn: the grid-wide executor takes %d samples per call (got %d); the host shim chunks larger batches", PIX_MB, B);
  // batch tile of the launch: the smallest of 8 / 16 / 32 / 64 samples that holds the batch (TS_PIX_TILE overrides);
  // every output is bit-identical whatever tile a sample runs in (same K slicing and reduction order)
  int MB = B <= 16 ? 16 : B <= 32 ? 32 : 64;    // the 8-sample tile stays opt-in (TS_PIX_TILE)
  if (const char* v = getenv("TS_PIX_TILE")) {
    const int t = atoi(v);
    if ((t == 8 || t == 16 || t == 32 || t == 64) && t >= B) MB = t;
  }
  const bool tracing = P->d_trace && P->trace_row >= 0;
  if (P->sched == 2 || (tracing && MB != 16)) MB = 64;   // schedule 2 / the stage trace: 64-sample tile (trace also 16)
  const PixLayout lay = make_layout(P->L, P->sched == 2 ? P->L : 2, MB);
  TS_CUDA(cudaMemsetAsync(P->d_arena, 0, (size_t)lay.total * sizeof(float), s));
  TS_CUDA(cudaMemsetAsync(P->d_barrier, 0, 4096, s));
  build_cls_kernel<<<e->sm_count, 256, 0, s>>>(P->d_cls, label, P->d_arena, lay.CLS, P->L, P->nclasses, B, MB);
  e->launches++;
  TS_CUDA(cudaGetLastError());

  PixArgs A;
  A.table = P->d_table; A.blob = P->d_blob; A.arena = P->d_arena; A.emb = P->d_emb;
  A.audv = audv; A.audh = audh; A.noise = noise; A.pre = pre; A.idx_out = idx_out; A.logits_out = logits_out;
  A.barrier = P->d_barrier; A.lay = lay;
  A.B = B; A.T0 = T0; A.Ttot = Ttot; A.log_r0 = logits_all ? 0 : T0; A.L = P->L; A.nstages = P->nstages; A.ncta = P->ncta;
  A.fused = P->fused ? 1 : 0;
  A.trace = P->d_trace; A.trace_row = P->trace_row;
  A.draw = d;
  A.cls_w = P->d_cls; A.ncls = P->nclasses;
  if (e->pixel_mode == 0) {
    void* fn = (void*)pixelcnn_kernel<true>;
    if (MB == 32) fn = (void*)pixelcnn_kernel<true, false, false, 32>;
    if (MB == 16) fn = (void*)pixelcnn_kernel<true, false, false, 16>;
    if (MB == 8) fn = (void*)pixelcnn_kernel<true, false, false, 8>;
    if (tracing) fn = MB == 16 ? (void*)pixelcnn_kernel<true, true, false, 16> : (void*)pixelcnn_kernel<true, true>;
    if (P->sched == 2) fn = tracing ? (void*)pixelcnn_kernel<true, true, true> : (void*)pixelcnn_kernel<true, false, true>;
    if (d.warp()) {   // the WARP instantiation of the default pipeline (no stage-trace variant)
      fn = MB == 8 ? (void*)pixelcnn_kernel<true, false, false, 8, true>
           : MB == 16 ? (void*)pixelcnn_kernel<true, false, false, 16, true>
           : MB == 32 ? (void*)pixelcnn_kernel<true, false, false, 32, true>
           : P->sched == 2 ? (void*)pixelcnn_kernel<true, false, true, 64, true>
                           : (void*)pixelcnn_kernel<true, false, false, 64, true>;
    }
    TS_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PIX_SMEM));
    int rs = 0, ss = 0;
    void* args[] = {&A, &rs, &ss};
    if (P->timing) TS_CUDA(cudaEventRecord(P->ev0, s));
    if (P->ncta < e->sm_count && (P->ncta & 1) == 0) {
      // partial-GPU plan: launched as CTA pairs (cluster 2x1x1) so that the kernel fills whole TPCs and the remaining TPCs
      // stay entirely free for the face path running next to it
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = dim3(P->ncta);
      cfg.blockDim = dim3(PIX_THREADS);
      cfg.dynamicSmemBytes = PIX_SMEM;
      cfg.stream = s;
      cudaLaunchAttribute at[2];
      at[0].id = cudaLaunchAttributeClusterDimension;
      at[0].val.clusterDim.x = 2; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
      at[1].id = cudaLaunchAttributeCooperative;
      at[1].val.cooperative = 1;
      cfg.attrs = at;
      cfg.numAttrs = 2;
      TS_CUDA(cudaLaunchKernelExC(&cfg, fn, args));
    } else {
      TS_CUDA(cudaLaunchCooperativeKernel(fn, dim3(P->ncta), dim3(PIX_THREADS), args, PIX_SMEM, s));
    }
    if (P->timing) { TS_CUDA(cudaEventRecord(P->ev1, s)); P->timed_rows += Ttot; P->timed_launches++; P->pending = true; }
    e->launches++;
  } else {
    void (*fn1)(PixArgs, int, int) = P->sched == 2 ? pixelcnn_kernel<false, false, true> : pixelcnn_kernel<false>;
    if (MB == 32) fn1 = pixelcnn_kernel<false, false, false, 32>;
    if (MB == 16) fn1 = pixelcnn_kernel<false, false, false, 16>;
    if (MB == 8) fn1 = pixelcnn_kernel<false, false, false, 8>;
    if (d.warp()) {
      fn1 = MB == 8 ? pixelcnn_kernel<false, false, false, 8, true>
            : MB == 16 ? pixelcnn_kernel<false, false, false, 16, true>
            : MB == 32 ? pixelcnn_kernel<false, false, false, 32, true>
            : P->sched == 2 ? pixelcnn_kernel<false, false, true, 64, true>
                            : pixelcnn_kernel<false, false, false, 64, true>;
    }
    TS_CUDA(cudaFuncSetAttribute(fn1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PIX_SMEM));
    for (int r = 0; r < Ttot; ++r)
      for (int st = 0; st < P->nstages; ++st) {
        fn1<<<P->ncta, PIX_THREADS, PIX_SMEM, s>>>(A, r, st);
        e->launches++;
      }
    TS_CUDA(cudaGetLastError());
  }
}

void pixel_destroy(ts_engine* e) {
  if (!e->pix) return;
  delete (Plan3*)e->pix->p3;
  tf_free(e->pix->tf);
  delete e->pix;
  e->pix = nullptr;
}

void pixelcnn_generate_act(ts_engine* e, const Act3& aud, const int64_t* label, const float* noise, int64_t* idx_out,
                           float* logits_out, int B, int T, const int64_t* pre, int T0, cudaStream_t s, bool logits_all,
                           const SampleCtl& d) {
  if (!e->pix) fail(TS_ERR_NOT_LOADED, "pixelcnn weights not loaded");
  // an anchored, styled, per-clip, shaped or guided call always runs the WARP kernels (d.warp()); without controls at
  // temperature 1, top_k 0 (the default draw's bits)
  // per-clip (guided: per-pair) controls, shaping and scales: host entries (validated by the caller) -> workspace, in
  // stream order before the sampler reads them
  SampleCtl dd = d;
  const size_t nd = d.guide ? (size_t)B / 2 : (size_t)B;
  ts_clip_ctl* dclip = d.clip_ctl ? e->ws.alloc<ts_clip_ctl>(nd) : nullptr;
  if (dclip && !e->ws.sizing)
    TS_CUDA(cudaMemcpyAsync(dclip, d.clip_ctl, nd * sizeof(ts_clip_ctl), cudaMemcpyHostToDevice, s));
  ts_clip_shape* dshape = d.clip_shape ? e->ws.alloc<ts_clip_shape>(nd) : nullptr;
  if (dshape && !e->ws.sizing)
    TS_CUDA(cudaMemcpyAsync(dshape, d.clip_shape, nd * sizeof(ts_clip_shape), cudaMemcpyHostToDevice, s));
  float* dguide = d.guide ? e->ws.alloc<float>(nd) : nullptr;
  if (dguide && !e->ws.sizing) TS_CUDA(cudaMemcpyAsync(dguide, d.guide, nd * sizeof(float), cudaMemcpyHostToDevice, s));
  dd.clip_ctl = dclip; dd.clip_shape = dshape; dd.guide = dguide;
  // guided: pre_latents [P][T0][2] -> one copy per branch [2P][T0][2], so every pre read stays on the branch's own index
  int64_t* dpre = d.guide && pre && T0 > 0 ? e->ws.alloc<int64_t>((size_t)B * T0 * 2) : nullptr;
  if (dpre && !e->ws.sizing) {
    const size_t row = (size_t)T0 * 2 * sizeof(int64_t);
    for (int k = 0; k < 2; ++k)
      TS_CUDA(cudaMemcpy2DAsync(reinterpret_cast<char*>(dpre) + k * row, 2 * row, pre, row, row, nd, cudaMemcpyDeviceToDevice, s));
  }
  generate_chunk(e, aud, 0, label, noise, B, idx_out, logits_out, B, T, dpre ? dpre : pre, T0, s, logits_all, dd);
}

void check_style(const ts_engine* e, const int64_t* label, const float* style, int ncls, const char* who) {
  if (!style) {
    if (!label) fail(TS_ERR_INVALID, "%s: label is NULL without a style schedule", who);
    return;
  }
  if (ncls < 1 || ncls > PIX_MAXCLS)
    fail(TS_ERR_INVALID, "%s: ncls = %d (styled calls take 1 to %d classes)", who, ncls, PIX_MAXCLS);
  if (ncls != e->pix->nclasses)
    fail(TS_ERR_INVALID, "%s: ncls = %d, the loaded prior has %d classes", who, ncls, e->pix->nclasses);
}

void check_sample_ctl(const SampleCtl& c, const float* noise, const int64_t* seeds) {
  if (!std::isfinite(c.temperature) || c.temperature < 0.f)
    fail(TS_ERR_INVALID, "pixelcnn sample: temperature %g (must be finite and >= 0)", (double)c.temperature);
  if (c.top_k < 0 || c.top_k > PIX_NCODE) fail(TS_ERR_INVALID, "pixelcnn sample: top_k %d outside [0, %d]", c.top_k, PIX_NCODE);
  if (c.temperature > 0.f && !noise && !seeds)
    fail(TS_ERR_INVALID, "pixelcnn sample: noise (or seeds) is NULL with temperature %g > 0", (double)c.temperature);
  if (!(c.top_p > 0.f && c.top_p <= 1.f)) fail(TS_ERR_INVALID, "pixelcnn sample: top_p %g outside (0, 1]", (double)c.top_p);
  if (!(c.min_p >= 0.f && c.min_p <= 1.f)) fail(TS_ERR_INVALID, "pixelcnn sample: min_p %g outside [0, 1]", (double)c.min_p);
}

void check_anchored_source(const SampleCtl* ctl, const float* noise, const int64_t* seeds, const char* who) {
  const bool greedy = ctl && ctl->temperature == 0.f;
  if (!greedy && (noise != nullptr) == (seeds != nullptr))
    fail(TS_ERR_INVALID, "%s: noise=%p seeds=%p (give exactly one; only greedy decoding runs without)", who, (const void*)noise,
         (const void*)seeds);
}

void check_clip_ctl(const ts_clip_ctl* clip_ctl, int B, const float* noise, const int64_t* seeds, const char* who) {
  bool sampled = false;
  for (int b = 0; b < B; ++b) {
    const ts_clip_ctl& c = clip_ctl[b];
    if (!std::isfinite(c.temperature) || c.temperature < 0.f)
      fail(TS_ERR_INVALID, "%s: clip %d: temperature %g (must be finite and >= 0)", who, b, (double)c.temperature);
    if (c.top_k < 0 || c.top_k > PIX_NCODE) fail(TS_ERR_INVALID, "%s: clip %d: top_k %d outside [0, %d]", who, b, c.top_k, PIX_NCODE);
    if (!(c.top_p > 0.f && c.top_p <= 1.f)) fail(TS_ERR_INVALID, "%s: clip %d: top_p %g outside (0, 1]", who, b, (double)c.top_p);
    if (!(c.min_p >= 0.f && c.min_p <= 1.f)) fail(TS_ERR_INVALID, "%s: clip %d: min_p %g outside [0, 1]", who, b, (double)c.min_p);
    sampled = sampled || c.temperature > 0.f;
  }
  if (sampled && (noise != nullptr) == (seeds != nullptr))
    fail(TS_ERR_INVALID, "%s: noise=%p seeds=%p (give exactly one; only a batch of greedy clips runs without)", who,
         (const void*)noise, (const void*)seeds);
}

SampleCtl shaped_ctl(const ts_sample_ctl* ctl, const ts_clip_ctl* clip_ctl, int B, const float* noise, const int64_t* seeds,
                     const char* who) {
  SampleCtl c;
  if (clip_ctl) {   // logp_out / kept_out of ctl; the draws' controls come from clip_ctl
    check_clip_ctl(clip_ctl, B, noise, seeds, who);
    if (ctl) { c.logp_out = ctl->logp_out; c.kept_out = ctl->kept_out; }
    return c;
  }
  if (ctl) c = sample_ctl_of(ctl);
  check_sample_ctl(c, noise, seeds);
  check_anchored_source(&c, noise, seeds, who);
  return c;
}

void check_clip_shape(const ts_clip_shape* clip_shape, int B, const char* who) {
  for (int b = 0; b < B; ++b) {
    const ts_clip_shape& c = clip_shape[b];
    if (!std::isfinite(c.repetition_penalty) || !(c.repetition_penalty >= 1.f))
      fail(TS_ERR_INVALID, "%s: clip %d: repetition_penalty %g (must be finite and >= 1)", who, b, (double)c.repetition_penalty);
    if (c.repetition_window < 1)
      fail(TS_ERR_INVALID, "%s: clip %d: repetition_window %d (must be >= 1)", who, b, c.repetition_window);
  }
}

void check_guidance(const float* guidance, int P, const char* who) {
  if (!guidance) fail(TS_ERR_INVALID, "%s: guidance is NULL", who);
  for (int p = 0; p < P; ++p)
    if (!std::isfinite(guidance[p]) || !(guidance[p] >= 0.f && guidance[p] <= TS_GUIDANCE_MAX))
      fail(TS_ERR_INVALID, "%s: pair %d: guidance %g (must be finite and in [0, %g])", who, p, (double)guidance[p],
           (double)TS_GUIDANCE_MAX);
}

SampleCtl sample_ctl_of(const ts_sample_ctl* c) {
  if (!c) fail(TS_ERR_INVALID, "pixelcnn sample: ctl is NULL");
  SampleCtl s;
  s.temperature = c->temperature; s.top_k = c->top_k; s.top_p = c->top_p; s.min_p = c->min_p;
  s.logp_out = c->logp_out; s.kept_out = c->kept_out;
  s.controls = true;
  return s;
}

}  // namespace ts

using namespace ts;

extern "C" int ts_load_pixelcnn(ts_engine* e, const ts_tensor* tensors, int n) {
  TS_API_BEGIN(e)
  Ckpt ck(tensors, n);
  const ts_tensor* emb = ck.get("embedding.weight");
  if (emb->ndim != 2 || emb->shape[0] != PIX_NCODE)
    fail(TS_ERR_UNSUPPORTED, "pixelcnn: embedding.weight must be [%d, dim]", PIX_NCODE);
  const int D = (int)emb->shape[1];
  int L = 0;
  while (ck.has("layers." + std::to_string(L) + ".vert_stack.weight")) ++L;
  if (L < 3 || L > 30) fail(TS_ERR_MISSING, "pixelcnn: %d layers found", L);
  const int ncls = (int)ck.get("layers.0.class_cond_embedding.weight")->shape[0];
  LoadScope scope(e, "pixelcnn");
  // the grid-wide executor (modes 0 / 1) is built for the shipped geometry dim = 256 only; every geometry runs on the
  // cluster-resident executor (mode 2)
  std::unique_ptr<PixelPlan> P(D == PIX_D ? build_plan(e, ck, e->pixel_fusion) : new PixelPlan());
  P->L = L; P->D = D; P->nclasses = ncls;
  plan_common(e, ck, P.get(), L, D);
  // an engine set up for a partial-GPU grid-wide plan (ts_set_pixelcnn_ctas) does not need the cluster-resident plan as well
  Plan3* Q = (P->has_v1 && e->pixel_ctas > 0) ? nullptr : build_plan3(e, ck, L, D, ncls);
  P->p3 = Q;
  if (!P->has_v1) { P->nstages = Q->nstages; P->ncta = C3_CL; }
  P->tf = tf_build(e, ck, L, D, ncls);
  pixel_destroy(e);
  e->pix = P.release();
  scope.commit();
  TS_API_END(e)
}

extern "C" int64_t ts_pixelcnn_row_bytes(ts_engine* e) { return (e && e->pix) ? e->pix->row_bytes : 0; }
extern "C" int64_t ts_pixelcnn_staged_row_bytes(ts_engine* e) {
  if (!e || !e->pix) return 0;
  if ((e->pixel_mode == 2 && e->pix->p3) || !e->pix->has_v1) return (int64_t)((Plan3*)e->pix->p3)->rank_stride * C3_CL * 4;
  return e->pix->staged_row_bytes;
}

// CUDA-event timing of the persistent kernel on its launch stream (bench.py roofline leg).
extern "C" int ts_pixelcnn_timing(ts_engine* e, int enable) {
  TS_API_BEGIN(e)
  ts::require_device(e);
  if (!e->pix) fail(TS_ERR_NOT_LOADED, "pixelcnn weights not loaded");
  PixelPlan* P = e->pix;
  if (enable && !P->ev0) {
    TS_CUDA(cudaEventCreate(&P->ev0));
    TS_CUDA(cudaEventCreate(&P->ev1));
  }
  P->timing = enable != 0;
  P->pending = false;
  TS_API_END(e)
}
// duration (ms) of the most recent timed persistent-kernel launch; synchronises on its end event.
extern "C" double ts_pixelcnn_last_ms(ts_engine* e) {
  if (!e || !e->pix || !e->pix->pending) return -1.0;
  float ms = 0.f;
  if (cudaEventSynchronize(e->pix->ev1) != cudaSuccess) return -1.0;
  if (cudaEventElapsedTime(&ms, e->pix->ev0, e->pix->ev1) != cudaSuccess) return -1.0;
  return (double)ms;
}

// Stage trace of one latent row (debug): row >= 0 arms it for the following ts_pixelcnn_generate calls (the
// TRACE instantiation of the persistent kernel runs instead of the default one), row < 0 disarms.
extern "C" int ts_pixelcnn_trace(ts_engine* e, int row) {
  TS_API_BEGIN(e)
  if (!e->pix) fail(TS_ERR_NOT_LOADED, "pixelcnn weights not loaded");
  if (e->host_only) fail(TS_ERR_UNSUPPORTED, "host-only engine cannot execute");
  PixelPlan* P = e->pix;
  const size_t n = (size_t)P->nstages * std::max(P->ncta, 16) * 4;
  if (row >= 0 && !P->d_trace) P->d_trace = (unsigned long long*)e->dmalloc(n * sizeof(unsigned long long));
  if (row >= 0) TS_CUDA(cudaMemset(P->d_trace, 0, n * sizeof(unsigned long long)));
  P->trace_row = row;
  TS_API_END(e)
}
// out[nstages][ncta][4] (ns): weights ready / left the grid barrier / task done / arrived.  *len in/out (elements).
extern "C" int ts_pixelcnn_trace_read(ts_engine* e, uint64_t* out, int64_t* len) {
  TS_API_BEGIN(e)
  if (!e->pix || !e->pix->d_trace) fail(TS_ERR_NOT_LOADED, "pixelcnn trace not armed");
  PixelPlan* P = e->pix;
  const int64_t n = (int64_t)P->nstages * std::max(P->ncta, 16) * 4;
  if (out) {
    if (*len < n) fail(TS_ERR_INVALID, "trace buffer too small");
    TS_CUDA(cudaDeviceSynchronize());
    TS_CUDA(cudaMemcpy(out, P->d_trace, (size_t)n * sizeof(uint64_t), cudaMemcpyDeviceToHost));
  }
  *len = n;
  TS_API_END(e)
}

extern "C" int ts_pixelcnn_plan_shape(ts_engine* e, int* nstages, int* ncta) {
  TS_API_BEGIN(e)
  if (!e->pix) fail(TS_ERR_NOT_LOADED, "pixelcnn weights not loaded");
  *nstages = e->pix->nstages;
  *ncta = e->pix->ncta;
  TS_API_END(e)
}

extern "C" int ts_debug_pixelcnn_plan(ts_engine* e, int32_t* table, int64_t* table_len, float* blob, int64_t* blob_len) {
  TS_API_BEGIN(e)
  if (!e->pix) fail(TS_ERR_NOT_LOADED, "pixelcnn weights not loaded");
  PixelPlan* P = e->pix;
  const int64_t hdr = 32;
  const int64_t tl = hdr + (int64_t)P->table.size() * 8, bl = (int64_t)P->blob.size();
  if (table) {
    if (*table_len < tl) fail(TS_ERR_INVALID, "table buffer too small");
    int32_t h[32] = {P->ncta, P->nstages, P->L, PIX_D, PIX_MB, P->lay.E, P->lay.XV1P, P->lay.XV, P->lay.HV, P->lay.V2H,
                     P->lay.G, P->lay.XHP, P->lay.XH, P->lay.Y, P->lay.LOG, P->lay.CLS, P->lay.total, PIX_NCODE, P->cl,
                     P->sched == 2 ? P->L : 2};
    memcpy(table, h, sizeof h);
    memcpy(table + hdr, P->table.data(), P->table.size() * sizeof(PixTask));
  }
  if (blob) {
    if (*blob_len < bl) fail(TS_ERR_INVALID, "blob buffer too small");
    memcpy(blob, P->blob.data(), P->blob.size() * sizeof(float));
  }
  *table_len = tl;
  *blob_len = bl;
  TS_API_END(e)
}

static void check_pix(ts_engine* e, int B, int T) {
  if (!e->pix) fail(TS_ERR_NOT_LOADED, "pixelcnn weights not loaded");
  if (e->host_only) fail(TS_ERR_UNSUPPORTED, "host-only engine cannot execute");
  if (B <= 0 || T <= 0) fail(TS_ERR_INVALID, "pixelcnn: B=%d T=%d", B, T);
}

// d: the draw inputs (SampleCtl), the default sampler (ts_pixelcnn_generate) when they are the defaults.
static void pixelcnn_generate_call(ts_engine* e, const float* aud, const int64_t* label, const float* noise, int64_t* idx_out,
                                   float* logits_out, int B, int T, const int64_t* pre_latents, int T0, void* stream,
                                   const SampleCtl& d = SampleCtl()) {
  check_pix(e, B, T);
  if (T0 < 0 || (T0 > 0 && !pre_latents)) fail(TS_ERR_INVALID, "pixelcnn: T0=%d without pre_latents", T0);
  if (d.controls && !d.clip_ctl) check_sample_ctl(d, noise, d.seeds);
  cudaStream_t s = (cudaStream_t)stream;
  auto body = [&] {
    Act3 a = new_act(e, B, T0 + T, 256, 0, s);
    nct_to_act(e, aud, 256, a, s);
    pixelcnn_generate_act(e, a, label, noise, idx_out, logits_out, B, T, pre_latents, T0, s, false, d);
  };
  e->ws.begin_sizing(); body();
  size_t need = e->ws.need;
  e->ws.buf.ensure(need + 256);
  e->ws.begin(need); body();
}

extern "C" int ts_pixelcnn_generate(ts_engine* e, const float* aud, const int64_t* label, const float* noise,
                                    int64_t* idx_out, float* logits_out, int B, int T, const int64_t* pre_latents, int T0,
                                    void* stream) {
  TS_API_BEGIN(e)
  pixelcnn_generate_call(e, aud, label, noise, idx_out, logits_out, B, T, pre_latents, T0, stream);
  TS_API_END(e)
}

extern "C" int ts_pixelcnn_sample(ts_engine* e, const float* aud, const int64_t* label, const float* noise,
                                  int64_t* idx_out, float* logits_out, int B, int T, const int64_t* pre_latents, int T0,
                                  float temperature, int top_k, float* logp_out, void* stream) {
  const ts_sample_ctl ctl = {temperature, top_k, 1.f, 0.f, logp_out, nullptr};
  return ts_pixelcnn_sample_ctl(e, aud, label, noise, idx_out, logits_out, B, T, pre_latents, T0, &ctl, stream);
}

extern "C" int ts_pixelcnn_sample_ctl(ts_engine* e, const float* aud, const int64_t* label, const float* noise,
                                      int64_t* idx_out, float* logits_out, int B, int T, const int64_t* pre_latents, int T0,
                                      const ts_sample_ctl* ctl, void* stream) {
  TS_API_BEGIN(e)
  const SampleCtl c = sample_ctl_of(ctl);
  pixelcnn_generate_call(e, aud, label, noise, idx_out, logits_out, B, T, pre_latents, T0, stream, c);
  TS_API_END(e)
}

// The Exp(1) values of the seeded sampler in the layout of `noise`: block (2 (r - T0) + c) B + m holds draw (r, c) of
// clip m.  One CTA of 256 threads per block, the thread <-> code mapping of the samplers.
__global__ void __launch_bounds__(256) sampler_noise_kernel(const int64_t* __restrict__ seeds, float* __restrict__ out, int B, int T0) {
  const int blk = blockIdx.x, m = blk % B, step = blk / B;
  float q[8];
  seeded_q(seeds[m], T0 + (step >> 1), step & 1, threadIdx.x, q);
  float* dst = out + (size_t)blk * PIX_NCODE;
#pragma unroll
  for (int j = 0; j < 8; ++j) dst[threadIdx.x + 256 * j] = q[j];
}

extern "C" int ts_sampler_noise(ts_engine* e, const int64_t* seeds, float* noise_out, int B, int T, int T0, void* stream) {
  TS_API_BEGIN(e)
  ts::require_device(e);
  if (B <= 0 || T <= 0 || T0 < 0 || (int64_t)2 * T * B > INT32_MAX || !seeds || !noise_out)
    fail(TS_ERR_INVALID, "ts_sampler_noise: B=%d T=%d T0=%d seeds=%p noise_out=%p", B, T, T0, (const void*)seeds, (void*)noise_out);
  sampler_noise_kernel<<<2 * T * B, 256, 0, (cudaStream_t)stream>>>(seeds, noise_out, B, T0);
  e->launches++;
  TS_CUDA(cudaGetLastError());
  TS_API_END(e)
}

extern "C" int ts_pixelcnn_sample_seeded(ts_engine* e, const float* aud, const int64_t* label, const int64_t* seeds,
                                         int64_t* idx_out, float* logits_out, int B, int T, const int64_t* pre_latents, int T0,
                                         const ts_sample_ctl* ctl, void* stream) {
  TS_API_BEGIN(e)
  check_pix(e, B, T);
  SampleCtl c;
  if (ctl) c = sample_ctl_of(ctl);
  else if (!seeds) fail(TS_ERR_INVALID, "ts_pixelcnn_sample_seeded: seeds is NULL (only greedy decoding runs without)");
  c.seeds = seeds;
  pixelcnn_generate_call(e, aud, label, nullptr, idx_out, logits_out, B, T, pre_latents, T0, stream, c);
  TS_API_END(e)
}

// anchors [B,T,2] (device): draws pinned to a code in [0, 2048), the others sampled; NULL: the entry point of the same
// noise, seeds and ctl (ts_pixelcnn_generate, _sample_ctl or _sample_seeded) with its launches and bits.
extern "C" int ts_pixelcnn_sample_anchored(ts_engine* e, const float* aud, const int64_t* label, const float* noise,
                                           const int64_t* seeds, const int64_t* anchors, int64_t* idx_out, float* logits_out,
                                           int B, int T, const int64_t* pre_latents, int T0, const ts_sample_ctl* ctl,
                                           void* stream) {
  TS_API_BEGIN(e)
  check_pix(e, B, T);
  SampleCtl c;
  if (ctl) c = sample_ctl_of(ctl);
  check_anchored_source(ctl ? &c : nullptr, noise, seeds, "ts_pixelcnn_sample_anchored");
  c.seeds = seeds; c.anchors = anchors;
  pixelcnn_generate_call(e, aud, label, noise, idx_out, logits_out, B, T, pre_latents, T0, stream, c);
  TS_API_END(e)
}

// style [B, T0+T, ncls] (device): per-row speaker weights blended into every gate's class term, label unread (may be
// NULL); NULL: ts_pixelcnn_sample_anchored with its launches and bits.
extern "C" int ts_pixelcnn_sample_styled(ts_engine* e, const float* aud, const int64_t* label, const float* style, int ncls,
                                         const float* noise, const int64_t* seeds, const int64_t* anchors, int64_t* idx_out,
                                         float* logits_out, int B, int T, const int64_t* pre_latents, int T0,
                                         const ts_sample_ctl* ctl, void* stream) {
  TS_API_BEGIN(e)
  check_pix(e, B, T);
  check_style(e, label, style, ncls, "ts_pixelcnn_sample_styled");
  SampleCtl c;
  if (ctl) c = sample_ctl_of(ctl);
  check_anchored_source(ctl ? &c : nullptr, noise, seeds, "ts_pixelcnn_sample_styled");
  c.seeds = seeds; c.anchors = anchors; c.style = style;
  pixelcnn_generate_call(e, aud, label, noise, idx_out, logits_out, B, T, pre_latents, T0, stream, c);
  TS_API_END(e)
}

// clip_ctl [B] (host): each clip's temperature, top_k, top_p and min_p, validated here and copied to the workspace on the
// call's stream; ctl (may be NULL) gives logp_out / kept_out only.  NULL: ts_pixelcnn_sample_styled with its launches and bits.
extern "C" int ts_pixelcnn_sample_clips(ts_engine* e, const float* aud, const int64_t* label, const float* style, int ncls,
                                        const float* noise, const int64_t* seeds, const int64_t* anchors, int64_t* idx_out,
                                        float* logits_out, int B, int T, const int64_t* pre_latents, int T0,
                                        const ts_sample_ctl* ctl, const ts_clip_ctl* clip_ctl, void* stream) {
  if (!clip_ctl)
    return ts_pixelcnn_sample_styled(e, aud, label, style, ncls, noise, seeds, anchors, idx_out, logits_out, B, T, pre_latents,
                                     T0, ctl, stream);
  TS_API_BEGIN(e)
  check_pix(e, B, T);
  check_style(e, label, style, ncls, "ts_pixelcnn_sample_clips");
  check_clip_ctl(clip_ctl, B, noise, seeds, "ts_pixelcnn_sample_clips");
  SampleCtl c;   // logp_out / kept_out of ctl; the draws' controls come from clip_ctl
  if (ctl) { c.logp_out = ctl->logp_out; c.kept_out = ctl->kept_out; }
  c.seeds = seeds; c.anchors = anchors; c.style = style; c.clip_ctl = clip_ctl;
  pixelcnn_generate_call(e, aud, label, noise, idx_out, logits_out, B, T, pre_latents, T0, stream, c);
  TS_API_END(e)
}

// clip_shape [B] (host): each clip's repetition penalty and window, validated here and copied to the workspace on the
// call's stream; code_bias [B,2,2048] (device).  clip_ctl NULL: ctl's scalar controls.  Both NULL: ts_pixelcnn_sample_clips
// with its launches and bits.
extern "C" int ts_pixelcnn_sample_shaped(ts_engine* e, const float* aud, const int64_t* label, const float* style, int ncls,
                                         const float* noise, const int64_t* seeds, const int64_t* anchors, int64_t* idx_out,
                                         float* logits_out, int B, int T, const int64_t* pre_latents, int T0,
                                         const ts_sample_ctl* ctl, const ts_clip_ctl* clip_ctl, const ts_clip_shape* clip_shape,
                                         const float* code_bias, void* stream) {
  if (!clip_shape && !code_bias)
    return ts_pixelcnn_sample_clips(e, aud, label, style, ncls, noise, seeds, anchors, idx_out, logits_out, B, T, pre_latents,
                                    T0, ctl, clip_ctl, stream);
  TS_API_BEGIN(e)
  check_pix(e, B, T);
  check_style(e, label, style, ncls, "ts_pixelcnn_sample_shaped");
  if (clip_shape) check_clip_shape(clip_shape, B, "ts_pixelcnn_sample_shaped");
  SampleCtl c = shaped_ctl(ctl, clip_ctl, B, noise, seeds, "ts_pixelcnn_sample_shaped");
  c.seeds = seeds; c.anchors = anchors; c.style = style; c.clip_ctl = clip_ctl; c.clip_shape = clip_shape; c.code_bias = code_bias;
  pixelcnn_generate_call(e, aud, label, noise, idx_out, logits_out, B, T, pre_latents, T0, stream, c);
  TS_API_END(e)
}

// P pairs = 2P branches: aud / label / style / idx_out / logits_out / logp / kept per branch, every draw input per pair.
// guidance [P] (host): checked here and copied to the workspace on the call's stream.
extern "C" int ts_pixelcnn_sample_guided(ts_engine* e, const float* aud, const int64_t* label, const float* style, int ncls,
                                         const float* noise, const int64_t* seeds, const int64_t* anchors, int64_t* idx_out,
                                         float* logits_out, int P, int T, const int64_t* pre_latents, int T0,
                                         const ts_sample_ctl* ctl, const ts_clip_ctl* clip_ctl, const ts_clip_shape* clip_shape,
                                         const float* code_bias, const float* guidance, void* stream) {
  TS_API_BEGIN(e)
  if (P < 1 || P > INT_MAX / 2) fail(TS_ERR_INVALID, "ts_pixelcnn_sample_guided: P=%d pairs", P);
  check_pix(e, 2 * P, T);
  check_style(e, label, style, ncls, "ts_pixelcnn_sample_guided");
  check_guidance(guidance, P, "ts_pixelcnn_sample_guided");
  if (clip_shape) check_clip_shape(clip_shape, P, "ts_pixelcnn_sample_guided");
  SampleCtl c = shaped_ctl(ctl, clip_ctl, P, noise, seeds, "ts_pixelcnn_sample_guided");
  c.seeds = seeds; c.anchors = anchors; c.style = style; c.clip_ctl = clip_ctl; c.clip_shape = clip_shape; c.code_bias = code_bias;
  c.guide = guidance;
  pixelcnn_generate_call(e, aud, label, noise, idx_out, logits_out, 2 * P, T, pre_latents, T0, stream, c);
  TS_API_END(e)
}

extern "C" int ts_pixelcnn_logits(ts_engine* e, const float* aud, const int64_t* label, const int64_t* codes,
                                  float* logits_out, int B, int T, void* stream) {
  TS_API_BEGIN(e)
  check_pix(e, B, T);
  cudaStream_t s = (cudaStream_t)stream;
  auto body = [&] {
    Act3 a = new_act(e, B, T, 256, 0, s);
    nct_to_act(e, aud, 256, a, s);
    float* steps = e->ws.alloc<float>((size_t)2 * T * B * PIX_NCODE);
    int64_t* dummy = e->ws.alloc<int64_t>(16);
    // all rows forced (T0 = T, nothing sampled), logits recorded for every row
    pixelcnn_generate_act(e, a, label, nullptr, dummy, steps, B, 0, codes, T, s, true);
    if (!e->ws.sizing) {
      long n = (long)2 * T * B * PIX_NCODE;
      logits_to_ref_kernel<<<(int)std::min<long>((n + 255) / 256, (long)e->sm_count * 16), 256, 0, s>>>(steps, logits_out, B, T);
      e->launches++;
      TS_CUDA(cudaGetLastError());
    }
  };
  e->ws.begin_sizing(); body();
  size_t need = e->ws.need;
  e->ws.buf.ensure(need + 256);
  e->ws.begin(need); body();
  TS_API_END(e)
}
