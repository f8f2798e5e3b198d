// talkshow_b200 — 1-D conv stacks of the body path: AudioEncoder (nets/spg/vqvae_1d.py:11-34),
// VQ-VAE Encoder (:66-92) + VectorQuantizerEMA lookup/argmin (vqvae_modules.py:311-323) and
// Decoder (:116-149).  BatchNorm (eval) and the parallel "residual" conv of every down/up block
// are folded into one weight matrix at load time:
//     LReLU(BN(conv(x)) + conv_res(x))  ==  LReLU(conv'(x)),  W' = a*W + W_res,
//     b' = a*(b - mean) + beta + b_res,  a = gamma / sqrt(var + eps)
// so each block is ONE implicit GEMM; ConvTranspose1d(k4,s2,p1) becomes two 2-tap convs (even /
// odd output phase) writing interleaved rows.
#include "convstack.h"

#include <cmath>

namespace ts {

static const double BN_EPS = 1e-5;

struct Folded {
  std::vector<double> a, b;  // per out channel: scale and shift
};

static Folded bn_fold(const Ckpt& ck, const std::string& p, int c) {
  const float* g = ck.f32(p + "weight", {c});
  const float* be = ck.f32(p + "bias", {c});
  const float* mu = ck.f32(p + "running_mean", {c});
  const float* var = ck.f32(p + "running_var", {c});
  Folded f;
  f.a.resize(c);
  f.b.resize(c);
  for (int i = 0; i < c; ++i) {
    double a = (double)g[i] / std::sqrt((double)var[i] + BN_EPS);
    f.a[i] = a;
    f.b[i] = (double)be[i] - (double)mu[i] * a;
  }
  return f;
}

// Conv1d weight [cout][cin][k] (+BN, + residual conv of the same shape) -> Layer [cout][k][cin_pad]
static Layer pack_conv(ts_engine* e, const Ckpt& ck, const std::string& p, int cin, int cout, int k, bool bn,
                       bool residual) {
  const float* w = ck.f32(p + "conv.weight", {cout, cin, k});
  const float* b = ck.f32(p + "conv.bias", {cout});
  const float* wr = residual ? ck.f32(p + "residual_layer.weight", {cout, cin, k}) : nullptr;
  const float* br = residual ? ck.f32(p + "residual_layer.bias", {cout}) : nullptr;
  Folded f;
  if (bn) f = bn_fold(ck, p + "norm.", cout);
  int cp = pad4(cin);
  std::vector<float> W((size_t)cout * k * cp, 0.f), B(cout);
  for (int o = 0; o < cout; ++o) {
    double a = bn ? f.a[o] : 1.0, sh = bn ? f.b[o] : 0.0;
    for (int c = 0; c < cin; ++c)
      for (int t = 0; t < k; ++t) {
        double v = a * (double)w[((size_t)o * cin + c) * k + t];
        if (wr) v += (double)wr[((size_t)o * cin + c) * k + t];
        W[((size_t)o * k + t) * cp + c] = (float)v;
      }
    double bb = a * (double)b[o] + sh;
    if (br) bb += (double)br[o];
    B[o] = (float)bb;
  }
  Layer L;
  L.N = cout;
  L.taps = k;
  L.cin = cp;
  L.K = k * cp;
  upload_weights(e, W, &L);
  L.bias = e->upload(B);
  return L;
}

// plain Conv1d without norm, key prefix p + "weight"/"bias"
static Layer pack_plain(ts_engine* e, const Ckpt& ck, const std::string& p, int cin, int cout, int k) {
  const float* w = ck.f32(p + "weight", {cout, cin, k});
  const float* b = ck.f32(p + "bias", {cout});
  int cp = pad4(cin);
  std::vector<float> W((size_t)cout * k * cp, 0.f), B(b, b + cout);
  for (int o = 0; o < cout; ++o)
    for (int c = 0; c < cin; ++c)
      for (int t = 0; t < k; ++t) W[((size_t)o * k + t) * cp + c] = w[((size_t)o * cin + c) * k + t];
  Layer L;
  L.N = cout;
  L.taps = k;
  L.cin = cp;
  L.K = k * cp;
  upload_weights(e, W, &L);
  L.bias = e->upload(B);
  return L;
}

// ConvTranspose1d(k=4,s=2,p=1) weight [cin][cout][4] + BN + residual ConvTranspose -> two 2-tap
// layers.  y[2m] = x[m-1]*W[..,3] + x[m]*W[..,1];  y[2m+1] = x[m]*W[..,2] + x[m+1]*W[..,0].
static void pack_up(ts_engine* e, const Ckpt& ck, const std::string& p, int cin, int cout, Layer* even, Layer* odd) {
  const float* w = ck.f32(p + "conv.weight", {cin, cout, 4});
  const float* b = ck.f32(p + "conv.bias", {cout});
  const float* wr = ck.f32(p + "residual_layer.weight", {cin, cout, 4});
  const float* br = ck.f32(p + "residual_layer.bias", {cout});
  Folded f = bn_fold(ck, p + "norm.", cout);
  const int tapk[2][2] = {{3, 1}, {2, 0}};
  for (int ph = 0; ph < 2; ++ph) {
    std::vector<float> W((size_t)cout * 2 * cin), B(cout);
    for (int o = 0; o < cout; ++o) {
      for (int t = 0; t < 2; ++t)
        for (int c = 0; c < cin; ++c) {
          size_t src = ((size_t)c * cout + o) * 4 + tapk[ph][t];
          W[((size_t)o * 2 + t) * cin + c] = (float)(f.a[o] * (double)w[src] + (double)wr[src]);
        }
      B[o] = (float)(f.a[o] * (double)b[o] + f.b[o] + (double)br[o]);
    }
    Layer L;
    L.N = cout;
    L.taps = 2;
    L.cin = cin;
    L.K = 2 * cin;
    upload_weights(e, W, &L);
    L.bias = e->upload(B);
    *(ph ? odd : even) = L;
  }
}

static void pack_stack(ts_engine* e, const Ckpt& ck, const std::string& p, int c, ResStack* s) {
  s->l0 = pack_conv(e, ck, p + "_layers.0.", c, c, 3, true, false);
  s->l1 = pack_conv(e, ck, p + "_layers.1.", c, c, 3, true, false);
  // final conv + norm of Res_CNR_Stack: keys p+"conv.*", p+"norm.*"
  s->fin = pack_conv(e, ck, p, c, c, 3, true, false);
}

void pack_trunk(ts_engine* e, const Ckpt& ck, const std::string& p, int in_dim, int hid, Trunk* t) {
  t->in_dim = in_dim;
  t->hid = hid;
  t->project = pack_conv(e, ck, p + "project.", in_dim, hid / 4, 3, true, false);
  pack_stack(e, ck, p + "_enc_1.", hid / 4, &t->s1);
  t->down1 = pack_conv(e, ck, p + "_down_1.", hid / 4, hid / 2, 4, true, true);
  pack_stack(e, ck, p + "_enc_2.", hid / 2, &t->s2);
  t->down2 = pack_conv(e, ck, p + "_down_2.", hid / 2, hid, 4, true, true);
  pack_stack(e, ck, p + "_enc_3.", hid, &t->s3);
}

void pack_vq(ts_engine* e, const Ckpt& ck, VQNet* v) {
  const ts_tensor* pw = ck.get("decoder.project.weight");
  int C = (int)pw->shape[0];
  v->out_dim = C;
  const int hid = 1024, emb = 64;
  const ts_tensor* cbt = ck.get("vq_layer.embeddings");
  v->ncodes = (int)cbt->shape[0];
  pack_trunk(e, ck, "encoder.", C, hid, &v->enc);
  v->pre_vq = pack_plain(e, ck, "encoder.pre_vq_conv.", hid, emb, 1);
  const float* cb = ck.f32("vq_layer.embeddings", {v->ncodes, emb});
  std::vector<float> CB(cb, cb + (size_t)v->ncodes * emb), EE(v->ncodes);
  for (int n = 0; n < v->ncodes; ++n) {
    // torch.sum(embeddings ** 2, dim=1): squares rounded to fp32 like ATen, summed exactly (double) and
    // rounded once -- within 1 ulp of ATen's vectorised fp32 sum whatever its order
    double s = 0.0;
    for (int c = 0; c < emb; ++c) s += (double)(cb[(size_t)n * emb + c] * cb[(size_t)n * emb + c]);
    EE[n] = (float)s;
  }
  v->codebook = e->upload(CB);
  v->ee = e->upload(EE);
  v->aft_vq = pack_plain(e, ck, "decoder.aft_vq_conv.", emb, hid, 1);
  pack_stack(e, ck, "decoder._dec_1.", hid, &v->d1);
  pack_up(e, ck, "decoder._up_2.", hid, hid / 2, &v->up2e, &v->up2o);
  pack_stack(e, ck, "decoder._dec_2.", hid / 2, &v->d2);
  pack_up(e, ck, "decoder._up_3.", hid / 2, hid / 4, &v->up3e, &v->up3o);
  pack_stack(e, ck, "decoder._dec_3.", hid / 4, &v->d3);
  v->project = pack_plain(e, ck, "decoder.project.", hid / 4, C, 1);
  v->loaded = true;
}

// ---- execution -------------------------------------------------------------------------------
Act3 new_act(ts_engine* e, int B, int T, int C, int pad, cudaStream_t s, bool split, int tail, bool planes_only) {
  Act3 a;
  a.B = B;
  a.T = T;
  a.C = C;
  a.pad = pad;
  a.tail = tail;
  a.split = split;
  // planes_only: the activation feeds tensor-core convs only -- no fp32 copy (half the bytes written and kept)
  if (!(planes_only && split && e->tc_f16 && e->use_tc)) a.p = e->ws.alloc<float>(a.numel());
  if (split && e->tc_f16) {
    a.h16 = e->ws.alloc<unsigned short>(a.numel());
    a.l16 = e->ws.alloc<unsigned short>(a.numel());
  } else if (split) {
    a.lo = e->ws.alloc<float>(a.numel());
  }
  zero_pads(e, a, s);
  return a;
}

static Act3 run_stack(ts_engine* e, const ResStack& st, const Act3& x, cudaStream_t s, bool tc = false) {
  // tc: activations kept as (hi, lo) pairs so the convs run on the tensor-core kernel (VQ decoder);
  // the audio / VQ encoders stay on the fp32 FFMA kernel (their outputs decide code indices)
  Act3 h0 = new_act(e, x.B, x.T, x.C, 1, s, tc);
  conv_auto(e, st.l0, x, 3, 1, 1, h0, x.T, ACT_LRELU, nullptr, s);
  Act3 h1 = new_act(e, x.B, x.T, x.C, 1, s, tc);
  conv_auto(e, st.l1, h0, 3, 1, 1, h1, x.T, ACT_LRELU, nullptr, s);
  Act3 y = new_act(e, x.B, x.T, x.C, 1, s, tc);
  conv_auto(e, st.fin, h1, 3, 1, 1, y, x.T, ACT_RELU, &x, s);  // relu(BN(conv(h)) + x), vqvae_modules.py:210-212
  return y;
}

Act3 run_trunk(ts_engine* e, const Trunk& t, const Act3& x, cudaStream_t s) {
  Act3 h = new_act(e, x.B, x.T, t.hid / 4, 1, s);
  conv1d(e, t.project, x, 3, 1, 1, h, x.T, ACT_LRELU, nullptr, s);
  h = run_stack(e, t.s1, h, s);
  int T1 = (h.T + 2 - 4) / 2 + 1;
  Act3 d1 = new_act(e, x.B, T1, t.hid / 2, 1, s);
  conv1d(e, t.down1, h, 4, 2, 1, d1, T1, ACT_LRELU, nullptr, s);
  h = run_stack(e, t.s2, d1, s);
  int T2 = (T1 + 2 - 4) / 2 + 1;
  Act3 d2 = new_act(e, x.B, T2, t.hid, 1, s);
  conv1d(e, t.down2, h, 4, 2, 1, d2, T2, ACT_LRELU, nullptr, s);
  return run_stack(e, t.s3, d2, s);
}

static Act3 run_up(ts_engine* e, const Layer& ev, const Layer& od, const Act3& x, cudaStream_t s, bool tc) {
  Act3 y = new_act(e, x.B, 2 * x.T, ev.N, 1, s, tc);
  conv_auto(e, ev, x, 2, 1, 1, y, x.T, ACT_LRELU, nullptr, s, 2, 0);   // rows m-1, m   -> y[2m]
  conv_auto(e, od, x, 2, 1, 0, y, x.T, ACT_LRELU, nullptr, s, 2, 1);   // rows m, m+1   -> y[2m+1]
  return y;
}

// q: quantised latents [B,T,64] channel-last -> decoder output Act3 [B,4T,C]
Act3 run_decoder(ts_engine* e, const VQNet& v, const Act3& q, cudaStream_t s) {
  const bool tc = e->use_tc;   // activations stored split for the tensor-core kernel
  Act3 h = new_act(e, q.B, q.T, 1024, 1, s, tc);
  conv_auto(e, v.aft_vq, q, 1, 1, 0, h, q.T, ACT_NONE, nullptr, s);
  h = run_stack(e, v.d1, h, s, tc);
  h = run_up(e, v.up2e, v.up2o, h, s, tc);
  h = run_stack(e, v.d2, h, s, tc);
  h = run_up(e, v.up3e, v.up3o, h, s, tc);
  h = run_stack(e, v.d3, h, s, tc);
  Act3 y = new_act(e, q.B, h.T, pad4(v.out_dim), 0, s);
  conv_auto(e, v.project, h, 1, 1, 0, y, h.T, ACT_NONE, nullptr, s);
  return y;
}

Act3 run_vq_decode(ts_engine* e, const VQNet& v, const int64_t* idx, int B, int T, cudaStream_t s) {
  Act3 q = new_act(e, B, T, 64, 0, s);
  gather_rows(e, v.codebook, 64, idx, q, s);
  return run_decoder(e, v, q, s);
}

}  // namespace ts

using namespace ts;

extern "C" int ts_latent_rows(int M) {
  int m = (M + 2 - 4) / 2 + 1;
  return (m + 2 - 4) / 2 + 1;
}

extern "C" int ts_load_audioenc(ts_engine* e, const ts_tensor* tensors, int n) {
  TS_API_BEGIN(e)
  Ckpt ck(tensors, n);
  if (!e->conv) e->conv = new ConvStacks();
  LoadScope scope(e, "audioenc");
  Trunk t;
  pack_trunk(e, ck, "", 64, 256, &t);
  e->conv->audio = t;
  e->conv->audio_loaded = true;
  scope.commit();
  TS_API_END(e)
}

extern "C" int ts_load_vq(ts_engine* e, int which, const ts_tensor* tensors, int n) {
  TS_API_BEGIN(e)
  if (which < 0 || which > 1) fail(TS_ERR_INVALID, "ts_load_vq: which must be 0 (body) or 1 (hand)");
  Ckpt ck(tensors, n);
  if (!e->conv) e->conv = new ConvStacks();
  LoadScope scope(e, which ? "vq1" : "vq0");
  VQNet v;
  pack_vq(e, ck, &v);
  e->conv->vq[which] = v;
  scope.commit();
  TS_API_END(e)
}

extern "C" int ts_audio_encode(ts_engine* e, const float* mfcc, float* out, int B, int M, void* stream) {
  TS_API_BEGIN(e)
  ts::require_device(e);
  if (!e->conv || !e->conv->audio_loaded) fail(TS_ERR_NOT_LOADED, "audio encoder weights not loaded");
  if (B <= 0 || M < 4) fail(TS_ERR_INVALID, "ts_audio_encode: B=%d M=%d", B, M);
  cudaStream_t s = (cudaStream_t)stream;
  run_sized(e, [&] {
    Act3 x = new_act(e, B, M, 64, 1, s);
    nct_to_act(e, mfcc, 64, x, s);
    Act3 y = run_trunk(e, e->conv->audio, x, s);
    act_to_nct(e, y, 256, out, s);
  });
  TS_API_END(e)
}

extern "C" int ts_vq_decode(ts_engine* e, int which, const int64_t* idx, float* out, int B, int T, void* stream) {
  TS_API_BEGIN(e)
  ts::require_device(e);
  if (which < 0 || which > 1 || !e->conv || !e->conv->vq[which].loaded) fail(TS_ERR_NOT_LOADED, "vq[%d] weights not loaded", which);
  if (B <= 0 || T <= 0) fail(TS_ERR_INVALID, "ts_vq_decode: B=%d T=%d", B, T);
  cudaStream_t s = (cudaStream_t)stream;
  const VQNet& v = e->conv->vq[which];
  run_sized(e, [&] {
    Act3 y = run_vq_decode(e, v, idx, B, T, s);
    act_to_nct(e, y, v.out_dim, out, s);
  });
  TS_API_END(e)
}

extern "C" int ts_vq_encode(ts_engine* e, int which, const float* poses, int64_t* idx, float* e_out, int B, int F,
                            void* stream) {
  TS_API_BEGIN(e)
  ts::require_device(e);
  if (which < 0 || which > 1 || !e->conv || !e->conv->vq[which].loaded) fail(TS_ERR_NOT_LOADED, "vq[%d] weights not loaded", which);
  if (B <= 0 || F < 4) fail(TS_ERR_INVALID, "ts_vq_encode: B=%d F=%d", B, F);
  cudaStream_t s = (cudaStream_t)stream;
  const VQNet& v = e->conv->vq[which];
  run_sized(e, [&] {
    Act3 x = new_act(e, B, F, pad4(v.out_dim), 1, s);
    btc_to_act(e, poses, v.out_dim, x, s);
    Act3 h = run_trunk(e, v.enc, x, s);
    Act3 z = new_act(e, B, h.T, 64, 0, s);
    conv1d(e, v.pre_vq, h, 1, 1, 0, z, h.T, ACT_NONE, nullptr, s);
    vq_argmin(e, v.codebook, v.ee, v.ncodes, z, idx, s);
    if (e_out) {
      Act3 q = new_act(e, B, h.T, 64, 0, s);
      gather_rows(e, v.codebook, 64, idx, q, s);
      act_to_nct(e, q, 64, e_out, s);
    }
  });
  TS_API_END(e)
}
