/* talkshow_b200 — C ABI of the H100-native (sm_90a) TalkSHOW speech-to-motion engine.
 *
 * The reference (yhw-yhw/TalkSHOW) is pure Python/PyTorch and has no FFI of its own; the boundary
 * this library replaces is the *module level* of nets/spg/ — the calls the wrappers
 * nets/smplx_body_pixel.py, nets/smplx_body_vq.py and nets/smplx_face.py make.  Each entry point
 * below cites the reference call it replaces.  The host-side mirror of the wrappers lives in
 * talkshow_b200/nets/ (ctypes binding: talkshow_b200/_lib.py, see INTEGRATION.md).
 *
 * Conventions
 *  - every function returns 0 (TS_OK) on success, a ts_status otherwise; ts_last_error() gives text;
 *  - all data pointers are DEVICE pointers on the engine's device unless the name says `host`;
 *    tensors are dense, fp32 / int64, in the reference's own layouts (channel-first [B,C,T]);
 *  - caller owns inputs/outputs; the engine owns packed weights + workspace;
 *  - work is enqueued on `stream` (a cudaStream_t passed as void*); no hidden synchronisation;
 *  - one engine per device, not thread-safe.
 */
#ifndef TALKSHOW_B200_H
#define TALKSHOW_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ts_engine ts_engine;

enum ts_status {
  TS_OK = 0,
  TS_ERR_INVALID = 1,    /* bad argument / shape */
  TS_ERR_NOT_LOADED = 2, /* weights for this module were not loaded */
  TS_ERR_MISSING = 3,    /* a checkpoint tensor is missing or has the wrong shape */
  TS_ERR_CUDA = 4,       /* CUDA runtime error */
  TS_ERR_UNSUPPORTED = 5
};

/* One checkpoint tensor, HOST memory, fp32 (dtype 0) or int64 (dtype 1), dense row-major, named
 * exactly as in the reference's state_dict() (SURVEY.md Appendix A) after 'module.' stripping
 * (nets/smplx_body_pixel.py:117-126). */
typedef struct ts_tensor {
  const char* name;
  const void* data;
  int32_t dtype;
  int32_t ndim;
  int64_t shape[6];
} ts_tensor;

int ts_engine_create(ts_engine** out, int device);
void ts_engine_destroy(ts_engine* e);
const char* ts_last_error(ts_engine* e); /* e may be NULL: error of the last failed create */
int ts_engine_sm_count(ts_engine* e);

/* ---- weights: replace nn.Module.load_state_dict for each sub-module ------------------------ */
/* GatedPixelCNN(2048, dim, n_layers, 4, audio=True, bh_model=True): nets/smplx_body_pixel.py:53,
 * keys of ckpt['generator']['generator'].  dim/n_layers are read from the tensor shapes. */
int ts_load_pixelcnn(ts_engine* e, const ts_tensor* tensors, int n);
/* AudioEncoder(64,256,2,256): nets/smplx_body_pixel.py:46, ckpt['generator']['audioencoder']. */
int ts_load_audioenc(ts_engine* e, const ts_tensor* tensors, int n);
/* VQVAE(39|90,64,2048,1024,2,512): nets/smplx_body_pixel.py:54-62, which = 0 g_body, 1 g_hand. */
int ts_load_vq(ts_engine* e, int which, const ts_tensor* tensors, int n);
/* s2g_face.Generator: nets/smplx_face.py:37-45, ckpt['generator']['generator'].  The positional
 * conv must be passed with its effective weight under
 * 'audio_encoder.encoder.pos_conv_embed.conv.weight' [768,48,128] (the host shim resolves the
 * weight_norm parametrisation). */
int ts_load_face(ts_engine* e, const ts_tensor* tensors, int n);

/* ---- hot path ------------------------------------------------------------------------------- */
/* AudioEncoder.forward, nets/spg/vqvae_1d.py:27-34.  mfcc [B,64,M] -> out [B,256,T],
 * T = ts_latent_rows(M). */
int ts_audio_encode(ts_engine* e, const float* mfcc, float* out, int B, int M, void* stream);
int ts_latent_rows(int M);

/* GatedPixelCNN.generate, nets/spg/gated_pixelcnn_v2.py:152-177, as an exact O(T) incremental
 * evaluation.  aud [B,256,T0+T] (the AudioEncoder output, incl. the T0 prefix rows when
 * pre_latents is given, :158-165), label [B] int64, noise [2T,B,2048] = the Exp(1) draws the
 * reference's multinomial would consume, one [B,2048] block per sampled position in the order
 * (i,0),(i,1) (RNG contract, DESIGN.md), pre_latents [B,T0,2] int64 or NULL (T0=0).
 * idx_out [B,T,2] int64.  logits_out (may be NULL) [2T,B,2048]: the logits each draw used.
 * Device data is not range-checked: pre_latents (and `codes` of ts_pixelcnn_logits) must lie in [0,2048) like the
 * indices nn.Embedding accepts; labels outside [0, num_classes) are clamped. */
int ts_pixelcnn_generate(ts_engine* e, const float* aud, const int64_t* label, const float* noise,
                         int64_t* idx_out, float* logits_out, int B, int T, const int64_t* pre_latents, int T0,
                         void* stream);
/* ts_pixelcnn_generate with sampling controls.  Let l be the 2048 raw logits of one draw (what logits_out holds).
 *  - top_k (0 = off, 1..2048): keep code i iff l_i >= v_k, v_k the k-th largest logit counting multiplicity (ties at the
 *    boundary are all kept; TopKLogitsWarper).  The comparison is on the raw logits, whatever the temperature.
 *  - temperature > 0: s = l / temperature (IEEE division), dropped codes -> -inf, then the default draw on s:
 *    argmax(softmax(s) / q) with first-index ties, same noise and RNG contract.  A dropped code is never drawn, even when
 *    every kept probability underflows to 0.  Any finite temperature > 0 is valid: one so small that max l / temperature
 *    overflows (e.g. a subnormal temperature) leaves every tempered probability NaN, and the code is then the greedy one,
 *    the limit of the tempered draw as the temperature goes to 0.  Codes always lie in [0, 2048).
 *  - temperature = 0 (greedy): code = first index of max l.  noise is not read and may be NULL.
 *  - logp_out (may be NULL) [B,T,2], laid out like idx_out: log_softmax(l)[code] of the untempered, untruncated model
 *    (= -nll of ts_pixelcnn_score), computed as (l[code] - max l) - logf(sum exp(l - max l)).  Rows forced by
 *    pre_latents have no entry.
 * temperature 1 with top_k 0 or 2048 gives codes bit-identical to ts_pixelcnn_generate.  The launches are those of
 * ts_pixelcnn_generate.  TS_ERR_INVALID: temperature < 0 or not finite, top_k outside [0, 2048], NULL noise with
 * temperature > 0. */
int ts_pixelcnn_sample(ts_engine* e, const float* aud, const int64_t* label, const float* noise,
                       int64_t* idx_out, float* logits_out, int B, int T, const int64_t* pre_latents, int T0,
                       float temperature, int top_k, float* logp_out, void* stream);
/* The sampling controls as one struct, with nucleus (top-p) and min-p truncation and the size of each draw's keep set.
 * The controls apply in the order temperature -> top_k -> top_p -> min_p.  Let l be the 2048 raw logits of one draw and
 * t = temperature > 0.
 *  1. keep0 = the top_k set of ts_pixelcnn_sample (on the raw logits, ties kept; every code when off).
 *  2. e_i = expf(l_i / t - max(l) / t) for the codes of keep0 and 0 for the others, in fp32 (the most likely code has e = 1).
 *  3. Integer mass w_i = e_i * 2^32 rounded to the nearest integer, ties to even, as uint64; W = sum w_i <= 2^43.  Every
 *     partial sum of masses is exact in uint64 and in a double, and integer addition is associative: the sums below do not
 *     depend on the order in which an implementation adds, so the keep set is the same in every executor, batch tile and
 *     batch.
 *  4. top_p in (0, 1), 1 = off: with A_i = sum { w_j : l_j > l_i } the mass strictly above code i (-0 compares equal to
 *     +0), keep i iff (double)A_i < (double)top_p * (double)W, one IEEE double multiplication.  This is the smallest set
 *     of most likely codes whose mass reaches top_p (TopPLogitsWarper), with the ties at the boundary all kept, like
 *     top_k.  The most likely code is always kept.
 *  5. min_p in (0, 1], 0 = off: keep i iff e_i >= min_p (fp32 comparison): probability at least min_p times that of the
 *     most likely code.  The final keep set is the intersection of 1, 4 and 5.
 *  6. The draw is that of ts_pixelcnn_sample over the final keep set: argmax((e_i / sum of kept e) / q_i), first-index
 *     ties, same noise and RNG contract, the same fallback to the greedy code when every e / q is NaN.  A dropped code
 *     is never drawn.
 *  7. temperature = 0 (greedy) ignores top_p and min_p as it ignores top_k.  logp_out is the log-softmax of the
 *     untempered, untruncated logits, as in ts_pixelcnn_sample.
 *  8. kept_out (may be NULL) [B,T,2] int32, laid out like idx_out: the size of the final keep set of each draw (1 for a
 *     greedy draw).  Rows forced by pre_latents have no entry.
 * With top_p = 1 and min_p = 0 the arithmetic is that of ts_pixelcnn_sample step for step. */
typedef struct ts_sample_ctl {
  float temperature;   /* as ts_pixelcnn_sample */
  int32_t top_k;       /* as ts_pixelcnn_sample */
  float top_p;         /* (0, 1]; 1 = off */
  float min_p;         /* [0, 1]; 0 = off */
  float* logp_out;     /* [B,T,2] or NULL */
  int32_t* kept_out;   /* [B,T,2] or NULL */
} ts_sample_ctl;
/* ts_pixelcnn_sample with the controls of ts_sample_ctl; ts_pixelcnn_sample is this call with top_p = 1, min_p = 0 and
 * kept_out = NULL.  The launches are those of ts_pixelcnn_generate.  TS_ERR_INVALID: ctl NULL, top_p outside (0, 1] or
 * NaN, min_p outside [0, 1] or NaN, and the conditions of ts_pixelcnn_sample. */
int ts_pixelcnn_sample_ctl(ts_engine* e, const float* aud, const int64_t* label, const float* noise, int64_t* idx_out,
                           float* logits_out, int B, int T, const int64_t* pre_latents, int T0,
                           const ts_sample_ctl* ctl, void* stream);
/* ---- seeded sampling: per-clip counter-based noise generated inside the sampler --------------------------------------
 * RNG contract.  The draw at absolute latent row r (rows forced by pre_latents count: a call with T0 prefix rows samples
 * rows T0 .. T0+T-1), column c in {0,1}, code n in [0,2048), of a clip with seed s (int64, used as its 64 bits) divides by
 *     x = Philox4x32-10(counter = (n & 511, r, c, 0), key = (s & 0xffffffff, s >> 32))[n >> 9]
 *     u = (float)((x >> 8) | 1) * 2^-24        an odd multiple of 2^-24: exact in fp32, in [2^-24, 1 - 2^-24]
 *     q = -logf(u)                             > 0, never inf
 * Philox4x32-10 is the Random123 / cuRAND generator (multipliers 0xD2511F53, 0xCD9E8D57; key increments 0x9E3779B9,
 * 0xBB67AE85).  A clip's noise depends only on its seed and the absolute position of the draw: not on B, T, the clip's
 * place in the batch, the executor or how the clip is split into chunks.  The draw itself (argmax(p / q), every
 * sampling control) is unchanged.
 *
 * The Exp(1) values of the seeded sampler in the layout of `noise` of ts_pixelcnn_generate: seeds [B] (device),
 * noise_out [2T,B,2048], block 2(r-T0)+c holds row r in [T0, T0+T).  One launch.  TS_ERR_INVALID: B, T <= 0, T0 < 0,
 * 2TB >= 2^31, NULL seeds or noise_out. */
int ts_sampler_noise(ts_engine* e, const int64_t* seeds, float* noise_out, int B, int T, int T0, void* stream);
/* ts_pixelcnn_sample_ctl with seeds [B] (device, int64) in place of noise: there is no noise tensor.  ctl may be NULL: the
 * default draw of ts_pixelcnn_generate.  Equivalences: with ctl, the call equals ts_pixelcnn_sample_ctl(noise =
 * ts_sampler_noise(seeds, B, T, T0)) bit for bit (codes, logits_out, logp_out, kept_out); with ctl = NULL it equals
 * ts_pixelcnn_generate on that noise.  The launches are those of ts_pixelcnn_generate (no extra kernel, no noise buffer).
 * seeds may be NULL only for greedy decoding (ctl->temperature = 0); otherwise TS_ERR_INVALID, like the conditions of
 * ts_pixelcnn_sample_ctl. */
int ts_pixelcnn_sample_seeded(ts_engine* e, const float* aud, const int64_t* label, const int64_t* seeds, int64_t* idx_out,
                              float* logits_out, int B, int T, const int64_t* pre_latents, int T0,
                              const ts_sample_ctl* ctl, void* stream);
/* ---- anchored sampling: pin chosen draws to given codes, sample the rest --------------------------------------------
 * anchors [B,T,2] int64 (device), laid out like idx_out over the sampled rows: with pre_latents, anchor row i is absolute
 * row T0+i.  Per draw (clip, row, column):
 *  - a value a in [0, 2048) PINS the draw: its code is a.  The code is written to idx_out, gathered into the embedding
 *    like a drawn code and conditions every later draw.
 *  - -1 samples the draw exactly as the call without anchors would (its noise or seeds, its controls).
 *  - any other value is treated as -1 by the kernel, so malformed device data never reaches the embedding gather (the
 *    Python layer rejects such values before the call).
 *  - A pinned draw reads no noise.  noise keeps its [2T,B,2048] shape (a pinned draw's block is not used); seeded noise is
 *    keyed by the absolute (row, column) as before.  Either way no sampled draw's noise changes.
 *  - logp_out of a pinned draw: (l[a] - max l) - logf(sum exp(l - max l)) on its raw logits, the arithmetic and reduction
 *    order of a sampled draw's logp (pinning a draw to the code it draws gives the same bits).  kept_out is 0 for a pinned
 *    draw.  logits_out is written as usual.
 *  - The prior is causal: a pinned code conditions the later draws only (later rows, and column 1 of its own row when it
 *    is in column 0).  This is not bidirectional infilling: nothing before a pinned draw depends on it.
 * An anchored call runs the kernels of ts_pixelcnn_sample_ctl (with ctl = NULL at temperature 1, top_k 0: the default
 * draw's codes) with the launches of ts_pixelcnn_generate.  Exactly one of noise and seeds must be given unless ctl is
 * greedy (temperature 0), even when every draw is pinned; otherwise TS_ERR_INVALID.  ctl may be NULL.  anchors = NULL:
 * the call makes the launches of, and equals bit for bit, ts_pixelcnn_generate (noise, ctl NULL),
 * ts_pixelcnn_sample_ctl (noise, ctl) or ts_pixelcnn_sample_seeded (seeds, ctl). */
int ts_pixelcnn_sample_anchored(ts_engine* e, const float* aud, const int64_t* label, const float* noise, const int64_t* seeds,
                                const int64_t* anchors, int64_t* idx_out, float* logits_out, int B, int T,
                                const int64_t* pre_latents, int T0, const ts_sample_ctl* ctl, void* stream);
/* ---- styled sampling: per-row mixtures of the speaker embeddings ----------------------------------------------------
 * style [B, Ttot, ncls] float32 (device), Ttot = T0 + T: every latent row the network sees, the pre_latents prefix
 * included.  Row r of clip b holds the speaker weights w[b,r,0..ncls) of every position (row r, columns 0 and 1) of every
 * layer.  At a gate of layer l, channel ch, position (b, r, .) the class term E_l[label[b]][ch] is replaced by
 *     acc = w0 * E_l[0][ch];  acc = acc + w_s * E_l[s][ch]  for s = 1 .. ncls-1,
 * every product and every sum rounded to fp32 with no FMA contraction (__fmul_rn / __fadd_rn).  A one-hot row gives
 * exactly E_l[s][ch] (up to the sign of a zero), so a one-hot schedule of class s equals the call labelled s bit for bit.
 *  - Weights are used as given: the kernel neither normalises nor checks them (every code stays in [0, 2048) whatever the
 *    logits).  The Python layer rejects non-finite or negative weights, rows whose sum differs from 1 by more than 1e-5
 *    and wrong shapes before any launch: only convex mixtures of the trained embeddings are offered.
 *  - With style, label is not read and may be NULL.  ncls must equal the loaded prior's class count and be at most 16,
 *    otherwise TS_ERR_INVALID (every shipped config has 4).  Without style, label is required.
 *  - The prior stays causal: a draw at row r depends only on the style rows <= r.
 * A styled call runs the kernels of an anchored call (noise, seeds, anchors and ctl keep their contracts) with its
 * launches.  style = NULL: the call equals ts_pixelcnn_sample_anchored bit for bit, with the same launches, and ncls is
 * not read. */
int ts_pixelcnn_sample_styled(ts_engine* e, const float* aud, const int64_t* label, const float* style, int ncls,
                              const float* noise, const int64_t* seeds, const int64_t* anchors, int64_t* idx_out,
                              float* logits_out, int B, int T, const int64_t* pre_latents, int T0, const ts_sample_ctl* ctl,
                              void* stream);
/* ---- per-clip sampling controls: each clip of a batch with its own temperature, top_k, top_p and min_p ----------------
 * One entry per clip: the four controls of ts_sample_ctl, with their ranges and their meaning. */
typedef struct ts_clip_ctl {
  float temperature;   /* >= 0, finite; 0 = greedy */
  int32_t top_k;       /* [0, 2048]; 0 or 2048 = off */
  float top_p;         /* (0, 1]; 1 = off */
  float min_p;         /* [0, 1]; 0 = off */
} ts_clip_ctl;
/* ts_pixelcnn_sample_styled where clip b draws with clip_ctl[b] in place of ctl's four controls.
 *  - clip_ctl [B] is HOST memory.  Every entry is checked on the host with the rules of ts_sample_ctl before any launch
 *    (TS_ERR_INVALID, the message names the clip), then the entries are copied to engine-owned device memory on `stream`
 *    (the caller's array may be reused when the call returns; no synchronisation).
 *  - ctl (may be NULL) supplies logp_out and kept_out only; its temperature, top_k, top_p and min_p are not read.
 *  - Clip b's codes, logp_out and kept_out equal bit for bit those of clip b run alone through ts_pixelcnn_sample_styled
 *    with ctl = clip_ctl[b] (the same noise column or seed, anchors, style rows and pre_latents): the logits of a clip do
 *    not depend on the batch, and the draw reads only the clip's own controls.
 *  - A greedy clip (temperature 0) reads no noise; noise keeps its [2T,B,2048] shape.  Exactly one of noise and seeds
 *    must be given when any clip has temperature > 0; neither is needed when every clip is greedy.
 * The call runs the kernels and launches of ts_pixelcnn_sample_styled (no extra kernel: one host-to-device copy).
 * clip_ctl = NULL: the call equals ts_pixelcnn_sample_styled with the same arguments, bit for bit and with its launches. */
int ts_pixelcnn_sample_clips(ts_engine* e, const float* aud, const int64_t* label, const float* style, int ncls,
                             const float* noise, const int64_t* seeds, const int64_t* anchors, int64_t* idx_out,
                             float* logits_out, int B, int T, const int64_t* pre_latents, int T0, const ts_sample_ctl* ctl,
                             const ts_clip_ctl* clip_ctl, void* stream);
/* ---- logit shaping: a repetition penalty over each clip's recent codes and an additive per-code bias ----------------
 * One entry per clip (clip_shape, HOST memory): */
typedef struct ts_clip_shape {
  float repetition_penalty;   /* theta: finite, >= 1; 1 = off */
  int32_t repetition_window;  /* W >= 1 latent rows */
} ts_clip_shape;
/* ts_pixelcnn_sample_clips where the raw logits l of every sampled draw are shaped before the controls act.
 * code_bias [B,2,2048] (DEVICE, may be NULL): one row per clip and column (0 = body codebook, 1 = hand codebook); each value
 * finite with |v| <= 1e4, or -inf, and each row with at least one finite value (the kernel survives any data: a row of
 * -inf draws code 0, the first-index argmax).  For the draw at absolute latent row r (pre_latents rows included), column
 * c, of clip b:
 *  1. Penalty.  H = the codes at column c in rows max(0, r - W) .. r - 1 of clip b: pre_latents rows and pinned draws
 *     included, column 1 of row r not seen by column 0 nor the other way.  Every code n in H (once, however often it
 *     occurs) gets l_n = l_n > 0 ? l_n / theta : l_n * theta, IEEE fp32, no contraction.
 *  2. Bias.  l_n = l_n + bias[b][c][n] (fp32 add, round to nearest).
 *  3. The controls of ts_pixelcnn_sample_clips (temperature, top_k, top_p, min_p, the argmax(p / q) draw, greedy as the
 *     first-index argmax, the overflow fallback) act on the shaped logits.
 *  4. A code whose shaped logit is -inf is never drawn and is not counted in kept_out.
 *  5. logp_out is still the log-probability under the raw (untempered, unshaped) prior, as in every sampling call.
 *  6. A pinned draw (anchors) is not shaped: its log p and kept_out = 0 are unchanged; its code enters later histories.
 * clip_shape [B] (HOST, may be NULL = theta 1 for every clip) is checked on the host (TS_ERR_INVALID, the message names
 * the clip) and copied to engine-owned device memory on `stream` with no synchronisation.  theta = 1 and no bias: the
 * clip draws what ts_pixelcnn_sample_clips draws, bit for bit.  clip_ctl = NULL: ctl's scalar controls (or the default
 * draw when ctl is NULL too).  Both clip_shape and code_bias NULL: the call equals ts_pixelcnn_sample_clips with the same
 * arguments, bit for bit and with its launches; otherwise it runs that call's kernels (one extra host-to-device copy). */
int ts_pixelcnn_sample_shaped(ts_engine* e, const float* aud, const int64_t* label, const float* style, int ncls,
                              const float* noise, const int64_t* seeds, const int64_t* anchors, int64_t* idx_out,
                              float* logits_out, int B, int T, const int64_t* pre_latents, int T0, const ts_sample_ctl* ctl,
                              const ts_clip_ctl* clip_ctl, const ts_clip_shape* clip_shape, const float* code_bias,
                              void* stream);
/* ---- guided sampling: each draw pushed away from a negative conditioning ------------------------------------------------
 * A guided call has P pairs.  Pair p has two branches: branch 2p is the clip (conditional), branch 2p + 1 its negative
 * conditioning (silence, another speaker, a style blend: the prior was trained without condition dropout, so this is
 * contrastive guidance, not classifier-free guidance against a learned unconditional model).
 *  - Conditioning is per branch (2P rows): aud [2P,256,T0+T], label [2P], style [2P,T0+T,ncls].
 *  - Draw inputs are per pair (P rows): noise [2T,P,2048] or seeds [P], clip_ctl [P], clip_shape [P], code_bias [P,2,2048],
 *    anchors [P,T,2], pre_latents [P,T0,2] (motion, fed to both branches) and guidance [P] (HOST memory).
 *  - Outputs are per branch (2P rows): idx_out [2P,T,2], logits_out [2T,2P,2048], ctl->logp_out / ctl->kept_out [2P,T,2].
 * For the draw at row r, column c of pair p:
 *  1. l_c, l_u = the raw logits of branches 2p and 2p + 1; with s = w_p - 1 (fp32 subtraction),
 *     g_n = l_c,n + s * (l_c,n - l_u,n) as three separately rounded fp32 operations (subtract, multiply, add; no
 *     contraction).  At w = 1, g = l_c (up to the sign of a zero, which the draw does not see).
 *  2. The pair's shaping (ts_pixelcnn_sample_shaped: penalty over the pair's history, then the bias) acts on g, then the
 *     pair's controls (temperature, top_k, top_p, min_p, greedy, the overflow fallback) with the pair's noise or seed.
 *  3. Both branches write the code to their idx_out rows and feed it to their own next rows: later draws of both branches
 *     see the guided code.
 *  4. logp_out of each branch is the log p of the code under that branch's raw prior (branch 2p: the conditional log p of
 *     every sampling call; branch 2p + 1: the negative one).  kept_out is the guided keep-set size, equal in both rows.
 *  5. A pinned draw (anchors[p]) pins both branches and is not guided.
 *  6. w must be finite and in [0, TS_GUIDANCE_MAX] (TS_ERR_INVALID, the message names the pair).  Whatever the logits,
 *     the code lies in [0, 2048).
 * Contract: a pair with w = 1 draws, bit for bit, the codes, conditional log p and kept sizes of ts_pixelcnn_sample_shaped
 * run on its conditional branch alone with the same draw inputs; a pair's results do not depend on the other pairs; a
 * seeded pair's q is keyed by (seed, row, column, code) as in ts_pixelcnn_sample_seeded.  The grid-wide executor takes at
 * most 64 branches (32 pairs) per call; the cluster executor any number.  TS_ERR_INVALID: P < 1, guidance NULL or a bad
 * w, or anything ts_pixelcnn_sample_shaped refuses. */
#define TS_GUIDANCE_MAX 100.0f
int ts_pixelcnn_sample_guided(ts_engine* e, const float* aud, const int64_t* label, const float* style, int ncls,
                              const float* noise, const int64_t* seeds, const int64_t* anchors, int64_t* idx_out,
                              float* logits_out, int P, int T, const int64_t* pre_latents, int T0, const ts_sample_ctl* ctl,
                              const ts_clip_ctl* clip_ctl, const ts_clip_shape* clip_shape, const float* code_bias,
                              const float* guidance, void* stream);
/* GatedPixelCNN.forward (teacher forced), :130-150, for rows [0,T): logits_out [B,2048,T,2]. */
int ts_pixelcnn_logits(ts_engine* e, const float* aud, const int64_t* label, const int64_t* codes,
                       float* logits_out, int B, int T, void* stream);
/* Teacher-forced GatedPixelCNN.forward (:130-150) over all rows at once + per-position cross-entropy
 * (nets/smplx_body_pixel.py:207-216 without the update).  aud [B,256,T], label [B], codes [B,T,2] int64 ->
 * nll_out [B,T,2] = -log softmax(logits)[code]; logits_out (may be NULL) [B,2048,T,2].  Any B, any T >= 1.
 * No serial dependency: a fixed number of launches (large GEMMs over all B*T*2 positions) whatever T is.
 * Dense layers run on the kernel ts_set_tensor_cores selects. */
int ts_pixelcnn_score(ts_engine* e, const float* aud, const int64_t* label, const int64_t* codes,
                      float* nll_out, float* logits_out, int B, int T, void* stream);
/* ts_pixelcnn_score under a style schedule [B,T,ncls] (the rule of ts_pixelcnn_sample_styled: the gates of row t blend row
 * t's weights, label is not read).  style = NULL equals ts_pixelcnn_score. */
int ts_pixelcnn_score_styled(ts_engine* e, const float* aud, const int64_t* label, const float* style, int ncls,
                             const int64_t* codes, float* nll_out, float* logits_out, int B, int T, void* stream);

/* VQVAE.decode(latents=...), nets/spg/vqvae_1d.py:201-208: idx [B,T] int64 -> out [B,C,4T]
 * (C = ts_vq_dim(which): 39 body / 90 hand, 78 / 180 for 6-D).  The indices are device data and are NOT range-checked (the
 * reference's F.embedding raises IndexError): every idx must lie in [0, num_embeddings) of the loaded codebook. */
int ts_vq_decode(ts_engine* e, int which, const int64_t* idx, float* out, int B, int T, void* stream);
/* VQVAE.encode, :196-199: poses [B,F,C] -> idx [B,T] int64 (T=F/4), e_out (may be NULL) [B,64,T].
 * Each index is the argmin over codes n of the fp32 distance (|z|^2 + |e_n|^2) - 2 z.e_n with torch.argmin's rule: the
 * lowest code among equal distances, and a latent row with a NaN distance gets the first such code, as torch.argmin
 * does.  Every index lies in [0, num_embeddings) whatever the poses hold. */
int ts_vq_encode(ts_engine* e, int which, const float* poses, int64_t* idx, float* e_out, int B, int F,
                 void* stream);

/* s2g_face.Generator.forward, nets/spg/s2g_face.py:196-224: wave [B,N] (16 kHz), id [B,4] float
 * one-hot (zeros = "no id", nets/smplx_face.py:205-206) -> out [B,frame,ts_face_dim(e)].
 * The net's geometry is read from the checkpoint by ts_load_face: with 'audio_middle.id_mlp.*' it is the identity net
 * (3-D jaw, 103 columns); without, the identity-free net of convert_to_6d configs (AudioEncoder identity=False, 6-D jaw,
 * 106 columns), which ignores `id` (it may be NULL). */
int ts_face_forward(ts_engine* e, const float* wave, const float* id, float* out, int B, int N, int frame,
                    void* stream);

/* ---- held-out scoring: the forward half of the reference's training steps, losses kept per clip ---------------
 * Reductions run in a fixed order without atomics (repeated calls give the same bits): elementwise terms in fp32 as the
 * reference forms them, accumulated in fp64; clip_out is fp64.
 *
 * VQVAE of s2g_body_vq.vq_train + get_loss (nets/smplx_body_vq.py:155-206) in eval mode: poses [B,F,C] (C = ts_vq_dim)
 * -> encoder + argmin (idx_out [B,T], T = F/4, bit-identical to ts_vq_encode, whose argmin rule applies: a latent row
 * with a NaN distance gets the first such code, as torch.argmin does) -> decoder on the quantised embeddings
 * (recon_out, may be NULL, [B,F,C], bit-identical to ts_vq_decode of those indices, transposed) and per clip
 * clip_out [B,3] = { sum |recon - gt| over (F,C), sum |d recon - d gt| over (F-1,C) (d = frame-to-frame difference),
 * sum ||z - e[idx]||^2 over the T latent rows (z = encoder output before quantisation) }.
 * F must be a positive multiple of 4 (otherwise TS_ERR_INVALID: the reference fails on the recon / gt shape mismatch). */
int ts_vq_score(ts_engine* e, int which, const float* poses, int64_t* idx_out, float* recon_out, double* clip_out, int B,
                int F, void* stream);
/* s2g_face.__call__ + get_loss (nets/smplx_face.py:95-167) in eval mode, frame = F: the ts_face_forward computation
 * (pred_out, may be NULL, [B,F,ts_face_dim], bit-identical to it) against gt [B,F,Cgt] (Cgt >= 100: pose columns then
 * the 100 expression columns) -> clip_out [B,2] = { sum |pred[:,:,:6] - gt[:,:,:6]|, sum (pred[:,:,-100:] - gt[:,:,-100:])^2 }.
 * Either net: id [B,4] is required by the identity net (103 columns) and may be NULL for the identity-free one (106). */
int ts_face_score(ts_engine* e, const float* wave, const float* id, const float* gt, int Cgt, float* pred_out,
                  double* clip_out, int B, int N, int F, void* stream);

/* output columns of the loaded face net: 103 (jaw 3 + expression 100) or 106 (6-D jaw 6 + expression 100);
 * 0 when no face is loaded. */
int ts_face_dim(ts_engine* e);

/* pose channels of the loaded VQ-VAE `which` (in_dim of nets/smplx_body_pixel.py:54-57: 39 / 90 axis-angle,
 * 78 / 180 with convert_to_6d); 0 when not loaded. */
int ts_vq_dim(ts_engine* e, int which);

/* s2g_body_pixel.infer_on_audio core, nets/smplx_body_pixel.py:270-285, fused:
 * mfcc [B,64,M] -> codes [B,T,2] (may be NULL), poses [B,4T,C] with C = ts_vq_dim(0) + ts_vq_dim(1)
 * (body 39 + hand 90 = 129; 258 for the 6-D configs). */
int ts_body_generate(ts_engine* e, const float* mfcc, const int64_t* label, const float* noise, int64_t* codes,
                     float* poses, int B, int M, void* stream);
/* ts_body_generate with the sampling controls of ts_pixelcnn_sample (same semantics, same error statuses):
 * temperature, top_k, logp_out [B,T,2] (may be NULL); noise may be NULL when temperature = 0. */
int ts_body_sample(ts_engine* e, const float* mfcc, const int64_t* label, const float* noise, int64_t* codes,
                   float* poses, int B, int M, float temperature, int top_k, float* logp_out, void* stream);
/* ts_body_generate with the controls of ts_pixelcnn_sample_ctl, same semantics and same error statuses;
 * ts_body_sample is this call with top_p = 1, min_p = 0 and kept_out = NULL. */
int ts_body_sample_ctl(ts_engine* e, const float* mfcc, const int64_t* label, const float* noise, int64_t* codes,
                       float* poses, int B, int M, const ts_sample_ctl* ctl, void* stream);
/* ts_body_sample_ctl with seeds [B] (device) in place of noise, the RNG contract of ts_pixelcnn_sample_seeded; ctl may be
 * NULL (the default draw of ts_body_generate).  Same launches as ts_body_generate; seeds may be NULL only for greedy
 * decoding (TS_ERR_INVALID otherwise). */
int ts_body_sample_seeded(ts_engine* e, const float* mfcc, const int64_t* label, const int64_t* seeds, int64_t* codes,
                          float* poses, int B, int M, const ts_sample_ctl* ctl, void* stream);
/* ts_body_generate with the anchors of ts_pixelcnn_sample_anchored ([B,T,2], T = ts_latent_rows(M)); the poses are decoded
 * from the resulting codes, pinned or drawn.  Same noise / seeds / ctl rules; anchors = NULL equals ts_body_generate,
 * ts_body_sample_ctl or ts_body_sample_seeded. */
int ts_body_sample_anchored(ts_engine* e, const float* mfcc, const int64_t* label, const float* noise, const int64_t* seeds,
                            const int64_t* anchors, int64_t* codes, float* poses, int B, int M, const ts_sample_ctl* ctl,
                            void* stream);
/* ts_body_sample_anchored under a style schedule [B,T,ncls] (T = ts_latent_rows(M); the rule of
 * ts_pixelcnn_sample_styled, label may be NULL).  style = NULL equals ts_body_sample_anchored. */
int ts_body_sample_styled(ts_engine* e, const float* mfcc, const int64_t* label, const float* style, int ncls,
                          const float* noise, const int64_t* seeds, const int64_t* anchors, int64_t* codes, float* poses,
                          int B, int M, const ts_sample_ctl* ctl, void* stream);
/* ts_body_sample_styled with the per-clip controls of ts_pixelcnn_sample_clips (clip_ctl [B] in host memory, ctl for
 * logp_out / kept_out only); the poses decode each clip's codes.  clip_ctl = NULL equals ts_body_sample_styled. */
int ts_body_sample_clips(ts_engine* e, const float* mfcc, const int64_t* label, const float* style, int ncls,
                         const float* noise, const int64_t* seeds, const int64_t* anchors, int64_t* codes, float* poses,
                         int B, int M, const ts_sample_ctl* ctl, const ts_clip_ctl* clip_ctl, void* stream);
/* ts_body_sample_clips with the logit shaping of ts_pixelcnn_sample_shaped (clip_shape [B] in host memory, code_bias
 * [B,2,2048] on the device); the poses decode each clip's codes.  Both NULL equals ts_body_sample_clips. */
int ts_body_sample_shaped(ts_engine* e, const float* mfcc, const int64_t* label, const float* style, int ncls,
                          const float* noise, const int64_t* seeds, const int64_t* anchors, int64_t* codes, float* poses,
                          int B, int M, const ts_sample_ctl* ctl, const ts_clip_ctl* clip_ctl,
                          const ts_clip_shape* clip_shape, const float* code_bias, void* stream);
/* ts_body_sample_shaped under the guidance of ts_pixelcnn_sample_guided: mfcc [2P,64,M], label / style per branch, every
 * draw input per pair, guidance [P] (HOST).  codes [2P,T,2] (may be NULL) gets every branch's codes (both rows of a pair
 * equal); poses [P,4T,C] decodes the conditional branches only. */
int ts_body_sample_guided(ts_engine* e, const float* mfcc, const int64_t* label, const float* style, int ncls,
                          const float* noise, const int64_t* seeds, const int64_t* anchors, int64_t* codes, float* poses,
                          int P, int M, const ts_sample_ctl* ctl, const ts_clip_ctl* clip_ctl,
                          const ts_clip_shape* clip_shape, const float* code_bias, const float* guidance, void* stream);

/* Audio front-end of get_mfcc_ta, data_utils/utils.py:148-177 (SURVEY.md §8f-1): wave [B,N] mono at
 * `sr` Hz -> torchaudio Resample(sr, 22000) -> MFCC(64 coefficients, n_fft 2048, hop 734 = 30 fps, 256 HTK
 * mels, top_db 80, DCT-II ortho) -> out [B,64,M], M = ts_mfcc_frames(N, sr). */
int ts_mfcc(ts_engine* e, const float* wave, float* out, int B, int N, int sr, void* stream);
int ts_mfcc_frames(int N, int sr);

/* scripts/demo.py:182-229 + data_utils/lower_body.py:68-87 (part2full): face [B,Ff,103],
 * body [B,Fb,129] -> out [B,Ff,265]; body is padded with its last frame / truncated to Ff. */
int ts_assemble_pose(ts_engine* e, const float* face, const float* body, float* out, int B, int Ff, int Fb,
                     int stand, void* stream);

/* The convert_to_6d form of ts_assemble_pose: face [B,Ff,106] (6-D jaw | expression), body [B,Fb,258] (43 joints x 6-D)
 * -> out [B,Ff,265].  Each jaw / body joint is converted to axis-angle inside the assembly kernel with the arithmetic of
 * ts_rot6d_to_axis_angle, so the result equals ts_rot6d_to_axis_angle followed by ts_assemble_pose bit for bit. */
int ts_assemble_pose6d(ts_engine* e, const float* face, const float* body, float* out, int B, int Ff, int Fb,
                       int stand, void* stream);

/* scripts/demo.py:185-188,216-219 (convert_to_6d configs): matrix_to_axis_angle(rotation_6d_to_matrix(x)),
 * data_utils/rotation_conversion.py:512-533,433-447.  d6 [n,6] -> aa [n,3] (device pointers). */
int ts_rot6d_to_axis_angle(ts_engine* e, const float* d6, float* aa, int64_t n, void* stream);

/* ---- multi-GPU: the single collective of the path (SURVEY.md §8b / §8e) ------------------------------
 * The reference generates diversity samples / clips in a Python loop (scripts/demo.py:195-204); here they are sharded
 * one process per GPU and the [b,F,265] pose shards are all-gathered ONCE over NCCL (NVLink / NVSwitch).  NCCL is
 * dlopen'ed (libnccl_path: e.g. torch's nvidia/nccl/lib/libnccl.so.2; NULL = "libnccl.so.2" from the loader path).
 * Bootstrap: rank 0 calls ts_nccl_unique_id, ships the 128 bytes to the other ranks, every rank calls ts_nccl_init. */
int ts_nccl_unique_id(ts_engine* e, const char* libnccl_path, void* id128_host);
int ts_nccl_init(ts_engine* e, const char* libnccl_path, const void* id128_host, int rank, int world);
/* out[world*count] = concat over ranks of in[count] (fp32 device pointers), on `stream`. */
int ts_allgather(ts_engine* e, const float* in, float* out, int64_t count, void* stream);

/* ---- batched SMPL-X evaluation (SURVEY.md §8 f4) ---------------------------------------------------
 * Replaces the per-frame smplx_model(...) calls of scripts/demo.py:122-152 (get_vertices) and data_utils/get_j.py:20-51
 * (get_joints): smplx 0.1.28 SMPLX.forward + lbs (use_pca=False, flat_hand_mean=False, 300 betas, 100 expression
 * coefficients, static face landmarks) for F frames per call, fp32.  Model tensors (host, fp32 / int64), named as in
 * oracle/smplx_oracle.py: v_template [V,3], shapedirs [V,3,400], posedirs [486,3V], J_regressor [55,V], lbs_weights [V,55],
 * pose_mean [165], parents [55], faces [Fc,3], lmk_faces_idx [L], lmk_bary_coords [L,3], extra_joint_idx [E]. */
int ts_load_smplx(ts_engine* e, const ts_tensor* tensors, int n);
int ts_smplx_dims(ts_engine* e, int* V, int* njoints);
/* poses [F,265] in the reference's argument layout (jaw | leye | reye | global | body | lhand | rhand | expression,
 * demo.py:129-138), betas [300] or NULL (zeros, demo.py:159) -> vertices [F,V,3] (may be NULL), joints
 * [F,55+E+L,3] (may be NULL); use_expression = 0 evaluates with zero expression (get_vertices(exp=False)). */
int ts_smplx_forward(ts_engine* e, const float* poses, const float* betas, int use_expression, float* vertices,
                     float* joints, int F, void* stream);

/* ---- introspection (tests / bench) ---------------------------------------------------------- */
/* number of kernel launches issued by this engine since creation */
int64_t ts_launch_count(ts_engine* e);
/* device time of the last ts_pixelcnn_generate persistent-kernel launch is measured by the caller
 * with events; this returns the algorithmic weight bytes one latent row touches (DESIGN.md). */
int64_t ts_pixelcnn_row_bytes(ts_engine* e);
/* bytes the kernel actually stages per row (packed blob incl. row padding / per-column duplication) */
int64_t ts_pixelcnn_staged_row_bytes(ts_engine* e);
/* enable CUDA-event timing around the persistent kernel (events on its launch stream) and read the
 * duration of the most recent launch in ms (synchronises on the end event; -1 if none). */
int ts_pixelcnn_timing(ts_engine* e, int enable);
double ts_pixelcnn_last_ms(ts_engine* e);
/* Export the PixelCNN execution plan (stage table + packed weight blob) to host buffers so a test
 * can interpret it on the CPU; sizes are returned when the buffers are NULL. */
int ts_debug_pixelcnn_plan(ts_engine* e, int32_t* table, int64_t* table_len, float* blob, int64_t* blob_len);
/* One Conv1d layer through one dense kernel, built as the nets build it (unit tests): production activation layouts and
 * operand splits (including the per-layer fp16 weight scale), and no fall-back between kernels.
 *   y(b, t * y_tmul + y_toff, coff + n) = act( sum_{c, j} W[n][c][j] x(b, t * stride + j - pd, c) + bias[n] + res(b, t, n) )
 * for t < T_out.  x [B,T,C] and res [B,T_out,N] (or NULL) are device fp32; W_host [N,C,k] (torch Conv1d layout) and
 * bias_host [N] (or NULL) are host fp32.  x is staged in an activation with x_pad zero rows before and after every item
 * and x_tail rows after those (filled with NaN in every plane: no conv reads them), res in one with res_pad zero rows.
 * y, y_plane_hi and y_plane_lo are the whole padded output [B, 2 y_pad + y_T, y_C]: their contents are copied in before
 * the conv and copied back after it, so rows and columns the conv must not write keep what the caller put there.
 *   mode 0 FFMA gemm_kernel, 1 wgmma 3xTF32, 6 wgmma fp16-split (the numbering of ts_set_tensor_cores);
 *   y_split: the output is also stored split in the mode's format -- modes 0 / 1: fp32 hi / lo planes (y unused, may be
 *     NULL), mode 6: fp16 planes (uint16) beside the full fp32 value in y;
 *   res_split: the residual is stored split in the mode's format;
 *   planes_only (mode 6): bit 0 the input, bit 1 the output has fp16 planes only, no fp32 copy (y unused);
 *   chunk: wgmma k-blocks accumulated before each round-to-nearest add (0 = production, K = 256).
 * Returns TS_ERR_INVALID, before any launch, for a geometry the mode's kernel does not run (modes 1 / 6: C a multiple of
 * the k-block of 32 / 64 values, rows per item and x_pad - pd multiples of the stride, y_C and coff multiples of 4).
 * The engine's ts_set_tensor_cores setting is unchanged afterwards. */
typedef struct ts_debug_conv {
  int32_t mode;
  int32_t B, T, C, x_pad, x_tail;
  int32_t N, k, stride, pd, T_out, act;  /* act: 0 none, 1 ReLU, 2 LeakyReLU(0.2), 3 GELU (erf) */
  int32_t y_T, y_C, y_pad, y_tmul, y_toff, coff;
  int32_t y_split;
  int32_t res_pad, res_split;
  int32_t chunk;
  int32_t planes_only;
} ts_debug_conv;
int ts_debug_conv1d(ts_engine* e, const ts_debug_conv* a, const float* x, const float* W_host, const float* bias_host,
                    const float* res, float* y, void* y_plane_hi, void* y_plane_lo, void* stream);
/* The face regressor's self-attention through one kernel (unit tests), as the face forward runs it: 12 heads of 64,
 *   out(b, t, 64 h + d) = sum_j softmax_j(q(b, t, h) . k(b, j, h) / 8) v(b, j, h)[d]
 * with qkv [B,T,2304] device fp32 in the layout of the fused projection, rows [q(768) | k(768) | v(768)], head h at
 * columns 64 h of each block.  qkv is staged in the workspace with 64 NaN rows after the last item (no kernel reads them).
 *   kernel: -1 the one the face forward runs for T frames (TS_ATT_MMA, default: 3 up to 384 frames, 4 beyond), 0 FFMA
 *     attention_kernel (T <= 3136), 1 tf32 3xTF32 attention_mma_kernel, 2 fp16-split attention_mma16_kernel,
 *     3 attention_mma16p_kernel (K / V resident, split once per CTA; 1, 2 and 3 hold T <= 384), 4 attention_mma16t_kernel
 *     (K / V staged `chunk` keys at a time, any T);
 *   chunk: kernel 4 only, a multiple of 64 in [64, 384]; 0 = the face forward's 320;
 *   out_format: 0 fp32 in out; 1 the 3xTF32 (hi, lo) pair of ts_set_tensor_cores(e, 1) in plane_hi / plane_lo (fp32,
 *     out unused, may be NULL); 2 (kernels 3 and 4, the default mode 6) fp32 in out plus its fp16 planes
 *     h = fp16(o), l = fp16(o - h) (uint16) in plane_hi / plane_lo.
 * Output buffers are [B,T,768]; their contents are copied in before the kernel and back after it.
 * Input contract of the fp16-split kernels (2, 3, 4): |q| / 8, |k| and |v| below 65504; every operand is carried to 22
 * significant bits only while its low fp16 plane is normal -- values below about 2^-3 pay an absolute error of up to
 * 2^-25, and below 2^-14 the high plane itself is subnormal.  Kernels 3 and 4 give the same bits at every T kernel 3 holds.
 * Returns TS_ERR_INVALID, before any launch, for a kernel that cannot hold T, a chunk off the grid above, or format 2 on
 * kernels 0 - 2.  The engine's ts_set_tensor_cores setting is unchanged afterwards. */
typedef struct ts_debug_att {
  int32_t kernel, B, T, chunk, out_format;
} ts_debug_att;
int ts_debug_attention(ts_engine* e, const ts_debug_att* a, const float* qkv, float* out, void* plane_hi, void* plane_lo,
                       void* stream);
/* The face regressor's positional conv (pos_conv_embed: Conv1d(768, 768, 128, padding 64, groups 16), last output
 * dropped, then erf-GELU) through one kernel (unit tests): x [B,T,768] device fp32, staged with the face forward's 64 zero
 * rows before and after every item; W_host [768,48,128] (torch layout) and bias_host [768] host fp32, packed as
 * ts_load_face packs them; y [B,T,768] device fp32, copied in before the kernel and back after it.
 *   mode 6 or 1: posconv_mma_kernel (fp16-split HMMA, weights pre-split and scaled per layer); 0: the FFMA GEMM with one
 *   grid slice per group.
 * The engine's ts_set_tensor_cores setting is unchanged afterwards. */
int ts_debug_posconv(ts_engine* e, int mode, const float* x, const float* W_host, const float* bias_host, float* y, int B,
                     int T, void* stream);
/* The four debug entries below share the conventions of the three above: sizes and pointers are checked before any launch
 * (TS_ERR_INVALID), host weights are packed as the load path packs them, output buffers are copied in before the kernels
 * and back after them, and the engine's ts_set_tensor_cores setting is unchanged afterwards.  mode is the activation
 * format of ts_set_tensor_cores: 0 fp32, 1 the 3xTF32 (hi, lo) pair (fp32 hi with its 13 low mantissa bits clear, lo =
 * v - hi), 6 fp32 + fp16 planes (h = fp16(v), l = fp16(v - h), uint16).
 *
 * The wav2vec2 feature extractor's first layer as the face forward runs it: Conv1d(1, 512, 10, stride 5, no bias) +
 * GroupNorm(512, 512) (per clip and channel over time, biased variance, eps 1e-5, affine g / b) + erf-GELU, through
 * conv0_stats_kernel (per-channel sums in fp64, 256 outputs per block merged with atomicAdd) and conv0_apply_kernel (the
 * variance is E[y^2] - mean^2, clamped at 0).  wave [B,N] device fp32, N >= 10; W_host [512,1,10], g_host / b_host [512]
 * host fp32.  The output has T0 = (N - 10) / 5 + 1 rows per clip, staged as the face forward stages it: T0 & 1 tail rows
 * after every clip, so every buffer is [B, T0 + (T0 & 1), 512].  The tail rows are set to NaN before the launch (no kernel
 * writes them).  Mode 0: fp32 in y; mode 1: the (hi, lo) pair in plane_hi / plane_lo (fp32), y unused; mode 6: the fp16
 * planes only in plane_hi / plane_lo (uint16), y unused.  Samples past the last window are not read.  For T0 <= 256 a clip's
 * statistics come from one block and repeated calls give the same bits; beyond, the order of the fp64 atomic merges
 * varies from call to call (DESIGN.md). */
int ts_debug_conv0_gn(ts_engine* e, int mode, const float* wave, const float* W_host, const float* g_host, const float* b_host,
                      float* y, void* plane_hi, void* plane_lo, int B, int N, void* stream);
/* The 50 -> 30 fps interpolation of the face forward (F.interpolate(mode='linear', align_corners=False) along time, with
 * ATen's fp32 source positions: src = (Tin / Tout) * (t + 0.5) - 0.5 as two rounded operations, clamped at 0):
 * x [B,Tin,C] device fp32, staged as conv6's output with Tin & 1 NaN tail rows after every clip (no read reaches them),
 * -> y [B,Tout,C] device fp32. */
int ts_debug_interp(ts_engine* e, const float* x, float* y, int B, int Tin, int Tout, int C, void* stream);
/* Every LayerNorm of the face net (ln_pre_kernel, one warp per row, eps 1e-5):
 *   y(b, t) = act( LN_C(x(b, t) + pre(b, t)) * g + b + res(b, t) ),  act 0 none, 1 ReLU,
 * with pre (has_pre) and res (has_res) optional.  x, pre, res [B,T,C] device fp32, C in [1, 768] (the kernel holds 24
 * values per lane; wider rows are TS_ERR_INVALID); g_host / b_host [C] host fp32.  x_split / res_split: x / res are
 * stored split in the mode's format (modes 0 / 1: the (hi, lo) pair, which the kernel adds back exactly; mode 6: fp32 +
 * planes, the kernel reads the fp32 copy).  The output is staged with one pad row before and after every clip, as the
 * first_net and decoder norms stage it: every output buffer is [B, T + 2, C] and the pad rows keep what the caller put
 * there.  y_split = 0: fp32 in y; modes 0 / 1: the (hi, lo) pair in plane_hi / plane_lo (fp32), y unused; mode 6: fp32
 * in y and its fp16 planes in plane_hi / plane_lo (uint16).
 * Input range: the mean is an fp32 sum of the row and the variance an fp32 sum of squared deviations, so |x| must stay
 * below about 1e17 (the sum of squares overflows to inf beyond; the reference's Welford does not). */
typedef struct ts_debug_ln {
  int32_t mode, B, T, C;
  int32_t has_pre, has_res, act;
  int32_t x_split, res_split, y_split;
} ts_debug_ln;
int ts_debug_layernorm(ts_engine* e, const ts_debug_ln* a, const float* x, const float* pre, const float* res,
                       const float* g_host, const float* b_host, float* y, void* plane_hi, void* plane_lo, void* stream);
/* VectorQuantizerEMA.get_code_indices (the argmin of ts_vq_encode / ts_vq_score) on caller data: codebook_host
 * [ncodes,64] host fp32 (uploaded with the squared row norms ts_load_vq computes), z [R,64] device fp32 staged as
 * ts_vq_encode stages its latents, -> idx [R] int64 device, in [0, ncodes), torch.argmin's rule (ts_vq_encode). */
int ts_debug_vq_argmin(ts_engine* e, const float* codebook_host, int ncodes, const float* z, int64_t* idx, int R, void* stream);
/* Dense-contraction kernel for the face network and the VQ decoder (csrc/gemm_tc.cu):
 *   6 (default) Hopper wgmma kernel (128x128 tile) on two-term fp16-split operands (three products per MAC: fp32-grade
 *       results at twice the tf32 rate; operands must stay below 65504 in magnitude -- weights are pre-scaled per layer),
 *   1 / 3 / 4 the same kernel on 3xTF32 operands pre-split in HBM by the producing epilogue (full fp32 range),
 *   0 everything on the fp32 FFMA kernel.  Other values return TS_ERR_UNSUPPORTED.
 * Every mode keeps the face outputs within 1e-4 of the reference (tests/test_gpu_parity.py). */
int ts_set_tensor_cores(ts_engine* e, int enable);
/* PixelCNN executor: 0 (default) = grid-wide persistent cooperative kernel (grid barrier; batch tile 16 / 32 / 64 picked per
 * launch), 1 = the same device code, one launch per stage (debug cross-check), 2 = cluster-resident executor: 16-CTA
 * clusters own 4 / 8 samples, TMA weight ring, stage hand-over through DSMEM mbarriers, any batch size and both
 * checkpoint geometries (dim 256 x 15 layers, dim 512 x 10 layers — the latter always runs here).  All three produce
 * bit-identical logits. */
int ts_set_pixelcnn_mode(ts_engine* e, int mode);
/* Debug: per-stage, per-CTA globaltimer stamps of one latent row of the persistent kernel.  ts_pixelcnn_trace(e, row)
 * arms it (row < 0 disarms) for the following ts_pixelcnn_generate calls; ts_pixelcnn_trace_read copies
 * out[stages][ctas][4] = {weights ready, left the grid barrier, task done, arrived} in ns (*len in/out, elements;
 * out may be NULL to query the size). */
/* stages per latent row and persistent CTAs of the loaded plan */
int ts_pixelcnn_plan_shape(ts_engine* e, int* nstages, int* ncta);
int ts_pixelcnn_trace(ts_engine* e, int row);
int ts_pixelcnn_trace_read(ts_engine* e, uint64_t* out, int64_t* len);

/* Persistent CTAs of the grid-wide plan built by the NEXT ts_load_pixelcnn (0 = one per SM).  A smaller even count (>= 64)
 * launches the sampler as CTA pairs on that many SMs and leaves the other TPCs free for kernels of another stream: with
 * the latency-bound sampler and the face regressor run side by side (talkshow_b200/pipeline.py: 64 clips 59.2 -> 51.0 ms). */
int ts_set_pixelcnn_ctas(ts_engine* e, int n);

/* ts_body_generate runs its two VQ-VAE decoders (body, hands — independent chains of ~20 small launches each) side by side
 * on two streams for batches of at most `max_batch` samples (default 16; 0 = one after the other on the caller's stream).  The
 * result is bit-identical either way (the chains share nothing but their input codes); the caller's stream is joined before the
 * call returns.  Measured: -0.6 ms per call at 1..16 samples, neutral at 32 / 64. */
int ts_set_vq_parallel(ts_engine* e, int max_batch);

/* Plan built by the NEXT ts_load_pixelcnn: 1 (default) = fused 52-stage plan (adjacent linear maps of the horizontal
 * stack multiplied together at load, layer-0 gate of column 1 gathered from a code table), 0 = plain 84-stage plan
 * (one stage per reference conv), 2 = EXPERIMENTAL: the fused plan with vert_to_horiz taken out of the vertical stages
 * (it runs one column at a time beside the horizontal stage before its consumer).  All evaluate
 * GatedPixelCNN.forward exactly up to fp32 rounding order. */
int ts_set_pixelcnn_fusion(ts_engine* e, int on);

#ifdef __cplusplus
}
#endif
#endif
