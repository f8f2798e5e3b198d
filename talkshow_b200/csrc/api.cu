// talkshow_b200 — engine lifetime, error reporting, pose assembly, fused body path entry.
#include "convstack.h"
#include <climits>
#include "pixelcnn.h"

using namespace ts;

static std::string g_create_err;

float* ts_engine::upload(const std::vector<float>& h) {
  if (host_only) return nullptr;
  void* d = dmalloc(h.size() * sizeof(float));
  TS_CUDA(cudaMemcpy(d, h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice));
  return (float*)d;
}
unsigned short* ts_engine::upload(const std::vector<unsigned short>& h) {
  if (host_only) return nullptr;
  void* d = dmalloc(h.size() * sizeof(unsigned short));
  TS_CUDA(cudaMemcpy(d, h.data(), h.size() * sizeof(unsigned short), cudaMemcpyHostToDevice));
  return (unsigned short*)d;
}
void* ts_engine::dmalloc(size_t bytes) {
  if (host_only) return nullptr;
  void* d = nullptr;
  TS_CUDA(cudaMalloc(&d, bytes ? bytes : 16));
  (alloc_sink ? *alloc_sink : owned).push_back(d);
  return d;
}

extern "C" int ts_engine_create(ts_engine** out, int device) {
  if (!out) return TS_ERR_INVALID;
  *out = nullptr;
  ts_engine* e = new ts_engine();
  try {
    e->device = device;
    if (device < 0) {  // host-only planning mode: weight packing / plan export without a GPU (tests)
      e->host_only = true;
      e->sm_count = -device > 1 ? -device : 132;
    } else {
      int n = 0;
      TS_CUDA(cudaGetDeviceCount(&n));
      if (device >= n) fail(TS_ERR_INVALID, "device %d out of range (%d devices)", device, n);
      cudaDeviceProp prop;   // no cudaSetDevice here: creating an engine does not change the caller's current device
      TS_CUDA(cudaGetDeviceProperties(&prop, device));
      if (prop.major != 9 || prop.minor != 0)
        fail(TS_ERR_UNSUPPORTED, "talkshow_b200 is built for sm_90a (Hopper, H100), found sm_%d%d", prop.major, prop.minor);
      e->sm_count = prop.multiProcessorCount;
    }
  } catch (const std::exception& ex) {
    g_create_err = ex.what();
    delete e;
    return TS_ERR_CUDA;
  }
  *out = e;
  return TS_OK;
}

extern "C" void ts_engine_destroy(ts_engine* e) {
  if (!e) return;
  if (!e->host_only) {
    ts::DeviceGuard g(e);
    cudaDeviceSynchronize();
    if (e->aux_stream) cudaStreamDestroy(e->aux_stream);
    if (e->aux_fork) cudaEventDestroy(e->aux_fork);
    if (e->aux_join) cudaEventDestroy(e->aux_join);
    for (void* p : e->owned) cudaFree(p);
    for (auto& kv : e->slot_mem)
      for (void* p : kv.second) cudaFree(p);
    e->ws.buf.release();
  }
  ts::pixel_destroy(e);
  delete e->conv;
  ts::face_destroy(e);
  ts::mfcc_destroy(e);
  ts::smplx_destroy(e);
  ts::nccl_destroy(e);
  delete e;
}

extern "C" const char* ts_last_error(ts_engine* e) { return e ? e->err.c_str() : g_create_err.c_str(); }
extern "C" int ts_engine_sm_count(ts_engine* e) { return e ? e->sm_count : 0; }
extern "C" int64_t ts_launch_count(ts_engine* e) { return e ? e->launches : 0; }
extern "C" int ts_set_pixelcnn_mode(ts_engine* e, int mode) {
  if (!e || mode < 0 || mode > 2) return TS_ERR_INVALID;
  e->pixel_mode = mode;
  return TS_OK;
}

extern "C" int ts_set_pixelcnn_ctas(ts_engine* e, int n) {
  if (!e || n < 0) return TS_ERR_INVALID;
  e->pixel_ctas = n;
  return TS_OK;
}

extern "C" int ts_set_vq_parallel(ts_engine* e, int max_batch) {
  if (!e || max_batch < 0) return TS_ERR_INVALID;
  e->vq_parallel_batch = max_batch;
  return TS_OK;
}

extern "C" int ts_set_pixelcnn_fusion(ts_engine* e, int on) {
  if (!e) return TS_ERR_INVALID;
  if (on < 0 || on > 2) return TS_ERR_INVALID;
  e->pixel_fusion = on;
  return TS_OK;
}

// ---- pose assembly: scripts/demo.py:182-229 + data_utils/lower_body.py:68-87 -------------------
__constant__ float c_lower_pose[33] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 3.0747f, -0.0158f, -0.0152f,
    -1.1826512813568115f, 0.23866955935955048f, 0.15146760642528534f, -1.2604516744613647f, -0.3160211145877838f,
    -0.1603458970785141f, 1.1654603481292725f, 0.0f, 0.0f, 1.2521806955337524f, 0.041598282754421234f,
    -0.06312154978513718f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};

// ---- 6-D rotation -> axis-angle: matrix_to_axis_angle(rotation_6d_to_matrix(x)) ----------------------
// (data_utils/rotation_conversion.py:512-533 Gram-Schmidt, :98-118 matrix_to_quaternion, :481-507
// quaternion_to_axis_angle; applied by scripts/demo.py:185-188,216-219 when convert_to_6d is set).
// One definition for rot6d_to_aa_kernel and the fused 6-D assembly, so the two give the same bits.
__device__ __forceinline__ void rot6d_to_aa(const float* __restrict__ p, float& ax, float& ay, float& az) {
  const float a1x = p[0], a1y = p[1], a1z = p[2], a2x = p[3], a2y = p[4], a2z = p[5];
  float n1 = fmaxf(sqrtf(a1x * a1x + a1y * a1y + a1z * a1z), 1e-12f);           // F.normalize eps
  const float b1x = a1x / n1, b1y = a1y / n1, b1z = a1z / n1;
  const float d = b1x * a2x + b1y * a2y + b1z * a2z;
  float b2x = a2x - d * b1x, b2y = a2y - d * b1y, b2z = a2z - d * b1z;
  float n2 = fmaxf(sqrtf(b2x * b2x + b2y * b2y + b2z * b2z), 1e-12f);
  b2x /= n2; b2y /= n2; b2z /= n2;
  const float b3x = b1y * b2z - b1z * b2y, b3y = b1z * b2x - b1x * b2z, b3z = b1x * b2y - b1y * b2x;
  // rows of the matrix are b1, b2, b3
  const float m00 = b1x, m11 = b2y, m22 = b3z;
  auto sqp = [](float v) { return v > 0.f ? sqrtf(v) : 0.f; };                     // _sqrt_positive_part
  const float q0 = 0.5f * sqp(1.f + m00 + m11 + m22);
  float q1 = 0.5f * sqp(1.f + m00 - m11 - m22);
  float q2 = 0.5f * sqp(1.f - m00 + m11 - m22);
  float q3 = 0.5f * sqp(1.f - m00 - m11 + m22);
  if (b3y - b2z < 0.f) q1 = -q1;        // _copysign(x, m21 - m12)
  if (b1z - b3x < 0.f) q2 = -q2;        // _copysign(y, m02 - m20)
  if (b2x - b1y < 0.f) q3 = -q3;        // _copysign(z, m10 - m01)
  const float nv = sqrtf(q1 * q1 + q2 * q2 + q3 * q3);
  const float half = atan2f(nv, q0), ang = 2.f * half;
  const float sh = fabsf(ang) < 1e-6f ? 0.5f - (ang * ang) / 48.f : sinf(half) / ang;
  ax = q1 / sh;
  ay = q2 / sh;
  az = q3 / sh;
}

// component c (0..2) of the axis-angle of the 6-D rotation at p
__device__ __forceinline__ float rot6d_aa_component(const float* __restrict__ p, int c) {
  float x, y, z;
  rot6d_to_aa(p, x, y, z);
  return c == 0 ? x : (c == 1 ? y : z);
}

// out column -> source: pred = cat[jaw(3), body(129), expr(100)] (232), part2full inserts lower-pose
// blocks: [pred 0:3 | lp 0:15 | pred 3:6 | lp 15:21 | pred 6:9 | lp 21:27 | pred 9:12 | lp 27:33 | pred 12:232]
// SIX = false: face [B,Ff,103] = jaw(3) | expr(100), body [B,Fb,129] axis-angle.
// SIX = true:  face [B,Ff,106] = jaw(6-D) | expr(100), body [B,Fb,258] = 43 joints x 6-D; each needed joint is converted
//              to axis-angle on the fly (demo.py:185-188,216-219 followed by the same assembly).
template <bool SIX>
__global__ void assemble_kernel(const float* __restrict__ face, const float* __restrict__ body, float* __restrict__ out,
                                int B, int Ff, int Fb, int stand) {
  constexpr int FD = SIX ? 106 : 103, BD = SIX ? 258 : 129, JW = SIX ? 6 : 3;
  long n = (long)B * Ff * 265;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    int c = i % 265;
    long bf = i / 265;
    int f = bf % Ff, b = bf / Ff;
    int pc = -1, lp = -1;  // index into pred (232) or into lower pose (33)
    if (c < 3) pc = c;
    else if (c < 18) lp = c - 3;
    else if (c < 21) pc = c - 15;
    else if (c < 27) lp = c - 21 + 15;
    else if (c < 30) pc = c - 21;
    else if (c < 36) lp = c - 30 + 21;
    else if (c < 39) pc = c - 27;
    else if (c < 45) lp = c - 39 + 27;
    else pc = c - 33;
    float v;
    if (lp >= 0) {
      v = stand ? ((lp >= 6 && lp < 9) ? c_lower_pose[lp] : 0.f) : c_lower_pose[lp];
    } else if (pc < 3) {
      const float* fr = face + ((long)b * Ff + f) * FD;
      v = SIX ? rot6d_aa_component(fr, pc) : fr[pc];
    } else if (pc < 132) {
      int fb = f < Fb ? f : Fb - 1;
      const float* br = body + ((long)b * Fb + fb) * BD;
      v = SIX ? rot6d_aa_component(br + (pc - 3) / 3 * 6, (pc - 3) % 3) : br[pc - 3];
    } else {
      v = face[((long)b * Ff + f) * FD + JW + (pc - 132)];
    }
    out[i] = v;
  }
}

static void launch_assemble(ts_engine* e, bool six, const float* face, const float* body, float* out, int B, int Ff, int Fb,
                            int stand, void* stream) {
  ts::require_device(e);
  if (B <= 0 || Ff <= 0 || Fb <= 0) fail(TS_ERR_INVALID, "%s: B=%d Ff=%d Fb=%d", six ? "ts_assemble_pose6d" : "ts_assemble_pose", B, Ff, Fb);
  long n = (long)B * Ff * 265;
  int blocks = (int)std::min<long>((n + 255) / 256, (long)e->sm_count * 8);
  if (six) assemble_kernel<true><<<blocks, 256, 0, (cudaStream_t)stream>>>(face, body, out, B, Ff, Fb, stand);
  else assemble_kernel<false><<<blocks, 256, 0, (cudaStream_t)stream>>>(face, body, out, B, Ff, Fb, stand);
  e->launches++;
  TS_CUDA(cudaGetLastError());
}

extern "C" int ts_assemble_pose(ts_engine* e, const float* face, const float* body, float* out, int B, int Ff, int Fb,
                                int stand, void* stream) {
  TS_API_BEGIN(e)
  launch_assemble(e, false, face, body, out, B, Ff, Fb, stand, stream);
  TS_API_END(e)
}

extern "C" int ts_assemble_pose6d(ts_engine* e, const float* face, const float* body, float* out, int B, int Ff, int Fb,
                                  int stand, void* stream) {
  TS_API_BEGIN(e)
  launch_assemble(e, true, face, body, out, B, Ff, Fb, stand, stream);
  TS_API_END(e)
}

__global__ void rot6d_to_aa_kernel(const float* __restrict__ d6, float* __restrict__ aa, long n) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
    rot6d_to_aa(d6 + i * 6, aa[i * 3 + 0], aa[i * 3 + 1], aa[i * 3 + 2]);
}

extern "C" int ts_rot6d_to_axis_angle(ts_engine* e, const float* d6, float* aa, int64_t n, void* stream) {
  TS_API_BEGIN(e)
  ts::require_device(e);
  if (n < 0) fail(TS_ERR_INVALID, "ts_rot6d_to_axis_angle: n=%lld", (long long)n);
  if (n > 0) {
    int blocks = (int)std::min<long>((n + 255) / 256, (long)e->sm_count * 8);
    rot6d_to_aa_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(d6, aa, (long)n);
    e->launches++;
    TS_CUDA(cudaGetLastError());
  }
  TS_API_END(e)
}

extern "C" int ts_vq_dim(ts_engine* e, int which) {
  if (!e || which < 0 || which > 1 || !e->conv || !e->conv->vq[which].loaded) return 0;
  return e->conv->vq[which].out_dim;
}

// ---- fused body path: audio encoder -> PixelCNN sampler -> two VQ decoders -------------------------
// ctl = nullptr: the default sampler (ts_body_generate); else the sampling controls of ts_body_sample.
// seeds (ts_body_sample_seeded): per-clip seeds in place of noise.  anchors (ts_body_sample_anchored): pinned draws.
// style (ts_body_sample_styled): per-row speaker weights in place of label.  clip_ctl (ts_body_sample_clips): per-clip
// controls (host, validated) in place of ctl's four.  clip_shape / code_bias (ts_body_sample_shaped): logit shaping.
// guide (ts_body_sample_guided): B = 2P branches sampled in pairs; codes gets every branch, poses the P conditional ones.
static void body_generate(ts_engine* e, const float* mfcc, const int64_t* label, const float* noise, int64_t* codes,
                          float* poses, int B, int M, void* stream, const SampleCtl* ctl, const int64_t* seeds = nullptr,
                          const int64_t* anchors = nullptr, const float* style = nullptr,
                          const ts_clip_ctl* clip_ctl = nullptr, const ts_clip_shape* clip_shape = nullptr,
                          const float* code_bias = nullptr, const float* guide = nullptr) {
  ts::require_device(e);
  if (!e->conv || !e->conv->audio_loaded) fail(TS_ERR_NOT_LOADED, "audio encoder weights not loaded");
  if (!e->conv->vq[0].loaded || !e->conv->vq[1].loaded) fail(TS_ERR_NOT_LOADED, "vq weights not loaded");
  if (!e->pix) fail(TS_ERR_NOT_LOADED, "pixelcnn weights not loaded");
  for (int w = 0; w < 2; ++w)   // the sampler emits indices in [0, 2048): F.embedding of the reference would raise on a smaller codebook
    if (e->conv->vq[w].ncodes < PIX_NCODE)
      fail(TS_ERR_INVALID, "ts_body_generate: vq[%d] codebook has %d codes, the PixelCNN samples %d", w, e->conv->vq[w].ncodes, PIX_NCODE);
  if (B <= 0 || M < 4) fail(TS_ERR_INVALID, "ts_body_generate: B=%d M=%d", B, M);
  cudaStream_t s = (cudaStream_t)stream;
  const int T = ts_latent_rows(M);
  auto body = [&] {
    Act3 x = new_act(e, B, M, 64, 1, s);
    nct_to_act(e, mfcc, 64, x, s);
    Act3 a = run_trunk(e, e->conv->audio, x, s);          // [B,T,256] channel-last, pad 1
    int64_t* idx = e->ws.alloc<int64_t>((size_t)B * T * 2);
    int64_t* idx_c = e->ws.alloc<int64_t>((size_t)B * T * 2);  // [2][B][T] column-split copy
    pixelcnn_generate_act(e, a, label, noise, idx, nullptr, B, T, nullptr, 0, s, false, ctl, seeds, anchors, style, clip_ctl,
                          clip_shape, code_bias, guide);
    if (guide) split_guided_codes(e, idx, idx_c, B / 2, T, codes, s);   // decode the conditional branches only
    else split_codes(e, idx, idx_c, B, T, codes, s);
    const int Bd = guide ? B / 2 : B;
    const int c0 = e->conv->vq[0].out_dim, c1 = e->conv->vq[1].out_dim;   // 39 + 90 (axis-angle) or 78 + 180 (6-D)
    // Small batches: each decoder is a chain of ~20 launches that fill a few SMs, so the hand decoder runs on a second
    // stream beside the body decoder (fork after the code split, join before the call returns to the caller's stream).
    // The two chains share nothing but their input codes: separate workspace blocks, disjoint columns of `poses`.
    const bool par = !e->ws.sizing && Bd <= e->vq_parallel_batch;
    if (par) {
      if (!e->aux_stream) {
        int prio = 0;
        TS_CUDA(cudaStreamGetPriority(s, &prio));      // the body path may run on a high-priority stream (pipeline.WholeBody)
        TS_CUDA(cudaStreamCreateWithPriority(&e->aux_stream, cudaStreamNonBlocking, prio));
        TS_CUDA(cudaEventCreateWithFlags(&e->aux_fork, cudaEventDisableTiming));
        TS_CUDA(cudaEventCreateWithFlags(&e->aux_join, cudaEventDisableTiming));
      }
      TS_CUDA(cudaEventRecord(e->aux_fork, s));
      TS_CUDA(cudaStreamWaitEvent(e->aux_stream, e->aux_fork, 0));
    }
    for (int w = 0; w < 2; ++w) {
      cudaStream_t sw = (w == 1 && par) ? e->aux_stream : s;
      Act3 y = run_vq_decode(e, e->conv->vq[w], idx_c + (size_t)w * Bd * T, Bd, T, sw);
      act_to_btc(e, y, e->conv->vq[w].out_dim, poses, c0 + c1, w ? c0 : 0, sw);
    }
    if (par) {
      TS_CUDA(cudaEventRecord(e->aux_join, e->aux_stream));
      TS_CUDA(cudaStreamWaitEvent(s, e->aux_join, 0));
    }
  };
  e->ws.begin_sizing();
  body();
  size_t need = e->ws.need;
  e->ws.buf.ensure(need + 256);
  e->ws.begin(need);
  body();
}

extern "C" int ts_body_generate(ts_engine* e, const float* mfcc, const int64_t* label, const float* noise,
                                int64_t* codes, float* poses, int B, int M, void* stream) {
  TS_API_BEGIN(e)
  body_generate(e, mfcc, label, noise, codes, poses, B, M, stream, nullptr);
  TS_API_END(e)
}

extern "C" int ts_body_sample(ts_engine* e, const float* mfcc, const int64_t* label, const float* noise, int64_t* codes,
                              float* poses, int B, int M, float temperature, int top_k, float* logp_out, void* stream) {
  const ts_sample_ctl ctl = {temperature, top_k, 1.f, 0.f, logp_out, nullptr};
  return ts_body_sample_ctl(e, mfcc, label, noise, codes, poses, B, M, &ctl, stream);
}

extern "C" int ts_body_sample_ctl(ts_engine* e, const float* mfcc, const int64_t* label, const float* noise, int64_t* codes,
                                  float* poses, int B, int M, const ts_sample_ctl* ctl, void* stream) {
  TS_API_BEGIN(e)
  const SampleCtl c = sample_ctl_of(ctl);
  check_sample_ctl(c, noise);
  body_generate(e, mfcc, label, noise, codes, poses, B, M, stream, &c);
  TS_API_END(e)
}

extern "C" int ts_body_sample_seeded(ts_engine* e, const float* mfcc, const int64_t* label, const int64_t* seeds, int64_t* codes,
                                     float* poses, int B, int M, const ts_sample_ctl* ctl, void* stream) {
  TS_API_BEGIN(e)
  ts::require_device(e);
  if (ctl) {
    const SampleCtl c = sample_ctl_of(ctl);
    check_sample_ctl(c, nullptr, seeds);
    body_generate(e, mfcc, label, nullptr, codes, poses, B, M, stream, &c, seeds);
  } else {
    if (!seeds) fail(TS_ERR_INVALID, "ts_body_sample_seeded: seeds is NULL (only greedy decoding runs without)");
    body_generate(e, mfcc, label, nullptr, codes, poses, B, M, stream, nullptr, seeds);
  }
  TS_API_END(e)
}

extern "C" int ts_body_sample_anchored(ts_engine* e, const float* mfcc, const int64_t* label, const float* noise,
                                       const int64_t* seeds, const int64_t* anchors, int64_t* codes, float* poses, int B, int M,
                                       const ts_sample_ctl* ctl, void* stream) {
  TS_API_BEGIN(e)
  ts::require_device(e);
  SampleCtl c;
  if (ctl) {
    c = sample_ctl_of(ctl);
    check_sample_ctl(c, noise, seeds);
  }
  check_anchored_source(ctl ? &c : nullptr, noise, seeds, "ts_body_sample_anchored");
  body_generate(e, mfcc, label, noise, codes, poses, B, M, stream, ctl ? &c : nullptr, seeds, anchors);
  TS_API_END(e)
}

extern "C" int ts_body_sample_styled(ts_engine* e, const float* mfcc, const int64_t* label, const float* style, int ncls,
                                     const float* noise, const int64_t* seeds, const int64_t* anchors, int64_t* codes,
                                     float* poses, int B, int M, const ts_sample_ctl* ctl, void* stream) {
  TS_API_BEGIN(e)
  ts::require_device(e);
  if (!e->pix) fail(TS_ERR_NOT_LOADED, "pixelcnn weights not loaded");
  check_style(e, label, style, ncls, "ts_body_sample_styled");
  SampleCtl c;
  if (ctl) {
    c = sample_ctl_of(ctl);
    check_sample_ctl(c, noise, seeds);
  }
  check_anchored_source(ctl ? &c : nullptr, noise, seeds, "ts_body_sample_styled");
  body_generate(e, mfcc, label, noise, codes, poses, B, M, stream, ctl ? &c : nullptr, seeds, anchors, style);
  TS_API_END(e)
}

extern "C" int ts_body_sample_clips(ts_engine* e, const float* mfcc, const int64_t* label, const float* style, int ncls,
                                    const float* noise, const int64_t* seeds, const int64_t* anchors, int64_t* codes,
                                    float* poses, int B, int M, const ts_sample_ctl* ctl, const ts_clip_ctl* clip_ctl,
                                    void* stream) {
  if (!clip_ctl)
    return ts_body_sample_styled(e, mfcc, label, style, ncls, noise, seeds, anchors, codes, poses, B, M, ctl, stream);
  TS_API_BEGIN(e)
  ts::require_device(e);
  if (!e->pix) fail(TS_ERR_NOT_LOADED, "pixelcnn weights not loaded");
  if (B <= 0) fail(TS_ERR_INVALID, "ts_body_sample_clips: B=%d", B);
  check_style(e, label, style, ncls, "ts_body_sample_clips");
  check_clip_ctl(clip_ctl, B, noise, seeds, "ts_body_sample_clips");
  SampleCtl c;   // logp_out / kept_out of ctl; the draws' controls come from clip_ctl
  if (ctl) { c.logp_out = ctl->logp_out; c.kept_out = ctl->kept_out; }
  body_generate(e, mfcc, label, noise, codes, poses, B, M, stream, &c, seeds, anchors, style, clip_ctl);
  TS_API_END(e)
}

extern "C" int ts_body_sample_shaped(ts_engine* e, const float* mfcc, const int64_t* label, const float* style, int ncls,
                                     const float* noise, const int64_t* seeds, const int64_t* anchors, int64_t* codes,
                                     float* poses, int B, int M, const ts_sample_ctl* ctl, const ts_clip_ctl* clip_ctl,
                                     const ts_clip_shape* clip_shape, const float* code_bias, void* stream) {
  if (!clip_shape && !code_bias)
    return ts_body_sample_clips(e, mfcc, label, style, ncls, noise, seeds, anchors, codes, poses, B, M, ctl, clip_ctl, stream);
  TS_API_BEGIN(e)
  ts::require_device(e);
  if (!e->pix) fail(TS_ERR_NOT_LOADED, "pixelcnn weights not loaded");
  if (B <= 0) fail(TS_ERR_INVALID, "ts_body_sample_shaped: B=%d", B);
  check_style(e, label, style, ncls, "ts_body_sample_shaped");
  if (clip_shape) check_clip_shape(clip_shape, B, "ts_body_sample_shaped");
  const SampleCtl c = shaped_ctl(ctl, clip_ctl, B, noise, seeds, "ts_body_sample_shaped");
  body_generate(e, mfcc, label, noise, codes, poses, B, M, stream, &c, seeds, anchors, style, clip_ctl, clip_shape, code_bias);
  TS_API_END(e)
}

extern "C" int ts_body_sample_guided(ts_engine* e, const float* mfcc, const int64_t* label, const float* style, int ncls,
                                     const float* noise, const int64_t* seeds, const int64_t* anchors, int64_t* codes,
                                     float* poses, int P, int M, const ts_sample_ctl* ctl, const ts_clip_ctl* clip_ctl,
                                     const ts_clip_shape* clip_shape, const float* code_bias, const float* guidance,
                                     void* stream) {
  TS_API_BEGIN(e)
  ts::require_device(e);
  if (!e->pix) fail(TS_ERR_NOT_LOADED, "pixelcnn weights not loaded");
  if (P < 1 || P > INT_MAX / 2) fail(TS_ERR_INVALID, "ts_body_sample_guided: P=%d pairs", P);
  check_style(e, label, style, ncls, "ts_body_sample_guided");
  check_guidance(guidance, P, "ts_body_sample_guided");
  if (clip_shape) check_clip_shape(clip_shape, P, "ts_body_sample_guided");
  const SampleCtl c = shaped_ctl(ctl, clip_ctl, P, noise, seeds, "ts_body_sample_guided");
  body_generate(e, mfcc, label, noise, codes, poses, 2 * P, M, stream, &c, seeds, anchors, style, clip_ctl, clip_shape,
                code_bias, guidance);
  TS_API_END(e)
}
