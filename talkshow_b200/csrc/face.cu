// talkshow_b200 — face regressor: s2g_face.Generator.forward (nets/spg/s2g_face.py:196-224) with the
// reference's wav2vec2 variant (nets/spg/wav2vec.py:76-143: HF Wav2Vec2Model whose CNN features are
// linearly interpolated from 50 to 30 fps before the transformer).  Everything runs channel-last
// ([B,T,C]) so that every Conv1d / Linear is one implicit GEMM (kernels.h); GroupNorm(512,512),
// LayerNorm, the 50->30 fps interpolation and the 12-head attention are small dedicated kernels.
// fp32 throughout (the parity bar is 1e-4 max-abs on the 103 outputs).
#include <cuda_fp16.h>
#include "convstack.h"

#include <memory>
#include "pixelcnn.h"

namespace ts {

static const int W2V_K[7] = {10, 3, 3, 3, 3, 2, 2};
static const int W2V_S[7] = {5, 2, 2, 2, 2, 2, 2};

struct EncLayer {
  Layer qkv, out, ff1, ff2;
  float *ln1_g, *ln1_b, *ln2_g, *ln2_b;
};

struct FaceNet {
  float* conv0_w = nullptr;  // [512][10]
  float *gn_g = nullptr, *gn_b = nullptr;
  Layer conv[7];  // 1..6 used
  float *fp_ln_g = nullptr, *fp_ln_b = nullptr;
  Layer fproj, posconv;
  unsigned short* pos_w16 = nullptr;   // posconv_mma_kernel's pre-split weights
  float pos_unscale = 1.f;
  float *enc_ln_g = nullptr, *enc_ln_b = nullptr;
  std::vector<EncLayer> layers;
  Layer feat_map;
  // identity net (audio_middle.id_mlp present): first_net layer 0 takes [feature 256 | id 64] and has a residual conv.
  // identity-free net (the convert_to_6d face, identity=False): layer 0 takes the 256 features, residual = input.
  bool identity = true;
  float *id_w = nullptr, *id_b = nullptr;  // [64][ncls], [64]
  int ncls = 4;
  Layer fn_conv[3], fn_res0;
  float *fn_g[3], *fn_b[3];
  Layer dec_conv[2][3];
  float *dec_g[2][3], *dec_b[2][3];
  Layer fin[2];
  int jaw_dim = 3, exp_dim = 100;
};

void face_destroy(ts_engine* e) {
  delete e->face;
  e->face = nullptr;
}

static float* up(ts_engine* e, const float* p, size_t n) { return e->upload(std::vector<float>(p, p + n)); }

// weight [cout][cin][k] -> Layer [cout][k][cin] (+ optional bias)
static Layer pack_ckc(ts_engine* e, const float* w, const float* b, int cout, int cin, int k) {
  int cp = pad4(cin);
  std::vector<float> W((size_t)cout * k * cp, 0.f);
  for (int o = 0; o < cout; ++o)
    for (int c = 0; c < cin; ++c)
      for (int t = 0; t < k; ++t) W[((size_t)o * k + t) * cp + c] = w[((size_t)o * cin + c) * k + t];
  Layer L;
  L.N = cout; L.taps = k; L.cin = cp; L.K = k * cp;
  upload_weights(e, W, &L);
  L.bias = b ? up(e, b, cout) : nullptr;
  return L;
}
static Layer pack_linear(ts_engine* e, const float* w, const float* b, int N, int K) {
  Layer L;
  L.N = N; L.K = K; L.taps = 1; L.cin = K;
  upload_weights(e, std::vector<float>(w, w + (size_t)N * K), &L);
  L.bias = b ? up(e, b, N) : nullptr;
  return L;
}

// ---- kernels ---------------------------------------------------------------------------------
// conv0 (1 -> 512 channels, k=10, s=5, no bias) statistics for GroupNorm(512 groups): per (b, c)
// sum and sum of squares over time, accumulated in fp64.
__global__ void __launch_bounds__(256) conv0_stats_kernel(const float* __restrict__ wave, const float* __restrict__ w, int N, int T0,
                                                          double* __restrict__ stats) {
  constexpr int TC = 256;  // outputs per block
  __shared__ float xs[TC * 5 + 16];
  const int b = blockIdx.y, t0 = blockIdx.x * TC, tid = threadIdx.x;
  const int nt = min(TC, T0 - t0);
  const float* x = wave + (size_t)b * N + (size_t)t0 * 5;
  for (int i = tid; i < nt * 5 + 5; i += 256) xs[i] = x[i];
  __syncthreads();
  for (int c = tid; c < 512; c += 256) {
    float wr[10];
#pragma unroll
    for (int j = 0; j < 10; ++j) wr[j] = w[c * 10 + j];
    double s = 0.0, ss = 0.0;
    for (int t = 0; t < nt; ++t) {
      float y = 0.f;
#pragma unroll
      for (int j = 0; j < 10; ++j) y = fmaf(wr[j], xs[t * 5 + j], y);
      s += (double)y;
      ss += (double)y * (double)y;
    }
    atomicAdd(&stats[((size_t)b * 512 + c) * 2], s);
    atomicAdd(&stats[((size_t)b * 512 + c) * 2 + 1], ss);
  }
}
// recompute conv0, normalise per (b,c), affine, GELU, write channel-last [B,T0,512]
__global__ void __launch_bounds__(256) conv0_apply_kernel(const float* __restrict__ wave, const float* __restrict__ w,
                                                          const double* __restrict__ stats, const float* __restrict__ g,
                                                          const float* __restrict__ bta, int N, int T0, Act3 out) {
  constexpr int TC = 64;
  __shared__ float xs[TC * 5 + 16];
  const int b = blockIdx.y, t0 = blockIdx.x * TC, tid = threadIdx.x;
  const int nt = min(TC, T0 - t0);
  const float* x = wave + (size_t)b * N + (size_t)t0 * 5;
  for (int i = tid; i < nt * 5 + 5; i += 256) xs[i] = x[i];
  __syncthreads();
  for (int c = tid; c < 512; c += 256) {
    float wr[10];
#pragma unroll
    for (int j = 0; j < 10; ++j) wr[j] = w[c * 10 + j];
    double s = stats[((size_t)b * 512 + c) * 2], ss = stats[((size_t)b * 512 + c) * 2 + 1];
    double mean = s / T0, var = ss / T0 - mean * mean;
    if (var < 0) var = 0;
    float rstd = (float)(1.0 / sqrt(var + 1e-5)), mu = (float)mean, gg = g[c], bb = bta[c];
    for (int t = 0; t < nt; ++t) {
      float y = 0.f;
#pragma unroll
      for (int j = 0; j < 10; ++j) y = fmaf(wr[j], xs[t * 5 + j], y);
      float v = (y - mu) * rstd * gg + bb;
      v = 0.5f * v * (1.0f + erff(v * 0.70710678118654752440f));
      if (out.h16) {
        if (out.p) out.row(b, t0 + t)[c] = v;
        split16(v, out.row_h16(b, t0 + t)[c], out.row_l16(b, t0 + t)[c]);
      } else if (out.lo) {
        float h = __uint_as_float(__float_as_uint(v) & 0xffffe000u);
        out.row(b, t0 + t)[c] = h;
        out.row_lo(b, t0 + t)[c] = v - h;
      } else {
        out.row(b, t0 + t)[c] = v;
      }
    }
  }
}

// F.interpolate(mode='linear', align_corners=False) along time, channel-last
__global__ void interp_kernel(Act3 in, Act3 out) {
  const float scale = (float)in.T / (float)out.T;
  long n = (long)out.B * out.T * out.C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    int c = i % out.C;
    long bt = i / out.C;
    int t = bt % out.T, b = bt / out.T;
    // ATen's area_pixel_compute_source_index in float, scale * (t + 0.5) - 0.5 rounded once (torch contracts it to an
    // FMA): at 100 s the source positions reach 5000 and a differently rounded position moves the interpolation
    // weights by up to 5e-4
    float src = fmaf(scale, (float)t + 0.5f, -0.5f);
    if (src < 0.f) src = 0.f;
    int i0 = (int)src;
    if (i0 > in.T - 1) i0 = in.T - 1;
    int i1 = i0 + (i0 < in.T - 1 ? 1 : 0);
    float l1 = src - (float)i0, l0 = 1.0f - l1;
    out.row(b, t)[c] = l0 * in.row(b, i0)[c] + l1 * in.row(b, i1)[c];
  }
}

// y = LayerNorm_C(x + pre) * g + b  (+ res) -> act ; one warp per row
__global__ void ln_pre_kernel(Act3 x, Act3 pre, int has_pre, const float* __restrict__ g, const float* __restrict__ bta, Act3 y,
                              Act3 res, int has_res, int act, float eps) {
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  int rows = x.B * x.T;
  if (warp >= rows) return;
  int b = warp / x.T, t = warp % x.T, C = x.C;
  const float* xr = x.row(b, t);
  const float* xl = x.lo ? x.row_lo(b, t) : nullptr;
  const float* pr = has_pre ? pre.row(b, t) : nullptr;
  float v[24];  // C <= 768
  float s = 0.f;
  int n = 0;
  for (int c = lane; c < C; c += 32, ++n) {
    float a = xr[c];
    if (xl) a += xl[c];
    if (pr) a += pr[c];
    v[n] = a;
    s += a;
  }
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  float mean = s / C, q = 0.f;
  for (int i = 0; i < n; ++i) { float d = v[i] - mean; q = fmaf(d, d, q); }
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  float rstd = 1.0f / sqrtf(q / C + eps);
  float* yr = y.row(b, t);
  float* yl = y.lo ? y.row_lo(b, t) : nullptr;
  const float* rr = has_res ? res.row(b, t) : nullptr;
  const float* rl = (has_res && res.lo) ? res.row_lo(b, t) : nullptr;
  n = 0;
  for (int c = lane; c < C; c += 32, ++n) {
    float o = (v[n] - mean) * rstd * g[c] + bta[c];
    if (rr) o += rl ? (rr[c] + rl[c]) : rr[c];
    if (act == ACT_RELU) o = o > 0.f ? o : 0.f;
    if (y.h16) {
      yr[c] = o;
      split16(o, y.row_h16(b, t)[c], y.row_l16(b, t)[c]);
    } else if (yl) {
      float h = __uint_as_float(__float_as_uint(o) & 0xffffe000u);
      yr[c] = h;
      yl[c] = o - h;
    } else {
      yr[c] = o;
    }
  }
}
// conv0 + GroupNorm(512, 512) + GELU of wave [B,N] into h [B,T0,512], T0 = (N - 10) / 5 + 1; stats: B * 512 * 2 doubles
static void conv0_gn(ts_engine* e, const float* wave, const float* w, const float* g, const float* b, double* stats, int B, int N,
                     const Act3& h, cudaStream_t s) {
  if (e->ws.sizing) return;
  const int T = h.T;
  TS_CUDA(cudaMemsetAsync(stats, 0, (size_t)B * 512 * 2 * sizeof(double), s));
  conv0_stats_kernel<<<dim3(cdiv(T, 256), B), 256, 0, s>>>(wave, w, N, T, stats);
  conv0_apply_kernel<<<dim3(cdiv(T, 64), B), 256, 0, s>>>(wave, w, stats, g, b, N, T, h);
  e->launches += 2;
  TS_CUDA(cudaGetLastError());
}
static void interp(ts_engine* e, const Act3& x, const Act3& y, cudaStream_t s) {
  if (e->ws.sizing) return;
  long n = (long)y.B * y.T * y.C;
  interp_kernel<<<(int)std::min<long>((n + 255) / 256, (long)e->sm_count * 16), 256, 0, s>>>(x, y);
  e->launches++;
  TS_CUDA(cudaGetLastError());
}
static void ln_pre(ts_engine* e, const Act3& x, const Act3* pre, const float* g, const float* b, const Act3& y, const Act3* res,
                   int act, cudaStream_t s) {
  if (e->ws.sizing) return;
  if (x.C > 768) fail(TS_ERR_INVALID, "layernorm width %d > 768", x.C);
  int rows = x.B * x.T;
  ln_pre_kernel<<<cdiv(rows, 8), 256, 0, s>>>(x, pre ? *pre : Act3(), pre ? 1 : 0, g, b, y, res ? *res : Act3(), res ? 1 : 0, act, 1e-5f);
  e->launches++;
  TS_CUDA(cudaGetLastError());
}

// id_mlp: Conv1d(ncls,64,1) on the id vector, broadcast over time into columns [off, off+64) of x
__global__ void id_cols_kernel(const float* __restrict__ idv, const float* __restrict__ w, const float* __restrict__ bias, int ncls,
                               Act3 x, int off) {
  int b = blockIdx.y;
  __shared__ float v[64];
  if (threadIdx.x < 64) {
    float a = bias[threadIdx.x];
    for (int k = 0; k < ncls; ++k) a = fmaf(w[threadIdx.x * ncls + k], idv[b * ncls + k], a);
    v[threadIdx.x] = a;
  }
  __syncthreads();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < x.T * 64; i += gridDim.x * blockDim.x) {
    x.row(b, i / 64)[off + (i & 63)] = v[i & 63];
    if (x.h16) split16(v[i & 63], x.row_h16(b, i / 64)[off + (i & 63)], x.row_l16(b, i / 64)[off + (i & 63)]);
  }
}

// multi-head self-attention, eager softmax(QK^T * scale) V, head_dim 64.  qkv rows are
// [q(768) | k(768) | v(768)], head h uses columns h*64.. in each block.  One CTA = QT queries of one
// (batch, head); scores for the QT rows live in shared memory.
template <int QT>
__global__ void __launch_bounds__(256) attention_kernel(const float* __restrict__ qkv, float* __restrict__ out, float* __restrict__ out_lo, int T,
                                                        int H, float scale) {
  extern __shared__ float sm[];
  const int Tp = (T + 63) & ~63;
  float* Qs = sm;                    // [QT][65]
  float* KVs = Qs + QT * 65;         // [64][65]
  float* S = KVs + 64 * 65;          // [QT][Tp]
  const int bh = blockIdx.y, b = bh / H, h = bh % H;
  const int q0 = blockIdx.x * QT, tid = threadIdx.x;
  const int ld = 3 * H * 64;
  const float* base = qkv + (size_t)b * T * ld;
  constexpr int RQ = QT / 16;        // query rows per thread
  const int ty = tid >> 4, tx = tid & 15;
  for (int i = tid; i < QT * 64; i += 256) {
    int r = i >> 6, d = i & 63;
    Qs[r * 65 + d] = (q0 + r < T) ? base[(size_t)(q0 + r) * ld + h * 64 + d] : 0.f;
  }
  // phase 1: scores
  for (int k0 = 0; k0 < T; k0 += 64) {
    __syncthreads();
    for (int i = tid; i < 64 * 64; i += 256) {
      int r = i >> 6, d = i & 63;
      KVs[r * 65 + d] = (k0 + r < T) ? base[(size_t)(k0 + r) * ld + H * 64 + h * 64 + d] : 0.f;
    }
    __syncthreads();
    float acc[RQ][4];
#pragma unroll
    for (int i = 0; i < RQ; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (int d = 0; d < 64; ++d) {
      float q[RQ], k[4];
#pragma unroll
      for (int i = 0; i < RQ; ++i) q[i] = Qs[(ty * RQ + i) * 65 + d];
#pragma unroll
      for (int j = 0; j < 4; ++j) k[j] = KVs[(tx * 4 + j) * 65 + d];
#pragma unroll
      for (int i = 0; i < RQ; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(q[i], k[j], acc[i][j]);
    }
#pragma unroll
    for (int i = 0; i < RQ; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        int kk = k0 + tx * 4 + j;
        S[(ty * RQ + i) * Tp + kk] = kk < T ? acc[i][j] * scale : -INFINITY;
      }
  }
  __syncthreads();
  // phase 2: softmax per row (warp per row)
  const int warp = tid >> 5, lane = tid & 31;
  for (int r = warp; r < QT; r += 8) {
    float* row = S + r * Tp;
    float mx = -INFINITY;
    for (int k = lane; k < T; k += 32) mx = fmaxf(mx, row[k]);
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int k = lane; k < T; k += 32) { float ev = expf(row[k] - mx); row[k] = ev; sum += ev; }
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    for (int k = lane; k < Tp; k += 32) row[k] = k < T ? row[k] / sum : 0.f;
  }
  // phase 3: O = P V
  float o[RQ][4];
#pragma unroll
  for (int i = 0; i < RQ; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) o[i][j] = 0.f;
  for (int k0 = 0; k0 < T; k0 += 64) {
    __syncthreads();
    for (int i = tid; i < 64 * 64; i += 256) {
      int r = i >> 6, d = i & 63;
      KVs[r * 65 + d] = (k0 + r < T) ? base[(size_t)(k0 + r) * ld + 2 * H * 64 + h * 64 + d] : 0.f;
    }
    __syncthreads();
    for (int kk = 0; kk < 64; ++kk) {
      float p[RQ], v[4];
#pragma unroll
      for (int i = 0; i < RQ; ++i) p[i] = S[(ty * RQ + i) * Tp + k0 + kk];
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = KVs[kk * 65 + tx * 4 + j];
#pragma unroll
      for (int i = 0; i < RQ; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) o[i][j] = fmaf(p[i], v[j], o[i][j]);
    }
  }
#pragma unroll
  for (int i = 0; i < RQ; ++i) {
    int q = q0 + ty * RQ + i;
    if (q < T)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        size_t at = ((size_t)b * T + q) * (H * 64) + h * 64 + tx * 4 + j;
        if (out_lo) {
          float hh = __uint_as_float(__float_as_uint(o[i][j]) & 0xffffe000u);
          out[at] = hh;
          out_lo[at] = o[i][j] - hh;
        } else {
          out[at] = o[i][j];
        }
      }
  }
}

// ---- tensor-core attention (legacy warp-level MMA, 3xTF32) -------------------------------------------
// One CTA per (batch, head): K and V of the head live in shared memory as fp32 (row stride 68 floats, which
// makes both fragment access patterns below bank-conflict free); every warp owns 16-query row blocks and runs
// an online-softmax pass over 64-key blocks with mma.sync.m16n8k8 (tf32 inputs, fp32 accumulate).  fp32 accuracy
// comes from the 3xTF32 split x = hi + lo (both rounded to tf32 with cvt.rna; products lo*hi + hi*lo + hi*hi),
// done in registers: Q once per row block, K / V / P on the fly.  The P accumulator fragment is fed to the PV
// product without shuffles by letting MMA k-slot t / t+4 stand for keys 2t / 2t+1 of the 8-key step (a
// permutation of the reduction index applied to both operands).
constexpr int ATT_LD = 68;
__device__ __forceinline__ uint32_t to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  hi = to_tf32(x);
  lo = to_tf32(x - __uint_as_float(hi));
}
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// 3xTF32 products of one A fragment (hi, lo) against four B fragments, small terms first; the four
// accumulators are independent, so each pass keeps four MMAs in flight per warp
__device__ __forceinline__ void mma3x4(float (&c0)[4], float (&c1)[4], float (&c2)[4], float (&c3)[4], const uint32_t (&ah)[4],
                                       const uint32_t (&al)[4], const float (&bf)[8]) {
  uint32_t bh[8], bl[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) split_tf32(bf[i], bh[i], bl[i]);
  mma_tf32(c0, al, bh[0], bh[1]); mma_tf32(c1, al, bh[2], bh[3]); mma_tf32(c2, al, bh[4], bh[5]); mma_tf32(c3, al, bh[6], bh[7]);
  mma_tf32(c0, ah, bl[0], bl[1]); mma_tf32(c1, ah, bl[2], bl[3]); mma_tf32(c2, ah, bl[4], bl[5]); mma_tf32(c3, ah, bl[6], bl[7]);
  mma_tf32(c0, ah, bh[0], bh[1]); mma_tf32(c1, ah, bh[2], bh[3]); mma_tf32(c2, ah, bh[4], bh[5]); mma_tf32(c3, ah, bh[6], bh[7]);
}

constexpr int ATT_WARPS = 10;
__global__ void __launch_bounds__(ATT_WARPS * 32, 1) attention_mma_kernel(const float* __restrict__ qkv, float* __restrict__ out,
                                                                          float* __restrict__ out_lo, int T, int H, float scale) {
  extern __shared__ __align__(16) float sm[];
  const int Tp = (T + 63) & ~63;      // keys padded to whole 64-key blocks (pad rows are zero and masked)
  float* Ks = sm;                     // [Tp][ATT_LD]
  float* Vs = sm + (size_t)Tp * ATT_LD;
  const int bh = blockIdx.x, b = bh / H, h = bh % H;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int ld = 3 * H * 64;
  const float* base = qkv + (size_t)b * T * ld + h * 64;
  for (int i = tid; i < Tp * 16; i += ATT_WARPS * 32) {
    const int r = i >> 4, c4 = (i & 15) * 4;
    float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
    if (r < T) {
      kv = *reinterpret_cast<const float4*>(base + (size_t)r * ld + H * 64 + c4);
      vv = *reinterpret_cast<const float4*>(base + (size_t)r * ld + 2 * H * 64 + c4);
    }
    *reinterpret_cast<float4*>(Ks + r * ATT_LD + c4) = kv;
    *reinterpret_cast<float4*>(Vs + r * ATT_LD + c4) = vv;
  }
  __syncthreads();
  const int nrb = (T + 15) >> 4;
  for (int rb = warp; rb < nrb; rb += ATT_WARPS) {
    const int ra = rb * 16 + g, rbw = ra + 8;     // the two query rows this thread holds fragments of
    uint32_t qh[8][4], ql[8][4];
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const float* qa = base + (size_t)ra * ld + ks * 8 + t;
      const float* qb = base + (size_t)rbw * ld + ks * 8 + t;
      const float a0 = ra < T ? qa[0] * scale : 0.f, a2 = ra < T ? qa[4] * scale : 0.f;
      const float a1 = rbw < T ? qb[0] * scale : 0.f, a3 = rbw < T ? qb[4] * scale : 0.f;
      split_tf32(a0, qh[ks][0], ql[ks][0]);
      split_tf32(a1, qh[ks][1], ql[ks][1]);
      split_tf32(a2, qh[ks][2], ql[ks][2]);
      split_tf32(a3, qh[ks][3], ql[ks][3]);
    }
    float o[8][4];
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) o[dt][0] = o[dt][1] = o[dt][2] = o[dt][3] = 0.f;
    float m_a = -INFINITY, m_b = -INFINITY, l_a = 0.f, l_b = 0.f;
    for (int kb = 0; kb < Tp; kb += 64) {
      float sc[8][4];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) sc[nt][0] = sc[nt][1] = sc[nt][2] = sc[nt][3] = 0.f;
      // S = Q K^T:  B fragment (k = d, n = key): b0 = K[key = kb + 8 nt + g][8 ks + t], b1 = ...[8 ks + t + 4]
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
#pragma unroll
        for (int n4 = 0; n4 < 8; n4 += 4) {
          const float* kr = Ks + (kb + n4 * 8 + g) * ATT_LD + ks * 8 + t;
          float bf[8];
#pragma unroll
          for (int i = 0; i < 4; ++i) { bf[2 * i] = kr[i * 8 * ATT_LD]; bf[2 * i + 1] = kr[i * 8 * ATT_LD + 4]; }
          mma3x4(sc[n4], sc[n4 + 1], sc[n4 + 2], sc[n4 + 3], qh[ks], ql[ks], bf);
        }
      }
      // mask the padded keys, block row maxima (accumulator columns: keys kb + 8 nt + 2t, +1; rows g / g+8)
      float mx_a = -INFINITY, mx_b = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int key = kb + nt * 8 + 2 * t;
        if (key >= T) sc[nt][0] = sc[nt][2] = -INFINITY;
        if (key + 1 >= T) sc[nt][1] = sc[nt][3] = -INFINITY;
        mx_a = fmaxf(mx_a, fmaxf(sc[nt][0], sc[nt][1]));
        mx_b = fmaxf(mx_b, fmaxf(sc[nt][2], sc[nt][3]));
      }
      mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 1));
      mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 2));
      mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 1));
      mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 2));
      const float mn_a = fmaxf(m_a, mx_a), mn_b = fmaxf(m_b, mx_b);   // finite: every key block holds a valid key
      const float ca = expf(m_a - mn_a), cb = expf(m_b - mn_b);
      m_a = mn_a; m_b = mn_b;
      l_a *= ca; l_b *= cb;
#pragma unroll
      for (int dt = 0; dt < 8; ++dt) { o[dt][0] *= ca; o[dt][1] *= ca; o[dt][2] *= cb; o[dt][3] *= cb; }
      // O += P V:  A fragment of key step j = accumulator fragment of n-tile j (slot t <-> key 2t, slot t+4 <-> key 2t+1);
      // B fragment (k-slot, n = d): b0 = V[kb + 8 j + 2t][8 dt + g], b1 = V[kb + 8 j + 2t + 1][8 dt + g]
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (kb + j * 8 >= T) break;       // whole 8-key step is padding (warp-uniform)
        const float p0 = expf(sc[j][0] - mn_a), p1 = expf(sc[j][1] - mn_a);
        const float p2 = expf(sc[j][2] - mn_b), p3 = expf(sc[j][3] - mn_b);
        l_a += p0 + p1;
        l_b += p2 + p3;
        uint32_t ph[4], pl[4];
        split_tf32(p0, ph[0], pl[0]);   // a0: row g,   slot t
        split_tf32(p2, ph[1], pl[1]);   // a1: row g+8, slot t
        split_tf32(p1, ph[2], pl[2]);   // a2: row g,   slot t+4
        split_tf32(p3, ph[3], pl[3]);   // a3: row g+8, slot t+4
        const float* vr = Vs + (kb + j * 8 + 2 * t) * ATT_LD + g;
#pragma unroll
        for (int d4 = 0; d4 < 8; d4 += 4) {
          float bf[8];
#pragma unroll
          for (int i = 0; i < 4; ++i) { bf[2 * i] = vr[(d4 + i) * 8]; bf[2 * i + 1] = vr[ATT_LD + (d4 + i) * 8]; }
          mma3x4(o[d4], o[d4 + 1], o[d4 + 2], o[d4 + 3], ph, pl, bf);
        }
      }
    }
    l_a += __shfl_xor_sync(0xffffffffu, l_a, 1);
    l_a += __shfl_xor_sync(0xffffffffu, l_a, 2);
    l_b += __shfl_xor_sync(0xffffffffu, l_b, 1);
    l_b += __shfl_xor_sync(0xffffffffu, l_b, 2);
    const float ia = 1.0f / l_a, ib = 1.0f / l_b;
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) {
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int row = half ? rbw : ra;
        if (row >= T) continue;
        const float inv = half ? ib : ia;
        const float v0 = o[dt][half * 2] * inv, v1 = o[dt][half * 2 + 1] * inv;
        const size_t at = ((size_t)b * T + row) * (H * 64) + h * 64 + dt * 8 + 2 * t;
        if (out_lo) {
          const float h0 = __uint_as_float(__float_as_uint(v0) & 0xffffe000u), h1 = __uint_as_float(__float_as_uint(v1) & 0xffffe000u);
          *reinterpret_cast<float2*>(out + at) = make_float2(h0, h1);
          *reinterpret_cast<float2*>(out_lo + at) = make_float2(v0 - h0, v1 - h1);
        } else {
          *reinterpret_cast<float2*>(out + at) = make_float2(v0, v1);
        }
      }
    }
  }
}

// ---- same algorithm on the fp16 MMA shape (m16n8k16, half the MMA count of the tf32 version) ---------
// fp32 accuracy from a two-term fp16 split x = h + l (h = fp16(x), l = fp16(x - h): 22 significant bits),
// products l*h + h*l + h*h accumulated in fp32.  P is scaled by 2^10 before the split so its low part stays
// out of the fp16 subnormal range; q/k/v of a wav2vec2 layer are O(1..100), far inside the fp16 range.
constexpr int ATT_LDK = 72;   // K row stride (floats): 64-bit fragment loads conflict-free per half-warp
constexpr int ATT_LDV = 68;   // V row stride: 32-bit fragment loads conflict-free
__device__ __forceinline__ void split_h2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(x0, x1);
  const float2 f = __half22float2(h);
  const __half2 l = __floats2half2_rn(x0 - f.x, x1 - f.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}
__device__ __forceinline__ void mma_f16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(ATT_WARPS * 32, 1) attention_mma16_kernel(const float* __restrict__ qkv, float* __restrict__ out,
                                                                            float* __restrict__ out_lo, int T, int H, float scale) {
  extern __shared__ __align__(16) float sm[];
  const int Tp = (T + 63) & ~63;
  float* Ks = sm;                                  // [Tp][ATT_LDK]
  float* Vs = sm + (size_t)Tp * ATT_LDK;           // [Tp][ATT_LDV]
  const int bh = blockIdx.x, b = bh / H, h = bh % H;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int ld = 3 * H * 64;
  const float* base = qkv + (size_t)b * T * ld + h * 64;
  for (int i = tid; i < Tp * 16; i += ATT_WARPS * 32) {
    const int r = i >> 4, c4 = (i & 15) * 4;
    float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
    if (r < T) {
      kv = *reinterpret_cast<const float4*>(base + (size_t)r * ld + H * 64 + c4);
      vv = *reinterpret_cast<const float4*>(base + (size_t)r * ld + 2 * H * 64 + c4);
    }
    *reinterpret_cast<float4*>(Ks + r * ATT_LDK + c4) = kv;
    *reinterpret_cast<float4*>(Vs + r * ATT_LDV + c4) = vv;
  }
  __syncthreads();
  const int nrb = (T + 15) >> 4;
  for (int rb = warp; rb < nrb; rb += ATT_WARPS) {
    const int ra = rb * 16 + g, rbw = ra + 8;
    // Q fragments per 16-wide d step: a0 = (row g, d 2t..2t+1), a1 = (row g+8, same), a2 = (row g, d 2t+8..9), a3 = (row g+8, same)
    uint32_t qh[4][4], ql[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      float2 x0 = make_float2(0.f, 0.f), x1 = x0, x2 = x0, x3 = x0;
      if (ra < T) {
        x0 = *reinterpret_cast<const float2*>(base + (size_t)ra * ld + ks * 16 + 2 * t);
        x2 = *reinterpret_cast<const float2*>(base + (size_t)ra * ld + ks * 16 + 2 * t + 8);
      }
      if (rbw < T) {
        x1 = *reinterpret_cast<const float2*>(base + (size_t)rbw * ld + ks * 16 + 2 * t);
        x3 = *reinterpret_cast<const float2*>(base + (size_t)rbw * ld + ks * 16 + 2 * t + 8);
      }
      split_h2(x0.x * scale, x0.y * scale, qh[ks][0], ql[ks][0]);
      split_h2(x1.x * scale, x1.y * scale, qh[ks][1], ql[ks][1]);
      split_h2(x2.x * scale, x2.y * scale, qh[ks][2], ql[ks][2]);
      split_h2(x3.x * scale, x3.y * scale, qh[ks][3], ql[ks][3]);
    }
    float o[8][4];
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) o[dt][0] = o[dt][1] = o[dt][2] = o[dt][3] = 0.f;
    float m_a = -INFINITY, m_b = -INFINITY, l_a = 0.f, l_b = 0.f;
    for (int kb = 0; kb < Tp; kb += 64) {
      float sc[8][4];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) sc[nt][0] = sc[nt][1] = sc[nt][2] = sc[nt][3] = 0.f;
      // S = Q K^T: B fragment (k = d, n = key): b0 = K[key = kb + 8 nt + g][16 ks + 2t .. +1], b1 = ...[16 ks + 2t + 8 .. +9]
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
          const float* kr = Ks + (kb + nt * 8 + g) * ATT_LDK + ks * 16 + 2 * t;
          const float2 k0 = *reinterpret_cast<const float2*>(kr), k1 = *reinterpret_cast<const float2*>(kr + 8);
          uint32_t bh0, bl0, bh1, bl1;
          split_h2(k0.x, k0.y, bh0, bl0);
          split_h2(k1.x, k1.y, bh1, bl1);
          mma_f16(sc[nt], ql[ks], bh0, bh1);
          mma_f16(sc[nt], qh[ks], bl0, bl1);
          mma_f16(sc[nt], qh[ks], bh0, bh1);
        }
      }
      float mx_a = -INFINITY, mx_b = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int key = kb + nt * 8 + 2 * t;
        if (key >= T) sc[nt][0] = sc[nt][2] = -INFINITY;
        if (key + 1 >= T) sc[nt][1] = sc[nt][3] = -INFINITY;
        mx_a = fmaxf(mx_a, fmaxf(sc[nt][0], sc[nt][1]));
        mx_b = fmaxf(mx_b, fmaxf(sc[nt][2], sc[nt][3]));
      }
      mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 1));
      mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 2));
      mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 1));
      mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 2));
      const float mn_a = fmaxf(m_a, mx_a), mn_b = fmaxf(m_b, mx_b);
      const float ca = expf(m_a - mn_a), cb = expf(m_b - mn_b);
      m_a = mn_a; m_b = mn_b;
      l_a *= ca; l_b *= cb;
#pragma unroll
      for (int dt = 0; dt < 8; ++dt) { o[dt][0] *= ca; o[dt][1] *= ca; o[dt][2] *= cb; o[dt][3] *= cb; }
      // O += P V per 16-key step j2: A = accumulator fragments of n-tiles 2 j2 (keys 2t, 2t+1) and 2 j2 + 1 (keys 2t+8, 2t+9);
      // B fragment (k = key, n = d): b0 = V[kb + 16 j2 + 2t .. +1][8 dt + g], b1 = V[kb + 16 j2 + 2t + 8 .. +9][8 dt + g]
#pragma unroll
      for (int j2 = 0; j2 < 4; ++j2) {
        if (kb + j2 * 16 >= T) break;     // whole 16-key step is padding (warp-uniform)
        float p[8];
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          p[q * 4 + 0] = expf(sc[2 * j2 + q][0] - mn_a);
          p[q * 4 + 1] = expf(sc[2 * j2 + q][1] - mn_a);
          p[q * 4 + 2] = expf(sc[2 * j2 + q][2] - mn_b);
          p[q * 4 + 3] = expf(sc[2 * j2 + q][3] - mn_b);
        }
        l_a += (p[0] + p[1]) + (p[4] + p[5]);
        l_b += (p[2] + p[3]) + (p[6] + p[7]);
        uint32_t ph[4], pl[4];
        split_h2(p[0] * 1024.f, p[1] * 1024.f, ph[0], pl[0]);   // a0: row g,   keys 2t, 2t+1
        split_h2(p[2] * 1024.f, p[3] * 1024.f, ph[1], pl[1]);   // a1: row g+8
        split_h2(p[4] * 1024.f, p[5] * 1024.f, ph[2], pl[2]);   // a2: row g,   keys 2t+8, 2t+9
        split_h2(p[6] * 1024.f, p[7] * 1024.f, ph[3], pl[3]);   // a3: row g+8
        const float* vr = Vs + (kb + j2 * 16 + 2 * t) * ATT_LDV + g;
#pragma unroll
        for (int dt = 0; dt < 8; ++dt) {
          uint32_t bh0, bl0, bh1, bl1;
          split_h2(vr[dt * 8], vr[ATT_LDV + dt * 8], bh0, bl0);
          split_h2(vr[8 * ATT_LDV + dt * 8], vr[9 * ATT_LDV + dt * 8], bh1, bl1);
          mma_f16(o[dt], pl, bh0, bh1);
          mma_f16(o[dt], ph, bl0, bl1);
          mma_f16(o[dt], ph, bh0, bh1);
        }
      }
    }
    l_a += __shfl_xor_sync(0xffffffffu, l_a, 1);
    l_a += __shfl_xor_sync(0xffffffffu, l_a, 2);
    l_b += __shfl_xor_sync(0xffffffffu, l_b, 1);
    l_b += __shfl_xor_sync(0xffffffffu, l_b, 2);
    const float ia = 1.0f / (l_a * 1024.f), ib = 1.0f / (l_b * 1024.f);
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) {
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int row = half ? rbw : ra;
        if (row >= T) continue;
        const float inv = half ? ib : ia;
        const float v0 = o[dt][half * 2] * inv, v1 = o[dt][half * 2 + 1] * inv;
        const size_t at = ((size_t)b * T + row) * (H * 64) + h * 64 + dt * 8 + 2 * t;
        if (out_lo) {
          const float h0 = __uint_as_float(__float_as_uint(v0) & 0xffffe000u), h1 = __uint_as_float(__float_as_uint(v1) & 0xffffe000u);
          *reinterpret_cast<float2*>(out + at) = make_float2(h0, h1);
          *reinterpret_cast<float2*>(out_lo + at) = make_float2(v0 - h0, v1 - h1);
        } else {
          *reinterpret_cast<float2*>(out + at) = make_float2(v0, v1);
        }
      }
    }
  }
}

// ---- fp16-split attention with K and V split ONCE per CTA -------------------------------------------
// attention_mma16_kernel re-splits every K / V fragment in every warp and row block (19 times per element at
// T = 300) and is issue-bound on those conversions (ncu: issue slots 52 % busy, HMMA pipe 33 %).  Here the fill
// phase stores K as two fp16 planes [key][d] (hi, lo) and V as two transposed fp16 planes [d][key], so a B
// fragment register is one 32-bit shared load (two adjacent d for K, two adjacent keys for V^T) and the inner
// loops are 4 LDS + 3 HMMA per product triple.  Same bytes of shared memory as the fp32 copies.
constexpr int ATT_KW = 36;    // K plane row stride in 32-bit words (72 halves): fragment loads conflict-free

// One 64-key block of the online softmax, the step of both kernels below: scores of the warp's 16 query rows (fragments
// qh / ql, already scaled) against keys [kb, kb + 64) of the shared planes -- clip keys key0 + kb + ... --, keys >= T
// masked, the running max / sum update, O += P V.  The tensor core's fp32 accumulator truncates, so P V of the block
// accumulates into a fresh fragment (12 MMAs deep) that is added to O with round-to-nearest adds: the truncation does not
// build up with the clip length, and a block gives the same bits however the keys are staged (whole clip or chunks).
__device__ __forceinline__ void att16_block(const uint32_t* Kh, const uint32_t* Kl, const uint32_t* Vh, const uint32_t* Vl, int VW, int kb,
                                            int key0, int T, const uint32_t (&qh)[4][4], const uint32_t (&ql)[4][4], float (&o)[8][4],
                                            float& m_a, float& m_b, float& l_a, float& l_b, int g, int t) {
  float sc[8][4];
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) sc[nt][0] = sc[nt][1] = sc[nt][2] = sc[nt][3] = 0.f;
  // b0 = K[key = kb + 8 nt + g][d = 16 ks + 2t, +1] = word (8 ks + t) of the key's row, b1 = word (8 ks + t + 4)
  // (the three products of one accumulator are issued a whole pass apart, so dependent HMMAs never queue back to back)
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    uint32_t bh0[8], bh1[8], bl0[8], bl1[8];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int w = (kb + nt * 8 + g) * ATT_KW + ks * 8 + t;
      bh0[nt] = Kh[w]; bh1[nt] = Kh[w + 4]; bl0[nt] = Kl[w]; bl1[nt] = Kl[w + 4];
    }
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) mma_f16(sc[nt], ql[ks], bh0[nt], bh1[nt]);
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) mma_f16(sc[nt], qh[ks], bl0[nt], bl1[nt]);
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) mma_f16(sc[nt], qh[ks], bh0[nt], bh1[nt]);
  }
  float mx_a = -INFINITY, mx_b = -INFINITY;
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) {
    const int key = key0 + kb + nt * 8 + 2 * t;
    if (key >= T) sc[nt][0] = sc[nt][2] = -INFINITY;
    if (key + 1 >= T) sc[nt][1] = sc[nt][3] = -INFINITY;
    mx_a = fmaxf(mx_a, fmaxf(sc[nt][0], sc[nt][1]));
    mx_b = fmaxf(mx_b, fmaxf(sc[nt][2], sc[nt][3]));
  }
  mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 1));
  mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 2));
  mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 1));
  mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 2));
  const float mn_a = fmaxf(m_a, mx_a), mn_b = fmaxf(m_b, mx_b);   // finite: every block holds a key < T
  const float ca = expf(m_a - mn_a), cb = expf(m_b - mn_b);
  m_a = mn_a; m_b = mn_b;
  l_a *= ca; l_b *= cb;
#pragma unroll
  for (int dt = 0; dt < 8; ++dt) { o[dt][0] *= ca; o[dt][1] *= ca; o[dt][2] *= cb; o[dt][3] *= cb; }
  float oc[8][4];
#pragma unroll
  for (int dt = 0; dt < 8; ++dt) oc[dt][0] = oc[dt][1] = oc[dt][2] = oc[dt][3] = 0.f;
  // b0 = V^T[d = 8 dt + g][keys kb + 16 j2 + 2t, +1] = word ((kb + 16 j2) / 2 + t) of row d, b1 = that + 4
#pragma unroll
  for (int j2 = 0; j2 < 4; ++j2) {
    if (key0 + kb + j2 * 16 >= T) break;     // whole 16-key step is padding (warp-uniform)
    float p[8];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      p[q * 4 + 0] = expf(sc[2 * j2 + q][0] - mn_a);
      p[q * 4 + 1] = expf(sc[2 * j2 + q][1] - mn_a);
      p[q * 4 + 2] = expf(sc[2 * j2 + q][2] - mn_b);
      p[q * 4 + 3] = expf(sc[2 * j2 + q][3] - mn_b);
    }
    l_a += (p[0] + p[1]) + (p[4] + p[5]);
    l_b += (p[2] + p[3]) + (p[6] + p[7]);
    uint32_t ph[4], pl[4];
    split_h2(p[0] * 1024.f, p[1] * 1024.f, ph[0], pl[0]);
    split_h2(p[2] * 1024.f, p[3] * 1024.f, ph[1], pl[1]);
    split_h2(p[4] * 1024.f, p[5] * 1024.f, ph[2], pl[2]);
    split_h2(p[6] * 1024.f, p[7] * 1024.f, ph[3], pl[3]);
    uint32_t bh0[8], bh1[8], bl0[8], bl1[8];
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) {
      const int w = (dt * 8 + g) * VW + (kb >> 1) + j2 * 8 + t;
      bh0[dt] = Vh[w]; bh1[dt] = Vh[w + 4]; bl0[dt] = Vl[w]; bl1[dt] = Vl[w + 4];
    }
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) mma_f16(oc[dt], pl, bh0[dt], bh1[dt]);
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) mma_f16(oc[dt], ph, bl0[dt], bl1[dt]);
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) mma_f16(oc[dt], ph, bh0[dt], bh1[dt]);
  }
#pragma unroll
  for (int dt = 0; dt < 8; ++dt) { o[dt][0] += oc[dt][0]; o[dt][1] += oc[dt][1]; o[dt][2] += oc[dt][2]; o[dt][3] += oc[dt][3]; }
}

__global__ void __launch_bounds__(ATT_WARPS * 32, 1) attention_mma16p_kernel(const float* __restrict__ qkv, float* __restrict__ out,
                                                                             float* __restrict__ out_lo, unsigned short* __restrict__ o_h16,
                                                                             unsigned short* __restrict__ o_l16, int T, int H, float scale) {
  extern __shared__ __align__(16) uint32_t smw[];
  const int Tp = (T + 63) & ~63;
  const int VW = Tp / 2 + 4;                       // V^T plane row stride in words (Tp halves + 8 pad)
  uint32_t* Kh = smw;                              // [Tp][ATT_KW]   pairs (d, d+1)
  uint32_t* Kl = Kh + (size_t)Tp * ATT_KW;
  uint32_t* Vh = Kl + (size_t)Tp * ATT_KW;         // [64][VW]       pairs (key, key+1)
  uint32_t* Vl = Vh + (size_t)64 * VW;
  const int bh = blockIdx.x, b = bh / H, h = bh % H;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int ld = 3 * H * 64;
  const float* base = qkv + (size_t)b * T * ld + h * 64;
  // fill K planes: one (key, d-pair) per iteration
  for (int i = tid; i < Tp * 32; i += ATT_WARPS * 32) {
    const int r = i >> 5, dp = i & 31;
    float2 kv = make_float2(0.f, 0.f);
    if (r < T) kv = *reinterpret_cast<const float2*>(base + (size_t)r * ld + H * 64 + 2 * dp);
    uint32_t hi, lo;
    split_h2(kv.x, kv.y, hi, lo);
    Kh[r * ATT_KW + dp] = hi;
    Kl[r * ATT_KW + dp] = lo;
  }
  // fill V^T planes: one (key-pair, d) per iteration, d fastest across lanes for coalesced global reads
  for (int i = tid; i < (Tp / 2) * 64; i += ATT_WARPS * 32) {
    const int kp = i >> 6, d = i & 63, r = 2 * kp;
    const float v0 = r < T ? base[(size_t)r * ld + 2 * H * 64 + d] : 0.f;
    const float v1 = r + 1 < T ? base[(size_t)(r + 1) * ld + 2 * H * 64 + d] : 0.f;
    uint32_t hi, lo;
    split_h2(v0, v1, hi, lo);
    Vh[d * VW + kp] = hi;
    Vl[d * VW + kp] = lo;
  }
  __syncthreads();
  const int nrb = (T + 15) >> 4;
  for (int rb = warp; rb < nrb; rb += ATT_WARPS) {
    const int ra = rb * 16 + g, rbw = ra + 8;
    uint32_t qh[4][4], ql[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      float2 x0 = make_float2(0.f, 0.f), x1 = x0, x2 = x0, x3 = x0;
      if (ra < T) {
        x0 = *reinterpret_cast<const float2*>(base + (size_t)ra * ld + ks * 16 + 2 * t);
        x2 = *reinterpret_cast<const float2*>(base + (size_t)ra * ld + ks * 16 + 2 * t + 8);
      }
      if (rbw < T) {
        x1 = *reinterpret_cast<const float2*>(base + (size_t)rbw * ld + ks * 16 + 2 * t);
        x3 = *reinterpret_cast<const float2*>(base + (size_t)rbw * ld + ks * 16 + 2 * t + 8);
      }
      split_h2(x0.x * scale, x0.y * scale, qh[ks][0], ql[ks][0]);
      split_h2(x1.x * scale, x1.y * scale, qh[ks][1], ql[ks][1]);
      split_h2(x2.x * scale, x2.y * scale, qh[ks][2], ql[ks][2]);
      split_h2(x3.x * scale, x3.y * scale, qh[ks][3], ql[ks][3]);
    }
    float o[8][4];
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) o[dt][0] = o[dt][1] = o[dt][2] = o[dt][3] = 0.f;
    float m_a = -INFINITY, m_b = -INFINITY, l_a = 0.f, l_b = 0.f;
    for (int kb = 0; kb < Tp; kb += 64) att16_block(Kh, Kl, Vh, Vl, VW, kb, 0, T, qh, ql, o, m_a, m_b, l_a, l_b, g, t);
    l_a += __shfl_xor_sync(0xffffffffu, l_a, 1);
    l_a += __shfl_xor_sync(0xffffffffu, l_a, 2);
    l_b += __shfl_xor_sync(0xffffffffu, l_b, 1);
    l_b += __shfl_xor_sync(0xffffffffu, l_b, 2);
    const float ia = 1.0f / (l_a * 1024.f), ib = 1.0f / (l_b * 1024.f);
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) {
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int row = half ? rbw : ra;
        if (row >= T) continue;
        const float inv = half ? ib : ia;
        const float v0 = o[dt][half * 2] * inv, v1 = o[dt][half * 2 + 1] * inv;
        const size_t at = ((size_t)b * T + row) * (H * 64) + h * 64 + dt * 8 + 2 * t;
        if (o_h16) {   // fp16-split copy for the out_proj GEMM; `out` keeps the full value
          *reinterpret_cast<float2*>(out + at) = make_float2(v0, v1);
          uint32_t hh, ll;
          split_h2(v0, v1, hh, ll);
          *reinterpret_cast<uint32_t*>(o_h16 + at) = hh;
          *reinterpret_cast<uint32_t*>(o_l16 + at) = ll;
        } else if (out_lo) {
          const float h0 = __uint_as_float(__float_as_uint(v0) & 0xffffe000u), h1 = __uint_as_float(__float_as_uint(v1) & 0xffffe000u);
          *reinterpret_cast<float2*>(out + at) = make_float2(h0, h1);
          *reinterpret_cast<float2*>(out_lo + at) = make_float2(v0 - h0, v1 - h1);
        } else {
          *reinterpret_cast<float2*>(out + at) = make_float2(v0, v1);
        }
      }
    }
  }
}

// Same arithmetic (att16_block: the same bits as the resident kernel at every T it can hold), KV-TILED for long clips (flash-attention style): the keys / values of a head are staged CH at a time,
// every warp owns ONE 16-row query block and keeps its online-softmax state in registers across the chunks; grid =
// (clip x head, query tiles of 16 x ATT_WARPS rows).  No limit on the clip length (the resident variant above needs the
// whole sequence in shared memory: <= 384 frames = 12.8 s).
__global__ void __launch_bounds__(ATT_WARPS * 32, 1) attention_mma16t_kernel(const float* __restrict__ qkv, float* __restrict__ out,
                                                                             float* __restrict__ out_lo, unsigned short* __restrict__ o_h16,
                                                                             unsigned short* __restrict__ o_l16, int T, int H, float scale, int CH) {
  extern __shared__ __align__(16) uint32_t smw[];
  const int Tp = CH;                               // keys resident per chunk (multiple of 64)
  const int VW = Tp / 2 + 4;                       // V^T plane row stride in words (Tp halves + 8 pad)
  uint32_t* Kh = smw;                              // [Tp][ATT_KW]   pairs (d, d+1)
  uint32_t* Kl = Kh + (size_t)Tp * ATT_KW;
  uint32_t* Vh = Kl + (size_t)Tp * ATT_KW;         // [64][VW]       pairs (key, key+1)
  uint32_t* Vl = Vh + (size_t)64 * VW;
  const int bh = blockIdx.x, b = bh / H, h = bh % H;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int ld = 3 * H * 64;
  const float* base = qkv + (size_t)b * T * ld + h * 64;
  const int nrb = (T + 15) >> 4;
  const int rb = blockIdx.y * ATT_WARPS + warp;      // one 16-row query block per warp
  const bool live = rb < nrb;
  {
    const int ra = rb * 16 + g, rbw = ra + 8;
    uint32_t qh[4][4], ql[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      float2 x0 = make_float2(0.f, 0.f), x1 = x0, x2 = x0, x3 = x0;
      if (ra < T) {
        x0 = *reinterpret_cast<const float2*>(base + (size_t)ra * ld + ks * 16 + 2 * t);
        x2 = *reinterpret_cast<const float2*>(base + (size_t)ra * ld + ks * 16 + 2 * t + 8);
      }
      if (rbw < T) {
        x1 = *reinterpret_cast<const float2*>(base + (size_t)rbw * ld + ks * 16 + 2 * t);
        x3 = *reinterpret_cast<const float2*>(base + (size_t)rbw * ld + ks * 16 + 2 * t + 8);
      }
      split_h2(x0.x * scale, x0.y * scale, qh[ks][0], ql[ks][0]);
      split_h2(x1.x * scale, x1.y * scale, qh[ks][1], ql[ks][1]);
      split_h2(x2.x * scale, x2.y * scale, qh[ks][2], ql[ks][2]);
      split_h2(x3.x * scale, x3.y * scale, qh[ks][3], ql[ks][3]);
    }
    float o[8][4];
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) o[dt][0] = o[dt][1] = o[dt][2] = o[dt][3] = 0.f;
    float m_a = -INFINITY, m_b = -INFINITY, l_a = 0.f, l_b = 0.f;
    for (int c0 = 0; c0 < T; c0 += CH) {
      if (c0) __syncthreads();                       // every warp is done with the previous chunk's planes
    // fill K planes: one (key, d-pair) per iteration
    for (int i = tid; i < Tp * 32; i += ATT_WARPS * 32) {
      const int r = i >> 5, dp = i & 31;
      float2 kv = make_float2(0.f, 0.f);
      if (c0 + r < T) kv = *reinterpret_cast<const float2*>(base + (size_t)(c0 + r) * ld + H * 64 + 2 * dp);
      uint32_t hi, lo;
      split_h2(kv.x, kv.y, hi, lo);
      Kh[r * ATT_KW + dp] = hi;
      Kl[r * ATT_KW + dp] = lo;
    }
    // fill V^T planes: one (key-pair, d) per iteration, d fastest across lanes for coalesced global reads
    for (int i = tid; i < (Tp / 2) * 64; i += ATT_WARPS * 32) {
      const int kp = i >> 6, d = i & 63, r = 2 * kp;
      const float v0 = c0 + r < T ? base[(size_t)(c0 + r) * ld + 2 * H * 64 + d] : 0.f;
      const float v1 = c0 + r + 1 < T ? base[(size_t)(c0 + r + 1) * ld + 2 * H * 64 + d] : 0.f;
      uint32_t hi, lo;
      split_h2(v0, v1, hi, lo);
      Vh[d * VW + kp] = hi;
      Vl[d * VW + kp] = lo;
    }
      __syncthreads();
      for (int kb = 0; live && kb < Tp && c0 + kb < T; kb += 64) att16_block(Kh, Kl, Vh, Vl, VW, kb, c0, T, qh, ql, o, m_a, m_b, l_a, l_b, g, t);
    }
    l_a += __shfl_xor_sync(0xffffffffu, l_a, 1);
    l_a += __shfl_xor_sync(0xffffffffu, l_a, 2);
    l_b += __shfl_xor_sync(0xffffffffu, l_b, 1);
    l_b += __shfl_xor_sync(0xffffffffu, l_b, 2);
    const float ia = 1.0f / (l_a * 1024.f), ib = 1.0f / (l_b * 1024.f);
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) {
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int row = half ? rbw : ra;
        if (!live || row >= T) continue;
        const float inv = half ? ib : ia;
        const float v0 = o[dt][half * 2] * inv, v1 = o[dt][half * 2 + 1] * inv;
        const size_t at = ((size_t)b * T + row) * (H * 64) + h * 64 + dt * 8 + 2 * t;
        if (o_h16) {   // fp16-split copy for the out_proj GEMM; `out` keeps the full value
          *reinterpret_cast<float2*>(out + at) = make_float2(v0, v1);
          uint32_t hh, ll;
          split_h2(v0, v1, hh, ll);
          *reinterpret_cast<uint32_t*>(o_h16 + at) = hh;
          *reinterpret_cast<uint32_t*>(o_l16 + at) = ll;
        } else if (out_lo) {
          const float h0 = __uint_as_float(__float_as_uint(v0) & 0xffffe000u), h1 = __uint_as_float(__float_as_uint(v1) & 0xffffe000u);
          *reinterpret_cast<float2*>(out + at) = make_float2(h0, h1);
          *reinterpret_cast<float2*>(out_lo + at) = make_float2(v0 - h0, v1 - h1);
        } else {
          *reinterpret_cast<float2*>(out + at) = make_float2(v0, v1);
        }
      }
    }
  }
}


// ---- positional conv embedding (Conv1d 768 -> 768, k = 128, groups = 16, pad 64) on HMMA ---------------------------
// Per (clip, group) the conv is a [T x 6144] Toeplitz matrix times a [6144 x 48] weight block: N = 48 is too narrow for a
// wgmma tile, and as an fp32 FFMA GEMM it is a large share of the face forward.  Here one CTA owns 320 output rows of
// one (clip, group): the group's 48 input channels of the 447-row window are split ONCE into two fp16 planes in shared
// memory (x = h + l, as everywhere else), a tap is a row shift of the window (A fragments are plain 32-bit shared loads at
// row m + tap), the weights arrive pre-split and pre-scaled in 4-tap chunks through a cp.async double buffer, and every
// (tap, 16-channel) step is 3 HMMA m16n8k16 per 16 x 8 output block (l*h + h*l + h*h).  Each chunk accumulates into fresh
// fp32 accumulators that are then added (round-to-nearest) to the running sum: the tensor core's accumulator truncates.
constexpr int PC_WARPS = 10, PC_MT = 2;
constexpr int PC_ROWS = PC_WARPS * PC_MT * 16;      // 320 output rows per CTA
constexpr int PC_XR = PC_ROWS + 128;                // window rows (127-row halo)
constexpr int PC_LD = 56;                           // row stride in halves (48 + 8 pad = 28 words: fragment loads conflict-free)
constexpr int PC_TAPS = 4;                          // taps per weight chunk
constexpr int PC_WCH = PC_TAPS * 2 * 48 * PC_LD;    // halves per chunk: [tap][plane][n][PC_LD]
constexpr size_t PC_SMEM = ((size_t)2 * PC_XR * PC_LD + (size_t)2 * PC_WCH) * sizeof(unsigned short);

__global__ void __launch_bounds__(PC_WARPS * 32, 1) posconv_mma_kernel(Act3 x, const unsigned short* __restrict__ W16,
                                                                       const float* __restrict__ bias, float unscale, Act3 out) {
  extern __shared__ __align__(16) unsigned short pcs[];
  unsigned short* Xh = pcs;
  unsigned short* Xl = Xh + PC_XR * PC_LD;
  unsigned short* Wb = Xl + PC_XR * PC_LD;          // two chunk buffers
  const int b = blockIdx.x / 16, grp = blockIdx.x % 16, t0 = blockIdx.y * PC_ROWS;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int T = out.T;
  const unsigned short* wsrc = W16 + (size_t)grp * 128 * 2 * 48 * PC_LD;
  auto fetch = [&](int ch) {
    const unsigned short* src = wsrc + (size_t)ch * PC_WCH;
    const uint32_t dst = (uint32_t)__cvta_generic_to_shared(Wb + (ch & 1) * PC_WCH);
    for (int i = tid; i < PC_WCH / 8; i += PC_WARPS * 32)
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + i * 16), "l"(src + i * 8) : "memory");
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  fetch(0);
  // window row r holds time t0 + r - 64 (the conv's left padding of 64 lives in the activation's pad rows)
  for (int i = tid; i < PC_XR * 12; i += PC_WARPS * 32) {
    const int r = i / 12, c4 = (i - r * 12) * 4, tt = t0 + r - 64;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (tt < T + 64) v = *reinterpret_cast<const float4*>(x.row(b, tt) + grp * 48 + c4);
    uint32_t h0, l0, h1, l1;
    split_h2(v.x, v.y, h0, l0);
    split_h2(v.z, v.w, h1, l1);
    *reinterpret_cast<uint2*>(Xh + r * PC_LD + c4) = make_uint2(h0, h1);
    *reinterpret_cast<uint2*>(Xl + r * PC_LD + c4) = make_uint2(l0, l1);
  }
  float acc[PC_MT][6][4];
#pragma unroll
  for (int mt = 0; mt < PC_MT; ++mt)
#pragma unroll
    for (int nt = 0; nt < 6; ++nt) acc[mt][nt][0] = acc[mt][nt][1] = acc[mt][nt][2] = acc[mt][nt][3] = 0.f;
  bool live[PC_MT];
#pragma unroll
  for (int mt = 0; mt < PC_MT; ++mt) live[mt] = t0 + (warp * PC_MT + mt) * 16 < T;   // warp-uniform

  for (int ch = 0; ch < 128 / PC_TAPS; ++ch) {
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();                                 // chunk ch landed; every warp is done with chunk ch - 1 (and, first time, the window is filled)
    if (ch + 1 < 128 / PC_TAPS) fetch(ch + 1);
    const unsigned short* Wc = Wb + (ch & 1) * PC_WCH;
    float fa[PC_MT][6][4];
#pragma unroll
    for (int mt = 0; mt < PC_MT; ++mt)
#pragma unroll
      for (int nt = 0; nt < 6; ++nt) fa[mt][nt][0] = fa[mt][nt][1] = fa[mt][nt][2] = fa[mt][nt][3] = 0.f;
#pragma unroll 1
    for (int tp = 0; tp < PC_TAPS; ++tp) {
      const int k = ch * PC_TAPS + tp;
      const unsigned short* Wh = Wc + (size_t)tp * 2 * 48 * PC_LD;
      const unsigned short* Wl = Wh + 48 * PC_LD;
#pragma unroll
      for (int cs = 0; cs < 3; ++cs) {
        const int c0 = cs * 16 + 2 * t;
        uint32_t bh0[6], bh1[6], bl0[6], bl1[6];
#pragma unroll
        for (int nt = 0; nt < 6; ++nt) {
          const int w = (nt * 8 + g) * PC_LD + c0;
          bh0[nt] = *reinterpret_cast<const uint32_t*>(Wh + w); bh1[nt] = *reinterpret_cast<const uint32_t*>(Wh + w + 8);
          bl0[nt] = *reinterpret_cast<const uint32_t*>(Wl + w); bl1[nt] = *reinterpret_cast<const uint32_t*>(Wl + w + 8);
        }
#pragma unroll
        for (int mt = 0; mt < PC_MT; ++mt) {
          if (!live[mt]) continue;
          const int r = (warp * PC_MT + mt) * 16 + g + k;
          uint32_t ah[4], al[4];
          ah[0] = *reinterpret_cast<const uint32_t*>(Xh + r * PC_LD + c0);       al[0] = *reinterpret_cast<const uint32_t*>(Xl + r * PC_LD + c0);
          ah[1] = *reinterpret_cast<const uint32_t*>(Xh + (r + 8) * PC_LD + c0); al[1] = *reinterpret_cast<const uint32_t*>(Xl + (r + 8) * PC_LD + c0);
          ah[2] = *reinterpret_cast<const uint32_t*>(Xh + r * PC_LD + c0 + 8);   al[2] = *reinterpret_cast<const uint32_t*>(Xl + r * PC_LD + c0 + 8);
          ah[3] = *reinterpret_cast<const uint32_t*>(Xh + (r + 8) * PC_LD + c0 + 8);
          al[3] = *reinterpret_cast<const uint32_t*>(Xl + (r + 8) * PC_LD + c0 + 8);
#pragma unroll
          for (int nt = 0; nt < 6; ++nt) mma_f16(fa[mt][nt], al, bh0[nt], bh1[nt]);
#pragma unroll
          for (int nt = 0; nt < 6; ++nt) mma_f16(fa[mt][nt], ah, bl0[nt], bl1[nt]);
#pragma unroll
          for (int nt = 0; nt < 6; ++nt) mma_f16(fa[mt][nt], ah, bh0[nt], bh1[nt]);
        }
      }
    }
#pragma unroll
    for (int mt = 0; mt < PC_MT; ++mt)
#pragma unroll
      for (int nt = 0; nt < 6; ++nt) {
        acc[mt][nt][0] += fa[mt][nt][0]; acc[mt][nt][1] += fa[mt][nt][1];
        acc[mt][nt][2] += fa[mt][nt][2]; acc[mt][nt][3] += fa[mt][nt][3];
      }
  }
#pragma unroll
  for (int mt = 0; mt < PC_MT; ++mt) {
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int row = t0 + (warp * PC_MT + mt) * 16 + g + half * 8;
      if (row >= T) continue;
      float* orow = out.row(b, row) + grp * 48;
#pragma unroll
      for (int nt = 0; nt < 6; ++nt) {
        const int n = nt * 8 + 2 * t;
        float v0 = acc[mt][nt][half * 2] * unscale + bias[grp * 48 + n];
        float v1 = acc[mt][nt][half * 2 + 1] * unscale + bias[grp * 48 + n + 1];
        v0 = 0.5f * v0 * (1.0f + erff(v0 * 0.70710678118654752440f));
        v1 = 0.5f * v1 * (1.0f + erff(v1 * 0.70710678118654752440f));
        *reinterpret_cast<float2*>(orow + n) = make_float2(v0, v1);
      }
    }
  }
}

// host pack of pos_conv_embed.conv.weight [768][48][128] -> fp16 planes [group][tap][plane][n][PC_LD] of W * 2^shift
static unsigned short* pack_posconv16(ts_engine* e, const float* w, float* unscale) {
  float mx = 0.f;
  for (size_t i = 0; i < (size_t)768 * 48 * 128; ++i) mx = std::max(mx, std::fabs(w[i]));
  const int shift = split16_shift(mx);
  const float sc = std::ldexp(1.0f, shift);
  *unscale = std::ldexp(1.0f, -shift);
  std::vector<unsigned short> P((size_t)16 * 128 * 2 * 48 * PC_LD, 0);
  for (int grp = 0; grp < 16; ++grp)
    for (int k = 0; k < 128; ++k)
      for (int n = 0; n < 48; ++n)
        for (int c = 0; c < 48; ++c) {
          const float v = w[((size_t)(grp * 48 + n) * 48 + c) * 128 + k] * sc;
          const __half h = __float2half_rn(v);
          const __half l = __float2half_rn(v - __half2float(h));
          const size_t at = ((((size_t)grp * 128 + k) * 2) * 48 + n) * PC_LD + c;
          P[at] = __half_as_ushort(h);
          P[at + (size_t)48 * PC_LD] = __half_as_ushort(l);
        }
  return e->upload(P);
}

// attention kernels by number (ts_debug_attention's numbering; TS_ATT_MMA 0..2 name the first three)
enum { ATT_FFMA = 0, ATT_TF32 = 1, ATT_MMA16 = 2, ATT_MMA16P = 3, ATT_MMA16T = 4 };
constexpr int ATT_CH = 320;                     // keys per chunk of the KV-tiled kernel in the face forward
constexpr size_t ATT_SMEM_MAX = 220 * 1024;
static size_t att_ffma_smem(int QT, int T) { return (size_t)(QT * 65 + 64 * 65 + QT * ((T + 63) & ~63)) * sizeof(float); }
// query rows per CTA of the FFMA kernel: the most whose score tile fits (0: none, T > 3136)
static int att_ffma_qt(int T) {
  for (int QT = 64; QT >= 16; QT /= 2)
    if (att_ffma_smem(QT, T) <= ATT_SMEM_MAX) return QT;
  return 0;
}
// dynamic shared memory of attention kernel `k` for a clip of T frames (ch: keys per chunk of ATT_MMA16T); 0 when the
// kernel cannot hold the clip
static size_t att_smem(int k, int T, int ch) {
  const size_t Tp = (size_t)((T + 63) & ~63);
  size_t b;
  switch (k) {
    case ATT_FFMA: { const int QT = att_ffma_qt(T); return QT ? att_ffma_smem(QT, T) : 0; }
    case ATT_TF32: b = 2 * Tp * ATT_LD * sizeof(float); break;
    case ATT_MMA16: b = Tp * (ATT_LDK + ATT_LDV) * sizeof(float); break;
    case ATT_MMA16P: b = (2 * Tp * ATT_KW + 2 * 64 * (Tp / 2 + 4)) * sizeof(uint32_t); break;
    default: b = ((size_t)2 * ch * ATT_KW + (size_t)2 * 64 * (ch / 2 + 4)) * sizeof(uint32_t); break;
  }
  return b <= ATT_SMEM_MAX ? b : 0;
}
// the kernel the face forward runs for a clip of T frames: TS_ATT_MMA picks the family, the clip length the member
static int att_kernel_for(int T) {
  static const int att_mode = getenv("TS_ATT_MMA") ? atoi(getenv("TS_ATT_MMA")) : 3;   // A/B switch: 0 FFMA, 1 tf32 MMA, 2 fp16-split MMA, 3 fp16-split MMA with K/V split once per CTA
  if (att_mode == 3) return att_smem(ATT_MMA16P, T, 0) ? ATT_MMA16P : ATT_MMA16T;   // longer than 12.8 s: keys / values staged in chunks
  if (att_mode == 2 && att_smem(ATT_MMA16, T, 0)) return ATT_MMA16;
  if (att_mode != 0 && att_smem(ATT_TF32, T, 0)) return ATT_TF32;
  return ATT_FFMA;
}

// o = softmax(q k^T / 8) v per head on kernel `kernel` (ch: keys per chunk of ATT_MMA16T), into o's format: plain fp32,
// 3xTF32 (hi, lo) pair, or fp32 with fp16 planes (ATT_MMA16P / ATT_MMA16T only)
static void attention(ts_engine* e, int kernel, int ch, const float* qkv, const Act3& o, int B, int T, int H, cudaStream_t s) {
  if (e->ws.sizing) return;
  const size_t smem = att_smem(kernel, T, ch);
  if (!smem) fail(TS_ERR_UNSUPPORTED, "attention: %d frames exceed the shared memory of kernel %d", T, kernel);
  if (o.h16 && kernel < ATT_MMA16P)
    fail(TS_ERR_UNSUPPORTED, "attention: kernel %d has no fp16-split output (use the default, or ts_set_tensor_cores(e, 1))", kernel);
  const float scale = 0.125f;  // head_dim ** -0.5
  auto smem_attr = [&](const void* fn) { TS_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); };
  switch (kernel) {
    case ATT_MMA16P:
      smem_attr((const void*)attention_mma16p_kernel);
      attention_mma16p_kernel<<<B * H, ATT_WARPS * 32, smem, s>>>(qkv, o.p, o.lo, o.h16, o.l16, T, H, scale);
      break;
    case ATT_MMA16T:
      smem_attr((const void*)attention_mma16t_kernel);
      attention_mma16t_kernel<<<dim3(B * H, cdiv(cdiv(T, 16), ATT_WARPS)), ATT_WARPS * 32, smem, s>>>(qkv, o.p, o.lo, o.h16, o.l16, T, H, scale, ch);
      break;
    case ATT_MMA16:
      smem_attr((const void*)attention_mma16_kernel);
      attention_mma16_kernel<<<B * H, ATT_WARPS * 32, smem, s>>>(qkv, o.p, o.lo, T, H, scale);
      break;
    case ATT_TF32:
      smem_attr((const void*)attention_mma_kernel);
      attention_mma_kernel<<<B * H, ATT_WARPS * 32, smem, s>>>(qkv, o.p, o.lo, T, H, scale);
      break;
    default: {
      const int QT = att_ffma_qt(T);
      if (QT == 64) {
        smem_attr((const void*)attention_kernel<64>);
        attention_kernel<64><<<dim3(cdiv(T, 64), B * H), 256, smem, s>>>(qkv, o.p, o.lo, T, H, scale);
      } else if (QT == 32) {
        smem_attr((const void*)attention_kernel<32>);
        attention_kernel<32><<<dim3(cdiv(T, 32), B * H), 256, smem, s>>>(qkv, o.p, o.lo, T, H, scale);
      } else {
        smem_attr((const void*)attention_kernel<16>);
        attention_kernel<16><<<dim3(cdiv(T, 16), B * H), 256, smem, s>>>(qkv, o.p, o.lo, T, H, scale);
      }
    }
  }
  e->launches++;
  TS_CUDA(cudaGetLastError());
}

// positional conv embedding (Conv1d 768 -> 768, k = 128, groups = 16, pad 64, last output dropped) + GELU: x [B,T,768] with
// 64 zero pad rows -> y [B,T,768].  posconv_mma_kernel on the pre-split weights when the tensor cores are on, else the FFMA
// GEMM with one grid z-slice per group on the packed Layer.
static void posconv(ts_engine* e, const Layer& L, const unsigned short* w16, float unscale, const Act3& x, const Act3& y, cudaStream_t s) {
  if (e->ws.sizing) return;
  if (x.pad != 64 || x.C != 768 || y.C != 768 || y.T != x.T || y.B != x.B) fail(TS_ERR_INVALID, "posconv: activation geometry");
  const int B = x.B, T = x.T;
  if (e->use_tc && w16) {
    TS_CUDA(cudaFuncSetAttribute(posconv_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PC_SMEM));
    posconv_mma_kernel<<<dim3(B * 16, cdiv(T, PC_ROWS)), PC_WARPS * 32, PC_SMEM, s>>>(x, w16, L.bias, unscale, y);
    e->launches++;
    TS_CUDA(cudaGetLastError());
    return;
  }
  GemmP p;
  p.A = x.row(0, -64); p.W = L.W; p.bias = L.bias; p.C = y.row(0, 0);
  p.M = B * T; p.N = 48; p.K = 128 * 48; p.mper = T;
  p.a_bs = x.bstride(); p.a_rs = 768; p.kc = 48; p.a_ts = 768;
  p.c_bs = y.bstride(); p.c_rs = 768; p.act = ACT_GELU; p.ldw = 128 * 48;
  p.groups = 16; p.a_goff = 48; p.w_goff = (long)48 * 128 * 48; p.n_goff = 48;
  launch_gemm(e, p, s);
}

// Linear on channel-last activations: y[:, coff:coff+N] = act(x W^T + b (+ res)) — a 1-tap conv
static void linear(ts_engine* e, const Layer& L, const Act3& x, const Act3& y, int act, const Act3* res, cudaStream_t s, int coff = 0) {
  if (L.K != x.C) fail(TS_ERR_INVALID, "linear: K %d vs C %d", L.K, x.C);
  conv_auto(e, L, x, 1, 1, 0, y, x.T, act, res, s, 1, 0, coff);
}

bool face_has_identity(const ts_engine* e) { return e->face && e->face->identity; }

void face_run(ts_engine* e, const float* wave, const float* idv, float* out, int B, int N, int frame, cudaStream_t s) {
  FaceNet& F = *e->face;
  // ---- wav2vec2 feature extractor ---------------------------------------------------------
  int T = (N - 10) / 5 + 1;
  double* stats = e->ws.alloc<double>((size_t)B * 512 * 2);
  const bool tc = e->use_tc;   // activations stored split for the tensor-core kernel
  Act3 h = new_act(e, B, T, 512, 0, s, tc, T & 1, true);     // rows per batch even for the stride-2 convs; read by tensor-core convs only
  conv0_gn(e, wave, F.conv0_w, F.gn_g, F.gn_b, stats, B, N, h, s);
  for (int i = 1; i < 7; ++i) {
    int To = (T - W2V_K[i]) / W2V_S[i] + 1;
    Act3 y = new_act(e, B, To, 512, 0, s, tc && i < 6, To & 1, true);   // conv6 output feeds the interpolation: plain
    conv_auto(e, F.conv[i], h, W2V_K[i], W2V_S[i], 0, y, To, ACT_GELU, nullptr, s);
    h = y;
    T = To;
  }
  // ---- 50 -> 30 fps interpolation, feature projection ------------------------------------------
  Act3 hi = new_act(e, B, frame, 512, 0, s);
  interp(e, h, hi, s);
  Act3 hn = new_act(e, B, frame, 512, 0, s, tc);
  ln_pre(e, hi, nullptr, F.fp_ln_g, F.fp_ln_b, hn, nullptr, ACT_NONE, s);
  Act3 x = new_act(e, B, frame, 768, 64, s);            // padded for the k=128 positional conv (FFMA kernel: plain)
  linear(e, F.fproj, hn, x, ACT_NONE, nullptr, s);
  // ---- positional conv embedding (k=128, groups=16, pad 64, last output dropped) + LN -----------
  Act3 pc = new_act(e, B, frame, 768, 0, s);
  posconv(e, F.posconv, F.pos_w16, F.pos_unscale, x, pc, s);
  Act3 hcur = new_act(e, B, frame, 768, 0, s, tc);
  ln_pre(e, x, &pc, F.enc_ln_g, F.enc_ln_b, hcur, nullptr, ACT_NONE, s);
  // ---- 12 post-LN transformer layers ------------------------------------------------------------
  Act3 qkv = new_act(e, B, frame, 2304, 0, s);
  Act3 att = new_act(e, B, frame, 768, 0, s, tc);
  Act3 t1 = new_act(e, B, frame, 768, 0, s);
  Act3 ff = new_act(e, B, frame, 3072, 0, s, tc);
  for (auto& L : F.layers) {
    linear(e, L.qkv, hcur, qkv, ACT_NONE, nullptr, s);
    attention(e, att_kernel_for(frame), ATT_CH, qkv.p, att, B, frame, 12, s);
    linear(e, L.out, att, t1, ACT_NONE, &hcur, s);                       // h + out_proj(attn)
    ln_pre(e, t1, nullptr, L.ln1_g, L.ln1_b, hcur, nullptr, ACT_NONE, s);
    linear(e, L.ff1, hcur, ff, ACT_GELU, nullptr, s);
    linear(e, L.ff2, ff, t1, ACT_NONE, &hcur, s);                        // h + ffn(h)
    ln_pre(e, t1, nullptr, L.ln2_g, L.ln2_b, hcur, nullptr, ACT_NONE, s);
  }
  // ---- audio_feature_map (+ id_mlp concat on an identity net) -> first_net ------------------------------
  const bool tcf = tc && e->tc_f16;                       // first_net / decoder convs on the tensor-core kernel too (fp16 planes)
  Act3 cat = new_act(e, B, frame, F.identity ? 320 : 256, 1, s, tcf);
  linear(e, F.feat_map, hcur, cat, ACT_NONE, nullptr, s, 0);
  if (F.identity && !e->ws.sizing) {
    id_cols_kernel<<<dim3(cdiv(frame * 64, 256), B), 256, 0, s>>>(idv, F.id_w, F.id_b, F.ncls, cat, 256);
    e->launches++;
    TS_CUDA(cudaGetLastError());
  }
  Act3 c0 = new_act(e, B, frame, 256, 0, s);
  Act3 f;
  if (F.identity) {
    Act3 r0 = new_act(e, B, frame, 256, 0, s);
    conv_auto(e, F.fn_conv[0], cat, 3, 1, 1, c0, frame, ACT_NONE, nullptr, s);
    conv_auto(e, F.fn_res0, cat, 3, 1, 1, r0, frame, ACT_NONE, nullptr, s);
    f = new_act(e, B, frame, 256, 1, s, tcf);
    ln_pre(e, c0, nullptr, F.fn_g[0], F.fn_b[0], f, &r0, ACT_RELU, s);     // relu(LN(conv(x)) + conv_res(x))
  } else {
    conv_auto(e, F.fn_conv[0], cat, 3, 1, 1, c0, frame, ACT_NONE, nullptr, s);
    f = new_act(e, B, frame, 256, 1, s, tcf);
    ln_pre(e, c0, nullptr, F.fn_g[0], F.fn_b[0], f, &cat, ACT_RELU, s);    // relu(LN(conv(x)) + x): residual is nn.Identity
  }
  for (int i = 1; i < 3; ++i) {
    conv_auto(e, F.fn_conv[i], f, 3, 1, 1, c0, frame, ACT_NONE, nullptr, s);
    Act3 g = new_act(e, B, frame, 256, 1, s, tcf);
    ln_pre(e, c0, nullptr, F.fn_g[i], F.fn_b[i], g, &f, ACT_RELU, s);      // relu(LN(conv(x)) + x)
    f = g;
  }
  // ---- two decoder branches -> [B, frame, jaw_dim + exp_dim] (103, or 106 with a 6-D jaw) ---------------
  Act3 yout;
  yout.p = out; yout.B = B; yout.T = frame; yout.C = F.jaw_dim + F.exp_dim; yout.pad = 0;
  for (int br = 0; br < 2; ++br) {
    int c = br ? 256 : 64;
    Act3 m = f;
    for (int i = 0; i < 3; ++i) {
      Act3 cc = new_act(e, B, frame, c, 0, s);
      conv_auto(e, F.dec_conv[br][i], m, 3, 1, 1, cc, frame, ACT_NONE, nullptr, s);
      Act3 nn = new_act(e, B, frame, c, 1, s, tcf);
      ln_pre(e, cc, nullptr, F.dec_g[br][i], F.dec_b[br][i], nn, nullptr, ACT_RELU, s);
      m = nn;
    }
    linear(e, F.fin[br], m, yout, ACT_NONE, nullptr, s, br ? F.jaw_dim : 0);
  }
}

}  // namespace ts

using namespace ts;

extern "C" int ts_load_face(ts_engine* e, const ts_tensor* tensors, int n) {
  TS_API_BEGIN(e)
  Ckpt ck(tensors, n);
  LoadScope scope(e, "face");
  std::unique_ptr<FaceNet> Fp(new FaceNet());   // a throw part-way through frees the net and (scope) its uploads
  FaceNet* F = Fp.get();
  const std::string a = "audio_encoder.";
  F->conv0_w = up(e, ck.f32(a + "feature_extractor.conv_layers.0.conv.weight", {512, 1, 10}), 5120);
  F->gn_g = up(e, ck.f32(a + "feature_extractor.conv_layers.0.layer_norm.weight", {512}), 512);
  F->gn_b = up(e, ck.f32(a + "feature_extractor.conv_layers.0.layer_norm.bias", {512}), 512);
  for (int i = 1; i < 7; ++i)
    F->conv[i] = pack_ckc(e, ck.f32(a + "feature_extractor.conv_layers." + std::to_string(i) + ".conv.weight", {512, 512, W2V_K[i]}),
                          nullptr, 512, 512, W2V_K[i]);
  F->fp_ln_g = up(e, ck.f32(a + "feature_projection.layer_norm.weight", {512}), 512);
  F->fp_ln_b = up(e, ck.f32(a + "feature_projection.layer_norm.bias", {512}), 512);
  F->fproj = pack_linear(e, ck.f32(a + "feature_projection.projection.weight", {768, 512}),
                         ck.f32(a + "feature_projection.projection.bias", {768}), 768, 512);
  const std::string en = a + "encoder.";
  F->posconv = pack_ckc(e, ck.f32(en + "pos_conv_embed.conv.weight", {768, 48, 128}), ck.f32(en + "pos_conv_embed.conv.bias", {768}),
                        768, 48, 128);
  F->pos_w16 = pack_posconv16(e, ck.f32(en + "pos_conv_embed.conv.weight", {768, 48, 128}), &F->pos_unscale);
  F->enc_ln_g = up(e, ck.f32(en + "layer_norm.weight", {768}), 768);
  F->enc_ln_b = up(e, ck.f32(en + "layer_norm.bias", {768}), 768);
  for (int l = 0; ck.has(en + "layers." + std::to_string(l) + ".attention.q_proj.weight"); ++l) {
    const std::string p = en + "layers." + std::to_string(l) + ".";
    EncLayer L;
    std::vector<float> W((size_t)2304 * 768), Bv(2304);
    const char* nm[3] = {"q_proj", "k_proj", "v_proj"};
    for (int j = 0; j < 3; ++j) {
      const float* w = ck.f32(p + "attention." + nm[j] + ".weight", {768, 768});
      const float* b = ck.f32(p + "attention." + nm[j] + ".bias", {768});
      std::copy(w, w + (size_t)768 * 768, W.begin() + (size_t)j * 768 * 768);
      std::copy(b, b + 768, Bv.begin() + j * 768);
    }
    L.qkv.N = 2304; L.qkv.K = 768; L.qkv.taps = 1; L.qkv.cin = 768;
    upload_weights(e, W, &L.qkv);
    L.qkv.bias = e->upload(Bv);
    L.out = pack_linear(e, ck.f32(p + "attention.out_proj.weight", {768, 768}), ck.f32(p + "attention.out_proj.bias", {768}), 768, 768);
    L.ln1_g = up(e, ck.f32(p + "layer_norm.weight", {768}), 768);
    L.ln1_b = up(e, ck.f32(p + "layer_norm.bias", {768}), 768);
    L.ff1 = pack_linear(e, ck.f32(p + "feed_forward.intermediate_dense.weight", {3072, 768}),
                        ck.f32(p + "feed_forward.intermediate_dense.bias", {3072}), 3072, 768);
    L.ff2 = pack_linear(e, ck.f32(p + "feed_forward.output_dense.weight", {768, 3072}),
                        ck.f32(p + "feed_forward.output_dense.bias", {768}), 768, 3072);
    L.ln2_g = up(e, ck.f32(p + "final_layer_norm.weight", {768}), 768);
    L.ln2_b = up(e, ck.f32(p + "final_layer_norm.bias", {768}), 768);
    F->layers.push_back(L);
  }
  if (F->layers.empty()) fail(TS_ERR_MISSING, "face: no transformer layers in checkpoint");
  F->feat_map = pack_linear(e, ck.f32("audio_feature_map.weight", {256, 768}), ck.f32("audio_feature_map.bias", {256}), 256, 768);
  // the geometry follows the tensors: id_mlp present -> identity net, absent -> identity-free (AudioEncoder identity=False)
  const std::string fn = "audio_middle.first_net.conv_layers.";
  F->identity = ck.has("audio_middle.id_mlp.weight");
  if (F->identity) {
    const ts_tensor* idw = ck.get("audio_middle.id_mlp.weight");
    F->ncls = (int)idw->shape[1];
    F->id_w = up(e, ck.f32("audio_middle.id_mlp.weight", {64, F->ncls, 1}), (size_t)64 * F->ncls);
    F->id_b = up(e, ck.f32("audio_middle.id_mlp.bias", {64}), 64);
    F->fn_res0 = pack_ckc(e, ck.f32(fn + "0.residual_layer.0.weight", {256, 320, 3}), ck.f32(fn + "0.residual_layer.0.bias", {256}), 256, 320, 3);
  } else if (ck.has(fn + "0.residual_layer.0.weight")) {
    fail(TS_ERR_MISSING, "face: checkpoint tensor '%s0.residual_layer.0.weight' present but 'audio_middle.id_mlp.weight' missing "
         "(an identity-free net has no residual conv in layer 0)", fn.c_str());
  }
  for (int i = 0; i < 3; ++i) {
    int cin = (i == 0 && F->identity) ? 320 : 256;
    const std::string p = fn + std::to_string(i) + ".";
    F->fn_conv[i] = pack_ckc(e, ck.f32(p + "conv.weight", {256, cin, 3}), ck.f32(p + "conv.bias", {256}), 256, cin, 3);
    F->fn_g[i] = up(e, ck.f32(p + "norm.weight", {256}), 256);
    F->fn_b[i] = up(e, ck.f32(p + "norm.bias", {256}), 256);
  }
  const ts_tensor* f0 = ck.get("final_out.0.weight");
  const ts_tensor* f1 = ck.get("final_out.1.weight");
  F->jaw_dim = (int)f0->shape[0];
  F->exp_dim = (int)f1->shape[0];
  for (int br = 0; br < 2; ++br) {
    int c = br ? 256 : 64;
    for (int i = 0; i < 3; ++i) {
      int cin = i == 0 ? 256 : c;
      const std::string p = "decoder." + std::to_string(br) + "." + std::to_string(i) + ".";
      F->dec_conv[br][i] = pack_ckc(e, ck.f32(p + "conv.weight", {c, cin, 3}), ck.f32(p + "conv.bias", {c}), c, cin, 3);
      F->dec_g[br][i] = up(e, ck.f32(p + "norm.weight", {c}), c);
      F->dec_b[br][i] = up(e, ck.f32(p + "norm.bias", {c}), c);
    }
    int od = br ? F->exp_dim : F->jaw_dim;
    const std::string p = "final_out." + std::to_string(br) + ".";
    F->fin[br] = pack_ckc(e, ck.f32(p + "weight", {od, c, 1}), ck.f32(p + "bias", {od}), od, c, 1);
  }
  delete e->face;
  e->face = Fp.release();
  scope.commit();
  TS_API_END(e)
}

extern "C" int ts_face_forward(ts_engine* e, const float* wave, const float* id, float* out, int B, int N, int frame, void* stream) {
  TS_API_BEGIN(e)
  ts::require_device(e);
  if (!e->face) fail(TS_ERR_NOT_LOADED, "face weights not loaded");
  if (B <= 0 || N < 400 || frame <= 0) fail(TS_ERR_INVALID, "ts_face_forward: B=%d N=%d frame=%d (need >= 400 samples)", B, N, frame);
  cudaStream_t s = (cudaStream_t)stream;
  e->ws.begin_sizing();
  face_run(e, wave, id, out, B, N, frame, s);
  size_t need = e->ws.need;
  e->ws.buf.ensure(need + 256);
  e->ws.begin(need);
  face_run(e, wave, id, out, B, N, frame, s);
  TS_API_END(e)
}

extern "C" int ts_face_dim(ts_engine* e) { return (e && e->face) ? e->face->jaw_dim + e->face->exp_dim : 0; }

extern "C" int ts_debug_attention(ts_engine* e, const ts_debug_att* a, const float* qkv, float* out, void* plane_hi, void* plane_lo,
                                  void* stream) {
  TS_API_BEGIN(e)
  require_device(e);
  if (!a || !qkv) fail(TS_ERR_INVALID, "ts_debug_attention: a and qkv are required");
  const ts_debug_att g = *a;
  const int H = 12;
  if (g.B < 1 || g.T < 1) fail(TS_ERR_INVALID, "ts_debug_attention: B %d, T %d (need >= 1)", g.B, g.T);
  if ((long)g.B * g.T > INT_MAX / (3 * H * 64)) fail(TS_ERR_INVALID, "ts_debug_attention: more than 2^31 - 1 qkv elements");
  if (g.kernel < -1 || g.kernel > ATT_MMA16T)
    fail(TS_ERR_INVALID, "ts_debug_attention: kernel %d (-1 the face forward's choice, 0 FFMA, 1 tf32, 2 mma16, 3 mma16p, 4 mma16t)", g.kernel);
  if (g.out_format < 0 || g.out_format > 2)
    fail(TS_ERR_INVALID, "ts_debug_attention: out_format %d (0 fp32, 1 fp32 hi / lo, 2 fp32 + fp16 planes)", g.out_format);
  const int kernel = g.kernel < 0 ? att_kernel_for(g.T) : g.kernel;
  if (g.chunk && (kernel != ATT_MMA16T || g.chunk % 64 || g.chunk < 64 || g.chunk > 384))
    fail(TS_ERR_INVALID, "ts_debug_attention: chunk %d (kernel 4 only: a multiple of 64 in [64, 384])", g.chunk);
  const int ch = g.chunk ? g.chunk : ATT_CH;
  if (!att_smem(kernel, g.T, ch)) fail(TS_ERR_INVALID, "ts_debug_attention: kernel %d cannot hold %d frames in shared memory", kernel, g.T);
  if (g.out_format == 2 && kernel < ATT_MMA16P) fail(TS_ERR_INVALID, "ts_debug_attention: kernel %d has no fp16-split output", kernel);
  if ((g.out_format != 1 && !out) || (g.out_format != 0 && (!plane_hi || !plane_lo)))
    fail(TS_ERR_INVALID, "ts_debug_attention: out_format %d needs %s", g.out_format,
         g.out_format == 0 ? "out" : g.out_format == 1 ? "plane_hi and plane_lo" : "out, plane_hi and plane_lo");

  TcModeGuard guard(e, g.out_format == 0 ? 0 : g.out_format == 1 ? 1 : 6);   // the activation format face_run gives `att`
  cudaStream_t s = (cudaStream_t)stream;
  const size_t nq = (size_t)g.B * g.T * 3 * H * 64, nguard = (size_t)64 * 3 * H * 64;
  float* q = nullptr;
  Act3 o;
  run_sized(e, [&] {
    q = e->ws.alloc<float>(nq + nguard);
    o = new_act(e, g.B, g.T, H * 64, 0, s, g.out_format != 0);
  });
  TS_CUDA(cudaMemcpyAsync(q, qkv, nq * sizeof(float), cudaMemcpyDeviceToDevice, s));
  TS_CUDA(cudaMemsetAsync(q + nq, 0xff, nguard * sizeof(float), s));   // 64 NaN rows after the last item: no kernel may read them
  debug_planes(o, out, plane_hi, plane_lo, false, s);
  attention(e, kernel, ch, q, o, g.B, g.T, H, s);
  debug_planes(o, out, plane_hi, plane_lo, true, s);
  TS_CUDA(cudaStreamSynchronize(s));
  TS_API_END(e)
}

extern "C" int ts_debug_posconv(ts_engine* e, int mode, const float* x, const float* W_host, const float* bias_host, float* y, int B, int T,
                                void* stream) {
  TS_API_BEGIN(e)
  require_device(e);
  if (!x || !W_host || !bias_host || !y) fail(TS_ERR_INVALID, "ts_debug_posconv: x, W_host, bias_host and y are required");
  if (mode != 0 && mode != 1 && mode != 6) fail(TS_ERR_INVALID, "ts_debug_posconv: mode %d (0 FFMA grouped GEMM, 1 / 6 HMMA kernel)", mode);
  if (B < 1 || T < 1) fail(TS_ERR_INVALID, "ts_debug_posconv: B %d, T %d (need >= 1)", B, T);
  if ((long)B * (T + 128) > INT_MAX / 768) fail(TS_ERR_INVALID, "ts_debug_posconv: more than 2^31 - 1 activation elements");
  LoadScope scope(e, "debug_posconv");   // this call's weights replace the previous call's
  const Layer L = pack_ckc(e, W_host, bias_host, 768, 48, 128);
  float unscale = 1.f;
  const unsigned short* w16 = pack_posconv16(e, W_host, &unscale);
  TcModeGuard guard(e, mode);
  cudaStream_t s = (cudaStream_t)stream;
  Act3 xa, ya;
  run_sized(e, [&] {
    xa = new_act(e, B, T, 768, 64, s);   // face_run's x: 64 zero pad rows around every item
    ya = new_act(e, B, T, 768, 0, s);
  });
  debug_fill(e, x, xa, s);
  debug_planes(ya, y, nullptr, nullptr, false, s);
  posconv(e, L, w16, unscale, xa, ya, s);
  debug_planes(ya, y, nullptr, nullptr, true, s);
  TS_CUDA(cudaStreamSynchronize(s));
  scope.commit();
  TS_API_END(e)
}

extern "C" int ts_debug_conv0_gn(ts_engine* e, int mode, const float* wave, const float* W_host, const float* g_host, const float* b_host,
                                 float* y, void* plane_hi, void* plane_lo, int B, int N, void* stream) {
  TS_API_BEGIN(e)
  require_device(e);
  if (!wave || !W_host || !g_host || !b_host) fail(TS_ERR_INVALID, "ts_debug_conv0_gn: wave, W_host, g_host and b_host are required");
  if (mode != 0 && mode != 1 && mode != 6) fail(TS_ERR_INVALID, "ts_debug_conv0_gn: mode %d (0 fp32, 1 3xTF32 pair, 6 fp16 planes)", mode);
  if (B < 1 || N < 10) fail(TS_ERR_INVALID, "ts_debug_conv0_gn: B %d, N %d (need B >= 1, N >= 10)", B, N);
  const int T = (N - 10) / 5 + 1;
  if ((long)B * (T + 1) > INT_MAX / 512) fail(TS_ERR_INVALID, "ts_debug_conv0_gn: more than 2^31 - 1 output elements");
  if (mode == 0 ? !y : (!plane_hi || !plane_lo))
    fail(TS_ERR_INVALID, "ts_debug_conv0_gn: mode %d needs %s", mode, mode == 0 ? "y" : "plane_hi and plane_lo");
  LoadScope scope(e, "debug_conv0");   // this call's weights replace the previous call's
  const float* w = up(e, W_host, 5120);
  const float* g = up(e, g_host, 512);
  const float* b = up(e, b_host, 512);
  TcModeGuard guard(e, mode);
  cudaStream_t s = (cudaStream_t)stream;
  double* stats = nullptr;
  Act3 h;
  run_sized(e, [&] {
    stats = e->ws.alloc<double>((size_t)B * 512 * 2);
    h = new_act(e, B, T, 512, 0, s, mode != 0, T & 1, true);   // face_run's h
  });
  debug_planes(h, y, plane_hi, plane_lo, false, s);
  debug_fill(e, nullptr, h, s);   // NaN tail rows: nothing may write them
  conv0_gn(e, wave, w, g, b, stats, B, N, h, s);
  debug_planes(h, y, plane_hi, plane_lo, true, s);
  TS_CUDA(cudaStreamSynchronize(s));
  scope.commit();
  TS_API_END(e)
}

extern "C" int ts_debug_interp(ts_engine* e, const float* x, float* y, int B, int Tin, int Tout, int C, void* stream) {
  TS_API_BEGIN(e)
  require_device(e);
  if (!x || !y) fail(TS_ERR_INVALID, "ts_debug_interp: x and y are required");
  if (B < 1 || Tin < 1 || Tout < 1 || C < 1) fail(TS_ERR_INVALID, "ts_debug_interp: B %d, Tin %d, Tout %d, C %d (need >= 1)", B, Tin, Tout, C);
  if ((long)B * (Tin + 1) * C > INT_MAX || (long)B * Tout * C > INT_MAX) fail(TS_ERR_INVALID, "ts_debug_interp: more than 2^31 - 1 elements");
  cudaStream_t s = (cudaStream_t)stream;
  Act3 xa, ya;
  run_sized(e, [&] {
    xa = new_act(e, B, Tin, C, 0, s, false, Tin & 1);   // conv6's output: plain, Tin & 1 tail rows
    ya = new_act(e, B, Tout, C, 0, s);
  });
  debug_fill(e, x, xa, s);
  debug_planes(ya, y, nullptr, nullptr, false, s);
  interp(e, xa, ya, s);
  debug_planes(ya, y, nullptr, nullptr, true, s);
  TS_CUDA(cudaStreamSynchronize(s));
  TS_API_END(e)
}

extern "C" int ts_debug_layernorm(ts_engine* e, const ts_debug_ln* a, const float* x, const float* pre, const float* res,
                                  const float* g_host, const float* b_host, float* y, void* plane_hi, void* plane_lo, void* stream) {
  TS_API_BEGIN(e)
  require_device(e);
  if (!a || !x || !g_host || !b_host) fail(TS_ERR_INVALID, "ts_debug_layernorm: a, x, g_host and b_host are required");
  const ts_debug_ln d = *a;
  if (d.mode != 0 && d.mode != 1 && d.mode != 6) fail(TS_ERR_INVALID, "ts_debug_layernorm: mode %d (0 fp32, 1 3xTF32 pair, 6 fp16 planes)", d.mode);
  if (d.B < 1 || d.T < 1 || d.C < 1) fail(TS_ERR_INVALID, "ts_debug_layernorm: B %d, T %d, C %d (need >= 1)", d.B, d.T, d.C);
  if (d.C > 768) fail(TS_ERR_INVALID, "ts_debug_layernorm: width %d > 768", d.C);
  if ((long)d.B * (d.T + 2) * d.C > INT_MAX) fail(TS_ERR_INVALID, "ts_debug_layernorm: more than 2^31 - 1 elements");
  if (d.act != ACT_NONE && d.act != ACT_RELU) fail(TS_ERR_INVALID, "ts_debug_layernorm: act %d (0 none, 1 ReLU)", d.act);
  if ((d.has_pre && !pre) || (d.has_res && !res)) fail(TS_ERR_INVALID, "ts_debug_layernorm: has_pre / has_res need pre / res");
  const bool y_pair = d.y_split && d.mode != 6;   // (hi, lo) planes, no fp32 copy
  if ((!y_pair && !y) || (d.y_split && (!plane_hi || !plane_lo)))
    fail(TS_ERR_INVALID, "ts_debug_layernorm: y_split %d in mode %d needs %s", d.y_split, d.mode,
         !d.y_split ? "y" : y_pair ? "plane_hi and plane_lo" : "y, plane_hi and plane_lo");
  LoadScope scope(e, "debug_ln");   // this call's weights replace the previous call's
  const float* g = up(e, g_host, d.C);
  const float* b = up(e, b_host, d.C);
  TcModeGuard guard(e, d.mode);
  cudaStream_t s = (cudaStream_t)stream;
  Act3 xa, pa, ra, ya;
  run_sized(e, [&] {
    xa = new_act(e, d.B, d.T, d.C, 0, s, d.x_split != 0);
    if (d.has_pre) pa = new_act(e, d.B, d.T, d.C, 0, s);
    if (d.has_res) ra = new_act(e, d.B, d.T, d.C, 0, s, d.res_split != 0);
    ya = new_act(e, d.B, d.T, d.C, 1, s, d.y_split != 0);   // one pad row around every item, as first_net / decoder outputs
  });
  debug_fill(e, x, xa, s);
  if (d.has_pre) debug_fill(e, pre, pa, s);
  if (d.has_res) debug_fill(e, res, ra, s);
  debug_planes(ya, y, plane_hi, plane_lo, false, s);
  ln_pre(e, xa, d.has_pre ? &pa : nullptr, g, b, ya, d.has_res ? &ra : nullptr, d.act, s);
  debug_planes(ya, y, plane_hi, plane_lo, true, s);
  TS_CUDA(cudaStreamSynchronize(s));
  scope.commit();
  TS_API_END(e)
}
