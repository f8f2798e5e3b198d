// talkshow_b200 — held-out scoring of the VQ-VAE pair and the face regressor: the forward half of the reference's
// training steps (nets/smplx_body_vq.py:155-206 vq_train + get_loss, nets/smplx_face.py:95-167 __call__ + get_loss)
// with the loss reductions kept per clip.
//
// The dense work is the existing encoder / argmin / decoder chain (convstack.cu) and face_run (face.cu); this file adds
// the reductions.  Every reduction has a fixed order and no atomics, so repeated calls give the same bits:
//   - elementwise terms are formed in fp32 exactly as the reference forms them (difference, then |.| or square);
//   - one warp per latent row sums the 64 squared commitment terms in fp32 through a fixed xor-shuffle tree;
//   - each thread of a per-clip block accumulates its strided share of the terms in fp64, and the block's partials are
//     combined by a fixed fp64 tree.  clip_out holds fp64 sums.
#include "convstack.h"
#include "pixelcnn.h"

using namespace ts;

namespace {

constexpr int CLIP_THREADS = 256;

// sums v[k][tid] over the block for k < K into v[k][0]; fixed pairwise tree
template <int K>
__device__ __forceinline__ void block_sum(double (*v)[CLIP_THREADS]) {
  for (int h = CLIP_THREADS / 2; h > 0; h >>= 1) {
    __syncthreads();
    if (threadIdx.x < h)
      for (int k = 0; k < K; ++k) v[k][threadIdx.x] += v[k][threadIdx.x + h];
  }
  __syncthreads();
}

// out[r] = sum_c (z[r][c] - cb[idx[r]][c])^2 over the 64 embedding dims; one warp per latent row r = b*T + t.
// Lane l takes dims l and l+32; the 32 lane sums meet through a fixed xor tree (e_latent_loss, vqvae_modules.py:302).
__global__ void vq_commit_kernel(Act3 z, const float* __restrict__ cb, const int64_t* __restrict__ idx,
                                 float* __restrict__ out, int rows) {
  const int r = (int)((blockIdx.x * (long)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (r >= rows) return;   // whole warps leave together
  const float* zr = z.row(r / z.T, r % z.T);
  const float* er = cb + idx[r] * 64;
  const float d0 = __fsub_rn(zr[lane], er[lane]), d1 = __fsub_rn(zr[lane + 32], er[lane + 32]);
  float s = __fadd_rn(__fmul_rn(d0, d0), __fmul_rn(d1, d1));
  for (int o = 16; o > 0; o >>= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
  if (lane == 0) out[r] = s;
}

// One block per clip b: recon y (decoder output, channel-last rows of width y.C >= C) against gt [B,F,C].
// clip[b] = { sum |y - gt| over (F, C),  sum |(y[f+1]-y[f]) - (gt[f+1]-gt[f])| over (F-1, C),  sum_t commit[b*T+t] }
// (get_loss, nets/smplx_body_vq.py:186-189, and the commitment term before its mean).
__global__ void __launch_bounds__(CLIP_THREADS) vq_clip_kernel(Act3 y, const float* __restrict__ gt, int C, int F,
                                                               const float* __restrict__ commit, int T,
                                                               double* __restrict__ clip) {
  __shared__ double v[3][CLIP_THREADS];
  const int b = blockIdx.x;
  const float* g = gt + (long)b * F * C;
  double rec = 0.0, vel = 0.0, com = 0.0;
  const long n = (long)F * C;
  for (long i = threadIdx.x; i < n; i += CLIP_THREADS) {
    const int f = (int)(i / C), c = (int)(i % C);
    const float r = y.row(b, f)[c], gv = g[i];
    rec += (double)fabsf(__fsub_rn(r, gv));
    if (f + 1 < F) {
      const float vr = __fsub_rn(y.row(b, f + 1)[c], r), vg = __fsub_rn(g[i + C], gv);
      vel += (double)fabsf(__fsub_rn(vr, vg));
    }
  }
  for (int t = threadIdx.x; t < T; t += CLIP_THREADS) com += (double)commit[(long)b * T + t];
  v[0][threadIdx.x] = rec;
  v[1][threadIdx.x] = vel;
  v[2][threadIdx.x] = com;
  block_sum<3>(v);
  if (threadIdx.x < 3) clip[b * 3 + threadIdx.x] = v[threadIdx.x][0];
}

// One block per clip b: pred [B,F,D] against gt [B,F,Cg] (nets/smplx_face.py:155-157).
// clip[b] = { sum |pred[:, :6] - gt[:, :6]|,  sum (pred[:, D-100:] - gt[:, Cg-100:])^2 }
__global__ void __launch_bounds__(CLIP_THREADS) face_clip_kernel(const float* __restrict__ pred, int D,
                                                                 const float* __restrict__ gt, int Cg, int F,
                                                                 double* __restrict__ clip) {
  __shared__ double v[2][CLIP_THREADS];
  const int b = blockIdx.x;
  const float* p = pred + (long)b * F * D;
  const float* g = gt + (long)b * F * Cg;
  double l1 = 0.0, se = 0.0;
  for (int i = threadIdx.x; i < F * 6; i += CLIP_THREADS) {
    const int f = i / 6, c = i % 6;
    l1 += (double)fabsf(__fsub_rn(p[(long)f * D + c], g[(long)f * Cg + c]));
  }
  for (int i = threadIdx.x; i < F * 100; i += CLIP_THREADS) {
    const int f = i / 100, c = i % 100;
    const float d = __fsub_rn(p[(long)f * D + D - 100 + c], g[(long)f * Cg + Cg - 100 + c]);
    se += (double)__fmul_rn(d, d);
  }
  v[0][threadIdx.x] = l1;
  v[1][threadIdx.x] = se;
  block_sum<2>(v);
  if (threadIdx.x < 2) clip[b * 2 + threadIdx.x] = v[threadIdx.x][0];
}

}  // namespace

extern "C" int ts_vq_score(ts_engine* e, int which, const float* poses, int64_t* idx, float* recon, double* clip, int B,
                           int F, void* stream) {
  TS_API_BEGIN(e)
  ts::require_device(e);
  if (which < 0 || which > 1 || !e->conv || !e->conv->vq[which].loaded) fail(TS_ERR_NOT_LOADED, "vq[%d] weights not loaded", which);
  if (B <= 0 || F < 4 || F % 4 != 0)
    fail(TS_ERR_INVALID, "ts_vq_score: B=%d F=%d (F must be a positive multiple of 4: the decoder returns 4*(latent rows) frames)", B, F);
  if (!poses || !idx || !clip) fail(TS_ERR_INVALID, "ts_vq_score: poses, idx and clip_out are required");
  cudaStream_t s = (cudaStream_t)stream;
  const VQNet& v = e->conv->vq[which];
  const int C = v.out_dim;
  run_sized(e, [&] {
    // VQVAE.encode exactly as ts_vq_encode runs it: same kernels, same arithmetic, same indices
    Act3 x = new_act(e, B, F, pad4(C), 1, s);
    btc_to_act(e, poses, C, x, s);
    Act3 h = run_trunk(e, v.enc, x, s);
    const int T = h.T;
    Act3 z = new_act(e, B, T, 64, 0, s);
    conv1d(e, v.pre_vq, h, 1, 1, 0, z, T, ACT_NONE, nullptr, s);
    vq_argmin(e, v.codebook, v.ee, v.ncodes, z, idx, s);
    float* commit = e->ws.alloc<float>((size_t)B * T);
    // the decoder on the quantised embeddings (eval: no straight-through add), as ts_vq_decode runs it
    Act3 q = new_act(e, B, T, 64, 0, s);
    gather_rows(e, v.codebook, 64, idx, q, s);
    Act3 y = run_decoder(e, v, q, s);
    if (e->ws.sizing) return;
    const int rows = B * T;
    vq_commit_kernel<<<cdiv(rows, 8), 256, 0, s>>>(z, v.codebook, idx, commit, rows);
    e->launches++;
    TS_CUDA(cudaGetLastError());
    if (recon) act_to_btc(e, y, C, recon, C, 0, s);
    vq_clip_kernel<<<B, CLIP_THREADS, 0, s>>>(y, poses, C, F, commit, T, clip);
    e->launches++;
    TS_CUDA(cudaGetLastError());
  });
  TS_API_END(e)
}

extern "C" int ts_face_score(ts_engine* e, const float* wave, const float* id, const float* gt, int Cgt, float* pred,
                             double* clip, int B, int N, int F, void* stream) {
  TS_API_BEGIN(e)
  ts::require_device(e);
  if (!e->face) fail(TS_ERR_NOT_LOADED, "face weights not loaded");
  const int D = ts_face_dim(e);
  if (B <= 0 || N < 400 || F <= 0) fail(TS_ERR_INVALID, "ts_face_score: B=%d N=%d F=%d (need >= 400 samples)", B, N, F);
  if (Cgt < 100 || D < 100)
    fail(TS_ERR_INVALID, "ts_face_score: gt has %d columns, the net %d (both need the 100 expression columns last)", Cgt, D);
  if (!wave || !gt || !clip) fail(TS_ERR_INVALID, "ts_face_score: wave, gt and clip_out are required");
  if (!id && face_has_identity(e)) fail(TS_ERR_INVALID, "ts_face_score: the identity net needs id");
  cudaStream_t s = (cudaStream_t)stream;
  run_sized(e, [&] {
    float* out = pred ? pred : e->ws.alloc<float>((size_t)B * F * D);
    face_run(e, wave, id, out, B, N, F, s);
    if (e->ws.sizing) return;
    face_clip_kernel<<<B, CLIP_THREADS, 0, s>>>(out, D, gt, Cgt, F, clip);
    e->launches++;
    TS_CUDA(cudaGetLastError());
  });
  TS_API_END(e)
}
