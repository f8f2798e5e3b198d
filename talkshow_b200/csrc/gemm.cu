// talkshow_b200 — fp32 implicit-GEMM conv kernel (FFMA, register tiled) and the small layout /
// normalisation kernels of the conv stacks.  The body path needs fp32 accumulation for bit-exact
// VQ indices (DESIGN.md §numerics), so these are CUDA-core kernels, not tensor-core ones.
#include "kernels.h"

namespace ts {

__device__ __forceinline__ float act_apply(float v, int act) {
  if (act == ACT_RELU) return v > 0.f ? v : 0.f;
  if (act == ACT_LRELU) return v > 0.f ? v : 0.2f * v;
  if (act == ACT_GELU) return 0.5f * v * (1.0f + erff(v * 0.70710678118654752440f));
  return v;
}

__device__ __forceinline__ float2 unpack2(unsigned long long v) {
  float2 r;
  asm("mov.b64 {%0, %1}, %2;" : "=f"(r.x), "=f"(r.y) : "l"(v));
  return r;
}
__device__ __forceinline__ unsigned long long pack2(float x, float y) {
  unsigned long long v;
  asm("mov.b64 %0, {%1, %2};" : "=l"(v) : "f"(x), "f"(y));
  return v;
}
// Two IEEE fp32 FMAs on a register pair: acc / b hold two adjacent output columns, the A element is the broadcast
// operand.  The pair layout keeps 64-bit shared / global loads; the pack / unpack moves compile to nothing.
__device__ __forceinline__ void fma2(unsigned long long& acc, float a, unsigned long long b) {
  const float2 c = unpack2(acc), x = unpack2(b);
  acc = pack2(fmaf(a, x.x, c.x), fmaf(a, x.y, c.y));
}

template <int BM, int BN, int TM, int TN>
__global__ void __launch_bounds__((BM / TM) * (BN / TN), 2) gemm_kernel(GemmP p) {
  constexpr int BK = 16;
  constexpr int NT = (BM / TM) * (BN / TN);
  constexpr int LA = BM * 4 / NT, LB = BN * 4 / NT;
  static_assert(LA >= 1 && LB >= 1, "tile too small");
  __shared__ __align__(16) float As[2][BK][BM + 4];
  __shared__ __align__(16) float Bs[2][BK][BN + 4];
  const int tid = threadIdx.x;
  const int g = blockIdx.z;
  const float* A = p.A + g * p.a_goff;
  const float* W = p.W + g * p.w_goff;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const bool dense = (p.a_ts == p.kc);

  const float* a_ptr[LA];
  const float* al_ptr[LA];
  const float* w_ptr[LB];
  const float* A_lo = p.A_lo ? p.A_lo + g * p.a_goff : nullptr;
#pragma unroll
  for (int i = 0; i < LA; ++i) {
    int row = (tid + i * NT) >> 2;
    int m = min(m0 + row, p.M - 1);
    int b = m / p.mper, t = m - b * p.mper;
    a_ptr[i] = A + b * p.a_bs + t * p.a_rs;
    al_ptr[i] = A_lo ? A_lo + b * p.a_bs + t * p.a_rs : nullptr;
  }
#pragma unroll
  for (int i = 0; i < LB; ++i) {
    int row = (tid + i * NT) >> 2;
    int n = min(n0 + row, p.N - 1);
    w_ptr[i] = W + (long)n * p.ldw;
  }
  float4 ra[LA], rb[LB];
  auto gload = [&](int k0) {
#pragma unroll
    for (int i = 0; i < LA; ++i) {
      int k = k0 + ((tid + i * NT) & 3) * 4;
      if (k < p.K) {
        int off = dense ? k : (k / p.kc) * p.a_ts + (k % p.kc);
        ra[i] = *reinterpret_cast<const float4*>(a_ptr[i] + off);
        if (A_lo) {  // split activation (hi, lo): x = hi + lo exactly
          float4 l = *reinterpret_cast<const float4*>(al_ptr[i] + off);
          ra[i].x += l.x; ra[i].y += l.y; ra[i].z += l.z; ra[i].w += l.w;
        }
      } else {
        ra[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
#pragma unroll
    for (int i = 0; i < LB; ++i) {
      int k = k0 + ((tid + i * NT) & 3) * 4;
      rb[i] = (k < p.K) ? *reinterpret_cast<const float4*>(w_ptr[i] + k) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int i = 0; i < LA; ++i) {
      int idx = tid + i * NT, row = idx >> 2, kq = (idx & 3) * 4;
      As[buf][kq + 0][row] = ra[i].x;
      As[buf][kq + 1][row] = ra[i].y;
      As[buf][kq + 2][row] = ra[i].z;
      As[buf][kq + 3][row] = ra[i].w;
    }
#pragma unroll
    for (int i = 0; i < LB; ++i) {
      int idx = tid + i * NT, row = idx >> 2, kq = (idx & 3) * 4;
      Bs[buf][kq + 0][row] = rb[i].x;
      Bs[buf][kq + 1][row] = rb[i].y;
      Bs[buf][kq + 2][row] = rb[i].z;
      Bs[buf][kq + 3][row] = rb[i].w;
    }
  };

  const int ty = tid / (BN / TN), tx = tid % (BN / TN);
  unsigned long long acc2[TM][TN / 2];   // column pairs (j, j+1)
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN / 2; ++j) acc2[i][j] = 0ull;

  gload(0);
  sstore(0);
  __syncthreads();
  for (int k0 = 0, it = 0; k0 < p.K; k0 += BK, ++it) {
    const int buf = it & 1;
    const bool more = k0 + BK < p.K;
    if (more) gload(k0 + BK);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[TM];
      unsigned long long b2[TN / 2];
#pragma unroll
      for (int i = 0; i < TM; i += 4) {
        float4 v = *reinterpret_cast<const float4*>(&As[buf][kk][ty * TM + i]);
        a[i] = v.x; a[i + 1] = v.y; a[i + 2] = v.z; a[i + 3] = v.w;
      }
#pragma unroll
      for (int j = 0; j < TN; j += 4) {
        ulonglong2 v = *reinterpret_cast<const ulonglong2*>(&Bs[buf][kk][tx * TN + j]);
        b2[j / 2] = v.x; b2[j / 2 + 1] = v.y;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN / 2; ++j) fma2(acc2[i][j], a[i], b2[j]);
    }
    if (more) sstore(buf ^ 1);
    __syncthreads();
  }

  const float* bias = p.bias ? p.bias + g * p.n_goff : nullptr;
  float* C = p.C + g * p.n_goff;
  float* C_lo = p.C_lo ? p.C_lo + g * p.n_goff : nullptr;
  unsigned short* C_h16 = p.C_h16 ? p.C_h16 + g * p.n_goff : nullptr;
  unsigned short* C_l16 = p.C_l16 ? p.C_l16 + g * p.n_goff : nullptr;
  const float* R = p.R ? p.R + g * p.n_goff : nullptr;
  const float* R_lo = p.R_lo ? p.R_lo + g * p.n_goff : nullptr;
  const bool vec = ((p.c_rs | p.c_bs | p.r_rs | p.r_bs | p.n_goff) & 3) == 0 && (p.N & 3) == 0 &&
                   ((reinterpret_cast<uintptr_t>(C) & 15) == 0) && (!R || (reinterpret_cast<uintptr_t>(R) & 15) == 0);
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    int m = m0 + ty * TM + i;
    if (m >= p.M) continue;
    int b = m / p.mper, t = m - b * p.mper;
    float* crow = C + b * p.c_bs + t * p.c_rs;
    float* crow_lo = C_lo ? C_lo + b * p.c_bs + t * p.c_rs : nullptr;
    unsigned short* crow_h16 = C_h16 ? C_h16 + b * p.c_bs + t * p.c_rs : nullptr;
    unsigned short* crow_l16 = C_h16 ? C_l16 + b * p.c_bs + t * p.c_rs : nullptr;
    const float* rrow = R ? R + b * p.r_bs + t * p.r_rs : nullptr;
    const float* rrow_lo = R_lo ? R_lo + b * p.r_bs + t * p.r_rs : nullptr;
#pragma unroll
    for (int j = 0; j < TN; j += 4) {
      int n = n0 + tx * TN + j;
      if (n >= p.N) continue;
      const float2 c01 = unpack2(acc2[i][j / 2]), c23 = unpack2(acc2[i][j / 2 + 1]);
      const float accq[4] = {c01.x, c01.y, c23.x, c23.y};
      float v[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        int nn = n + q;
        float x = accq[q];
        if (nn < p.N) {
          if (bias) x += bias[nn];
          if (rrow) x += rrow_lo ? (rrow[nn] + rrow_lo[nn]) : rrow[nn];
          x = act_apply(x, p.act);
        }
        v[q] = x;
      }
      if (crow_h16) {
#pragma unroll
        for (int q = 0; q < 4; ++q)
          if (n + q < p.N) {
            crow[n + q] = v[q];
            split16(v[q], crow_h16[n + q], crow_l16[n + q]);
          }
      } else if (crow_lo) {
#pragma unroll
        for (int q = 0; q < 4; ++q)
          if (n + q < p.N) {
            float h = __uint_as_float(__float_as_uint(v[q]) & 0xffffe000u);
            crow[n + q] = h;
            crow_lo[n + q] = v[q] - h;
          }
      } else if (vec) {
        *reinterpret_cast<float4*>(crow + n) = make_float4(v[0], v[1], v[2], v[3]);
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q)
          if (n + q < p.N) crow[n + q] = v[q];
      }
    }
  }
}

void launch_gemm(ts_engine* e, const GemmP& p, cudaStream_t s) {
  if (e->ws.sizing) return;
  if (p.M <= 0 || p.N <= 0) return;
  if ((p.K & 3) || (p.kc & 3) || (p.a_ts & 3) || (p.a_rs & 3) || (p.a_bs & 3) || (p.ldw & 3) || (p.a_goff & 3) ||
      (p.w_goff & 3))
    fail(TS_ERR_INVALID, "gemm: K/strides must be multiples of 4 (K=%d kc=%d a_ts=%d a_rs=%ld)", p.K, p.kc, p.a_ts,
         p.a_rs);
  if (p.N <= 64) {
    dim3 grid(cdiv(p.M, 128), cdiv(p.N, 64), p.groups);
    gemm_kernel<128, 64, 8, 4><<<grid, 256, 0, s>>>(p);
  } else {
    dim3 grid(cdiv(p.M, 128), cdiv(p.N, 128), p.groups);
    gemm_kernel<128, 128, 8, 8><<<grid, 256, 0, s>>>(p);
  }
  e->launches++;
  TS_CUDA(cudaGetLastError());
}

void conv1d(ts_engine* e, const Layer& L, const Act3& x, int k, int stride, int pd, const Act3& y, int T_out, int act,
            const Act3* res, cudaStream_t s, int y_tmul, int y_toff, int x_toff, int coff) {
  if (L.taps != k || L.cin != x.C) fail(TS_ERR_INVALID, "conv1d: layer (taps %d, cin %d) vs input (k %d, C %d)", L.taps, L.cin, k, x.C);
  if (x.pad < pd) fail(TS_ERR_INVALID, "conv1d: input pad %d < conv pad %d", x.pad, pd);
  if (!e->ws.sizing && (!x.p || !y.p)) fail(TS_ERR_INVALID, "conv1d: activation without an fp32 copy (fp16 planes only) on the FFMA path");
  GemmP p;
  p.A = x.row(0, 0) + (long)(x_toff - pd) * x.C;
  if (x.lo) p.A_lo = x.row_lo(0, 0) + (long)(x_toff - pd) * x.C;
  if (y.lo) p.C_lo = y.row_lo(0, y_toff) + coff;
  if (y.h16) { p.C_h16 = y.row_h16(0, y_toff) + coff; p.C_l16 = y.row_l16(0, y_toff) + coff; }
  p.W = L.W;
  p.bias = L.bias;
  p.C = y.row(0, y_toff) + coff;
  p.M = x.B * T_out;
  p.N = L.N;
  p.K = L.K;
  p.mper = T_out;
  p.a_bs = x.bstride();
  p.a_rs = (long)stride * x.C;
  p.kc = L.K;
  p.a_ts = L.K;
  p.c_bs = y.bstride();
  p.c_rs = (long)y_tmul * y.C;
  p.act = act;
  p.ldw = L.K;
  if (res) {
    p.R = res->row(0, 0);
    if (res->lo) p.R_lo = res->row_lo(0, 0);
    p.r_bs = res->bstride();
    p.r_rs = res->C;
  }
  launch_gemm(e, p, s);
}

// ---- layout kernels ------------------------------------------------------------------------
__global__ void nct_to_act_kernel(const float* __restrict__ in, int C, Act3 out) {
  // one block per (b, 32-row tile); tile transpose through smem
  __shared__ float tile[32][33];
  int b = blockIdx.z, t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  int tx = threadIdx.x, ty = threadIdx.y;
  for (int i = ty; i < 32; i += 8) {
    int c = c0 + i, t = t0 + tx;
    tile[i][tx] = (c < C && t < out.T) ? in[((long)b * C + c) * out.T + t] : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    int t = t0 + i, c = c0 + tx;
    if (t < out.T && c < out.C) out.row(b, t)[c] = tile[tx][i];
  }
}
__global__ void act_to_nct_kernel(Act3 in, int C, float* __restrict__ out) {
  __shared__ float tile[32][33];
  int b = blockIdx.z, t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  int tx = threadIdx.x, ty = threadIdx.y;
  for (int i = ty; i < 32; i += 8) {
    int t = t0 + i, c = c0 + tx;
    tile[i][tx] = (t < in.T && c < C) ? in.row(b, t)[c] : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    int c = c0 + i, t = t0 + tx;
    if (c < C && t < in.T) out[((long)b * C + c) * in.T + t] = tile[tx][i];
  }
}
__global__ void btc_to_act_kernel(const float* __restrict__ in, int C, Act3 out) {
  long n = (long)out.B * out.T * out.C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    int c = i % out.C;
    long bt = i / out.C;
    int t = bt % out.T, b = bt / out.T;
    out.row(b, t)[c] = c < C ? in[((long)b * out.T + t) * C + c] : 0.f;
  }
}
__global__ void act_to_btc_kernel(Act3 in, int C, float* __restrict__ out, int ldo, int ooff) {
  long n = (long)in.B * in.T * C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    int c = i % C;
    long bt = i / C;
    int t = bt % in.T, b = bt / in.T;
    out[((long)b * in.T + t) * ldo + ooff + c] = in.row(b, t)[c];
  }
}
__global__ void zero_pads_kernel(Act3 a) {
  int per = 2 * a.pad * a.C;
  long n = (long)a.B * per;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    int b = i / per, r = i % per;
    int row = r / a.C, c = r % a.C;
    int t = row < a.pad ? row - a.pad : a.T + (row - a.pad);
    if (a.p) a.row(b, t)[c] = 0.f;
    if (a.lo) a.row_lo(b, t)[c] = 0.f;
    if (a.h16) { a.row_h16(b, t)[c] = 0; a.row_l16(b, t)[c] = 0; }
  }
}

static inline int gs_blocks(long n) { return (int)std::min<long>((n + 255) / 256, 132 * 16); }

void nct_to_act(ts_engine* e, const float* in, int C, const Act3& out, cudaStream_t s) {
  if (e->ws.sizing) return;
  zero_pads(e, out, s);
  dim3 grid(cdiv(out.T, 32), cdiv(out.C, 32), out.B);
  nct_to_act_kernel<<<grid, dim3(32, 8), 0, s>>>(in, C, out);
  e->launches++;
  TS_CUDA(cudaGetLastError());
}
void act_to_nct(ts_engine* e, const Act3& in, int C, float* out, cudaStream_t s) {
  if (e->ws.sizing) return;
  dim3 grid(cdiv(in.T, 32), cdiv(C, 32), in.B);
  act_to_nct_kernel<<<grid, dim3(32, 8), 0, s>>>(in, C, out);
  e->launches++;
  TS_CUDA(cudaGetLastError());
}
void btc_to_act(ts_engine* e, const float* in, int C, const Act3& out, cudaStream_t s) {
  if (e->ws.sizing) return;
  zero_pads(e, out, s);
  btc_to_act_kernel<<<gs_blocks((long)out.B * out.T * out.C), 256, 0, s>>>(in, C, out);
  e->launches++;
  TS_CUDA(cudaGetLastError());
}
void act_to_btc(ts_engine* e, const Act3& in, int C, float* out, int ldo, int ooff, cudaStream_t s) {
  if (e->ws.sizing) return;
  act_to_btc_kernel<<<gs_blocks((long)in.B * in.T * C), 256, 0, s>>>(in, C, out, ldo, ooff);
  e->launches++;
  TS_CUDA(cudaGetLastError());
}
void zero_pads(ts_engine* e, const Act3& a, cudaStream_t s) {
  if (e->ws.sizing) return;
  if (a.pad == 0) return;
  zero_pads_kernel<<<gs_blocks((long)a.B * 2 * a.pad * a.C), 256, 0, s>>>(a);
  e->launches++;
  TS_CUDA(cudaGetLastError());
}

// ---- VQ kernels ----------------------------------------------------------------------------
__global__ void gather_rows_kernel(const float* __restrict__ table, int C, const int64_t* __restrict__ idx, Act3 out) {
  int bt = blockIdx.x;
  int b = bt / out.T, t = bt % out.T;
  long code = idx[bt];
  for (int c = threadIdx.x; c < out.C; c += blockDim.x) out.row(b, t)[c] = c < C ? table[code * C + c] : 0.f;
}
void gather_rows(ts_engine* e, const float* table, int C, const int64_t* idx, const Act3& out, cudaStream_t s) {
  if (e->ws.sizing) return;
  zero_pads(e, out, s);
  gather_rows_kernel<<<out.B * out.T, 64, 0, s>>>(table, C, idx, out);
  e->launches++;
  TS_CUDA(cudaGetLastError());
}

// torch.argmin's order on (distance, code): a NaN distance beats everything, then the smaller distance, then the lower
// code.  On non-NaN distances this is `d < bd || (d == bd && i < bi)`.
__device__ __forceinline__ bool vq_better(float d, int i, float bd, int bi) {
  const bool dn = d != d, bn = bd != bd;
  if (dn != bn) return dn;
  return (dn || d == bd) ? i < bi : d < bd;
}

// distances = sum(x^2) + sum(e^2) - 2 x.e ; argmin in torch.argmin's order (vqvae_modules.py:311-319): first index on
// ties, the first NaN distance when there is one, so the index is in [0, ncodes) whatever the latent row holds
__global__ void __launch_bounds__(256) vq_argmin_kernel(const float* __restrict__ cb, const float* __restrict__ ee,
                                                        int ncodes, Act3 z, int64_t* __restrict__ idx) {
  __shared__ float xs[64];
  __shared__ float best_d[8];
  __shared__ int best_i[8];
  int bt = blockIdx.x, b = bt / z.T, t = bt % z.T;
  const float* x = z.row(b, t);
  if (threadIdx.x < 64) xs[threadIdx.x] = x[threadIdx.x];
  __syncthreads();
  float xx = 0.f;
  for (int c = 0; c < 64; ++c) xx = fmaf(xs[c], xs[c], xx);
  float bd = INFINITY;
  int bi = 0x7fffffff;
  for (int n = threadIdx.x; n < ncodes; n += 256) {
    const float4* e4 = reinterpret_cast<const float4*>(cb + (long)n * 64);
    float dot = 0.f;
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      float4 v = e4[c];
      dot = fmaf(xs[4 * c], v.x, dot);
      dot = fmaf(xs[4 * c + 1], v.y, dot);
      dot = fmaf(xs[4 * c + 2], v.z, dot);
      dot = fmaf(xs[4 * c + 3], v.w, dot);
    }
    float d = (xx + ee[n]) - 2.0f * dot;
    if (vq_better(d, n, bd, bi)) { bd = d; bi = n; }
  }
  for (int o = 16; o > 0; o >>= 1) {
    float od = __shfl_xor_sync(0xffffffffu, bd, o);
    int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (vq_better(od, oi, bd, bi)) { bd = od; bi = oi; }
  }
  int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { best_d[w] = bd; best_i[w] = bi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < 8; ++i)
      if (vq_better(best_d[i], best_i[i], bd, bi)) { bd = best_d[i]; bi = best_i[i]; }
    idx[bt] = bi;
  }
}
void vq_argmin(ts_engine* e, const float* codebook, const float* ee, int ncodes, const Act3& z, int64_t* idx,
               cudaStream_t s) {
  if (e->ws.sizing) return;
  if (z.C != 64) fail(TS_ERR_INVALID, "vq_argmin: embedding dim %d != 64", z.C);
  vq_argmin_kernel<<<z.B * z.T, 256, 0, s>>>(codebook, ee, ncodes, z, idx);
  e->launches++;
  TS_CUDA(cudaGetLastError());
}

}  // namespace ts
