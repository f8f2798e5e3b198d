// talkshow_b200 — device kernels shared by the conv stacks and the face network (host launchers).
#pragma once
#include "common.h"
#ifdef __CUDACC__
#include <cuda_fp16.h>
#endif

namespace ts {

enum Act { ACT_NONE = 0, ACT_RELU = 1, ACT_LRELU = 2, ACT_GELU = 3 };

// Channel-last activation with explicit zero rows before/after every batch item:
// element (b, t, c) lives at p[(b*(T+2*pad) + pad + t)*C + c].
struct Act3 {
  float* p = nullptr;
  int B = 0, T = 0, C = 0, pad = 0;
  int tail = 0;          // extra (unused) rows after the back padding so rows-per-batch is a multiple of a stride
  bool split = false;    // stored as (hi, lo) pair, see lo
  float* lo = nullptr;   // when set the activation is stored split for the 3xTF32 tensor-core GEMM:
                         // p = hi part (low 13 mantissa bits clear), lo = x - hi, x == p + lo exactly
  // fp16-split storage (ts_set_tensor_cores(e, 6), the default): p holds the FULL fp32 value (what every non-tensor-core
  // reader uses; lo stays null) and the tensor-core GEMM reads the two half planes h16 = fp16(x), l16 = fp16(x - h16)
  unsigned short* h16 = nullptr;
  unsigned short* l16 = nullptr;
  __host__ __device__ long bstride() const { return (long)(T + 2 * pad + tail) * C; }
  __host__ __device__ float* row(int b, int t) const { return p + ((long)b * (T + 2 * pad + tail) + pad + t) * C; }
  __host__ __device__ float* row_lo(int b, int t) const { return lo + ((long)b * (T + 2 * pad + tail) + pad + t) * C; }
  __host__ __device__ unsigned short* row_h16(int b, int t) const { return h16 + ((long)b * (T + 2 * pad + tail) + pad + t) * C; }
  __host__ __device__ unsigned short* row_l16(int b, int t) const { return l16 + ((long)b * (T + 2 * pad + tail) + pad + t) * C; }
  __host__ __device__ size_t numel() const { return (size_t)B * (T + 2 * pad + tail) * C; }
};

// C[m][n] = act( sum_k A(m,k) * W[n][k] + bias[n] + R(m,n) ), fp32 FFMA, fp32 accumulate.
//   row m -> (b = m / mper, t = m % mper);  A(m,k) = A[b*a_bs + t*a_rs + (k/kc)*a_ts + k%kc]
//   C(m,n) = C[b*c_bs + t*c_rs + n];  R likewise with r_bs/r_rs (R may be null)
// gridDim.z = groups: A += g*a_goff, W += g*w_goff, bias += g*n_goff, C/R += g*n_goff.
struct GemmP {
  const float* A = nullptr;
  const float* W = nullptr;
  const float* bias = nullptr;
  const float* R = nullptr;
  float* C = nullptr;
  const float* A_lo = nullptr;  // optional split operands / outputs (x = hi + lo), same indexing as A / R / C
  const float* R_lo = nullptr;
  float* C_lo = nullptr;
  unsigned short* C_h16 = nullptr;   // fp16-split copy of the output (C itself then holds the full value)
  unsigned short* C_l16 = nullptr;
  int M = 0, N = 0, K = 0, mper = 1;
  long a_bs = 0, a_rs = 0;
  int kc = 0, a_ts = 0;
  long c_bs = 0, c_rs = 0, r_bs = 0, r_rs = 0;
  int act = 0, ldw = 0;
  int groups = 1;
  long a_goff = 0, w_goff = 0, n_goff = 0;
};

void launch_gemm(ts_engine* e, const GemmP& p, cudaStream_t s);

// Conv1d (kernel k, stride s, zero padding p) as one GEMM over a padded channel-last input.
// x.pad must be >= p.  Output (b,t,n) is written to y.row(b, t*y_tmul + y_toff)[n] so a transposed
// conv can interleave its even/odd phases.  res (optional) is added before the activation and is
// indexed like y with y_tmul/y_toff = 1/0.
void conv1d(ts_engine* e, const Layer& L, const Act3& x, int k, int stride, int p, const Act3& y, int T_out,
            int act, const Act3* res, cudaStream_t s, int y_tmul = 1, int y_toff = 0, int x_toff = 0, int coff = 0);

// [B,C,T] -> padded channel-last Act3 (pads and channel padding zeroed); and back.
void nct_to_act(ts_engine* e, const float* in, int C, const Act3& out, cudaStream_t s);
void btc_to_act(ts_engine* e, const float* in, int C, const Act3& out, cudaStream_t s);   // in [B,T,C]
void act_to_nct(ts_engine* e, const Act3& in, int C, float* out, cudaStream_t s);          // out [B,C,T]
void act_to_btc(ts_engine* e, const Act3& in, int C, float* out, int ldo, int ooff, cudaStream_t s);
void zero_pads(ts_engine* e, const Act3& a, cudaStream_t s);

// codebook gather: idx [B*T] int64 -> out rows (C = 64)
void gather_rows(ts_engine* e, const float* table, int C, const int64_t* idx, const Act3& out, cudaStream_t s);
// VectorQuantizerEMA.get_code_indices (vqvae_modules.py:311-319): z rows -> argmin index
void vq_argmin(ts_engine* e, const float* codebook, const float* ee, int ncodes, const Act3& z, int64_t* idx,
               cudaStream_t s);

// ---- tensor-core path (gemm_tc.cu): Hopper wgmma on fp16-split or 3xTF32 operands, TMA-staged ------
bool tc_conv_supported(ts_engine* e, const Layer& L, const Act3& x, int stride, int pd);
void tc_conv1d(ts_engine* e, const Layer& L, const Act3& x, int k, int stride, int pd, const Act3& y, int T_out, int act,
               const Act3* res, cudaStream_t s, int y_tmul = 1, int y_toff = 0, int coff = 0, int chunk = 0);
void split_hi_lo(ts_engine* e, const float* x, float* hi, float* lo, long n, cudaStream_t s);
void split_host(const std::vector<float>& w, std::vector<float>* hi, std::vector<float>* lo);
// power-of-two exponent of a layer's fp16-split weight scale: max|W| * 2^shift lands in [2^13, 2^14) (0 for an all-zero layer)
int split16_shift(float max_abs);
// upload W and its (hi, lo) split copies into a Layer
void upload_weights(ts_engine* e, const std::vector<float>& W, Layer* L);
// conv through the tensor-core kernel when the geometry allows (and e->use_tc), else the FFMA kernel
void conv_auto(ts_engine* e, const Layer& L, const Act3& x, int k, int stride, int pd, const Act3& y, int T_out, int act,
               const Act3* res, cudaStream_t s, int y_tmul = 1, int y_toff = 0, int coff = 0);

// ---- debug entry points (ts_debug_*): one kernel on caller data, staged as the nets stage it ----------------------------
// x [B, a.T, a.C] -> rows [0, a.T) of every item of `a`, in a's storage format (fp32, 3xTF32 pair or fp32 + fp16 planes);
// the tail rows of every plane get NaN (no kernel may read them), pad rows keep new_act's zeros; x = NULL writes the tail
// rows only
void debug_fill(ts_engine* e, const float* x, const Act3& a, cudaStream_t s);
// copy the caller's output buffers into a's planes (back = false) or a's planes out to them (back = true): y <-> a.p, or
// plane_hi / plane_lo <-> the (hi, lo) pair (a.p, a.lo) or the fp16 planes (a.h16, a.l16) beside y <-> a.p
void debug_planes(const Act3& a, float* y, void* plane_hi, void* plane_lo, bool back, cudaStream_t s);
// the engine's dense-kernel switches (ts_set_tensor_cores numbering) for one call, restored however the call ends
struct TcModeGuard {
  ts_engine* e;
  bool use_tc, tc_f16;
  TcModeGuard(ts_engine* e_, int mode) : e(e_), use_tc(e_->use_tc), tc_f16(e_->tc_f16) {
    e->use_tc = mode != 0;
    e->tc_f16 = mode == 6;
  }
  ~TcModeGuard() {
    e->use_tc = use_tc;
    e->tc_f16 = tc_f16;
  }
};

#ifdef __CUDACC__
// two-term fp16 split of an fp32 value: h = fp16(x), l = fp16(x - h) (22 significant bits while l stays normal)
__device__ __forceinline__ void split16(float x, unsigned short& h, unsigned short& l) {
  const __half hh = __float2half_rn(x);
  h = __half_as_ushort(hh);
  l = __half_as_ushort(__float2half_rn(x - __half2float(hh)));
}
#endif

inline int cdiv(int a, int b) { return (a + b - 1) / b; }
inline int pad4(int c) { return (c + 3) & ~3; }

}  // namespace ts
