// talkshow_b200 — tensor-core implicit-GEMM for the dense contractions (face wav2vec2 convs /
// transformer, VQ decoder convs): Hopper wgmma with fp32-grade accuracy by a two-term operand split
//   x = hi + lo,  A*B ~= A_lo*B_hi + A_hi*B_lo + A_hi*B_hi  (fp32 accumulate).
//
//  * operands arrive pre-split as K-major tiles: TMA (cp.async.bulk.tensor, 128B swizzle) stages one
//    128-byte k-block of A_hi, A_lo, W_hi, W_lo per stage into a 3-stage shared-memory ring (mbarrier
//    full / empty handshake);
//  * warpgroup 0 is the TMA producer; warpgroups 1 and 2 each own 64 rows of the 128 x 128 CTA tile and
//    issue 12 wgmma.mma_async per stage (4 k-steps x 3 products) straight from the swizzled tiles;
//  * the same two warpgroups run the epilogue: bias / residual, activation, and either plain fp32 or the
//    split pair the next tensor-core GEMM consumes.
//  A Conv1d(k, stride s) is the same kernel: the A tensor map is 3-D {C, s, rows/s} over the padded
//  channel-last buffer, tap t reads box (c0, t % s, j + t / s); GEMM rows are indexed by the padded row
//  index j, rows that fall on padding are computed and discarded by the epilogue.
//
// Two operand formats, one kernel:
//  * fp16 split (ts_set_tensor_cores(e, 6), the default): h = fp16(x), l = fp16(x - h) — 11 + 11 significant bits, the
//    same as two tf32 terms — products as wgmma f16 (k16), which runs at twice the tf32 rate: a 128-byte k-block holds 64 K
//    values instead of 32.  Range: |x| < 65504 (fp16); the weights of every layer are pre-scaled by the power of two
//    (split16_shift) that puts max|W| in [2^13, 2^14) whatever the layer's magnitude -- the high plane cannot overflow and
//    the low plane stays normal for every weight within about 2^-16 of max|W| -- and the epilogue undoes it exactly;
//    activations whose low plane underflows lose absolute accuracy below 2^-25 only.
//  * 3xTF32 (modes 1 / 3 / 4): hi = fp32 with the 13 low mantissa bits cleared, lo = x - hi (exact), wgmma tf32 (k8).
#include <cuda.h>
#include <cuda_fp16.h>

#include <climits>

#include "convstack.h"

namespace ts {

constexpr int TC_BM = 128, TC_BN = 128;
constexpr int TC_BK = 32;                                   // fp32 values per 128-byte k-block row (64 for fp16 planes)
constexpr int TC_STAGES = 3;
constexpr int TC_TILE_BYTES = 128 * 128;                    // 16 KB: 128 rows x 128 bytes (A and B tiles alike)
constexpr int TC_STAGE_BYTES = 4 * TC_TILE_BYTES;           // A_hi, A_lo, B_hi, B_lo = 64 KB
constexpr int TC_THREADS = 384;                             // warpgroup 0: TMA; warpgroups 1, 2: wgmma + epilogue
constexpr int TC_SMEM = TC_STAGES * TC_STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
constexpr int TC_SLD = TC_BN + 4;                           // padded row of the parked output tile (floats)
static_assert(TC_BM * TC_SLD * 4 + 2 * TC_BM * 8 <= TC_STAGES * TC_STAGE_BYTES, "parked tile must fit in the operand ring");
static_assert(TC_SMEM <= 227 * 1024, "shared memory per block");
// The tensor core's fp32 accumulation is not round-to-nearest (error grows linearly with K, biased toward zero), so K
// is accumulated by wgmma only over chunks of P.chunk k-blocks (K = 256); each chunk is then added into a second set of
// fp32 registers with round-to-nearest adds.

struct TcArgs {
  int taps, cblocks, stride;        // K loop = taps x (C / k-block)
  int C;                            // input channels (K per tap)
  int rows_in, off, T_out, nbatch;  // epilogue row mapping (see header)
  int Rs;                           // GEMM rows (padded row index / stride)
  int N;
  float* c_hi;                      // output (plain fp32 when c_lo == nullptr)
  float* c_lo;
  long c_bs, c_rs;
  const float* bias;
  const float* r_hi;                // residual: plain (r_lo null) or split
  const float* r_lo;
  long r_bs, r_rs;
  int act;
  int chunk;                        // k-blocks accumulated by wgmma before the round-to-nearest add (K = 256)
  float oscale;                     // accumulator scale (undoes the power-of-two weight scale of the fp16 split), 1 for tf32
  unsigned short* c_h16;            // fp16-split copy of the output (c_hi then holds the full value, c_lo is null)
  unsigned short* c_l16;
};

__device__ __forceinline__ uint32_t s_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mb_init(uint64_t* b, int c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s_u32(b)), "r"(c)); }
__device__ __forceinline__ void mb_expect(uint64_t* b, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s_u32(b)), "r"(bytes) : "memory");
}
// lane 0 arrives; predicated rather than branched, so the wgmma loop around it stays free of divergent control flow
__device__ __forceinline__ void mb_arrive_lane0(uint64_t* b, int lane) {
  asm volatile("{\n.reg .pred p;\nsetp.eq.s32 p, %1, 0;\n@p mbarrier.arrive.shared::cta.b64 _, [%0];\n}\n" ::"r"(s_u32(b)), "r"(lane) : "memory");
}
__device__ __forceinline__ void mb_wait(uint64_t* b, uint32_t parity) {
  asm volatile(
      "{\n.reg .pred p;\nTCW:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra TCD;\nbra TCW;\nTCD:\n}\n" ::"r"(s_u32(b)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_3d(void* dst, const CUtensorMap* m, int c0, int c1, int c2, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(s_u32(dst)),
               "l"(m), "r"(c0), "r"(c1), "r"(c2), "r"(s_u32(bar))
               : "memory");
}
__device__ __forceinline__ void tma_2d(void* dst, const CUtensorMap* m, int c0, int c1, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(s_u32(dst)),
               "l"(m), "r"(c0), "r"(c1), "r"(s_u32(bar))
               : "memory");
}
// wgmma shared-memory descriptor of a K-major, 128B-swizzled tile: 8-row groups 1024 B apart (SBO), LBO unused (1)
__device__ __forceinline__ uint64_t wg_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3fff);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;  // SWIZZLE_128B
  return d;
}
#define TC_ACC64                                                                                                              \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, " \
  "%26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, "   \
  "%50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
#define TC_ACC64_OPS(d)                                                                                                       \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),     \
      "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),    \
      "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),    \
      "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),    \
      "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),    \
      "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),    \
      "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
// D[64 x 128] (+)= A[64 x k] * B[128 x k]^T, both operands K-major in shared memory; scale_d == 0 overwrites D
template <bool F16>
__device__ __forceinline__ void wgmma_64x128(float (&d)[64], uint64_t a, uint64_t b, int scale_d) {
  if constexpr (F16)
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " TC_ACC64 ", %64, %65, p, 1, 1, 0, 0;\n}\n"
                 : TC_ACC64_OPS(d)
                 : "l"(a), "l"(b), "r"(scale_d));
  else
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 " TC_ACC64 ", %64, %65, p, 1, 1;\n}\n"
                 : TC_ACC64_OPS(d)
                 : "l"(a), "l"(b), "r"(scale_d));
}
#undef TC_ACC64
#undef TC_ACC64_OPS
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ float tc_act(float v, int act) {
  if (act == ACT_RELU) return v > 0.f ? v : 0.f;
  if (act == ACT_LRELU) return v > 0.f ? v : 0.2f * v;
  if (act == ACT_GELU) return 0.5f * v * (1.0f + erff(v * 0.70710678118654752440f));
  return v;
}

// Write-out of the parked tile by the 256 epilogue threads (threads 128..383).  Thread -> 4 fixed columns (bias loaded
// once), rows strided by 256 / CG: coalesced bias / residual loads and float4 stores from a compact loop instead of a
// fully unrolled per-register epilogue.  CG = float4 column groups per parked row, SLD = parked row stride.
template <int ACT, int CG, int SLD>
__device__ __forceinline__ void tc_writeout(const TcArgs& P, const float* S, const long* rowc, const long* rowr, int n0) {
  const int et = threadIdx.x - 128;
  const int c4 = (et % CG) * 4, n = n0 + c4;
  if (n >= P.N) return;
  const int nv = min(4, P.N - n);                   // valid columns of this thread (4 except at a ragged N edge)
  float bv[4] = {0.f, 0.f, 0.f, 0.f};
  if (P.bias)
    for (int q = 0; q < nv; ++q) bv[q] = P.bias[n + q];
  const float osc = P.oscale;
  const bool rvec = nv == 4 && P.r_hi && (((P.r_bs | P.r_rs) & 3) == 0) && ((reinterpret_cast<uintptr_t>(P.r_hi) & 15) == 0) &&
                    (!P.r_lo || (reinterpret_cast<uintptr_t>(P.r_lo) & 15) == 0);
#pragma unroll 4
  for (int r = et / CG; r < TC_BM; r += 256 / CG) {
    const long co = rowc[r];
    if (co < 0) continue;
    const float4 sv = *reinterpret_cast<const float4*>(&S[r * SLD + c4]);
    float o[4] = {sv.x * osc + bv[0], sv.y * osc + bv[1], sv.z * osc + bv[2], sv.w * osc + bv[3]};
    if (P.r_hi) {
      const long roff = rowr[r] + n;
      if (rvec) {
        const float4 rh = *reinterpret_cast<const float4*>(P.r_hi + roff);
        if (P.r_lo) {
          const float4 rl = *reinterpret_cast<const float4*>(P.r_lo + roff);
          o[0] += rh.x + rl.x; o[1] += rh.y + rl.y; o[2] += rh.z + rl.z; o[3] += rh.w + rl.w;
        } else {
          o[0] += rh.x; o[1] += rh.y; o[2] += rh.z; o[3] += rh.w;
        }
      } else {
        for (int q = 0; q < nv; ++q) o[q] += P.r_lo ? (P.r_hi[roff + q] + P.r_lo[roff + q]) : P.r_hi[roff + q];
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (ACT == ACT_GELU) o[q] = 0.5f * o[q] * (1.0f + erff(o[q] * 0.70710678118654752440f));
      else if (ACT != ACT_NONE) o[q] = tc_act(o[q], P.act);
    }
    const long coff = co + n;
    if (nv == 4) {
      if (P.c_h16) {
        if (P.c_hi) *reinterpret_cast<float4*>(P.c_hi + coff) = make_float4(o[0], o[1], o[2], o[3]);
        ushort4 h, l;
        split16(o[0], h.x, l.x); split16(o[1], h.y, l.y); split16(o[2], h.z, l.z); split16(o[3], h.w, l.w);
        *reinterpret_cast<ushort4*>(P.c_h16 + coff) = h;
        *reinterpret_cast<ushort4*>(P.c_l16 + coff) = l;
      } else if (P.c_lo) {
        float4 h, l;
        h.x = __uint_as_float(__float_as_uint(o[0]) & 0xffffe000u); l.x = o[0] - h.x;
        h.y = __uint_as_float(__float_as_uint(o[1]) & 0xffffe000u); l.y = o[1] - h.y;
        h.z = __uint_as_float(__float_as_uint(o[2]) & 0xffffe000u); l.z = o[2] - h.z;
        h.w = __uint_as_float(__float_as_uint(o[3]) & 0xffffe000u); l.w = o[3] - h.w;
        *reinterpret_cast<float4*>(P.c_hi + coff) = h;
        *reinterpret_cast<float4*>(P.c_lo + coff) = l;
      } else {
        *reinterpret_cast<float4*>(P.c_hi + coff) = make_float4(o[0], o[1], o[2], o[3]);
      }
    } else {
      for (int q = 0; q < nv; ++q) {
        if (P.c_h16) {
          if (P.c_hi) P.c_hi[coff + q] = o[q];
          split16(o[q], P.c_h16[coff + q], P.c_l16[coff + q]);
        } else if (P.c_lo) {
          const float h = __uint_as_float(__float_as_uint(o[q]) & 0xffffe000u);
          P.c_hi[coff + q] = h;
          P.c_lo[coff + q] = o[q] - h;
        } else {
          P.c_hi[coff + q] = o[q];
        }
      }
    }
  }
}

// One 128 x 128 output tile per CTA.  N tiles vary fastest (blockIdx.x): the CTAs that share an A row block run together
// and hit it in L2.
template <bool F16>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_gemm_kernel(const __grid_constant__ CUtensorMap mA_hi, const __grid_constant__ CUtensorMap mA_lo,
               const __grid_constant__ CUtensorMap mB_hi, const __grid_constant__ CUtensorMap mB_lo, TcArgs P) {
  extern __shared__ unsigned char tc_smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(tc_smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + TC_STAGES * TC_STAGE_BYTES);
  uint64_t* empty = full + TC_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int j0 = blockIdx.y * TC_BM, n0 = blockIdx.x * TC_BN;
  const int nk = P.taps * P.cblocks;
  constexpr int BK = F16 ? 2 * TC_BK : TC_BK;      // K values per 128-byte k-block row

  if (threadIdx.x == 0) {
    // empty: one arrival per consumer warp (2 warpgroups x 4 warps)
    for (int i = 0; i < TC_STAGES; ++i) { mb_init(&full[i], 1); mb_init(&empty[i], 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mA_hi) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mA_lo) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mB_hi) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mB_lo) : "memory");
  }
  __syncthreads();

  if (warp < 4) {
    if (threadIdx.x == 0) {  // ===== TMA producer =====
      for (int kb = 0; kb < nk; ++kb) {
        const int st = kb % TC_STAGES, ph = (kb / TC_STAGES) & 1;
        mb_wait(&empty[st], ph ^ 1);
        const int tap = kb / P.cblocks, cb = kb - tap * P.cblocks;
        unsigned char* base = smem + st * TC_STAGE_BYTES;
        mb_expect(&full[st], TC_STAGE_BYTES);
        const int c0 = cb * BK, c1 = tap % P.stride, c2 = j0 + tap / P.stride;
        const int kcol = tap * P.C + cb * BK;
        tma_3d(base, &mA_hi, c0, c1, c2, &full[st]);
        tma_3d(base + TC_TILE_BYTES, &mA_lo, c0, c1, c2, &full[st]);
        tma_2d(base + 2 * TC_TILE_BYTES, &mB_hi, kcol, n0, &full[st]);
        tma_2d(base + 3 * TC_TILE_BYTES, &mB_lo, kcol, n0, &full[st]);
      }
    }
    return;
  }

  // ===== consumers: warpgroup wg owns rows [64 wg, +64) of the tile =====
  const int wg = (warp >> 2) - 1;
  float acc[64], sum[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) sum[i] = 0.f;
  for (int c0 = 0; c0 < nk; c0 += P.chunk) {
    const int cend = min(nk, c0 + P.chunk);
    for (int kb = c0; kb < cend; ++kb) {
      const int st = kb % TC_STAGES, ph = (kb / TC_STAGES) & 1;
      mb_wait(&full[st], ph);
      const uint32_t a_hi = s_u32(smem + st * TC_STAGE_BYTES) + wg * 64 * 128, a_lo = a_hi + TC_TILE_BYTES;
      const uint32_t b_hi = s_u32(smem + st * TC_STAGE_BYTES) + 2 * TC_TILE_BYTES, b_lo = b_hi + TC_TILE_BYTES;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t o = k * 32;    // 32 bytes along K inside the 128 B swizzle atom: 8 tf32 or 16 fp16 = one wgmma's K
        wgmma_64x128<F16>(acc, wg_desc(a_lo + o), wg_desc(b_hi + o), (kb > c0) | k);
        wgmma_64x128<F16>(acc, wg_desc(a_hi + o), wg_desc(b_lo + o), 1);
        wgmma_64x128<F16>(acc, wg_desc(a_hi + o), wg_desc(b_hi + o), 1);
      }
      wgmma_commit();
      wgmma_wait<1>();                             // the previous k-block's products are done with its stage
      __syncwarp();
      if (kb > c0) mb_arrive_lane0(&empty[(kb + TC_STAGES - 1) % TC_STAGES], lane);
    }
    wgmma_wait<0>();                               // chunk accumulated: drain it with round-to-nearest adds
    __syncwarp();
    mb_arrive_lane0(&empty[(cend - 1) % TC_STAGES], lane);
#pragma unroll
    for (int i = 0; i < 64; ++i) sum[i] += acc[i];
  }

  // ---- park the tile S[row][col] in the (now idle) operand ring, plus the output / residual offset of every GEMM row ----
  asm volatile("bar.sync 1, 256;" ::: "memory");   // both consumer warpgroups are done reading the ring
  float* S = reinterpret_cast<float*>(smem);
  long* rowc = reinterpret_cast<long*>(S + TC_BM * TC_SLD);
  long* rowr = rowc + TC_BM;
  {
    // wgmma m64nN f32 accumulator layout: register i of lane l in warp w (of the warpgroup) holds
    // row 16 w + l / 4 + 8 ((i / 2) % 2), column 8 (i / 4) + 2 (l % 4) + i % 2
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
      const int r = r0 + 8 * ((i >> 1) & 1), c = c0 + 8 * (i >> 2);
      *reinterpret_cast<float2*>(&S[r * TC_SLD + c]) = make_float2(sum[i], sum[i + 1]);
    }
  }
  const int et = threadIdx.x - 128;
  if (et < TC_BM) {  // GEMM row j <-> padded input row j*stride -> (batch, output step)
    const int j = j0 + et;
    long co = -1, ro = 0;
    if (j < P.Rs) {
      const long in_row = (long)j * P.stride;
      const int bb = (int)(in_row / P.rows_in);
      const int tin = (int)(in_row - (long)bb * P.rows_in) - P.off;
      if (bb < P.nbatch && tin >= 0 && (tin % P.stride) == 0 && tin / P.stride < P.T_out) {
        const int t = tin / P.stride;
        co = (long)bb * P.c_bs + (long)t * P.c_rs;
        ro = (long)bb * P.r_bs + (long)t * P.r_rs;
      }
    }
    rowc[et] = co;
    rowr[et] = ro;
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");
  if (P.act == ACT_NONE) tc_writeout<ACT_NONE, TC_BN / 4, TC_SLD>(P, S, rowc, rowr, n0);
  else if (P.act == ACT_GELU) tc_writeout<ACT_GELU, TC_BN / 4, TC_SLD>(P, S, rowc, rowr, n0);
  else tc_writeout<-1, TC_BN / 4, TC_SLD>(P, S, rowc, rowr, n0);
}

// ---- split kernels ------------------------------------------------------------------------------
__global__ void split_kernel(const float* __restrict__ x, float* __restrict__ hi, float* __restrict__ lo, long n) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    float v = x[i];
    float h = __uint_as_float(__float_as_uint(v) & 0xffffe000u);
    hi[i] = h;
    lo[i] = v - h;
  }
}
void split_hi_lo(ts_engine* e, const float* x, float* hi, float* lo, long n, cudaStream_t s) {
  if (e->ws.sizing || n <= 0) return;
  split_kernel<<<(int)std::min<long>((n + 255) / 256, (long)e->sm_count * 16), 256, 0, s>>>(x, hi, lo, n);
  e->launches++;
  TS_CUDA(cudaGetLastError());
}
int split16_shift(float max_abs) {
  if (!(max_abs > 0.f) || !std::isfinite(max_abs)) return 0;   // all-zero (or non-finite) layer: unscaled
  int ex;
  std::frexp(max_abs, &ex);                                       // max_abs = m * 2^ex, m in [0.5, 1)
  return std::min(100, std::max(-100, 14 - ex));                  // 2^+-100 stays a normal float
}
// fp16 planes of W * 2^shift (split16_shift); returns the epilogue's 2^-shift
static float split16_host(const std::vector<float>& w, std::vector<unsigned short>* h, std::vector<unsigned short>* l) {
  float mx = 0.f;
  for (float v : w) mx = std::max(mx, std::fabs(v));
  const int shift = split16_shift(mx);
  const float sc = std::ldexp(1.0f, shift);
  h->resize(w.size());
  l->resize(w.size());
  for (size_t i = 0; i < w.size(); ++i) {
    const float v = w[i] * sc;
    const __half hh = __float2half_rn(v);
    const __half ll = __float2half_rn(v - __half2float(hh));
    (*h)[i] = __half_as_ushort(hh);
    (*l)[i] = __half_as_ushort(ll);
  }
  return std::ldexp(1.0f, -shift);
}
void split_host(const std::vector<float>& w, std::vector<float>* hi, std::vector<float>* lo) {
  hi->resize(w.size());
  lo->resize(w.size());
  for (size_t i = 0; i < w.size(); ++i) {
    uint32_t u;
    memcpy(&u, &w[i], 4);
    u &= 0xffffe000u;
    float h;
    memcpy(&h, &u, 4);
    (*hi)[i] = h;
    (*lo)[i] = w[i] - h;
  }
}

// ---- host launcher -------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    TS_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
    if (!p || q != cudaDriverEntryPointSuccess) fail(TS_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
    fn = (EncodeTiledFn)p;
  }
  return fn;
}
static CUtensorMap make_map(const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes, const cuuint32_t* box,
                            bool f16 = false) {
  CUtensorMap m;
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = get_encode()(&m, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, rank, (void*)base, dims, strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) fail(TS_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) rank %d dims %llu,%llu", (int)r, rank, (unsigned long long)dims[0],
                              (unsigned long long)dims[1]);
  return m;
}

bool tc_conv_supported(ts_engine* e, const Layer& L, const Act3& x, int stride, int pd) {
  if (e->tc_f16) {   // fp16 planes
    if (!L.W_h16 || !x.h16 || x.C % (2 * TC_BK)) return false;
  } else {           // 3xTF32: operands pre-split in HBM
    if (!L.W_hi || !x.lo || x.C % TC_BK) return false;
  }
  const int rows_in = x.T + 2 * x.pad + x.tail;
  if (rows_in % stride || (x.pad - pd) % stride || x.pad < pd) return false;
  return true;
}

// y(b, t*y_tmul + y_toff, :) = act( conv(x)(b,t,:) + bias + res(b,t,:) );  x and W must be split (hi/lo)
void tc_conv1d(ts_engine* e, const Layer& L, const Act3& x, int k, int stride, int pd, const Act3& y, int T_out, int act, const Act3* res,
               cudaStream_t s, int y_tmul, int y_toff, int coff, int chunk) {
  if (e->ws.sizing) return;
  if (!tc_conv_supported(e, L, x, stride, pd)) fail(TS_ERR_INVALID, "tc_conv1d: unsupported geometry");
  if (!y.p && !y.h16) fail(TS_ERR_INVALID, "tc_conv1d: output without storage");
  const bool f16 = e->tc_f16;
  const int esz = f16 ? 2 : 4, bk = f16 ? 2 * TC_BK : TC_BK;
  if (L.taps != k || L.cin != x.C) fail(TS_ERR_INVALID, "tc_conv1d: layer/input mismatch");
  const int rows_in = x.T + 2 * x.pad + x.tail;
  const long R = (long)x.B * rows_in;
  const long Rs = R / stride;
  const void* base_hi = f16 ? (const void*)x.h16 : (const void*)x.p;   // first padded row of batch 0 (allocation start)
  const void* base_lo = f16 ? (const void*)x.l16 : (const void*)x.lo;
  cuuint64_t adims[3] = {(cuuint64_t)x.C, (cuuint64_t)stride, (cuuint64_t)Rs};
  cuuint64_t astr[2] = {(cuuint64_t)x.C * esz, (cuuint64_t)x.C * esz * stride};
  const int tiles_n = (L.N + TC_BN - 1) / TC_BN, tiles_m = (int)((Rs + TC_BM - 1) / TC_BM);
  cuuint32_t abox[3] = {(cuuint32_t)bk, 1, (cuuint32_t)TC_BM};
  CUtensorMap mAh = make_map(base_hi, 3, adims, astr, abox, f16), mAl = make_map(base_lo, 3, adims, astr, abox, f16);
  cuuint64_t bdims[2] = {(cuuint64_t)L.K, (cuuint64_t)L.N};
  cuuint64_t bstr[1] = {(cuuint64_t)L.K * esz};
  cuuint32_t bbox[2] = {(cuuint32_t)bk, (cuuint32_t)TC_BN};
  const void* wh = f16 ? (const void*)L.W_h16 : (const void*)L.W_hi;
  const void* wl = f16 ? (const void*)L.W_l16 : (const void*)L.W_lo;
  CUtensorMap mBh = make_map(wh, 2, bdims, bstr, bbox, f16), mBl = make_map(wl, 2, bdims, bstr, bbox, f16);
  TcArgs P;
  if (chunk < 0) fail(TS_ERR_INVALID, "tc_conv1d: chunk %d < 0", chunk);
  P.chunk = chunk ? chunk : 256 / bk;  // default: K = 256 per wgmma accumulation chunk
  P.oscale = f16 ? L.w_unscale : 1.f;
  P.c_h16 = y.h16 ? y.row_h16(0, y_toff) + coff : nullptr;
  P.c_l16 = y.h16 ? y.row_l16(0, y_toff) + coff : nullptr;
  P.taps = k; P.cblocks = x.C / bk; P.stride = stride; P.C = x.C;
  P.rows_in = rows_in; P.off = x.pad - pd; P.T_out = T_out; P.nbatch = x.B; P.Rs = (int)Rs; P.N = L.N;
  P.c_hi = y.p ? y.row(0, y_toff) + coff : nullptr; P.c_lo = y.lo ? y.row_lo(0, y_toff) + coff : nullptr;
  P.c_bs = y.bstride(); P.c_rs = (long)y_tmul * y.C;
  P.bias = L.bias;
  P.r_hi = res ? res->row(0, 0) : nullptr;
  P.r_lo = (res && res->lo) ? res->row_lo(0, 0) : nullptr;
  P.r_bs = res ? res->bstride() : 0; P.r_rs = res ? res->C : 0;
  P.act = act;
  if (!e->tc_attr_set) {   // the max-dynamic-smem attribute is per device: cached per engine, not per process
    TS_CUDA(cudaFuncSetAttribute(tc_gemm_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM));
    TS_CUDA(cudaFuncSetAttribute(tc_gemm_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM));
    e->tc_attr_set = true;
  }
  // surplus rows of the last M tile fall outside Rs and are masked (TMA zero-fills out-of-bounds boxes)
  const dim3 grid((unsigned)tiles_n, (unsigned)tiles_m);
  if (f16) tc_gemm_kernel<true><<<grid, TC_THREADS, TC_SMEM, s>>>(mAh, mAl, mBh, mBl, P);
  else tc_gemm_kernel<false><<<grid, TC_THREADS, TC_SMEM, s>>>(mAh, mAl, mBh, mBl, P);
  e->launches++;
  TS_CUDA(cudaGetLastError());
}

void upload_weights(ts_engine* e, const std::vector<float>& W, Layer* L) {
  L->W = e->upload(W);
  std::vector<float> hi, lo;
  split_host(W, &hi, &lo);
  L->W_hi = e->upload(hi);
  L->W_lo = e->upload(lo);
  std::vector<unsigned short> h16, l16;
  L->w_unscale = split16_host(W, &h16, &l16);
  L->W_h16 = e->upload(h16);
  L->W_l16 = e->upload(l16);
}

void conv_auto(ts_engine* e, const Layer& L, const Act3& x, int k, int stride, int pd, const Act3& y, int T_out, int act, const Act3* res,
               cudaStream_t s, int y_tmul, int y_toff, int coff) {
  if (e->use_tc && (y.C % 4) == 0 && (coff % 4) == 0 && tc_conv_supported(e, L, x, stride, pd)) tc_conv1d(e, L, x, k, stride, pd, y, T_out, act, res, s, y_tmul, y_toff, coff);
  else conv1d(e, L, x, k, stride, pd, y, T_out, act, res, s, y_tmul, y_toff, 0, coff);
}

}  // namespace ts

using namespace ts;

extern "C" int ts_set_tensor_cores(ts_engine* e, int enable) {
  if (!e) return TS_ERR_INVALID;
  if (enable < 0 || enable > 6 || enable == 2 || enable == 5) {
    e->err = "ts_set_tensor_cores: modes are 0 (FFMA), 1 / 3 / 4 (3xTF32 wgmma) and 6 (fp16-split wgmma)";
    return TS_ERR_UNSUPPORTED;
  }
  e->use_tc = enable != 0;
  e->tc_f16 = enable == 6;   // 6 (default): fp16-split operands (see the file header); 1 / 3 / 4: 3xTF32
  return TS_OK;
}

namespace ts {
// x [B, a.T, a.C] -> rows [0, a.T) of every batch item of `a`, in a's storage format (fp32, 3xTF32 pair or fp32 + fp16
// planes); the tail rows of every plane get NaN: no conv may read them.  Pad rows keep new_act's zeros.  x = NULL: rows
// [0, a.T) are left as they are (only the tail rows are written).
__global__ void debug_fill_kernel(const float* __restrict__ x, Act3 a) {
  const int rows = a.T + 2 * a.pad + a.tail;
  const long n = (long)a.B * rows * a.C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % a.C), r = (int)((i / a.C) % rows), b = (int)(i / ((long)a.C * rows));
    const int t = r - a.pad;
    float v;
    if (t >= 0 && t < a.T) {
      if (!x) continue;
      v = x[((long)b * a.T + t) * a.C + c];
    }
    else if (r >= a.T + 2 * a.pad) v = __int_as_float(0x7fffffff);
    else continue;
    if (a.lo) {
      const float h = __uint_as_float(__float_as_uint(v) & 0xffffe000u);
      a.p[i] = h;
      a.lo[i] = v - h;
    } else {
      if (a.p) a.p[i] = v;
      if (a.h16) split16(v, a.h16[i], a.l16[i]);
    }
  }
}

void debug_fill(ts_engine* e, const float* x, const Act3& a, cudaStream_t s) {
  debug_fill_kernel<<<(int)std::min<long>((long)(a.numel() + 255) / 256, (long)e->sm_count * 16), 256, 0, s>>>(x, a);
  e->launches++;
  TS_CUDA(cudaGetLastError());
}

void debug_planes(const Act3& a, float* y, void* plane_hi, void* plane_lo, bool back, cudaStream_t s) {
  const size_t n = a.numel();
  struct Plane { void* dev; void* user; size_t bytes; };
  const Plane planes[4] = {{a.p, a.lo ? plane_hi : (void*)y, n * 4}, {a.lo, plane_lo, n * 4}, {a.h16, plane_hi, n * 2}, {a.l16, plane_lo, n * 2}};
  for (const Plane& p : planes)
    if (p.dev) TS_CUDA(cudaMemcpyAsync(back ? p.user : p.dev, back ? p.dev : p.user, p.bytes, cudaMemcpyDeviceToDevice, s));
}
}  // namespace ts

extern "C" int ts_debug_conv1d(ts_engine* e, const ts_debug_conv* a, const float* x, const float* W_host, const float* bias_host,
                               const float* res, float* y, void* y_plane_hi, void* y_plane_lo, void* stream) {
  TS_API_BEGIN(e)
  require_device(e);
  if (!a || !x || !W_host) fail(TS_ERR_INVALID, "ts_debug_conv1d: a, x and W_host are required");
  const ts_debug_conv g = *a;
  const int mode = g.mode;
  if (mode != 0 && mode != 1 && mode != 6) fail(TS_ERR_INVALID, "ts_debug_conv1d: mode %d (0 = FFMA, 1 = wgmma 3xTF32, 6 = wgmma fp16-split)", mode);
  if (g.B < 1 || g.T < 1 || g.C < 1 || g.N < 1 || g.k < 1 || g.stride < 1 || g.T_out < 1 || g.x_pad < 0 || g.x_tail < 0 || g.pd < 0 ||
      g.y_T < 1 || g.y_C < 1 || g.y_pad < 0 || g.y_tmul < 1 || g.y_toff < 0 || g.coff < 0 || g.res_pad < 0 || g.chunk < 0)
    fail(TS_ERR_INVALID, "ts_debug_conv1d: an empty or negative size");
  if (g.act < ACT_NONE || g.act > ACT_GELU) fail(TS_ERR_INVALID, "ts_debug_conv1d: act %d (0 none, 1 ReLU, 2 LReLU 0.2, 3 GELU)", g.act);
  if (g.pd > g.x_pad) fail(TS_ERR_INVALID, "ts_debug_conv1d: conv padding %d > input pad rows %d", g.pd, g.x_pad);
  if ((long)(g.T_out - 1) * g.stride + g.k > (long)g.T + g.x_pad + g.pd)
    fail(TS_ERR_INVALID, "ts_debug_conv1d: the window of output %d reaches past the input's back pad rows", g.T_out - 1);
  if ((long)(g.T_out - 1) * g.y_tmul + g.y_toff >= g.y_T || (long)g.coff + g.N > g.y_C)
    fail(TS_ERR_INVALID, "ts_debug_conv1d: outputs fall outside y [%d rows, %d columns]", g.y_T, g.y_C);
  const long rows_in = (long)g.T + 2L * g.x_pad + g.x_tail;
  if ((long)g.B * rows_in > INT_MAX || (long)g.B * (g.y_T + 2L * g.y_pad) > INT_MAX)
    fail(TS_ERR_INVALID, "ts_debug_conv1d: more than 2^31 - 1 rows");
  if (mode == 0) {
    if (g.C % 4) fail(TS_ERR_INVALID, "ts_debug_conv1d: the FFMA kernel needs C %% 4 == 0 (C = %d)", g.C);
  } else {
    const int bk = mode == 6 ? 2 * TC_BK : TC_BK;
    if (g.C % bk) fail(TS_ERR_INVALID, "ts_debug_conv1d: C %d is not a multiple of the %d-value k-block of mode %d", g.C, bk, mode);
    if (rows_in % g.stride || (g.x_pad - g.pd) % g.stride)
      fail(TS_ERR_INVALID, "ts_debug_conv1d: rows per item (%ld) and x_pad - pd (%d) must be multiples of the stride %d", rows_in,
           g.x_pad - g.pd, g.stride);
    if (g.y_C % 4 || g.coff % 4)
      fail(TS_ERR_INVALID, "ts_debug_conv1d: the wgmma epilogue stores 4 columns at a time: y_C %d and coff %d must be multiples of 4", g.y_C,
           g.coff);
  }
  const bool x_planes = (g.planes_only & 1) != 0, y_planes = (g.planes_only & 2) != 0;
  if (g.planes_only & ~3) fail(TS_ERR_INVALID, "ts_debug_conv1d: planes_only %d (bit 0 input, bit 1 output)", g.planes_only);
  if ((x_planes || y_planes) && mode != 6) fail(TS_ERR_INVALID, "ts_debug_conv1d: planes-only activations exist in mode 6 only");
  if (y_planes && !g.y_split) fail(TS_ERR_INVALID, "ts_debug_conv1d: a planes-only output needs y_split");
  if (g.y_split && (!y_plane_hi || !y_plane_lo)) fail(TS_ERR_INVALID, "ts_debug_conv1d: y_split needs y_plane_hi and y_plane_lo");
  const bool y_full = !g.y_split || (mode == 6 && !y_planes);   // an fp32 copy of the full value exists
  if (y_full && !y) fail(TS_ERR_INVALID, "ts_debug_conv1d: y is required");

  // torch Conv1d weight [N][C][k] -> the packed layout [N][k][C] (tap-major), production split
  std::vector<float> W((size_t)g.N * g.k * g.C);
  for (int n = 0; n < g.N; ++n)
    for (int c = 0; c < g.C; ++c)
      for (int t = 0; t < g.k; ++t) W[((size_t)n * g.k + t) * g.C + c] = W_host[((size_t)n * g.C + c) * g.k + t];
  LoadScope scope(e, "debug_conv");   // this call's weights replace the previous call's
  Layer L;
  L.N = g.N; L.K = g.k * g.C; L.taps = g.k; L.cin = g.C;
  upload_weights(e, W, &L);
  if (bias_host) L.bias = e->upload(std::vector<float>(bias_host, bias_host + g.N));

  TcModeGuard guard(e, mode);
  cudaStream_t s = (cudaStream_t)stream;
  Act3 xa, ya, ra;
  run_sized(e, [&] {
    xa = new_act(e, g.B, g.T, g.C, g.x_pad, s, mode != 0, g.x_tail, x_planes);
    ya = new_act(e, g.B, g.y_T, g.y_C, g.y_pad, s, g.y_split != 0, 0, y_planes);
    if (res) ra = new_act(e, g.B, g.T_out, g.N, g.res_pad, s, g.res_split != 0);
  });
  debug_fill(e, x, xa, s);
  if (res) debug_fill(e, res, ra, s);
  debug_planes(ya, y, y_plane_hi, y_plane_lo, false, s);
  if (mode == 0) conv1d(e, L, xa, g.k, g.stride, g.pd, ya, g.T_out, g.act, res ? &ra : nullptr, s, g.y_tmul, g.y_toff, 0, g.coff);
  else tc_conv1d(e, L, xa, g.k, g.stride, g.pd, ya, g.T_out, g.act, res ? &ra : nullptr, s, g.y_tmul, g.y_toff, g.coff, g.chunk);
  debug_planes(ya, y, y_plane_hi, y_plane_lo, true, s);
  TS_CUDA(cudaStreamSynchronize(s));
  scope.commit();
  TS_API_END(e)
}
