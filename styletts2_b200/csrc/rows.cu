// Row-layout ops of the style denoiser and the duration encoder (fp32 SIMT path):
// fused (concat / +mapping) -> LayerNorm x2, Linear (SGEMM), attention, token mean.
#include "common.cuh"

namespace st2 {
extern long long g_launches;

// ------------------------------------------------------------------------------------------
// rows_ln: one warp per row, row kept in registers (C <= 1024, C % 32 == 0).
// PACKED: M packed token rows, the utterance of row r is row_utt[r] (no padding rows, so nothing is masked).
template <bool PACKED>
__global__ void __launch_bounds__(256) rows_ln_kernel(const st2_rows_args a, const int* __restrict__ row_utt, int M) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= (PACKED ? M : a.B * a.N)) return;
  const int b = PACKED ? row_utt[row] : row / a.N;
  const bool masked = !PACKED && a.lengths && row - b * a.N >= a.lengths[b];
  const int per = a.C >> 5;
  float v[32];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    v[i] = 0.f;
    if (i < per) {
      const int c = lane + 32 * i;
      float h;
      if (a.h_in) h = a.h_in[(long long)row * a.h_in_ld + c];
      else h = c < a.Cx ? a.xs * a.x[b * a.Cx + c] : a.emb[(long long)row * a.emb_ld + (c - a.Cx)];
      if (a.add) h += a.add[(long long)b * a.C + c];
      v[i] = h;
      s += h;
      if (a.h_out) a.h_out[(long long)row * a.h_out_ld + c] = masked ? 0.f : h;
    }
  }
  if (!a.out1) return;
  const float mean = warp_sum(s) / (float)a.C;
  float m2 = 0.f;
#pragma unroll
  for (int i = 0; i < 32; ++i)
    if (i < per) {
      const float d = v[i] - mean;
      m2 = fmaf(d, d, m2);
    }
  const float rstd = 1.0f / sqrtf(warp_sum(m2) / (float)a.C + a.eps);
  const float one = a.ada ? 1.0f : 0.0f;
  const long long go = (long long)b * a.gb_bstride;
#pragma unroll
  for (int i = 0; i < 32; ++i)
    if (i < per) {
      const int c = lane + 32 * i;
      const float z = (v[i] - mean) * rstd;
      float g = a.g1 ? a.g1[go + c] + one : 1.0f;
      float o = z * g + (a.b1 ? a.b1[go + c] : 0.f);
      a.out1[(long long)row * a.out1_ld + c] = masked ? 0.f : o;
      if (a.out2) {
        g = a.g2 ? a.g2[go + c] + one : 1.0f;
        o = z * g + (a.b2 ? a.b2[go + c] : 0.f);
        a.out2[(long long)row * a.out2_ld + c] = masked ? 0.f : o;
      }
    }
}

__global__ void bcast_cols_kernel(float* __restrict__ dst, long long ld, int col0, const float* __restrict__ src, int B, int N,
                                  int W, const int* __restrict__ lengths) {
  const long long total = (long long)B * N * W;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(i % W);
    const long long r = i / W;
    const int b = (int)(r / N), n = (int)(r % N);
    const bool masked = lengths && n >= lengths[b];
    dst[r * ld + col0 + j] = masked ? 0.f : src[(long long)b * W + j];
  }
}

// out[b,c] = mean_n h[(b,n),c]; fixed-order serial sum per (b,c) (N <= 512), coalesced over c.
__global__ void mean_rows_kernel(const float* __restrict__ h, long long ld, int N, int C, float* __restrict__ out) {
  const int b = blockIdx.y;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float* p = h + (long long)b * N * ld + c;
  float s = 0.f;
  for (int n = 0; n < N; ++n) s += p[(long long)n * ld];
  out[(long long)b * C + c] = s / (float)N;
}

// out[b,c] = mean of rows offsets[b] .. offsets[b+1]-1 of h; the summation order of mean_rows_kernel.
__global__ void mean_segments_kernel(const float* __restrict__ h, long long ld, const int* __restrict__ offsets, int C,
                                     float* __restrict__ out) {
  const int b = blockIdx.y;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const int r0 = offsets[b], n_b = offsets[b + 1] - r0;
  const float* p = h + (long long)r0 * ld + c;
  float s = 0.f;
  for (int n = 0; n < n_b; ++n) s += p[(long long)n * ld];
  out[(long long)b * C + c] = s / (float)n_b;
}

// ------------------------------------------------------------------------------------------
// SGEMM  C[M,Nf] = act(A W^T + bias) + R ; 64x64x16 tiles, 4x4 register micro-tiles.
constexpr int GBM = 64, GBN = 64, GBK = 16;

__global__ void __launch_bounds__(256) linear_kernel(const float* __restrict__ A, long long a_bs, long long a_ls, long long a_ks,
                                                     int a_L, const float* __restrict__ W, const float* __restrict__ bias,
                                                     const float* __restrict__ R, long long ldr, float* __restrict__ C,
                                                     long long ldc, int M, int Nf, int K, int act) {
  __shared__ __align__(16) float As[GBK][GBM + 4];
  __shared__ __align__(16) float Ws[GBK][GBN + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * GBM, n0 = blockIdx.x * GBN;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  const bool kcontig = (a_ks == 1);
  for (int k0 = 0; k0 < K; k0 += GBK) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int m, k;
      if (kcontig) { k = tid & 15; m = (tid >> 4) + 16 * i; }
      else { m = tid & 63; k = (tid >> 6) + 4 * i; }
      const int mg = m0 + m, kg = k0 + k;
      float v = 0.f;
      if (mg < M && kg < K) {
        const int bi = mg / a_L, l = mg - bi * a_L;
        v = A[(long long)bi * a_bs + (long long)l * a_ls + (long long)kg * a_ks];
      }
      As[k][m] = v;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int k = tid & 15, n = (tid >> 4) + 16 * i;
      const int ng = n0 + n, kg = k0 + k;
      Ws[k][n] = (ng < Nf && kg < K) ? W[(long long)ng * K + kg] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < GBK; ++kk) {
      const float4 av = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      const float4 wv = *reinterpret_cast<const float4*>(&Ws[kk][tx * 4]);
      const float a4[4] = {av.x, av.y, av.z, av.w};
      const float w4[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a4[i], w4[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= Nf) continue;
      float v = acc[i][j] + (bias ? bias[n] : 0.f);
      if (act == ST2_ACT_GELU) v = gelu_erf(v);
      else if (act == ST2_ACT_TANH) v = tanhf(v);
      else if (act == ST2_ACT_GELU_TANH) v = gelu_tanh(v);
      if (R) v += R[(long long)m * ldr + n];
      C[(long long)m * ldc + n] = v;
    }
  }
}


// ------------------------------------------------------------------------------------------
// Small-M Linear (M <= 64 rows: the per-utterance vectors of the path -- time/feature mapping MLP of the denoiser,
// AdaLayerNorm / AdaIN style projections): a weight-streaming split-K kernel.  The 64x64-tile SGEMM above gives such a
// shape 16 CTAs that each walk K serially (~100 us for 32x1024x1024).  Here a CTA of 8 warps owns 8 output features;
// warp w owns the K chunks {w, w+8, ...} (128 floats per chunk: one float4 per lane, weights read exactly once,
// coalesced) for all rows, two features at a time; row loads are issued in batches of 8 so that their latency
// overlaps; the 2 x 32 per-lane partial sums are folded with a transpose-reduce (31 shuffles per feature), the 8
// per-warp partials are summed in a fixed order through shared memory (deterministic) and one thread finishes each
// (row, feature) with bias / activation / residual.
constexpr int SM_MT = 32;   // rows per pass
constexpr int SM_NF = 8;    // features per CTA
constexpr int SM_NW = 8;    // warps per CTA (K slices)

template <bool VEC>
__global__ void __launch_bounds__(SM_NW * 32) linear_smallm_kernel(const float* __restrict__ A, long long a_bs, long long a_ls,
                                                                  int a_L, const float* __restrict__ W,
                                                                  const float* __restrict__ bias, const float* __restrict__ R,
                                                                  long long ldr, float* __restrict__ C, long long ldc, int M, int Nf,
                                                                  int K, int act) {
  __shared__ float part[SM_NW][SM_NF][SM_MT];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nb = blockIdx.x * SM_NF;
  constexpr int CH = VEC ? 128 : 32;     // floats of K per warp-wide step
  for (int mt = 0; mt < M; mt += SM_MT) {
    const int mrows = min(SM_MT, M - mt);
    // row base pointers of this pass (rows beyond M alias the last valid row: loaded but never stored)
    const float* rowp[SM_MT];
#pragma unroll
    for (int m = 0; m < SM_MT; ++m) {
      const int mg = mt + min(m, mrows - 1);
      const int bi = mg / a_L, l = mg - bi * a_L;
      rowp[m] = A + (long long)bi * a_bs + (long long)l * a_ls;
    }
#pragma unroll 1
    for (int fp = 0; fp < SM_NF; fp += 2) {
      const int n0 = min(nb + fp, Nf - 1), n1 = min(nb + fp + 1, Nf - 1);
      const float* w0 = W + (long long)n0 * K;
      const float* w1 = W + (long long)n1 * K;
      float acc0[SM_MT], acc1[SM_MT];
#pragma unroll
      for (int m = 0; m < SM_MT; ++m) { acc0[m] = 0.f; acc1[m] = 0.f; }
      for (int k0 = warp * CH; k0 < K; k0 += SM_NW * CH) {
        if (VEC) {
          const int k = k0 + lane * 4;
          if (k < K) {
            const float4 wa = __ldg(reinterpret_cast<const float4*>(w0 + k));
            const float4 wb = __ldg(reinterpret_cast<const float4*>(w1 + k));
#pragma unroll
            for (int m8 = 0; m8 < SM_MT; m8 += 8) {
              float4 av[8];
#pragma unroll
              for (int i = 0; i < 8; ++i) av[i] = __ldg(reinterpret_cast<const float4*>(rowp[m8 + i] + k));
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                float a0 = acc0[m8 + i], a1 = acc1[m8 + i];
                a0 = fmaf(av[i].x, wa.x, a0); a0 = fmaf(av[i].y, wa.y, a0); a0 = fmaf(av[i].z, wa.z, a0); a0 = fmaf(av[i].w, wa.w, a0);
                a1 = fmaf(av[i].x, wb.x, a1); a1 = fmaf(av[i].y, wb.y, a1); a1 = fmaf(av[i].z, wb.z, a1); a1 = fmaf(av[i].w, wb.w, a1);
                acc0[m8 + i] = a0; acc1[m8 + i] = a1;
              }
            }
          }
        } else {
          const int k = k0 + lane;
          if (k < K) {
            const float wa = __ldg(w0 + k), wb = __ldg(w1 + k);
#pragma unroll
            for (int m8 = 0; m8 < SM_MT; m8 += 8) {
              float av[8];
#pragma unroll
              for (int i = 0; i < 8; ++i) av[i] = __ldg(rowp[m8 + i] + k);
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                acc0[m8 + i] = fmaf(av[i], wa, acc0[m8 + i]);
                acc1[m8 + i] = fmaf(av[i], wb, acc1[m8 + i]);
              }
            }
          }
        }
      }
      // transpose-reduce over the 32 lanes: afterwards lane m holds this warp's partial sums of row (mt + m)
#define ST2_TRED(ACC, NV, OFF)                                                  \
  {                                                                             \
    const bool up = (lane & OFF) != 0;                                          \
    _Pragma("unroll") for (int i = 0; i < NV / 2; ++i) {                        \
      const float send = up ? ACC[i] : ACC[i + NV / 2];                         \
      const float keep = up ? ACC[i + NV / 2] : ACC[i];                         \
      ACC[i] = keep + __shfl_xor_sync(0xffffffffu, send, OFF);                  \
    }                                                                           \
  }
      ST2_TRED(acc0, 32, 16) ST2_TRED(acc0, 16, 8) ST2_TRED(acc0, 8, 4) ST2_TRED(acc0, 4, 2) ST2_TRED(acc0, 2, 1)
      ST2_TRED(acc1, 32, 16) ST2_TRED(acc1, 16, 8) ST2_TRED(acc1, 8, 4) ST2_TRED(acc1, 4, 2) ST2_TRED(acc1, 2, 1)
#undef ST2_TRED
      part[warp][fp][lane] = acc0[0];
      part[warp][fp + 1][lane] = acc1[0];
    }
    __syncthreads();
    {
      const int f = threadIdx.x >> 5, m = threadIdx.x & 31;   // 256 threads = 8 features x 32 rows
      const int n = nb + f;
      if (n < Nf && m < mrows) {
        float v = 0.f;
#pragma unroll
        for (int w = 0; w < SM_NW; ++w) v += part[w][f][m];
        v += bias ? bias[n] : 0.f;
        if (act == ST2_ACT_GELU) v = gelu_erf(v);
        else if (act == ST2_ACT_TANH) v = tanhf(v);
        else if (act == ST2_ACT_GELU_TANH) v = gelu_tanh(v);
        const long long mg = mt + m;
        if (R) v += R[mg * ldr + n];
        C[mg * ldc + n] = v;
      }
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------
// Tiny-M Linear (M <= 8 rows, 16-byte aligned operands: the time / feature mapping MLP of the denoiser at 8 utterances per
// GPU runs 100+ of these per step with K = 256): a warp owns TWO output features over the whole K (one float4 of each
// weight row per lane and 128-float step, weights read once, coalesced), the 8 x 2 per-lane partial sums are folded with a
// transposing shuffle tree (31 shuffles): lane f*8 + m ends up with (row m, feature f).  No shared memory, no block barrier,
// 16 features per CTA; latency = two rounds of loads + the tree (the 32-row kernel above needs ~20 us for such a shape:
// four sequential feature pairs per CTA, six of eight warps idle at K = 256).
constexpr int TM_ROWS = 8;
__global__ void __launch_bounds__(256) linear_tinym_kernel(const float* __restrict__ A, long long a_bs, long long a_ls, int a_L,
                                                           const float* __restrict__ W, const float* __restrict__ bias,
                                                           const float* __restrict__ R, long long ldr, float* __restrict__ C, long long ldc,
                                                           int M, int Nf, int K, int act) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n0 = blockIdx.x * 16 + warp * 2;
  if (n0 >= Nf) return;
  const int n1 = min(n0 + 1, Nf - 1);
  const float* rowp[TM_ROWS];
#pragma unroll
  for (int m = 0; m < TM_ROWS; ++m) {
    const int mg = min(m, M - 1);
    const int bi = mg / a_L, l = mg - bi * a_L;
    rowp[m] = A + (long long)bi * a_bs + (long long)l * a_ls;
  }
  const float* w0 = W + (long long)n0 * K;
  const float* w1 = W + (long long)n1 * K;
  float acc[2 * TM_ROWS];
#pragma unroll
  for (int i = 0; i < 2 * TM_ROWS; ++i) acc[i] = 0.f;
  for (int k = lane * 4; k < K; k += 128) {
    const float4 wa = __ldg(reinterpret_cast<const float4*>(w0 + k));
    const float4 wb = __ldg(reinterpret_cast<const float4*>(w1 + k));
    float4 av[TM_ROWS];
#pragma unroll
    for (int m = 0; m < TM_ROWS; ++m) av[m] = __ldg(reinterpret_cast<const float4*>(rowp[m] + k));
#pragma unroll
    for (int m = 0; m < TM_ROWS; ++m) {
      float a0 = acc[m], a1 = acc[TM_ROWS + m];
      a0 = fmaf(av[m].x, wa.x, a0); a0 = fmaf(av[m].y, wa.y, a0); a0 = fmaf(av[m].z, wa.z, a0); a0 = fmaf(av[m].w, wa.w, a0);
      a1 = fmaf(av[m].x, wb.x, a1); a1 = fmaf(av[m].y, wb.y, a1); a1 = fmaf(av[m].z, wb.z, a1); a1 = fmaf(av[m].w, wb.w, a1);
      acc[m] = a0; acc[TM_ROWS + m] = a1;
    }
  }
  // lanes L and L^16 first add their 16 sums, then four halving steps leave value (lane & 15) in acc[0]
#pragma unroll
  for (int i = 0; i < 16; ++i) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], 16);
#define ST2_TRED(NV, OFF)                                                       \
  {                                                                             \
    const bool up = (lane & OFF) != 0;                                          \
    _Pragma("unroll") for (int i = 0; i < NV / 2; ++i) {                        \
      const float send = up ? acc[i] : acc[i + NV / 2];                         \
      const float keep = up ? acc[i + NV / 2] : acc[i];                         \
      acc[i] = keep + __shfl_xor_sync(0xffffffffu, send, OFF);                  \
    }                                                                           \
  }
  ST2_TRED(16, 8) ST2_TRED(8, 4) ST2_TRED(4, 2) ST2_TRED(2, 1)
#undef ST2_TRED
  if (lane < 16) {
    const int f = lane >> 3, m = lane & 7;
    const int n = n0 + f;
    if (n < Nf && m < M) {
      float v = acc[0] + (bias ? bias[n] : 0.f);
      if (act == ST2_ACT_GELU) v = gelu_erf(v);
      else if (act == ST2_ACT_TANH) v = tanhf(v);
      else if (act == ST2_ACT_GELU_TANH) v = gelu_tanh(v);
      if (R) v += R[(long long)m * ldr + n];
      C[(long long)m * ldc + n] = v;
    }
  }
}

// ------------------------------------------------------------------------------------------
// Attention (no mask), D = 64.  CTA = 4 warps, 16 queries (4 per warp); keys streamed in chunks of
// 32 through shared memory; lane-per-key dot products, online softmax, P V through shared memory.
constexpr int ATT_D = 64, ATT_QW = 4, ATT_WARPS = 4, ATT_KC = 32;

__global__ void __launch_bounds__(128) attention_kernel(const float* __restrict__ q, long long q_ld, const float* __restrict__ kp,
                                                        const float* __restrict__ vp, long long kv_ld, float* __restrict__ out,
                                                        long long out_ld, const int* __restrict__ lengths, int N, int H, float scale) {
  __shared__ __align__(16) float Qs[ATT_WARPS * ATT_QW][ATT_D];
  __shared__ __align__(16) float Ks[ATT_KC][ATT_D + 4];
  __shared__ __align__(16) float Vs[ATT_KC][ATT_D];
  __shared__ float Ps[ATT_WARPS][ATT_QW][ATT_KC];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int bh = blockIdx.y, b = bh / H, h = bh - b * H;
  const int q0 = blockIdx.x * (ATT_WARPS * ATT_QW);
  const int NK = lengths ? min(N, lengths[b]) : N;  // keys beyond the utterance length are masked out
  for (int i = tid; i < ATT_WARPS * ATT_QW * ATT_D; i += 128) {
    const int qi = i / ATT_D, d = i - qi * ATT_D;
    const int n = q0 + qi;
    Qs[qi][d] = n < N ? q[((long long)b * N + n) * q_ld + h * ATT_D + d] : 0.f;
  }
  float m[ATT_QW], l[ATT_QW], o0[ATT_QW], o1[ATT_QW];
#pragma unroll
  for (int i = 0; i < ATT_QW; ++i) { m[i] = -INFINITY; l[i] = 0.f; o0[i] = 0.f; o1[i] = 0.f; }
  for (int k0 = 0; k0 < NK; k0 += ATT_KC) {
    __syncthreads();
    for (int i = tid; i < ATT_KC * ATT_D; i += 128) {
      const int kj = i / ATT_D, d = i - kj * ATT_D;
      const int n = k0 + kj;
      const long long base = ((long long)b * N + n) * kv_ld + h * ATT_D + d;
      Ks[kj][d] = n < NK ? kp[base] : 0.f;
      Vs[kj][d] = n < NK ? vp[base] : 0.f;
    }
    __syncthreads();
    float s[ATT_QW];
#pragma unroll
    for (int i = 0; i < ATT_QW; ++i) s[i] = 0.f;
#pragma unroll 4
    for (int d = 0; d < ATT_D; d += 4) {
      const float4 kk = *reinterpret_cast<const float4*>(&Ks[lane][d]);
#pragma unroll
      for (int i = 0; i < ATT_QW; ++i) {
        const float4 qq = *reinterpret_cast<const float4*>(&Qs[warp * ATT_QW + i][d]);
        s[i] = fmaf(qq.x, kk.x, s[i]);
        s[i] = fmaf(qq.y, kk.y, s[i]);
        s[i] = fmaf(qq.z, kk.z, s[i]);
        s[i] = fmaf(qq.w, kk.w, s[i]);
      }
    }
    const bool kvalid = (k0 + lane) < NK;
#pragma unroll
    for (int i = 0; i < ATT_QW; ++i) {
      const float sv = kvalid ? s[i] * scale : -INFINITY;
      const float mn = fmaxf(m[i], warp_max(sv));
      const float p = kvalid ? expf(sv - mn) : 0.f;
      const float corr = expf(m[i] - mn);
      l[i] = l[i] * corr + warp_sum(p);
      o0[i] *= corr;
      o1[i] *= corr;
      m[i] = mn;
      Ps[warp][i][lane] = p;
    }
    __syncwarp();
#pragma unroll 8
    for (int j = 0; j < ATT_KC; ++j) {
      const float2 vv = *reinterpret_cast<const float2*>(&Vs[j][2 * lane]);
#pragma unroll
      for (int i = 0; i < ATT_QW; ++i) {
        const float p = Ps[warp][i][j];
        o0[i] = fmaf(p, vv.x, o0[i]);
        o1[i] = fmaf(p, vv.y, o1[i]);
      }
    }
    __syncwarp();
  }
#pragma unroll
  for (int i = 0; i < ATT_QW; ++i) {
    const int n = q0 + warp * ATT_QW + i;
    if (n < N) {
      const float inv = 1.0f / l[i];
      float2 r = make_float2(o0[i] * inv, o1[i] * inv);
      *reinterpret_cast<float2*>(&out[((long long)b * N + n) * out_ld + h * ATT_D + 2 * lane]) = r;
    }
  }
}

}  // namespace st2

using namespace st2;

extern "C" {

int st2_rows_ln(const st2_rows_args* a, void* stream) {
  ST2_REQUIRE(a && (a->h_in || (a->x && a->emb)), "st2_rows_ln", "no input");
  ST2_REQUIRE(a->C % 32 == 0 && a->C <= 1024 && a->C > 0 && a->B > 0 && a->N > 0, "st2_rows_ln", "C must be a multiple of 32, <= 1024");
  const int rows = a->B * a->N;
  rows_ln_kernel<false><<<cdiv(rows, 8), 256, 0, (cudaStream_t)stream>>>(*a, nullptr, 0);
  ++g_launches;
  ST2_CHECK_LAUNCH("st2_rows_ln");
  return 0;
}

int st2_rows_ln_packed(const st2_rows_args* a, const int* row_utt, int M, void* stream) {
  ST2_REQUIRE(a && (a->h_in || (a->x && a->emb)), "st2_rows_ln_packed", "no input");
  ST2_REQUIRE(row_utt && M > 0 && a->B > 0, "st2_rows_ln_packed", "bad args");
  ST2_REQUIRE(a->C % 32 == 0 && a->C <= 1024 && a->C > 0, "st2_rows_ln_packed", "C must be a multiple of 32, <= 1024");
  rows_ln_kernel<true><<<cdiv(M, 8), 256, 0, (cudaStream_t)stream>>>(*a, row_utt, M);
  ++g_launches;
  ST2_CHECK_LAUNCH("st2_rows_ln_packed");
  return 0;
}

int st2_bcast_cols(float* dst, long long ld, int col0, const float* src, int B, int N, int W, const int* lengths, void* stream) {
  ST2_REQUIRE(dst && src && B > 0 && N > 0 && W > 0, "st2_bcast_cols", "bad args");
  const long long total = (long long)B * N * W;
  bcast_cols_kernel<<<(int)((total + 255) / 256 > 2048 ? 2048 : (total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      dst, ld, col0, src, B, N, W, lengths);
  ++g_launches;
  ST2_CHECK_LAUNCH("st2_bcast_cols");
  return 0;
}

int st2_mean_rows(const float* h, long long ld, int B, int N, int C, float* out, void* stream) {
  ST2_REQUIRE(h && out && B > 0 && N > 0 && C > 0, "st2_mean_rows", "bad args");
  mean_rows_kernel<<<dim3(cdiv(C, 128), B), 128, 0, (cudaStream_t)stream>>>(h, ld, N, C, out);
  ++g_launches;
  ST2_CHECK_LAUNCH("st2_mean_rows");
  return 0;
}

int st2_mean_segments(const float* h, long long ld, const int* offsets, int B, int C, float* out, void* stream) {
  ST2_REQUIRE(h && offsets && out && B > 0 && C > 0, "st2_mean_segments", "bad args");
  mean_segments_kernel<<<dim3(cdiv(C, 128), B), 128, 0, (cudaStream_t)stream>>>(h, ld, offsets, C, out);
  ++g_launches;
  ST2_CHECK_LAUNCH("st2_mean_segments");
  return 0;
}

int st2_linear(const float* A, long long a_bs, long long a_ls, long long a_ks, int a_L, const float* W, const float* bias,
               const float* R, long long ldr, float* C, long long ldc, int M, int Nf, int K, int act, void* stream) {
  ST2_REQUIRE(A && W && C && M > 0 && Nf > 0 && K > 0 && a_L > 0, "st2_linear", "bad args");
  if (M <= 64 && a_ks == 1) {
    const bool vec = (K % 4 == 0) && (a_bs % 4 == 0) && (a_ls % 4 == 0) && ((reinterpret_cast<size_t>(A) & 15) == 0) &&
                     ((reinterpret_cast<size_t>(W) & 15) == 0);
    if (vec && M <= TM_ROWS) {
      linear_tinym_kernel<<<cdiv(Nf, 16), 256, 0, (cudaStream_t)stream>>>(A, a_bs, a_ls, a_L, W, bias, R, ldr, C, ldc, M, Nf, K, act);
      ++g_launches;
      ST2_CHECK_LAUNCH("st2_linear (tiny M)");
      return 0;
    }
    const int grid = cdiv(Nf, SM_NF);
    if (vec) linear_smallm_kernel<true><<<grid, SM_NW * 32, 0, (cudaStream_t)stream>>>(A, a_bs, a_ls, a_L, W, bias, R, ldr, C, ldc, M, Nf, K, act);
    else linear_smallm_kernel<false><<<grid, SM_NW * 32, 0, (cudaStream_t)stream>>>(A, a_bs, a_ls, a_L, W, bias, R, ldr, C, ldc, M, Nf, K, act);
    ++g_launches;
    ST2_CHECK_LAUNCH("st2_linear (small M)");
    return 0;
  }
  dim3 grid(cdiv(Nf, GBN), cdiv(M, GBM));
  linear_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(A, a_bs, a_ls, a_ks, a_L, W, bias, R, ldr, C, ldc, M, Nf, K, act);
  ++g_launches;
  ST2_CHECK_LAUNCH("st2_linear");
  return 0;
}

int st2_attention_ex(const float* q, long long q_ld, const float* k, const float* v, long long kv_ld, float* out, long long out_ld,
                     const int* lengths, int B, int N, int H, int D, float scale, void* stream) {
  ST2_REQUIRE(q && k && v && out && B > 0 && N > 0 && H > 0, "st2_attention_ex", "bad args");
  ST2_REQUIRE(D == ATT_D, "st2_attention_ex", "head_features must be 64");
  ST2_REQUIRE((out_ld & 1) == 0, "st2_attention_ex", "out_ld must be even");
  dim3 grid(cdiv(N, ATT_WARPS * ATT_QW), B * H);
  attention_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(q, q_ld, k, v, kv_ld, out, out_ld, lengths, N, H, scale);
  ++g_launches;
  ST2_CHECK_LAUNCH("st2_attention_ex");
  return 0;
}

int st2_attention(const float* q, const float* kv, float* out, int B, int N, int H, int D, float scale, void* stream) {
  ST2_REQUIRE(q && kv, "st2_attention", "bad args");
  const long long HD = (long long)H * D;
  return st2_attention_ex(q, HD, kv, kv + HD, 2 * HD, out, HD, nullptr, B, N, H, D, scale, stream);
}

}  // extern "C"
