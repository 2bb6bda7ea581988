// Fused Conv1d / ConvTranspose1d for the AdaIN-conditioned decoder and vocoder (fp32 SIMT path).
//
//   y = epi( bias + sum_{ci,k} W * pre(x) )      -- see include/styletts2_b200.h
//
// Design (sm_90a, 132 SMs): one CTA = 256 threads computes a [CO_T x 256] output tile of one
// utterance.  Lanes stride the time axis (conflict-free shared-memory reads of the staged frame
// window for any dilation), warps stride output channels (weights are warp-broadcast 128-bit
// loads).  The AdaIN affine + Snake/LeakyReLU prologue is applied ONCE while the window is staged
// into shared memory; the epilogue fuses bias, residual, MRF mean accumulation and the per-(b,c)
// InstanceNorm partial statistics of what it stores, so no tensor makes an extra HBM round trip
// for normalisation or activation.  Partial statistics are (count, mean, M2) per 256-column tile,
// reduced with warp shuffles in a fixed order (deterministic; no atomics).
#include "common.cuh"

namespace st2 {

long long g_launches = 0;

constexpr int CONV_THREADS = 256;
constexpr int TQ = 256;  // output positions per CTA
constexpr int NJ = 8;    // positions per lane

struct EpiOut {
  float v;
};

__device__ __forceinline__ float conv_finish(const st2_conv_args& a, float acc, float bias, int b, int co, int oidx,
                                             float* yb) {
  float v = acc + bias;
  if (a.res) v += a.res[(long long)b * a.res_bstride + (long long)co * a.res_len + (oidx >> a.res_shift)];
  if (a.out_div != 1.0f) v = __fdiv_rn(v, a.out_div);
  float* p = yb + (long long)co * a.y_len + oidx;
  if (a.accum_mode == 1) v = *p + v;
  else if (a.accum_mode == 2) v = __fdiv_rn(*p + v, a.accum_div);
  if (a.out_act == ST2_ACT_TANH) v = tanhf(v);
  *p = v;
  return v;
}

template <int COW>
__global__ void __launch_bounds__(CONV_THREADS, 2) conv1d_kernel(const st2_conv_args a, const int ci_chunk, const int XT) {
  extern __shared__ __align__(16) float smem[];
  constexpr int CO_T = 8 * COW;
  float* xs = smem;                  // [ci_chunk][XT]
  float* ws = smem + ci_chunk * XT;  // [ci_chunk][K][CO_T]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int q0 = blockIdx.x * TQ;
  const int co0 = blockIdx.y * CO_T;
  const int b = blockIdx.z;
  const float* xb = a.x + (long long)b * a.x_bstride;
  const int in0 = q0 * a.stride - a.pad;
  const int K = a.K;

  float acc[COW][NJ];
#pragma unroll
  for (int i = 0; i < COW; ++i)
#pragma unroll
    for (int j = 0; j < NJ; ++j) acc[i][j] = 0.f;

  for (int c0 = 0; c0 < a.Cin; c0 += ci_chunk) {
    const int nci = min(ci_chunk, a.Cin - c0);
    // ---- stage the (activated) frame window
    for (int ci = 0; ci < nci; ++ci) {
      const int c = c0 + ci;
      const float* xr = xb + (long long)c * a.Lin;
      float pa = 1.f, pb = 0.f, al = 1.f;
      const bool affine = a.pre_a != nullptr;
      if (affine) {
        pa = a.pre_a[b * a.Cin + c];
        pb = a.pre_b[b * a.Cin + c];
      }
      if (a.pre_act == ST2_ACT_SNAKE) al = a.pre_alpha[c];
      float* xd = xs + ci * XT;
      for (int p = tid; p < XT; p += CONV_THREADS) {
        const int g = in0 + p;
        float v = 0.f;
        if (g >= 0 && g < a.Lin) {
          v = xr[g];
          if (affine) v = fmaf(v, pa, pb);
          v = act_apply(v, a.pre_act, a.pre_slope, al);
        }
        xd[p] = v;
      }
    }
    // ---- stage the weight slab  ws[(ci*K+k)*CO_T + co]
    {
      const int rmax = nci * K;
      const int wn = rmax * CO_T;
      const float* wsrc = a.w + (long long)c0 * K * a.Cout + co0;
      for (int idx = tid; idx < wn; idx += CONV_THREADS) {
        const int co = idx % CO_T;
        const int r = idx / CO_T;
        float v = 0.f;
        if (co0 + co < a.Cout) v = wsrc[(long long)r * a.Cout + co];
        ws[idx] = v;
      }
    }
    __syncthreads();
    for (int ci = 0; ci < nci; ++ci) {
      const float* xr = xs + ci * XT + lane * a.stride;
      const float* wr = ws + ci * K * CO_T + warp * COW;
      for (int k = 0; k < K; ++k) {
        float wv[COW];
        if constexpr (COW % 4 == 0) {
#pragma unroll
          for (int i = 0; i < COW; i += 4) {
            const float4 t = *reinterpret_cast<const float4*>(wr + i);
            wv[i] = t.x; wv[i + 1] = t.y; wv[i + 2] = t.z; wv[i + 3] = t.w;
          }
        } else {
#pragma unroll
          for (int i = 0; i < COW; ++i) wv[i] = wr[i];
        }
        float xv[NJ];
        const float* xk = xr + k * a.dil;
#pragma unroll
        for (int j = 0; j < NJ; ++j) xv[j] = xk[j * 32 * a.stride];
#pragma unroll
        for (int i = 0; i < COW; ++i)
#pragma unroll
          for (int j = 0; j < NJ; ++j) acc[i][j] = fmaf(wv[i], xv[j], acc[i][j]);
        wr += CO_T;
      }
    }
    __syncthreads();
  }

  // ---- epilogue
  float* yb = a.y + (long long)b * a.y_bstride;
#pragma unroll
  for (int i = 0; i < COW; ++i) {
    const int co = co0 + warp * COW + i;
    if (co >= a.Cout) continue;  // warp-uniform
    const float bias = a.bias ? a.bias[co] : 0.f;
    float vals[NJ + 1];
    float s = 0.f;
    int n = 0;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int q = q0 + lane + 32 * j;
      vals[j] = 0.f;
      if (q < a.Lq) {
        const float v = conv_finish(a, acc[i][j], bias, b, co, q * a.y_tstride + a.y_toffset, yb);
        vals[j] = v;
        s += v;
        ++n;
      }
    }
    const bool dup = (a.dup_q0_to >= 0) && (q0 == 0) && (lane == 0);
    vals[NJ] = 0.f;
    if (dup) {
      const float v = conv_finish(a, acc[i][0], bias, b, co, a.dup_q0_to, yb);
      vals[NJ] = v;
      s += v;
      ++n;
    }
    if (a.stats) {
      const float nt = warp_sum((float)n);
      const float mean = warp_sum(s) / nt;
      float m2 = 0.f;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const int q = q0 + lane + 32 * j;
        if (q < a.Lq) {
          const float d = vals[j] - mean;
          m2 = fmaf(d, d, m2);
        }
      }
      if (dup) {
        const float d = vals[NJ] - mean;
        m2 = fmaf(d, d, m2);
      }
      m2 = warp_sum(m2);
      if (lane == 0) {
        float* sp = a.stats + (((long long)b * a.Cout + co) * a.stats_nparts + a.stats_part_offset + blockIdx.x) * 3;
        sp[0] = nt;
        sp[1] = mean;
        sp[2] = m2;
      }
    }
  }
}

static int conv_launch(const st2_conv_args& a, cudaStream_t st) {
  const int cow = a.Cout >= 48 ? 8 : (a.Cout >= 12 ? 4 : 1);
  const int co_t = 8 * cow;
  int xt = (TQ - 1) * a.stride + (a.K - 1) * a.dil + 1;
  xt = (xt + 3) & ~3;
  int ci_chunk = a.K <= 5 ? 16 : 8;
  if (ci_chunk > a.Cin) ci_chunk = a.Cin;
  auto smem_of = [&](int cc) { return (size_t)(cc * xt + cc * a.K * co_t) * sizeof(float); };
  while (ci_chunk > 1 && smem_of(ci_chunk) > 96 * 1024) ci_chunk >>= 1;
  const size_t smem = smem_of(ci_chunk);
  if (smem > 200 * 1024) {
    set_error_msg("st2_conv1d", "tile does not fit in shared memory");
    return (int)cudaErrorInvalidValue;
  }
  dim3 grid(cdiv(a.Lq, TQ), cdiv(a.Cout, co_t), a.B);
  static PerDevice once;
  if (once.first()) {
    cudaFuncSetAttribute(conv1d_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(conv1d_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(conv1d_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  }
  if (cow == 8) conv1d_kernel<8><<<grid, CONV_THREADS, smem, st>>>(a, ci_chunk, xt);
  else if (cow == 4) conv1d_kernel<4><<<grid, CONV_THREADS, smem, st>>>(a, ci_chunk, xt);
  else conv1d_kernel<1><<<grid, CONV_THREADS, smem, st>>>(a, ci_chunk, xt);
  ++g_launches;
  return 0;
}

// ------------------------------------------------------------------------------------------
// weight preparation
// sum of squares of one row, fp64 accumulation, fixed reduction order (shared by the fold and the row-norm kernel so that
// a weight exported folded and re-imported as (v = w, g = ||w||) folds back to exactly w: scale == 1.0f)
__device__ __forceinline__ double row_sumsq_block(const float* __restrict__ vr, int cols, double* red) {
  double ss = 0.0;
  for (int c = threadIdx.x; c < cols; c += blockDim.x) ss += (double)vr[c] * (double)vr[c];
  ss = warp_sum_d(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  if (threadIdx.x < 32) {
    double t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.0;
    t = warp_sum_d(t);
    if (threadIdx.x == 0) red[0] = t;
  }
  __syncthreads();
  return red[0];
}

__global__ void row_norm_kernel(const float* __restrict__ v, float* __restrict__ out, int rows, int cols) {
  __shared__ double red[32];
  const int r = blockIdx.x;
  const double ss = row_sumsq_block(v + (long long)r * cols, cols, red);
  if (threadIdx.x == 0) out[r] = (float)sqrt(ss);
}

__global__ void weight_norm_fold_kernel(const float* __restrict__ v, const float* __restrict__ g, float* __restrict__ w,
                                        int rows, int cols) {
  const int r = blockIdx.x;
  const float* vr = v + (long long)r * cols;
  // two-pass, fp64 accumulation: folded once at load, accuracy over speed
  __shared__ double red[32];
  row_sumsq_block(vr, cols, red);
  const float scale = g[r] / (float)sqrt(red[0]);  // torch: v * (g / norm)
  for (int c = threadIdx.x; c < cols; c += blockDim.x) w[(long long)r * cols + c] = vr[c] * scale;
}

__global__ void conv_weight_layout_kernel(const float* __restrict__ w, float* __restrict__ wt, int Cout, int Cin, int K) {
  const long long n = (long long)Cout * Cin * K;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int co = (int)(i % Cout);
    const long long r = i / Cout;
    const int k = (int)(r % K);
    const int ci = (int)(r / K);
    wt[i] = w[((long long)co * Cin + ci) * K + k];
  }
}

__global__ void convT_weight_layout_kernel(const float* __restrict__ w, float* __restrict__ wp, int Cin, int Cout, int K,
                                           int S, int P, int J) {
  const long long n = (long long)S * Cin * J * Cout;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int co = (int)(i % Cout);
    long long r = i / Cout;
    const int kp = (int)(r % J);
    r /= J;
    const int ci = (int)(r % Cin);
    const int ph = (int)(r / Cin);
    const int kk = (J - 1 - kp) * S + ((ph + P) % S);
    wp[i] = kk < K ? w[((long long)ci * Cout + co) * K + kk] : 0.f;
  }
}

// ------------------------------------------------------------------------------------------
// InstanceNorm statistics for tensors not produced by conv1d_kernel: one CTA per (b,c) row.
__global__ void instance_stats_kernel(const float* __restrict__ x, long long bstride, int C, int L, float* __restrict__ stats) {
  const int c = blockIdx.x, b = blockIdx.y;
  const float* xr = x + (long long)b * bstride + (long long)c * L;
  __shared__ double red[32];
  __shared__ double mean_s;
  double s = 0.0;
  for (int i = threadIdx.x; i < L; i += blockDim.x) s += (double)xr[i];
  s = warp_sum_d(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    double t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.0;
    t = warp_sum_d(t);
    if (threadIdx.x == 0) mean_s = t / (double)L;
  }
  __syncthreads();
  const double mean = mean_s;
  double m2 = 0.0;
  for (int i = threadIdx.x; i < L; i += blockDim.x) {
    const double d = (double)xr[i] - mean;
    m2 += d * d;
  }
  m2 = warp_sum_d(m2);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m2;
  __syncthreads();
  if (threadIdx.x < 32) {
    double t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.0;
    t = warp_sum_d(t);
    if (threadIdx.x == 0) {
      float* sp = stats + ((long long)b * C + c) * 3;
      sp[0] = (float)L;
      sp[1] = (float)mean;
      sp[2] = (float)t;
    }
  }
}

// Merge partials (Chan et al.) in fp64; biased variance; AdaIN coefficients.  One WARP per (b,c): lanes take every
// 32nd partial (coalesced 12-byte records), then a fixed shuffle tree merges the 32 lane results (deterministic).
__device__ __forceinline__ void chan_merge(double& n, double& mean, double& m2, double nb, double mb, double m2b) {
  if (nb <= 0.0) return;
  const double nn = n + nb;
  const double delta = mb - mean;
  mean += delta * (nb / nn);
  m2 += m2b + delta * delta * (n * nb / nn);
  n = nn;
}

__global__ void adain_coef_kernel(const float* __restrict__ stats, int nparts, const float* __restrict__ gb,
                                  long long gb_stride, int B, int C, float eps, float* __restrict__ a,
                                  float* __restrict__ bo) {
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (i >= B * C) return;
  const int b = i / C, c = i - b * C;
  const float* sp = stats + (long long)i * nparts * 3;
  double n = 0.0, mean = 0.0, m2 = 0.0;
  for (int p = lane; p < nparts; p += 32) chan_merge(n, mean, m2, sp[p * 3 + 0], sp[p * 3 + 1], sp[p * 3 + 2]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double nb = __shfl_down_sync(0xffffffffu, n, o);
    const double mb = __shfl_down_sync(0xffffffffu, mean, o);
    const double m2b = __shfl_down_sync(0xffffffffu, m2, o);
    chan_merge(n, mean, m2, nb, mb, m2b);
  }
  if (lane == 0) {
    const double var = m2 / n;
    const float rstd = (float)(1.0 / sqrt(var + (double)eps));
    const float gamma = gb[(long long)b * gb_stride + c];
    const float beta = gb[(long long)b * gb_stride + C + c];
    const float av = (1.0f + gamma) * rstd;
    a[i] = av;
    bo[i] = beta - (float)mean * av;
  }
}

// AdaIN -> LeakyReLU -> depthwise ConvTranspose1d(k3,s2,p1,op1): y[2i] = w1*z[i] + pb,
// y[2i+1] = w2*z[i] + w0*z[i+1] + pb  (z[L] = 0), z = lrelu(a*x+b).
__global__ void adain_lrelu_pool_kernel(const float* __restrict__ x, long long x_bstride, const float* __restrict__ a,
                                        const float* __restrict__ bc, const float* __restrict__ pw,
                                        const float* __restrict__ pb, float slope, int C, int L, float* __restrict__ y,
                                        long long y_bstride) {
  const int c = blockIdx.y, b = blockIdx.z;
  const float* xr = x + (long long)b * x_bstride + (long long)c * L;
  float* yr = y + (long long)b * y_bstride + (long long)c * 2 * L;
  const float pa = a[b * C + c], pbv = bc[b * C + c];
  const float w0 = pw[c * 3 + 0], w1 = pw[c * 3 + 1], w2 = pw[c * 3 + 2], bias = pb[c];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < L; i += gridDim.x * blockDim.x) {
    float z0 = fmaf(xr[i], pa, pbv);
    z0 = z0 > 0.f ? z0 : z0 * slope;
    float z1 = 0.f;
    if (i + 1 < L) {
      z1 = fmaf(xr[i + 1], pa, pbv);
      z1 = z1 > 0.f ? z1 : z1 * slope;
    }
    yr[2 * i] = w1 * z0 + bias;
    yr[2 * i + 1] = w2 * z0 + w0 * z1 + bias;
  }
}

// LayerNorm over channels of [B,C,L] + LeakyReLU + length mask: one thread per (b,t) column.
__global__ void channel_layernorm_lrelu_kernel(const float* __restrict__ x, float* __restrict__ y,
                                               const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                               float slope, const int* __restrict__ lengths, int C, int L) {
  const int b = blockIdx.y;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= L) return;
  const float* xc = x + (long long)b * C * L + t;
  float* yc = y + (long long)b * C * L + t;
  if (lengths && t >= lengths[b]) {
    for (int c = 0; c < C; ++c) yc[(long long)c * L] = 0.f;
    return;
  }
  float s = 0.f;
  for (int c = 0; c < C; ++c) s += xc[(long long)c * L];
  const float mean = s / (float)C;
  float m2 = 0.f;
  for (int c = 0; c < C; ++c) {
    const float d = xc[(long long)c * L] - mean;
    m2 = fmaf(d, d, m2);
  }
  const float rstd = rsqrtf(m2 / (float)C + eps);
  for (int c = 0; c < C; ++c) {
    float v = (xc[(long long)c * L] - mean) * rstd * gamma[c] + beta[c];
    yc[(long long)c * L] = v > 0.f ? v : v * slope;
  }
}

}  // namespace st2

using namespace st2;

extern "C" {

int st2_conv_stats_parts(int Lq) { return cdiv(Lq, TQ); }

int st2_conv1d(const st2_conv_args* a, void* stream) {
  ST2_REQUIRE(a && a->x && a->w && a->y, "st2_conv1d", "null pointer");
  ST2_REQUIRE(a->B > 0 && a->Cin > 0 && a->Cout > 0 && a->Lq > 0 && a->K > 0 && a->stride > 0 && a->dil > 0,
              "st2_conv1d", "bad shape");
  ST2_REQUIRE(a->pre_act != ST2_ACT_SNAKE || a->pre_alpha, "st2_conv1d", "snake prologue needs alpha");
  ST2_REQUIRE(!a->stats || a->stats_nparts >= a->stats_part_offset + st2_conv_stats_parts(a->Lq), "st2_conv1d",
              "stats buffer too small");
  int rc = conv_launch(*a, (cudaStream_t)stream);
  if (rc) return rc;
  ST2_CHECK_LAUNCH("st2_conv1d");
  return 0;
}

int st2_conv_transpose1d(const st2_conv_args* a0, const float* wp, int K, int S, int P, int reflect_left1, void* stream) {
  ST2_REQUIRE(a0 && a0->x && wp && a0->y, "st2_conv_transpose1d", "null pointer");
  ST2_REQUIRE(K > 0 && S > 0 && P >= 0, "st2_conv_transpose1d", "bad shape");
  const int J = (K + S - 1) / S;
  const int parts = st2_conv_stats_parts(a0->Lin);
  ST2_REQUIRE(!a0->stats || a0->stats_nparts >= S * parts, "st2_conv_transpose1d", "stats buffer too small");
  for (int r = 0; r < S; ++r) {
    st2_conv_args a = *a0;
    const int cr = (r + P) / S;
    a.K = J;
    a.stride = 1;
    a.dil = 1;
    a.pad = (J - 1) - cr;
    a.Lq = a0->Lin;
    a.y_tstride = S;
    a.y_toffset = r + (reflect_left1 ? 1 : 0);
    a.y_len = a0->Lin * S + (reflect_left1 ? 1 : 0);
    a.w = wp + (long long)r * a0->Cin * J * a0->Cout;
    a.stats_part_offset = r * parts;
    a.dup_q0_to = (reflect_left1 && r == 1) ? 0 : -1;
    int rc = conv_launch(a, (cudaStream_t)stream);
    if (rc) return rc;
  }
  ST2_CHECK_LAUNCH("st2_conv_transpose1d");
  return 0;
}

int st2_row_norm(const float* v, float* out, int rows, int cols, void* stream) {
  ST2_REQUIRE(v && out && rows > 0 && cols > 0, "st2_row_norm", "bad args");
  row_norm_kernel<<<rows, 256, 0, (cudaStream_t)stream>>>(v, out, rows, cols);
  ++g_launches;
  ST2_CHECK_LAUNCH("st2_row_norm");
  return 0;
}

int st2_weight_norm_fold(const float* v, const float* g, float* w, int rows, int cols, void* stream) {
  ST2_REQUIRE(v && g && w && rows > 0 && cols > 0, "st2_weight_norm_fold", "bad args");
  weight_norm_fold_kernel<<<rows, 256, 0, (cudaStream_t)stream>>>(v, g, w, rows, cols);
  ++g_launches;
  ST2_CHECK_LAUNCH("st2_weight_norm_fold");
  return 0;
}

int st2_conv_weight_layout(const float* w, float* wt, int Cout, int Cin, int K, void* stream) {
  ST2_REQUIRE(w && wt && Cout > 0 && Cin > 0 && K > 0, "st2_conv_weight_layout", "bad args");
  const long long n = (long long)Cout * Cin * K;
  conv_weight_layout_kernel<<<(int)((n + 255) / 256 > 4096 ? 4096 : (n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      w, wt, Cout, Cin, K);
  ++g_launches;
  ST2_CHECK_LAUNCH("st2_conv_weight_layout");
  return 0;
}

int st2_convT_weight_layout(const float* w, float* wp, int Cin, int Cout, int K, int S, int P, void* stream) {
  ST2_REQUIRE(w && wp && Cout > 0 && Cin > 0 && K > 0 && S > 0, "st2_convT_weight_layout", "bad args");
  const int J = (K + S - 1) / S;
  const long long n = (long long)S * Cin * J * Cout;
  convT_weight_layout_kernel<<<(int)((n + 255) / 256 > 4096 ? 4096 : (n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      w, wp, Cin, Cout, K, S, P, J);
  ++g_launches;
  ST2_CHECK_LAUNCH("st2_convT_weight_layout");
  return 0;
}

int st2_instance_stats(const float* x, long long bstride, int B, int C, int L, float* stats, void* stream) {
  ST2_REQUIRE(x && stats && B > 0 && C > 0 && L > 0, "st2_instance_stats", "bad args");
  instance_stats_kernel<<<dim3(C, B), 256, 0, (cudaStream_t)stream>>>(x, bstride, C, L, stats);
  ++g_launches;
  ST2_CHECK_LAUNCH("st2_instance_stats");
  return 0;
}

int st2_adain_coef(const float* stats, int nparts, const float* gb, long long gb_stride, int B, int C, float eps,
                   float* a, float* b, void* stream) {
  ST2_REQUIRE(stats && gb && a && b && nparts > 0 && B > 0 && C > 0, "st2_adain_coef", "bad args");
  adain_coef_kernel<<<cdiv(B * C, 8), 256, 0, (cudaStream_t)stream>>>(stats, nparts, gb, gb_stride, B, C, eps, a, b);
  ++g_launches;
  ST2_CHECK_LAUNCH("st2_adain_coef");
  return 0;
}

int st2_adain_lrelu_pool(const float* x, long long x_bstride, const float* a, const float* b, const float* pw,
                         const float* pb, float slope, int B, int C, int L, float* y, long long y_bstride, void* stream) {
  ST2_REQUIRE(x && a && b && pw && pb && y && B > 0 && C > 0 && L > 0, "st2_adain_lrelu_pool", "bad args");
  adain_lrelu_pool_kernel<<<dim3(cdiv(L, 256), C, B), 256, 0, (cudaStream_t)stream>>>(x, x_bstride, a, b, pw, pb, slope, C,
                                                                                       L, y, y_bstride);
  ++g_launches;
  ST2_CHECK_LAUNCH("st2_adain_lrelu_pool");
  return 0;
}

int st2_channel_layernorm_lrelu(const float* x, float* y, const float* gamma, const float* beta, float eps, float slope,
                                const int* lengths, int B, int C, int L, void* stream) {
  ST2_REQUIRE(x && y && gamma && beta && B > 0 && C > 0 && L > 0, "st2_channel_layernorm_lrelu", "bad args");
  channel_layernorm_lrelu_kernel<<<dim3(cdiv(L, 128), B), 128, 0, (cudaStream_t)stream>>>(x, y, gamma, beta, eps, slope,
                                                                                         lengths, C, L);
  ++g_launches;
  ST2_CHECK_LAUNCH("st2_channel_layernorm_lrelu");
  return 0;
}

}  // extern "C"
