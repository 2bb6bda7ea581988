// Bidirectional LSTM recurrence (fp32).  The input projection x W_ih^T + b is one batched GEMM
// (st2_linear) done beforehand; this file runs the serial part: for every step,
//   gates = gx[:, t] + h_{t-1} W_hh^T ; (i,f,g,o) ; c = f*c + i*g ; h = o*tanh(c)
// v1: one launch per time step covering both directions (grid.y) and all utterances; a CTA owns
// 4 hidden units x 32 utterances, stages its 16 W_hh rows and the 32 previous hidden vectors in
// shared memory and does 128-bit conflict-free reads.  The sequential depth (N token steps,
// T frame steps) makes this latency-bound, not bandwidth-bound (SURVEY section 8d).
#include <cooperative_groups.h>

#include "common.cuh"

namespace st2 {
extern long long g_launches;

constexpr int LSTM_UT = 4;   // hidden units per CTA
constexpr int LSTM_BT = 32;  // utterances per CTA

__global__ void __launch_bounds__(LSTM_UT* LSTM_BT) lstm_step_kernel(
    const float* __restrict__ gx, const float* __restrict__ whh, float* __restrict__ out, long long o_bs, long long o_ts,
    long long o_cs, const int* __restrict__ lengths, int B, int L, int H, int step, const float* __restrict__ h_prev,
    float* __restrict__ h_next, float* __restrict__ c_state) {
  extern __shared__ __align__(16) float sm[];
  const int HP = H + 4;
  float* ws = sm;                       // [4 gates][UT][HP]
  float* hs = sm + 4 * LSTM_UT * HP;    // [BT][HP]
  const int dir = blockIdx.y;
  const int j0 = blockIdx.x * LSTM_UT;
  const int b0 = blockIdx.z * LSTM_BT;
  const int tid = threadIdx.x;
  const float* wd = whh + (long long)dir * 4 * H * H;
  // vectorised, unrolled staging: every thread has several independent 128-bit loads in flight
  // (a scalar loop with div/mod serialised ~100 dependent global loads per thread: 50 us per step)
  const int H4 = H >> 2;
  {
    const int n4 = 4 * LSTM_UT * H4;  // float4 count of the W slab
#pragma unroll 4
    for (int i = tid; i < n4; i += LSTM_UT * LSTM_BT) {
      const int k4 = i % H4;
      const int r = i / H4;  // g*UT + u
      const int g = r / LSTM_UT, u = r - g * LSTM_UT;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (j0 + u < H) v = __ldg(reinterpret_cast<const float4*>(wd + ((long long)g * H + j0 + u) * H) + k4);
      *reinterpret_cast<float4*>(ws + r * HP + 4 * k4) = v;
    }
  }
  const float* hp = h_prev + (long long)dir * B * H;
  {
    const int n4 = LSTM_BT * H4;
#pragma unroll 8
    for (int i = tid; i < n4; i += LSTM_UT * LSTM_BT) {
      const int k4 = i % H4, bl = i / H4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (b0 + bl < B) v = *(reinterpret_cast<const float4*>(hp + (long long)(b0 + bl) * H) + k4);
      *reinterpret_cast<float4*>(hs + bl * HP + 4 * k4) = v;
    }
  }
  __syncthreads();
  const int u = tid % LSTM_UT, bl = tid / LSTM_UT;
  const int b = b0 + bl, j = j0 + u;
  if (b >= B || j >= H) return;
  const int len = lengths ? lengths[b] : L;
  float* hn = h_next + (long long)dir * B * H + (long long)b * H + j;
  if (step >= len) {  // padded step: state carried through unchanged, no output
    *hn = hs[bl * HP + j];
    return;
  }
  const int t = dir == 0 ? step : (len - 1 - step);
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  const float* hr = hs + bl * HP;
  const float* w0 = ws + (0 * LSTM_UT + u) * HP;
  const float* w1 = ws + (1 * LSTM_UT + u) * HP;
  const float* w2 = ws + (2 * LSTM_UT + u) * HP;
  const float* w3 = ws + (3 * LSTM_UT + u) * HP;
#pragma unroll 4
  for (int k = 0; k < H; k += 4) {
    const float4 hv = *reinterpret_cast<const float4*>(hr + k);
    const float4 x0 = *reinterpret_cast<const float4*>(w0 + k);
    const float4 x1 = *reinterpret_cast<const float4*>(w1 + k);
    const float4 x2 = *reinterpret_cast<const float4*>(w2 + k);
    const float4 x3 = *reinterpret_cast<const float4*>(w3 + k);
    a0 = fmaf(hv.x, x0.x, a0); a0 = fmaf(hv.y, x0.y, a0); a0 = fmaf(hv.z, x0.z, a0); a0 = fmaf(hv.w, x0.w, a0);
    a1 = fmaf(hv.x, x1.x, a1); a1 = fmaf(hv.y, x1.y, a1); a1 = fmaf(hv.z, x1.z, a1); a1 = fmaf(hv.w, x1.w, a1);
    a2 = fmaf(hv.x, x2.x, a2); a2 = fmaf(hv.y, x2.y, a2); a2 = fmaf(hv.z, x2.z, a2); a2 = fmaf(hv.w, x2.w, a2);
    a3 = fmaf(hv.x, x3.x, a3); a3 = fmaf(hv.y, x3.y, a3); a3 = fmaf(hv.z, x3.z, a3); a3 = fmaf(hv.w, x3.w, a3);
  }
  const float* g = gx + ((long long)b * L + t) * (8 * H) + (long long)dir * 4 * H + j;
  const float gi = sigmoidf_(g[0] + a0);
  const float gf = sigmoidf_(g[H] + a1);
  const float gg = tanhf(g[2 * H] + a2);
  const float go = sigmoidf_(g[3 * H] + a3);
  float* cp = c_state + (long long)dir * B * H + (long long)b * H + j;
  const float c = gf * (*cp) + gi * gg;
  *cp = c;
  const float h = go * tanhf(c);
  *hn = h;
  out[(long long)b * o_bs + (long long)t * o_ts + (long long)(dir * H + j) * o_cs] = h;
}

// Persistent variant: ONE cooperative launch for the whole sequence.  Each CTA keeps its 16 W_hh rows in shared
// memory for all steps (no per-step re-staging, no per-step launch); the previous hidden state is exchanged through
// L2 with one grid-wide barrier per step (cooperative groups grid.sync()).  grid = (H/4, 2 directions) <= 132 CTAs.
__global__ void __launch_bounds__(LSTM_UT* LSTM_BT) lstm_persistent_kernel(
    const float* __restrict__ gx, const float* __restrict__ whh, float* __restrict__ out, long long o_bs, long long o_ts,
    long long o_cs, const int* __restrict__ lengths, int B, int L, int H, float* __restrict__ h0, float* __restrict__ h1,
    float* __restrict__ c_state, unsigned int* __restrict__ step_bar) {
  extern __shared__ __align__(16) float sm[];
  const int HP = H + 4;
  float* ws = sm;
  float* hs = sm + 4 * LSTM_UT * HP;
  const int dir = blockIdx.y;
  const int j0 = blockIdx.x * LSTM_UT;
  const int tid = threadIdx.x;
  const int H4 = H >> 2;
  const float* wd = whh + (long long)dir * 4 * H * H;
  {
    const int n4 = 4 * LSTM_UT * H4;
#pragma unroll 4
    for (int i = tid; i < n4; i += LSTM_UT * LSTM_BT) {
      const int k4 = i % H4;
      const int r = i / H4;
      const int g = r / LSTM_UT, u = r - g * LSTM_UT;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (j0 + u < H) v = __ldg(reinterpret_cast<const float4*>(wd + ((long long)g * H + j0 + u) * H) + k4);
      *reinterpret_cast<float4*>(ws + r * HP + 4 * k4) = v;
    }
  }
  const int u = tid % LSTM_UT, bl = tid / LSTM_UT;
  const int j = j0 + u;
  const float* w0 = ws + (0 * LSTM_UT + u) * HP;
  const float* w1 = ws + (1 * LSTM_UT + u) * HP;
  const float* w2 = ws + (2 * LSTM_UT + u) * HP;
  const float* w3 = ws + (3 * LSTM_UT + u) * HP;
  const int nbt = (B + LSTM_BT - 1) / LSTM_BT;
  const unsigned int nct = gridDim.x;                 // CTAs of this direction
  unsigned int* bar = step_bar + dir * 32;            // one 128-byte line per direction
  float creg = 0.f;                                   // cell state lives in a register when one batch tile covers B
  for (int step = 0; step < L; ++step) {
    const float* hprev = ((step & 1) ? h1 : h0) + (long long)dir * B * H;
    float* hnext = ((step & 1) ? h0 : h1) + (long long)dir * B * H;
    for (int bt = 0; bt < nbt; ++bt) {
      const int b0 = bt * LSTM_BT;
      const int b = b0 + bl;
      const bool live = b < B && j < H;
      // everything that does not depend on h_{t-1} is fetched first, under the latency of the h staging
      int len = L, t = 0;
      float g0 = 0.f, g1 = 0.f, g2 = 0.f, g3 = 0.f, cprev = creg;
      float* cp = c_state + (long long)dir * B * H + (long long)b * H + j;
      if (live) {
        len = lengths ? lengths[b] : L;
        if (step < len) {
          t = dir == 0 ? step : (len - 1 - step);
          const float* g = gx + ((long long)b * L + t) * (8 * H) + (long long)dir * 4 * H + j;
          g0 = __ldg(g); g1 = __ldg(g + H); g2 = __ldg(g + 2 * H); g3 = __ldg(g + 3 * H);
          if (nbt > 1) cprev = *cp;
        }
      }
      __syncthreads();  // previous users of hs are done (also orders the one-time ws staging)
      {
        const int n4 = LSTM_BT * H4;
#pragma unroll 8
        for (int i = tid; i < n4; i += LSTM_UT * LSTM_BT) {
          const int k4 = i % H4, bb = i / H4;
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          // L2 (cache-global) loads: written by other CTAs in the previous step, must not hit a stale L1 line
          if (b0 + bb < B) v = __ldcg(reinterpret_cast<const float4*>(hprev + (long long)(b0 + bb) * H) + k4);
          *reinterpret_cast<float4*>(hs + bb * HP + 4 * k4) = v;
        }
      }
      __syncthreads();
      if (live) {
        float* hn = hnext + (long long)b * H + j;
        if (step >= len) {
          *hn = hs[bl * HP + j];
        } else {
          float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
          const float* hr = hs + bl * HP;
#pragma unroll 4
          for (int k = 0; k < H; k += 4) {
            const float4 hv = *reinterpret_cast<const float4*>(hr + k);
            const float4 x0 = *reinterpret_cast<const float4*>(w0 + k);
            const float4 x1 = *reinterpret_cast<const float4*>(w1 + k);
            const float4 x2 = *reinterpret_cast<const float4*>(w2 + k);
            const float4 x3 = *reinterpret_cast<const float4*>(w3 + k);
            a0 = fmaf(hv.x, x0.x, a0); a0 = fmaf(hv.y, x0.y, a0); a0 = fmaf(hv.z, x0.z, a0); a0 = fmaf(hv.w, x0.w, a0);
            a1 = fmaf(hv.x, x1.x, a1); a1 = fmaf(hv.y, x1.y, a1); a1 = fmaf(hv.z, x1.z, a1); a1 = fmaf(hv.w, x1.w, a1);
            a2 = fmaf(hv.x, x2.x, a2); a2 = fmaf(hv.y, x2.y, a2); a2 = fmaf(hv.z, x2.z, a2); a2 = fmaf(hv.w, x2.w, a2);
            a3 = fmaf(hv.x, x3.x, a3); a3 = fmaf(hv.y, x3.y, a3); a3 = fmaf(hv.z, x3.z, a3); a3 = fmaf(hv.w, x3.w, a3);
          }
          const float gi = sigmoidf_(g0 + a0);
          const float gf = sigmoidf_(g1 + a1);
          const float gg = tanhf(g2 + a2);
          const float go = sigmoidf_(g3 + a3);
          const float c = gf * cprev + gi * gg;
          if (nbt > 1) *cp = c; else creg = c;
          const float h = go * tanhf(c);
          *hn = h;
          out[(long long)b * o_bs + (long long)t * o_ts + (long long)(dir * H + j) * o_cs] = h;
        }
      }
    }
    // per-direction step barrier (the two directions never exchange data): release our h writes, then wait
    // until all `nct` CTAs of this direction have arrived `step+1` times.  Co-residency of the CTAs is
    // guaranteed by the cooperative launch.
    __syncthreads();
    if (tid == 0) {
      __threadfence();
      atomicAdd(bar, 1u);
      const unsigned int want = nct * (unsigned int)(step + 1);
      unsigned int seen;
      do {
        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(bar) : "memory");
      } while (seen < want);
    }
    __syncthreads();
  }
}


// ------------------------------------------------------------------------------------------------
// v3 (H == 256): thread-block clusters + distributed shared memory.  One cluster of 8 CTAs owns
// (direction, group of BG utterances): CTA r keeps the W_hh rows of hidden units [32r, 32r+32) x 4 gates
// entirely in REGISTERS (64 weights per thread: unit u x 16-way k-slice) and the previous hidden vectors
// of its utterances (BG x 256, double-buffered) in shared memory.  After each step the 32 new h values
// of a CTA go straight into the shared memory of all 8 CTAs with st.async (remote store that also
// completes bytes on the destination CTA's mbarrier), so the only synchronisation on the serial chain is
// a local mbarrier wait: no global-memory round trip, no device-wide or cluster-wide barrier per step.
// (Measured alternatives: barrier.cluster per step 4.3 us/step, staged cp.async.bulk rows 4.7 us/step,
// st.async 3.7 us/step at B=32; the cooperative-launch kernel with an L2 barrier was 8.8 us/step.)
// Step cost = BG*64 FMAs/thread + a 15-shuffle transpose-reduce + gate math + one DSMEM hop (~215 cycles).
// Utterances are independent, so groups never synchronise with each other (B=32 -> 2 x 8 clusters = 128 SMs).
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_barrier() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t mapa_u32(uint32_t local_smem_addr, uint32_t rank) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local_smem_addr), "r"(rank));
  return remote;
}
// remote 4-byte store that completes 4 tx-bytes on the mbarrier of the SAME destination CTA
__device__ __forceinline__ void st_async_f32(uint32_t remote_addr, float v, uint32_t remote_mbar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(remote_addr),
               "r"(__float_as_uint(v)), "r"(remote_mbar)
               : "memory");
}
__device__ long long* g_lstm_trace = nullptr;   // [8] cycle sums of CTA 0 / thread 0 (st2_debug_lstm_trace)
__device__ __forceinline__ void lc_mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void lc_mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void lc_mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
  } while (!done);
}

constexpr int LC_H = 256, LC_CTAS = 8, LC_THREADS = 512, LC_GMAX = 8;

// BG utterances per pass (1..4), `npass` (1 or 2) passes per step: a cluster serves up to 8 utterances so that all
// clusters of a call are co-resident (the occupancy query below says how many 8-CTA clusters fit; a second wave would double the time).
template <int BG>
__global__ void __cluster_dims__(LC_CTAS, 1, 1) __launch_bounds__(LC_THREADS, 1)
    lstm_cluster_kernel(const float* __restrict__ gx, const float* __restrict__ whh, float* __restrict__ out, long long o_bs,
                        long long o_ts, long long o_cs, const int* __restrict__ lengths, int B, int L, int npass, int gsize) {
  constexpr int H = LC_H;
  __shared__ __align__(16) float hs[2][LC_GMAX][H];
  __shared__ __align__(8) unsigned long long full_bar[2];   // full_bar[b]: buffer b holds the complete h of a step
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int s = lane & 15;                    // k-slice: float4 columns {s, 16+s, 32+s, 48+s}
  const int u = warp * 2 + (lane >> 4);       // hidden unit inside this CTA
  const uint32_t rank = cluster_ctarank();
  const int ci = blockIdx.x / LC_CTAS;
  const int dir = ci & 1, grp = ci >> 1;
  const int j = (int)rank * 32 + u;
  const int b0 = grp * gsize;   // gsize <= BG * npass utterances per cluster
  const int nlive = min(gsize, B - b0);
  const uint32_t fill_bytes = (uint32_t)nlive * H * 4u;     // 8 CTAs x 32 units x nlive utterances x 4 B

  // W_hh rows of unit j, 4 gates, this thread's 16 k's, as (even k, odd k) pairs (two independent FMA chains)
  float2 w[4][8];
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    const float4* wr = reinterpret_cast<const float4*>(whh + ((long long)(dir * 4 + g) * H + j) * H);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 v = __ldg(wr + q * 16 + s);
      w[g][q * 2 + 0] = make_float2(v.x, v.y);
      w[g][q * 2 + 1] = make_float2(v.z, v.w);
    }
  }
  for (int i = tid; i < 2 * LC_GMAX * H; i += LC_THREADS) (&hs[0][0][0])[i] = 0.f;
  const uint32_t bar0 = (uint32_t)__cvta_generic_to_shared(&full_bar[0]);
  if (tid == 0) {
    lc_mbar_init(bar0, 1);
    lc_mbar_init(bar0 + 8, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }

  // after the transpose-reduce, lane gl = bb*4 + gate of each 16-lane half holds that pre-activation sum: every lane
  // applies its own gate non-linearity (branch-free: sigma(x) = 1/(1+e^-x), tanh(x) = 2/(1+e^-2x) - 1), then the
  // gate-0 lane of each utterance gathers f, g, o from its neighbours and finishes the cell.
  const int gl = lane & 15;
  const int bbl = gl >> 2, gate = gl & 3;
  const float act_k = gate == 2 ? 2.f : 1.f, act_b = gate == 2 ? -1.f : 0.f;
  bool valid[2];
  int len[2];
  const float* gxl[2];
  float c[2] = {0.f, 0.f};
  float nx[2] = {0.f, 0.f};   // this lane's gate pre-activation input of the coming step (fetched one step ahead)
#pragma unroll
  for (int p = 0; p < 2; ++p) {
    const int ub = p * BG + bbl;
    const int b = b0 + ub;
    valid[p] = p < npass && bbl < BG && ub < gsize && b < B;
    len[p] = L;
    if (valid[p] && lengths) len[p] = lengths[b];
    gxl[p] = gx + (long long)(valid[p] ? b : 0) * L * (8 * H) + (long long)dir * 4 * H + gate * H + j;
    if (valid[p] && len[p] > 0) nx[p] = __ldg(gxl[p] + (long long)(dir == 0 ? 0 : len[p] - 1) * (8 * H));
  }
  long long* trace = (blockIdx.x == 0 && tid == 0) ? g_lstm_trace : nullptr;
  long long tr[5] = {0, 0, 0, 0, 0};
  cluster_barrier();  // buffers zeroed and barriers initialised in every CTA before any remote store may land

  for (int step = 0; step < L; ++step) {
    const int cur = step & 1;
    if (tid == 0) lc_mbar_expect_tx(bar0 + 8 * (cur ^ 1), fill_bytes);   // arm this step's fill of the other buffer
    float gxv[2];
#pragma unroll
    for (int p = 0; p < 2; ++p) {
      gxv[p] = nx[p];
      if (valid[p] && step + 1 < len[p]) nx[p] = __ldg(gxl[p] + (long long)(dir == 0 ? step + 1 : len[p] - 2 - step) * (8 * H));
    }
    long long tc = trace ? clock64() : 0;
    if (step > 0) lc_mbar_wait(bar0 + 8 * cur, (uint32_t)(((step - 1) >> 1) & 1));
    if (trace) { const long long n = clock64(); tr[0] += n - tc; tc = n; }
#pragma unroll
    for (int p = 0; p < 2; ++p) {
      if (p < npass) {
        float2 acc[BG][4];
#pragma unroll
        for (int bb = 0; bb < BG; ++bb)
#pragma unroll
          for (int g = 0; g < 4; ++g) acc[bb][g] = make_float2(0.f, 0.f);
#pragma unroll
        for (int bb = 0; bb < BG; ++bb) {
          const float4* hr = reinterpret_cast<const float4*>(&hs[cur][p * BG + bb][0]);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float4 hv = hr[q * 16 + s];
            const float2 h01 = make_float2(hv.x, hv.y), h23 = make_float2(hv.z, hv.w);
#pragma unroll
            for (int g = 0; g < 4; ++g) {
              acc[bb][g].x = fmaf(h01.x, w[g][q * 2 + 0].x, acc[bb][g].x);
              acc[bb][g].y = fmaf(h01.y, w[g][q * 2 + 0].y, acc[bb][g].y);
              acc[bb][g].x = fmaf(h23.x, w[g][q * 2 + 1].x, acc[bb][g].x);
              acc[bb][g].y = fmaf(h23.y, w[g][q * 2 + 1].y, acc[bb][g].y);
            }
          }
        }
        float v[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) v[i] = (i >> 2) < BG ? acc[(i >> 2) < BG ? (i >> 2) : 0][i & 3].x + acc[(i >> 2) < BG ? (i >> 2) : 0][i & 3].y : 0.f;
        if (trace) { const long long n = clock64(); tr[1] += n - tc; tc = n; }
        // transpose-reduce over the 16 k-slices: 8+4+2+1 shuffles leave value #(lane&15) on each lane
#define ST2_RED(NV, OFF)                                                        \
  {                                                                             \
    const bool up = (lane & OFF) != 0;                                          \
    _Pragma("unroll") for (int i = 0; i < NV / 2; ++i) {                        \
      const float send = up ? v[i] : v[i + NV / 2];                             \
      const float keep = up ? v[i + NV / 2] : v[i];                             \
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, OFF);                    \
    }                                                                           \
  }
        ST2_RED(16, 8)
        ST2_RED(8, 4)
        ST2_RED(4, 2)
        ST2_RED(2, 1)
#undef ST2_RED
        if (trace) { const long long n = clock64(); tr[2] += n - tc; tc = n; }
        const float x = v[0] + gxv[p];
        const float a = __fdiv_rn(act_k, 1.0f + expf(-act_k * x)) + act_b;
        const float af = __shfl_down_sync(0xffffffffu, a, 1);
        const float ag = __shfl_down_sync(0xffffffffu, a, 2);
        const float ao = __shfl_down_sync(0xffffffffu, a, 3);
        if (gate == 0 && valid[p]) {
          const int ub = p * BG + bbl;
          const bool act = step < len[p];
          float hnew;
          if (!act) {
            hnew = hs[cur][ub][j];   // pack_padded_sequence: state frozen past the utterance's length
          } else {
            c[p] = af * c[p] + a * ag;
            hnew = ao * (__fdiv_rn(2.0f, 1.0f + expf(-2.0f * c[p])) - 1.0f);
          }
          if (trace) { const long long n = clock64(); tr[3] += n - tc; tc = n; }
          const uint32_t laddr = (uint32_t)__cvta_generic_to_shared(&hs[cur ^ 1][ub][j]);
          const uint32_t lbar = bar0 + 8 * (cur ^ 1);
#pragma unroll
          for (uint32_t r = 0; r < (uint32_t)LC_CTAS; ++r) st_async_f32(mapa_u32(laddr, r), hnew, mapa_u32(lbar, r));
          if (act) {
            const int t = dir == 0 ? step : (len[p] - 1 - step);
            out[(long long)(b0 + ub) * o_bs + (long long)t * o_ts + (long long)(dir * H + j) * o_cs] = hnew;
          }
          if (trace) { const long long n = clock64(); tr[4] += n - tc; tc = n; }
        }
      }
    }
  }
  if (trace) {
    for (int i = 0; i < 5; ++i) trace[i] = tr[i];
    trace[5] = L;
  }
  // drain: the last step's rows have landed here (so every copy INTO this CTA is complete), then meet the peers so
  // that every store OUT of this CTA has completed at its destination before any CTA of the cluster retires
  lc_mbar_wait(bar0 + 8 * (L & 1), (uint32_t)(((L - 1) >> 1) & 1));
  cluster_barrier();
}

}  // namespace st2

using namespace st2;

static int g_lstm_cluster = 1;
// testing / A-B hook: 0 selects the cooperative-launch kernel for every shape
// profiling aid: device buffer of 8 int64 receiving, for CTA 0 / thread 0 of the cluster kernel, the cycle sums of
// {mbarrier wait, h loads + FMAs, transpose-reduce, gate math, remote stores} and the step count; NULL disables
extern "C" int st2_debug_lstm_trace(void* buf) {
  long long* p = (long long*)buf;
  cudaError_t e = cudaMemcpyToSymbol(g_lstm_trace, &p, sizeof(p));
  if (e != cudaSuccess) { set_error("st2_debug_lstm_trace", e); return (int)e; }
  return 0;
}
extern "C" int st2_debug_lstm_cluster(int enable) {
  g_lstm_cluster = enable;
  return 0;
}

extern "C" int st2_lstm_bidir(const float* gx, const float* whh, float* out, long long o_bs, long long o_ts, long long o_cs,
                              const int* lengths, int B, int L, int H, float* work, void* stream) {
  ST2_REQUIRE(gx && whh && out && work && B > 0 && L > 0 && H > 0 && H % 4 == 0, "st2_lstm_bidir", "bad args");
  cudaStream_t st = (cudaStream_t)stream;
  if (H == LC_H && g_lstm_cluster) {
    // how many 8-CTA clusters the device holds at once (GPC geometry); a second wave would double the time
    static int max_clusters = 0;
    if (max_clusters == 0) {
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = dim3(LC_CTAS * 16);
      cfg.blockDim = dim3(LC_THREADS);
      cudaLaunchAttribute at[1];
      at[0].id = cudaLaunchAttributeClusterDimension;
      at[0].val.clusterDim.x = LC_CTAS;
      at[0].val.clusterDim.y = 1;
      at[0].val.clusterDim.z = 1;
      cfg.attrs = at;
      cfg.numAttrs = 1;
      int nc = 0;
      if (cudaOccupancyMaxActiveClusters(&nc, lstm_cluster_kernel<4>, &cfg) != cudaSuccess || nc < 2) {
        cudaGetLastError();
        nc = 8;
      }
      max_clusters = nc;
    }
    const int groups_fit = max_clusters / 2 > 0 ? max_clusters / 2 : 1;   // two directions per utterance group
    int gsize = cdiv(B, groups_fit);
    if (gsize > LC_GMAX) gsize = LC_GMAX;                                  // larger batches run in waves of co-resident clusters
    const int npass = gsize > 4 ? 2 : 1;
    const int bg = cdiv(gsize, npass);
    const int groups = cdiv(B, gsize);
    dim3 grid(LC_CTAS * 2 * groups);
    if (bg == 1) lstm_cluster_kernel<1><<<grid, LC_THREADS, 0, st>>>(gx, whh, out, o_bs, o_ts, o_cs, lengths, B, L, npass, gsize);
    else if (bg == 2) lstm_cluster_kernel<2><<<grid, LC_THREADS, 0, st>>>(gx, whh, out, o_bs, o_ts, o_cs, lengths, B, L, npass, gsize);
    else if (bg == 3) lstm_cluster_kernel<3><<<grid, LC_THREADS, 0, st>>>(gx, whh, out, o_bs, o_ts, o_cs, lengths, B, L, npass, gsize);
    else lstm_cluster_kernel<4><<<grid, LC_THREADS, 0, st>>>(gx, whh, out, o_bs, o_ts, o_cs, lengths, B, L, npass, gsize);
    ++g_launches;
    ST2_CHECK_LAUNCH("st2_lstm_bidir (cluster)");
    return 0;
  }
  const size_t n = (size_t)2 * B * H;
  float* h0 = work;
  float* h1 = work + n;
  float* c = work + 2 * n;
  unsigned int* step_bar = reinterpret_cast<unsigned int*>(work + 3 * n);   // 64 words: per-direction step barriers
  cudaError_t e = cudaMemsetAsync(work, 0, (3 * n + 64) * sizeof(float), st);
  if (e != cudaSuccess) { set_error("st2_lstm_bidir", e); return (int)e; }
  const size_t smem = (size_t)(4 * LSTM_UT + LSTM_BT) * (H + 4) * sizeof(float);
  static PerDevice once_step;
  if (once_step.first()) cudaFuncSetAttribute(lstm_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
  ST2_REQUIRE(smem <= 160 * 1024, "st2_lstm_bidir", "hidden size too large");
  // persistent cooperative kernel when the grid fits on the device (H/4 * 2 CTAs), else one launch per step
  static PerDevice once_p, sms_p;
  if (once_p.first()) {
    const int d = once_p.dev();
    cudaDeviceGetAttribute(&once_p.value[d], cudaDevAttrCooperativeLaunch, d);
    cudaDeviceGetAttribute(&sms_p.value[d], cudaDevAttrMultiProcessorCount, d);
    cudaFuncSetAttribute(lstm_persistent_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
  }
  const int coop = once_p.value[once_p.dev()], num_sms = sms_p.value[once_p.dev()];
  if (coop && cdiv(H, LSTM_UT) * 2 <= num_sms) {
    dim3 pgrid(cdiv(H, LSTM_UT), 2);
    void* args[] = {(void*)&gx, (void*)&whh, (void*)&out, (void*)&o_bs, (void*)&o_ts, (void*)&o_cs, (void*)&lengths,
                    (void*)&B,  (void*)&L,   (void*)&H,   (void*)&h0,   (void*)&h1,   (void*)&c,
                    (void*)&step_bar};
    e = cudaLaunchCooperativeKernel((const void*)lstm_persistent_kernel, pgrid, dim3(LSTM_UT * LSTM_BT), args, smem, st);
    if (e != cudaSuccess) { set_error("st2_lstm_bidir (cooperative launch)", e); return (int)e; }
    ++g_launches;
    return 0;
  }
  dim3 grid(cdiv(H, LSTM_UT), 2, cdiv(B, LSTM_BT));
  for (int s = 0; s < L; ++s) {
    const float* hp = (s & 1) ? h1 : h0;
    float* hn = (s & 1) ? h0 : h1;
    lstm_step_kernel<<<grid, LSTM_UT * LSTM_BT, smem, st>>>(gx, whh, out, o_bs, o_ts, o_cs, lengths, B, L, H, s, hp, hn, c);
    ++g_launches;
  }
  ST2_CHECK_LAUNCH("st2_lstm_bidir");
  return 0;
}
