// Tensor-core (wgmma) GEMM for the row-layout Linears of the style denoiser -- sm_90a.
//
//   C[m, n] = act( sum_k A[m,k] * W[n,k] + bias[n] ) + R[m,n]         A,C,R row-major, W = torch Linear weight [Nf,K]
//
// fp32-ACCURATE on 16-bit tensor cores: the predicted integer durations are downstream of the denoiser, so its
// arithmetic must stay at fp32 accuracy (DESIGN.md section 2).  Every operand is split into TWO fp16 planes,
// x = h + l * 2^-11 with h = fp16(x) and l = fp16((x - h) * 2^11): 22 significand bits, and the 2^11 pre-scaling keeps
// the low plane out of fp16's subnormal range for every |x| >= 2^-14.  A product needs the three MMAs h*h, h*l, l*h
// (l*l is 2^-22 relative); h*h accumulates in one register accumulator and the two scaled correction products in a
// second one that the epilogue folds in with an exact * 2^-11 (the tensor core truncates when it adds into an
// accumulator, so keeping the small terms out of the big running sum keeps the error at the fp32-SIMT level).
// Range: |x| must stay below fp16's 65504 (activations and weights of this model are O(1..10)); larger values
// produce inf/NaN loudly rather than a silently wrong result.
//
// Mapping: a tile is 128 out-features x 64 tokens.  A operand = weight block [64 n x 16 k] per warpgroup, B operand =
// activation block [64 tokens x 16 k], both K-major no-swizzle "interleave" layout (16-byte rows of 8 fp16).  Weights are
// pre-split and pre-arranged so that one K-block stage (32 features x 2 planes) is one contiguous 16 KB 1-D TMA bulk copy.
// Activations are staged by 8 warps (four threads per token row, 32 contiguous bytes each, software-pipelined one block
// ahead) or arrive pre-split as one bulk copy per stage.
// Warp roles: warps 0-7 = two consumer warpgroups (wgmma over out-features 0-63 / 64-127, accumulators in registers, then
// the epilogue), warp 8 = TMA producer, warps 9-16 = stagers; persistent CTAs.
#include <cuda_fp16.h>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace st2 {
extern long long g_launches;

namespace ltc {

constexpr int TMF = 128;   // out features per tile (two warpgroups of M = 64)
constexpr int TNT = 64;    // tokens per tile (wgmma N)
constexpr int KB = 32;     // K block (4 chunks of 8)
constexpr int NPL = 2;     // fp16 planes per operand (high, low * 2^11)
constexpr float LO_SCALE = 2048.0f, LO_UNSCALE = 1.0f / 2048.0f;
constexpr int W_STAGES = 6;
constexpr int W_PLANE_BYTES = 4 * TMF * 16;          // 8 KB
constexpr int W_STAGE_BYTES = NPL * W_PLANE_BYTES;   // 16 KB
constexpr int RWP = TNT + 2;                         // chunk pitch in rows (== 2 mod 8: conflict-free 128-bit stores)
constexpr int A_PLANE_BYTES = 4 * RWP * 16;          // 4224 B
constexpr int A_BUF_BYTES = NPL * A_PLANE_BYTES;
constexpr int A_BUFS = 4;
constexpr int PRE_PLANE_BYTES = 4 * TNT * 16;         // pre-split stage: no row padding, 4 KB per plane, 8 KB per stage
constexpr int PRE_STAGE_BYTES = NPL * PRE_PLANE_BYTES;
constexpr int NUM_CONS = 256;                        // two consumer warpgroups
constexpr int NUM_STAGERS = 256;
constexpr int THREADS = NUM_CONS + 32 + NUM_STAGERS;  // 544

constexpr int SM_W = 0;
constexpr int SM_A = SM_W + W_STAGES * W_STAGE_BYTES;
constexpr int SM_BAR = SM_A + A_BUFS * A_BUF_BYTES;
constexpr int SM_TOTAL = SM_BAR + 256;
constexpr int B_WFULL = 0, B_WEMPTY = 6, B_AFULL = 12, B_AEMPTY = 16, B_COUNT = 20;

using namespace st2::ptx;

// Range guard: the fp16 planes hold |x| < 65504; larger activations become inf (and the product NaN/inf).  Every thread
// that splits activations keeps one predicate over the values it converts and raises this flag once;
// st2_range_flag_fetch() reports and clears it (the host checks it after a pass, styletts2_b200.ops.check_range).
// Weights are checked when they are laid out.  The predicate is an AND of fabsf(x) < FP16_MAX, which is false for NaN
// (a running fmaxf maximum is not: fmaxf drops a NaN argument).
__device__ int g_range_flag = 0;
constexpr float FP16_MAX = 65504.0f;
__device__ __forceinline__ bool in_fp16_range(float x) { return fabsf(x) < FP16_MAX; }
__device__ __forceinline__ void range_note(bool in_range) {
  if (!in_range) atomicExch(&g_range_flag, 1);
}

// x0,x1 -> two packed fp16 pairs: p0 = fp16(x), p1 = fp16((x - p0) * 2^11)   (x = p0 + p1 * 2^-11 to ~2^-22 |x|)
__device__ __forceinline__ void split2(float x0, float x1, uint32_t& p0, uint32_t& p1) {
  const __half2 h = __floats2half2_rn(x0, x1);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn((x0 - hf.x) * LO_SCALE, (x1 - hf.y) * LO_SCALE);
  p0 = *reinterpret_cast<const uint32_t*>(&h);
  p1 = *reinterpret_cast<const uint32_t*>(&l);
}

struct LinArgs {
  const float* A; long long lda;
  const uint8_t* planes;   // pre-split activation stages (st2_linear_tc_split) or NULL: split on the fly by the stager warps
  const uint8_t* wtc;
  const float* bias;
  const float* R; long long ldr;
  float* C; long long ldc;
  int M, Nf, K, act;
};

__global__ void __launch_bounds__(THREADS, 1) linear_tc_kernel(const LinArgs a, const int ncb, const int ntiles, const int n_tq) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bar0 = sbase + SM_BAR;
  auto BAR = [&](int i) { return bar0 + 8u * i; };
  if (tid == 0) {
    for (int i = 0; i < W_STAGES; ++i) { mbar_init(BAR(B_WFULL + i), 1); mbar_init(BAR(B_WEMPTY + i), 2); }
    for (int i = 0; i < A_BUFS; ++i) { mbar_init(BAR(B_AFULL + i), a.planes ? 1 : NUM_STAGERS); mbar_init(BAR(B_AEMPTY + i), 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < NUM_CONS / 32) {
    // ================================================================ consumers: wgmma + epilogue
    const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t4 = lane & 3;
    const bool leader = (tid & 127) == 0;
    const uint32_t lbo_a = TMF * 16, lbo_b = (a.planes ? TNT : RWP) * 16;
    const uint32_t a_plane = a.planes ? (uint32_t)PRE_PLANE_BYTES : (uint32_t)A_PLANE_BYTES;
    const int M_ = a.M, Nf_ = a.Nf, act_ = a.act;
    int ws = 0, wph = 0, as = 0, aph = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      const int cob = tile / n_tq, tq = tile % n_tq;
      float dh[32], dl[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) { dh[i] = 0.f; dl[i] = 0.f; }
      int pws = -1, pas = -1;
      for (int cb = 0; cb < ncb; ++cb) {
        mbar_wait(BAR(B_AFULL + as), aph);
        mbar_wait(BAR(B_WFULL + ws), wph);
        wg_fence();
        const uint32_t wa = sbase + SM_W + ws * W_STAGE_BYTES + wg * 64 * 16, ab = sbase + SM_A + as * A_BUF_BYTES;
#pragma unroll
        for (int k16 = 0; k16 < 2; ++k16) {
          const uint64_t a0 = make_desc(wa + 2 * k16 * lbo_a, lbo_a, 128), a1 = make_desc(wa + 2 * k16 * lbo_a + W_PLANE_BYTES, lbo_a, 128);
          const uint64_t b0 = make_desc(ab + 2 * k16 * lbo_b, lbo_b, 128), b1 = make_desc(ab + 2 * k16 * lbo_b + a_plane, lbo_b, 128);
          const uint32_t acc = (cb | k16) ? 1u : 0u;
          wgmma_f16_n64(dh, a0, b0, acc);
          wgmma_f16_n64(dl, a0, b1, acc);
          wgmma_f16_n64(dl, a1, b0, 1u);
        }
        wg_commit();
        // keep one stage of MMAs in flight: the previous stage's operands are free once at most one group is pending
        wg_wait<1>();
        if (pws >= 0 && leader) { mbar_arrive(BAR(B_WEMPTY + pws)); mbar_arrive(BAR(B_AEMPTY + pas)); }
        pws = ws; pas = as;
        if (++ws == W_STAGES) { ws = 0; wph ^= 1; }
        if (++as == A_BUFS) { as = 0; aph ^= 1; }
      }
      wg_wait<0>();
      wg_fence_regs(dh);
      wg_fence_regs(dl);
      if (leader) { mbar_arrive(BAR(B_WEMPTY + pws)); mbar_arrive(BAR(B_AEMPTY + pas)); }
      // epilogue from the fragments: feature n = row, token m = column
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int n = cob * TMF + wg * 64 + w * 16 + g + 8 * i;
        const bool nok = n < Nf_;
        const float bias = (a.bias && nok) ? a.bias[n] : 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int m = tq * TNT + 8 * j + 2 * t4 + c;
            const int r = 4 * j + 2 * i + c;
            float val = fmaf(dl[r], LO_UNSCALE, dh[r]) + bias;
            if (act_ == ST2_ACT_GELU) val = gelu_erf(val);
            else if (act_ == ST2_ACT_TANH) val = tanhf(val);
            else if (act_ == ST2_ACT_GELU_TANH) val = gelu_tanh(val);
            if (nok && m < M_) {
              if (a.R) val += a.R[(long long)m * a.ldr + n];
              a.C[(long long)m * a.ldc + n] = val;
            }
          }
        }
      }
    }
  } else if (warp == NUM_CONS / 32) {
    // ================================================================ weight producer
    if (lane == 0) {
      int ws = 0, wph = 0;
      for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int cob = tile / n_tq;
        for (int cb = 0; cb < ncb; ++cb) {
          mbar_wait(BAR(B_WEMPTY + ws), wph ^ 1);
          const uint8_t* src = a.wtc + ((size_t)cob * ncb + cb) * W_STAGE_BYTES;
          mbar_expect_tx(BAR(B_WFULL + ws), W_STAGE_BYTES);
          bulk_g2s(sbase + SM_W + ws * W_STAGE_BYTES, src, W_STAGE_BYTES, BAR(B_WFULL + ws));
          if (++ws == W_STAGES) { ws = 0; wph ^= 1; }
        }
      }
    }
  } else {
    // ================================================================ activation stagers
    // thread -> token row (st >> 2) and 8-feature chunk (st & 3) of the 32-feature block: 8 contiguous floats = 2 x 128-bit
    // loads; the loads of block cb+1 are issued before block cb is converted (software pipeline).
    const int st = tid - (NUM_CONS + 32);
    const int row = st >> 2, kc = st & 3;
    const int K_ = a.K, M_ = a.M;
    int as = 0, aph = 0;
    if (a.planes) {
      // pre-split activations: every (token block, K block) stage is one contiguous image of the operand buffer
      if (st == 0) {
        for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
          const int tq = tile % n_tq;
          for (int cb = 0; cb < ncb; ++cb) {
            mbar_wait(BAR(B_AEMPTY + as), aph ^ 1);
            mbar_expect_tx(BAR(B_AFULL + as), PRE_STAGE_BYTES);
            bulk_g2s(sbase + SM_A + as * A_BUF_BYTES, a.planes + ((size_t)tq * ncb + cb) * PRE_STAGE_BYTES, PRE_STAGE_BYTES,
                     BAR(B_AFULL + as));
            if (++as == A_BUFS) { as = 0; aph ^= 1; }
          }
        }
      }
    } else
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      const int tq = tile % n_tq;
      const int m = tq * TNT + row;
      const bool mok = m < M_;
      const float* ar = a.A + (long long)(mok ? m : 0) * a.lda + kc * 8;
      const bool vec_ok = ((a.lda & 3) == 0) && ((reinterpret_cast<size_t>(a.A) & 15) == 0);
      float4 cur[2], nxt[2];
      auto load_blk = [&](int cb, float4 (&dst)[2]) {
        const int k0 = cb * KB + kc * 8;
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const int k = k0 + 4 * q;
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (mok) {
            if (vec_ok && k + 3 < K_) v = __ldg(reinterpret_cast<const float4*>(ar + cb * KB) + q);
            else {
              const float* p = ar + cb * KB + 4 * q;
              if (k < K_) v.x = __ldg(p);
              if (k + 1 < K_) v.y = __ldg(p + 1);
              if (k + 2 < K_) v.z = __ldg(p + 2);
              if (k + 3 < K_) v.w = __ldg(p + 3);
            }
          }
          dst[q] = v;
        }
      };
      load_blk(0, cur);
      bool in_range = true;
      for (int cb = 0; cb < ncb; ++cb) {
#pragma unroll
        for (int q = 0; q < 2; ++q)
          in_range &= in_fp16_range(cur[q].x) & in_fp16_range(cur[q].y) & in_fp16_range(cur[q].z) & in_fp16_range(cur[q].w);
        if (cb + 1 < ncb) load_blk(cb + 1, nxt);
        mbar_wait(BAR(B_AEMPTY + as), aph ^ 1);
        uint8_t* base = smem + SM_A + as * A_BUF_BYTES;
        uint32_t p0[4], p1[4];
        split2(cur[0].x, cur[0].y, p0[0], p1[0]);
        split2(cur[0].z, cur[0].w, p0[1], p1[1]);
        split2(cur[1].x, cur[1].y, p0[2], p1[2]);
        split2(cur[1].z, cur[1].w, p0[3], p1[3]);
        const size_t off = (size_t)(kc * RWP + row) * 16;
        *reinterpret_cast<uint4*>(base + off) = make_uint4(p0[0], p0[1], p0[2], p0[3]);
        *reinterpret_cast<uint4*>(base + A_PLANE_BYTES + off) = make_uint4(p1[0], p1[1], p1[2], p1[3]);
        fence_proxy_async();
        mbar_arrive(BAR(B_AFULL + as));
        if (++as == A_BUFS) { as = 0; aph ^= 1; }
#pragma unroll
        for (int q = 0; q < 2; ++q) cur[q] = nxt[q];
      }
      range_note(in_range);
    }
  }
}

// A [M,K] fp32 (row stride lda) -> pre-split operand stages [n_tq][ncb][2 planes][4 kc][128 rows][8 k] fp16, zero padded:
// done ONCE per activation matrix instead of once per 128-feature output block inside the GEMM
__global__ void linear_tc_split_kernel(const float* __restrict__ A, long long lda, int M, int K, int n_tq, int ncb,
                                       uint4* __restrict__ out) {
  const long long total = (long long)n_tq * ncb * 4 * TNT;
  const bool vec_ok = ((lda & 3) == 0) && ((reinterpret_cast<size_t>(A) & 15) == 0);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int row = (int)(i % TNT);
    long long r = i / TNT;
    const int kc = (int)(r % 4); r /= 4;
    const int cb = (int)(r % ncb);
    const int tq = (int)(r / ncb);
    const int m = tq * TNT + row, k0 = cb * KB + kc * 8;
    float x[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) x[j] = 0.f;
    if (m < M) {
      const float* p = A + (long long)m * lda + k0;
      if (vec_ok && k0 + 7 < K) {
        const float4 v0 = __ldg(reinterpret_cast<const float4*>(p)), v1 = __ldg(reinterpret_cast<const float4*>(p) + 1);
        x[0] = v0.x; x[1] = v0.y; x[2] = v0.z; x[3] = v0.w; x[4] = v1.x; x[5] = v1.y; x[6] = v1.z; x[7] = v1.w;
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (k0 + j < K) x[j] = __ldg(p + j);
      }
    }
    bool in_range = true;
#pragma unroll
    for (int j = 0; j < 8; ++j) in_range &= in_fp16_range(x[j]);
    range_note(in_range);
    uint32_t p0[4], p1[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) split2(x[2 * q], x[2 * q + 1], p0[q], p1[q]);
    const long long stage = (long long)tq * ncb + cb;
    uint4* hi = out + (stage * NPL * 4 + kc) * TNT + row;       // 16-byte units
    hi[0] = make_uint4(p0[0], p0[1], p0[2], p0[3]);
    hi[4 * TNT] = make_uint4(p1[0], p1[1], p1[2], p1[3]);
  }
}

// W [Nf,K] fp32 -> [n_cob][ncb][2 planes][4 kc][128 n][8 k] fp16
__global__ void linear_tc_weight_layout_kernel(const float* __restrict__ w, __half* __restrict__ out, int Nf, int K, int n_cob,
                                               int ncb) {
  const long long total = (long long)n_cob * ncb * NPL * 4 * TMF * 8;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long r = i;
    const int j = (int)(r % 8); r /= 8;
    const int col = (int)(r % TMF); r /= TMF;
    const int kc = (int)(r % 4); r /= 4;
    const int pl = (int)(r % NPL); r /= NPL;
    const int cb = (int)(r % ncb); r /= ncb;
    const int cob = (int)r;
    const int n = cob * TMF + col, k = cb * KB + kc * 8 + j;
    float v = 0.f;
    if (n < Nf && k < K) v = w[(long long)n * K + k];
    range_note(in_fp16_range(v));
    const __half h0 = __float2half_rn(v);
    const __half h1 = __float2half_rn((v - __half2float(h0)) * LO_SCALE);
    out[i] = pl == 0 ? h0 : h1;
  }
}

}  // namespace ltc
}  // namespace st2

using namespace st2;

extern "C" {

int st2_range_flag_fetch(int* flag_out) {
  ST2_REQUIRE(flag_out, "st2_range_flag_fetch", "bad args");
  int v = 0, zero = 0;
  cudaError_t e = cudaMemcpyFromSymbol(&v, ltc::g_range_flag, sizeof(int));     // synchronises with the device
  if (e == cudaSuccess && v) e = cudaMemcpyToSymbol(ltc::g_range_flag, &zero, sizeof(int));
  int vc = 0, va = 0;
  if (e == cudaSuccess) e = conv_tc_range_flag_fetch(&vc);                       // the tensor-core convs' flag (conv_tc.cu)
  if (e == cudaSuccess) e = attention_tc_range_flag_fetch(&va);                  // the tensor-core attention's (attention_tc.cu)
  if (e != cudaSuccess) { set_error("st2_range_flag_fetch", e); return (int)e; }
  *flag_out = v | vc | va;
  return 0;
}

long long st2_linear_tc_weight_bytes(int Nf, int K) {
  return (long long)cdiv(Nf, ltc::TMF) * cdiv(K, ltc::KB) * ltc::W_STAGE_BYTES;
}

int st2_linear_tc_weight_layout(const float* w, void* out, int Nf, int K, void* stream) {
  ST2_REQUIRE(w && out && Nf > 0 && K > 0, "st2_linear_tc_weight_layout", "bad args");
  ltc::linear_tc_weight_layout_kernel<<<1024, 256, 0, (cudaStream_t)stream>>>(w, (__half*)out, Nf, K, cdiv(Nf, ltc::TMF),
                                                                              cdiv(K, ltc::KB));
  ++g_launches;
  ST2_CHECK_LAUNCH("st2_linear_tc_weight_layout");
  return 0;
}

long long st2_linear_tc_split_bytes(int M, int K) {
  return (long long)cdiv(M, ltc::TNT) * cdiv(K, ltc::KB) * ltc::PRE_STAGE_BYTES;
}

int st2_linear_tc_split(const float* A, long long lda, int M, int K, void* planes, void* stream) {
  ST2_REQUIRE(A && planes && M > 0 && K > 0, "st2_linear_tc_split", "bad args");
  const int n_tq = cdiv(M, ltc::TNT), ncb = cdiv(K, ltc::KB);
  const long long total = (long long)n_tq * ncb * 4 * ltc::TNT;
  const int grid = (int)((total + 255) / 256 > 8192 ? 8192 : (total + 255) / 256);
  ltc::linear_tc_split_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(A, lda, M, K, n_tq, ncb, (uint4*)planes);
  ++g_launches;
  ST2_CHECK_LAUNCH("st2_linear_tc_split");
  return 0;
}

int st2_linear_tc(const float* A, long long lda, const void* wtc, const float* bias, const float* R, long long ldr, float* C,
                  long long ldc, int M, int Nf, int K, int act, void* stream) {
  return st2_linear_tc_pre(A, lda, nullptr, wtc, bias, R, ldr, C, ldc, M, Nf, K, act, stream);
}

int st2_linear_tc_pre(const float* A, long long lda, const void* planes, const void* wtc, const float* bias, const float* R,
                      long long ldr, float* C, long long ldc, int M, int Nf, int K, int act, void* stream) {
  ST2_REQUIRE((A || planes) && wtc && C && M > 0 && Nf > 0 && K > 0, "st2_linear_tc", "bad args");
  ltc::LinArgs a;
  a.planes = (const uint8_t*)planes;
  a.A = A; a.lda = lda; a.wtc = (const uint8_t*)wtc; a.bias = bias; a.R = R; a.ldr = ldr; a.C = C; a.ldc = ldc;
  a.M = M; a.Nf = Nf; a.K = K; a.act = act;
  const int n_tq = cdiv(M, ltc::TNT), n_cob = cdiv(Nf, ltc::TMF), ncb = cdiv(K, ltc::KB);
  const int ntiles = n_tq * n_cob;
  static PerDevice once;
  if (once.first()) {
    const int d = once.dev();
    cudaDeviceGetAttribute(&once.value[d], cudaDevAttrMultiProcessorCount, d);
    cudaFuncSetAttribute(ltc::linear_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ltc::SM_TOTAL);
  }
  const int num_sms = once.value[once.dev()];
  const int grid = ntiles < num_sms ? ntiles : num_sms;
  ltc::linear_tc_kernel<<<grid, ltc::THREADS, ltc::SM_TOTAL, (cudaStream_t)stream>>>(a, ncb, ntiles, n_tq);
  ++g_launches;
  ST2_CHECK_LAUNCH("st2_linear_tc");
  return 0;
}

}  // extern "C"
