// Tensor-core (wgmma) multi-head attention for the style denoiser and PL-BERT -- sm_90a.
//
//   out[b, n, h, :] = softmax_m( scale * q[b,n,h,:] . k[b,m,h,:] ) v[b,m,h,:]        head dimension 64, N <= 4096 keys
//   (Modules/diffusion/modules.py:523-535; transformers.AlbertModel's attention for PL-BERT, with a key-padding mask)
//
// The predicted integer durations are downstream, so both contractions run at fp32 accuracy on the 16-bit tensor
// cores with the recipe of linear_tc.cu: every operand is split into two fp16 planes, x = h + l * 2^-11 with h = fp16(x),
// l = fp16((x - h) * 2^11); a product is h*h (accumulator MAIN) + h*l + l*h (accumulator CORR, 2^11 too large, folded in
// by the reader with an exact 2^-11) -- three MMAs, two register accumulators, so the small terms never get truncated
// against the large running sum.
//
// One CTA = one warpgroup = (64 query rows, one head, one utterance):
//   S  = Q K^T   M = 64 queries, N = 128 keys per block, K = 64:  4 K-steps x 3 wgmmas, accumulators S_main / S_corr
//   P  = exp(scale * (S - rowmax))            a row lives in the four lanes of a quad: row max / row sum need two shuffles
//   O += P V     M = 64 queries, N = 64 (d), K = 128 keys:         8 K-steps x 3 wgmmas, accumulators O_main / O_corr
// Keys are processed in blocks of 128.  With more than one block the row maxima are found in a first sweep over S (QK^T is
// recomputed in the second sweep: cheap, and O never needs rescaling); N <= 128 takes a single sweep.
// Operands are staged into the K-major no-swizzle ("interleave") layout by the same threads: Q / K / P as
// [k-chunk][row][8 x fp16], V transposed on the fly to [key-chunk][d][8 keys] (lanes run over d: coalesced global reads).
// Range: the fp16 planes hold |q|, |k|, |v| < 65504; a larger (or NaN) staged value makes the output inf/NaN and raises a
// range flag (as linear_tc.cu does), which st2_range_flag_fetch() reports and clears.  Masked keys and padded query rows
// are staged as zeros and never raise it.  Every length must be >= 1: with no valid key the row sum is 0 and the output
// non-finite (the SIMT kernel st2_attention_ex gives NaN there too).
//
// Packed rows (PACKED = true, st2_attention_tc_packed): utterance b owns rows offsets[b] .. offsets[b+1] - 1 of q / k / v /
// out, concatenated without padding (varlen layout).  The kernel body is the same with N = n_b and the row base taken from
// the offsets: rows and keys are clamped to the utterance's last row, keys >= n_b are masked, query rows >= n_b (the next
// utterance's rows) are never stored, and a CTA whose query block starts at or beyond n_b exits.  With offsets[b] = b * N
// it does the arithmetic of the padded kernel with lengths = NULL.
#include <cuda_fp16.h>

#include <type_traits>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace st2 {
extern long long g_launches;

namespace atc {

using namespace st2::ptx;

constexpr int QB = 64, KB = 128, HD = 64;
constexpr int THREADS = 128;
constexpr float LO_SCALE = 2048.0f, LO_UNSCALE = 1.0f / 2048.0f;
constexpr int ROWS16 = 16;                                   // bytes per operand row chunk (8 fp16)
constexpr int Q_LBO = QB * ROWS16;                           // 1024: distance between 8-wide k-chunks of Q and of P
constexpr int K_LBO = KB * ROWS16;                           // 2048: distance between 8-wide k-chunks of K
constexpr int V_LBO = HD * ROWS16;                           // 1024: distance between 8-key chunks of V^T
constexpr int Q_PLANE = (HD / 8) * Q_LBO;                    // 8 KB
constexpr int K_PLANE = (HD / 8) * K_LBO;                    // 16 KB
constexpr int V_PLANE = (KB / 8) * V_LBO;                    // 16 KB
constexpr int P_PLANE = (KB / 8) * Q_LBO;                    // 16 KB
constexpr int SM_Q = 0, SM_K = SM_Q + 2 * Q_PLANE, SM_V = SM_K + 2 * K_PLANE, SM_P = SM_V + 2 * V_PLANE, SM_TOTAL = SM_P + 2 * P_PLANE;

__device__ int g_range_flag = 0;
constexpr float FP16_MAX = 65504.0f;

struct Args {
  const float* q; long long q_ld;
  const float* k; const float* v; long long kv_ld;
  float* out; long long out_ld;
  const int* lengths;      // key lengths [B] or NULL (padded layout)
  int N, H;
  float scale;
  const int* offsets;      // row offsets [B + 1] (packed layout)
};

__device__ __forceinline__ void split2(float x0, float x1, uint32_t& p0, uint32_t& p1) {
  const __half2 h = __floats2half2_rn(x0, x1);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn((x0 - hf.x) * LO_SCALE, (x1 - hf.y) * LO_SCALE);
  p0 = *reinterpret_cast<const uint32_t*>(&h);
  p1 = *reinterpret_cast<const uint32_t*>(&l);
}
// 8 fp32 -> one 16-byte row of each plane; with CHECK, in_range stays true while every value fits the fp16 planes (false
// for NaN)
template <bool CHECK = true>
__device__ __forceinline__ void store_row8(uint8_t* plane0, int plane_bytes, size_t off, const float (&x)[8], bool& in_range) {
  uint32_t a[4], b[4];
  if (CHECK) {
#pragma unroll
    for (int i = 0; i < 8; ++i) in_range &= fabsf(x[i]) < FP16_MAX;
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) split2(x[2 * i], x[2 * i + 1], a[i], b[i]);
  *reinterpret_cast<uint4*>(plane0 + off) = make_uint4(a[0], a[1], a[2], a[3]);
  *reinterpret_cast<uint4*>(plane0 + plane_bytes + off) = make_uint4(b[0], b[1], b[2], b[3]);
}
__device__ __forceinline__ void load8(const float* p, float (&x)[8]) {
  const float4 v0 = __ldg(reinterpret_cast<const float4*>(p)), v1 = __ldg(reinterpret_cast<const float4*>(p + 4));
  x[0] = v0.x; x[1] = v0.y; x[2] = v0.z; x[3] = v0.w; x[4] = v1.x; x[5] = v1.y; x[6] = v1.z; x[7] = v1.w;
}

template <bool PACKED>
__global__ void __launch_bounds__(THREADS, 1) attention_tc_kernel(const Args a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
  const uint32_t sbase = smem_u32(smem);
  const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int N = PACKED ? a.offsets[b + 1] - a.offsets[b] : a.N;     // rows of this utterance
  if (PACKED && qb * QB >= N) return;
  const int klen = PACKED ? N : (a.lengths ? min(a.lengths[b], N) : N);
  const int nkb = max(1, (klen + KB - 1) / KB);
  const long long rowbase = PACKED ? (long long)a.offsets[b] : (long long)b * N;
  bool in_range = true;

  // ---- stage Q (once): thread t -> query row t % 64, four 8-wide chunks of d
  {
    const int r = tid & 63, row = qb * QB + r;
    const float* qr = a.q + (rowbase + min(row, N - 1)) * a.q_ld + h * HD;
#pragma unroll
    for (int c = (tid >> 6) * 4; c < (tid >> 6) * 4 + 4; ++c) {
      float x[8];
      load8(qr + 8 * c, x);
      if (row >= N) {
#pragma unroll
        for (int j = 0; j < 8; ++j) x[j] = 0.f;
      }
      store_row8(smem + SM_Q, Q_PLANE, (size_t)c * Q_LBO + (size_t)r * ROWS16, x, in_range);
    }
  }
  // thread t -> key kb*128 + t.  check = std::true_type range-checks the keys; sweep 1 stages the same keys as sweep 2 and
  // passes std::false_type
  auto stage_k = [&](int kb, auto check) {
    const int key = kb * KB + tid;
    const float* kr = a.k + (rowbase + min(key, N - 1)) * a.kv_ld + h * HD;
#pragma unroll
    for (int c = 0; c < HD / 8; ++c) {
      float x[8];
      load8(kr + 8 * c, x);
      if (key >= klen) {
#pragma unroll
        for (int j = 0; j < 8; ++j) x[j] = 0.f;
      }
      store_row8<decltype(check)::value>(smem + SM_K, K_PLANE, (size_t)c * K_LBO + (size_t)tid * ROWS16, x, in_range);
    }
  };
  auto stage_v = [&](int kb) {      // thread t -> d = t % 64, key chunks (t / 64) * 8 .. + 7; V^T rows of 8 keys
    const int d = tid & 63, c0 = (tid >> 6) * 8;
#pragma unroll 2
    for (int c = c0; c < c0 + 8; ++c) {
      float x[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int key = kb * KB + c * 8 + i;
        x[i] = key < klen ? __ldg(a.v + (rowbase + key) * a.kv_ld + h * HD + d) : 0.f;
      }
      store_row8(smem + SM_V, V_PLANE, (size_t)c * V_LBO + (size_t)d * ROWS16, x, in_range);
    }
  };
  float sm[64], sc[64];             // S fragment: row 16 w + g + 8 i, key 8 j + 2 t4 + c  ->  index 4 j + 2 i + c
  auto compute_s = [&]() {          // S_main = Qh Kh^T ; S_corr = Qh Kl'^T + Ql' Kh^T
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < HD / 16; ++ks) {
      const uint64_t qh = make_desc(sbase + SM_Q + ks * 2 * Q_LBO, Q_LBO, 128), ql = make_desc(sbase + SM_Q + Q_PLANE + ks * 2 * Q_LBO, Q_LBO, 128);
      const uint64_t kh = make_desc(sbase + SM_K + ks * 2 * K_LBO, K_LBO, 128), kl = make_desc(sbase + SM_K + K_PLANE + ks * 2 * K_LBO, K_LBO, 128);
      wgmma_f16_n128(sm, qh, kh, ks ? 1u : 0u);
      wgmma_f16_n128(sc, qh, kl, ks ? 1u : 0u);
      wgmma_f16_n128(sc, ql, kh, 1u);
    }
    wg_commit();
    wg_wait<0>();
    wg_fence_regs(sm);
    wg_fence_regs(sc);
#pragma unroll
    for (int r = 0; r < 64; ++r) sm[r] = fmaf(sc[r], LO_UNSCALE, sm[r]) * a.scale;
  };
  float om[32], oc[32];
  auto compute_o = [&](bool first) {  // O_main += Ph Vh ; O_corr += Ph Vl' + Pl' Vh
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < KB / 16; ++ks) {
      const uint32_t po = (uint32_t)ks * 2 * Q_LBO, vo = (uint32_t)ks * 2 * V_LBO;
      const uint64_t ph = make_desc(sbase + SM_P + po, Q_LBO, 128), pl = make_desc(sbase + SM_P + P_PLANE + po, Q_LBO, 128);
      const uint64_t vh = make_desc(sbase + SM_V + vo, V_LBO, 128), vl = make_desc(sbase + SM_V + V_PLANE + vo, V_LBO, 128);
      const uint32_t acc = (first && ks == 0) ? 0u : 1u;
      wgmma_f16_n64(om, ph, vh, acc);
      wgmma_f16_n64(oc, ph, vl, acc);
      wgmma_f16_n64(oc, pl, vh, 1u);
    }
    wg_commit();
    wg_wait<0>();
    wg_fence_regs(om);
    wg_fence_regs(oc);
  };
#pragma unroll
  for (int r = 0; r < 32; ++r) { om[r] = 0.f; oc[r] = 0.f; }

  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  auto row_max = [&](int kb) {
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int c = 0; c < 2; ++c)
          if (kb * KB + 8 * j + 2 * t4 + c < klen) m[i] = fmaxf(m[i], sm[4 * j + 2 * i + c]);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      m[i] = fmaxf(m[i], __shfl_xor_sync(0xffffffffu, m[i], 1));
      m[i] = fmaxf(m[i], __shfl_xor_sync(0xffffffffu, m[i], 2));
    }
  };
  const bool two_pass = nkb > 1;
  // ---- sweep 1 (only when there are several key blocks): row maxima
  if (two_pass) {
    for (int kb = 0; kb < nkb; ++kb) {
      stage_k(kb, std::false_type{});
      fence_proxy_async();
      __syncthreads();
      compute_s();
      row_max(kb);
      __syncthreads();       // K buffer free
    }
  }
  // ---- sweep 2: P and O
  for (int kb = 0; kb < nkb; ++kb) {
    stage_k(kb, std::true_type{});
    stage_v(kb);
    fence_proxy_async();
    __syncthreads();
    compute_s();
    if (!two_pass) row_max(kb);
    // P planes: this thread's two keys (8 j + 2 t4, + 1) of rows 16 w + g + 8 i -> 4 bytes of the row's 16-byte line in chunk j
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float p[2];
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          p[c] = (kb * KB + 8 * j + 2 * t4 + c < klen) ? expf(sm[4 * j + 2 * i + c] - m[i]) : 0.f;
          l[i] += p[c];
        }
        uint32_t p0, p1;
        split2(p[0], p[1], p0, p1);
        const size_t off = (size_t)j * Q_LBO + (size_t)(16 * w + g + 8 * i) * ROWS16 + 4 * t4;
        *reinterpret_cast<uint32_t*>(smem + SM_P + off) = p0;
        *reinterpret_cast<uint32_t*>(smem + SM_P + P_PLANE + off) = p1;
      }
    fence_proxy_async();
    __syncthreads();
    compute_o(kb == 0);
    __syncthreads();         // K / V / P buffers free
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    l[i] += __shfl_xor_sync(0xffffffffu, l[i], 1);
    l[i] += __shfl_xor_sync(0xffffffffu, l[i], 2);
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int row = qb * QB + 16 * w + g + 8 * i;
    const float inv = 1.0f / l[i];
    float* orow = a.out + (rowbase + min(row, N - 1)) * a.out_ld + h * HD;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int r = 4 * j + 2 * i;
      const float2 o = make_float2(fmaf(oc[r], LO_UNSCALE, om[r]) * inv, fmaf(oc[r + 1], LO_UNSCALE, om[r + 1]) * inv);
      if (row < N) *reinterpret_cast<float2*>(orow + 8 * j + 2 * t4) = o;
    }
  }
  if (!in_range) atomicExch(&g_range_flag, 1);
}

}  // namespace atc

cudaError_t attention_tc_range_flag_fetch(int* flag) {
  int v = 0, zero = 0;
  cudaError_t e = cudaMemcpyFromSymbol(&v, atc::g_range_flag, sizeof(int));   // synchronises with the device
  if (e == cudaSuccess && v) e = cudaMemcpyToSymbol(atc::g_range_flag, &zero, sizeof(int));
  *flag = v;
  return e;
}

}  // namespace st2

using namespace st2;

extern "C" {

int st2_attention_tc_supported(long long q_ld, long long kv_ld, long long out_ld, int D) {
  return D == atc::HD && (q_ld % 4) == 0 && (kv_ld % 4) == 0 && (out_ld % 4) == 0;
}

int st2_attention_tc(const float* q, long long q_ld, const float* k, const float* v, long long kv_ld, float* out, long long out_ld,
                     const int* lengths, int B, int N, int H, int D, float scale, void* stream) {
  ST2_REQUIRE(q && k && v && out && B > 0 && N > 0 && H > 0, "st2_attention_tc", "bad args");
  ST2_REQUIRE(st2_attention_tc_supported(q_ld, kv_ld, out_ld, D), "st2_attention_tc", "head_features must be 64, row strides multiples of 4");
  ST2_REQUIRE(((reinterpret_cast<size_t>(q) | reinterpret_cast<size_t>(k) | reinterpret_cast<size_t>(v) | reinterpret_cast<size_t>(out)) & 15) == 0,
              "st2_attention_tc", "pointers must be 16-byte aligned");
  static bool attr_done[64] = {false};
  int dev = 0;
  cudaGetDevice(&dev);
  dev &= 63;
  if (!attr_done[dev]) {
    cudaFuncSetAttribute(atc::attention_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, atc::SM_TOTAL);
    attr_done[dev] = true;
  }
  atc::Args a;
  a.q = q; a.q_ld = q_ld; a.k = k; a.v = v; a.kv_ld = kv_ld; a.out = out; a.out_ld = out_ld; a.lengths = lengths; a.offsets = nullptr;
  a.N = N; a.H = H; a.scale = scale;
  dim3 grid(cdiv(N, atc::QB), H, B);
  atc::attention_tc_kernel<false><<<grid, atc::THREADS, atc::SM_TOTAL, (cudaStream_t)stream>>>(a);
  ++g_launches;
  ST2_CHECK_LAUNCH("st2_attention_tc");
  return 0;
}

int st2_attention_tc_packed(const float* q, long long q_ld, const float* k, const float* v, long long kv_ld, float* out,
                            long long out_ld, const int* offsets, int B, int max_len, int H, int D, float scale, void* stream) {
  ST2_REQUIRE(q && k && v && out && offsets && B > 0 && max_len > 0 && H > 0, "st2_attention_tc_packed", "bad args");
  ST2_REQUIRE(st2_attention_tc_supported(q_ld, kv_ld, out_ld, D), "st2_attention_tc_packed",
              "head_features must be 64, row strides multiples of 4");
  ST2_REQUIRE(((reinterpret_cast<size_t>(q) | reinterpret_cast<size_t>(k) | reinterpret_cast<size_t>(v) | reinterpret_cast<size_t>(out)) & 15) == 0,
              "st2_attention_tc_packed", "pointers must be 16-byte aligned");
  static bool attr_done[64] = {false};
  int dev = 0;
  cudaGetDevice(&dev);
  dev &= 63;
  if (!attr_done[dev]) {
    cudaFuncSetAttribute(atc::attention_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, atc::SM_TOTAL);
    attr_done[dev] = true;
  }
  atc::Args a;
  a.q = q; a.q_ld = q_ld; a.k = k; a.v = v; a.kv_ld = kv_ld; a.out = out; a.out_ld = out_ld; a.lengths = nullptr; a.offsets = offsets;
  a.N = max_len; a.H = H; a.scale = scale;
  dim3 grid(cdiv(max_len, atc::QB), H, B);
  atc::attention_tc_kernel<true><<<grid, atc::THREADS, atc::SM_TOTAL, (cudaStream_t)stream>>>(a);
  ++g_launches;
  ST2_CHECK_LAUNCH("st2_attention_tc_packed");
  return 0;
}

}  // extern "C"
