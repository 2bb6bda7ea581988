// Tensor-core (wgmma) implicit-GEMM Conv1d for the vocoder's AdaIN ResBlocks -- sm_90a.
//
//   D[co (M=128), t (N=128)] = sum_{tap} sum_{ci} W_tap[co, ci] * z[ci, t + tap*dil - pad],   z = snake/lrelu(a*x+b)
//
// Precision recipes (decided with the CPU oracle by emulation, DESIGN.md "precision"; tools/emulate_precision.py):
// operands are pre-scaled by exact powers of two, w' = w * 2^12 and z' = z * 2^6 (the epilogue multiplies by 2^-18), so
// that the fp16 "high" planes h = fp16(.) and the remainders l = (.) - h stay far away from fp16's subnormal range.
//   ST2_TC_FAST  (vocoder / decoder, 2 MMAs per product):
//       D0 += h(w') h(z')                                   one f16 wgmma   (K = 16 channels)
//       D1 += [l(w')*2^4 | h(w')*2^-8] . [h(z')*2^-4 ; l(z')*2^8]   one e4m3 wgmma (K = 32 = both corrections)
//     the correction terms are 2^-11 of the leading one and e4m3 keeps 4 of their bits: ~15-16 operand bits in total.
//     The e4m3 wgmma keeps fewer accumulator bits than the f16 one, so the corrections get their own accumulator
//     (folded in by the epilogue): added into D0 they would round the large running sum.
//   ST2_TC_ACCURATE (F0/N predictor: its F0 curve is integrated into a phase of 1e4..1e6 rad downstream):
//       D0 += h(w') h(z');   D1 += h(w') l(z')*2^8 + l(w')*2^8 h(z')      three f16 wgmmas, TWO register accumulators
//     (the tensor core truncates when it adds into an accumulator: keeping the small terms out of the big running sum
//     brings the error to the fp32-SIMT level, see linear_tc.cu); the epilogue folds D1 in with an exact 2^-8.
//   ST2_TC_F16X3: the accurate planes accumulated into ONE accumulator (3 MMAs; kept for A/B tests).
//
// Mapping:
//  * A operand = weights  [64 co x 16 ci] per consumer warpgroup, K-major, no-swizzle "interleave" layout (8-row x 16-byte
//    core matrices, rows contiguous at 16 B pitch).  Pre-arranged in HBM so that one pipeline stage (taps, 16 ci, both
//    planes) is ONE contiguous block moved by a single 1-D TMA bulk copy (cp.async.bulk) that signals an mbarrier.
//  * B operand = activations [128 t x 16 ci], K-major, same interleave layout: for each K chunk the frame window is a
//    column of 16-byte rows, so a conv tap is just a descriptor start address shifted by tap*dil rows (16 B
//    granularity) -- the window is staged ONCE per 16-channel block (AdaIN affine + Snake/LeakyReLU + plane split
//    fused into the staging) and re-used by all K taps.
//  * Raw fp32 frame windows travel HBM -> shared memory as 16-byte cp.async copies of the ALIGNED superset window of
//    every channel row (rows of odd length start at any 4-byte phase; the phase becomes a per-channel offset of the
//    scalar shared-memory reads of the conversion), a ring of four blocks per SM.
//  * D accumulators live in the registers of two consumer warpgroups (output channels 0-63 / 64-127 of the tile, 128 frames
//    each: m64n128 MMAs); the epilogue fuses bias, residual, MRF accumulation and the InstanceNorm partial statistics
//    (count, mean, M2) exactly like the SIMT kernel.  Its global traffic goes through a shared-memory transpose (SM_SLOT,
//    epi_rows: whole channel rows per warp), its statistics work on the fragments.  A 128-frame tile writes two partials, one per
//    64 frames, so the statistics layout does not depend on the tile width.  Output positions are contiguous
//    (y_tstride = 1, no reflection duplicate): a ConvTranspose1d runs its phases into phase-major scratch rows that
//    convT_interleave_kernel interleaves (st2_conv_transpose1d_tc2).
//  * Warp roles in whole warpgroups: warps 0-7 = consumers (wgmma + epilogue), warp 8 = weight TMA producer, warps 9-14 =
//    activation stagers, warp 15 idle.  setmaxnreg moves registers from warpgroups 2-3 to the consumers (arithmetic at
//    THREADS below).  Persistent CTAs (one per SM) loop over tiles.
//
// TWO kernels share this pipeline (barriers, producer roles and the consumer K-loop, device functions below): the
// channel-major conv1d_tc_kernel described above and the TIME-MAJOR conv1d_tct_kernel further down (FAST recipe,
// Cout <= 128: frames on the MMA's M axis, output channels on N; its header comment has the mapping).  They differ in the
// MMAs of one tap, the taps per weight stage and their epilogues.  One layout kernel writes the weight blocks of both, for
// a conv and for the phases of a ConvTranspose1d.
#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace st2 {
extern long long g_launches;

namespace tc {

constexpr int MODE_FAST = ST2_TC_FAST, MODE_ACC = ST2_TC_ACCURATE, MODE_X3 = ST2_TC_F16X3;

constexpr int TN = 128;                         // frames per tile (wgmma N of the channel-major kernel; 2 x M = 64 of the time-major one)
constexpr int TP = 64;                          // frames per InstanceNorm statistics partial: a tile writes TN / TP of them
constexpr int TM = 128;                        // output channels per tile of the channel-major kernel (two warpgroups of M = 64)
constexpr int CB = 16;                          // input channels per pipeline block (one UMMA K step of the fp16 planes)
constexpr int KCB = CB / 8;                     // 16-byte K chunks per plane and block
constexpr int W_PLANE_BYTES = KCB * TM * 16;    // 4 KB
constexpr int W_STEP_BYTES = 2 * W_PLANE_BYTES; // one (16 ci, tap) step: plane 0 (fp16 high) | plane 1 (fp8 corrections or fp16 low) = 8 KB
constexpr int TPS = 2;                          // taps per pipeline stage: one wait / one commit / one bulk copy per 2 taps (the
                                                // per-stage handshake of the two single-thread roles costs ~300 cycles, as much
                                                // as the 2 MMAs of one tap)
constexpr int W_STAGE_BYTES = TPS * W_STEP_BYTES;  // 16 KB
constexpr int W_STAGES = 3;                     // 48 KB (6 taps) of weights in flight per SM
constexpr int RW_MAX = 312;                     // TN + (K-1)*dil rounded up to 8, max: (K-1)*dil <= 184 (the models need <= 50)
constexpr int RWP_MAX = RW_MAX + 2;             // chunk pitch in rows of the staged planes
constexpr int ACT_PLANE_BYTES = KCB * RWP_MAX * 16;  // one plane of one 16-channel block
constexpr int ACT_BUF_BYTES = 2 * ACT_PLANE_BYTES;
constexpr int RAW_STAGES = 4;                   // cp.async ring of raw fp32 frame windows: 3 blocks (63 KB) in flight per SM
constexpr int RAW_CHUNKS = 84;                  // 16-byte chunks copied per channel row: 336 floats >= RW_MAX + 3
constexpr int RAW_PITCH = 336;                  // floats per channel row of a raw block: pitch = 64 bytes mod 128.  The 32 cp.async
                                                // destinations of a warp cover chunk runs of 12 (one row each) at row offsets that
                                                // alternate between 0 and 64 bytes mod 128, which puts exactly 4 of them on every
                                                // 16-byte bank group (ncu, earlier layout: 3x excess shared-memory wavefronts of the
                                                // LDGSTS at a pitch of 1280 bytes; the shared-memory data pipe is shared with the
                                                // tensor core's operand reads)
constexpr int RAW_BYTES = CB * RAW_PITCH * 4;   // 21 KB
constexpr int CIN_PAD_MAX = 1120;
// Warp roles in whole warpgroups, so that each can set its own register budget (setmaxnreg):
//   warpgroups 0-1 (warps 0-7): consumers, 64 frames x Cout (time-major) or 64 channels x 128 frames (channel-major) each
//   warp 8: weight TMA producer; warps 9-14: activation stagers; warp 15: idle
// The launch allocates 512 threads x 128 registers = 64 K, the whole register file.  The producer warpgroups give
// 2 x 128 x (128 - 64) registers back, which the consumers take: 2 x 128 x 192 + 2 x 128 x 64 = 65536.  A consumer holds two
// 64-register fp32 accumulators (FAST / ACCURATE; 64 x 128 per warpgroup).
constexpr int NUM_CONS = 256;                   // two consumer warpgroups
constexpr int NUM_STAGERS = 192;                // 6 warps: an even count (the conversion mapping pairs warps over the K chunks)
constexpr int ST_PER_CH = NUM_STAGERS / CB;     // issue mapping: threads per channel row of a raw block
constexpr int ROWS_PER_PASS = (NUM_STAGERS / 64) * 32;  // conversion mapping: rows covered per pass
constexpr int ST0 = NUM_CONS + 32;              // first stager thread (warp 8 is the weight producer)
constexpr int THREADS = 512;                    // 4 warpgroups
constexpr int REG_LAUNCH = 128, REG_CONS = 192, REG_AUX = 64;
static_assert(ST0 + NUM_STAGERS <= THREADS && THREADS * REG_LAUNCH <= 65536, "thread roles");
static_assert(NUM_CONS * REG_CONS + (THREADS - NUM_CONS) * REG_AUX <= THREADS * REG_LAUNCH, "register budget");

// power-of-two operand scaling (exact): w' = w * 2^12, z' = z * 2^6; accumulators hold 2^18 x the convolution
constexpr float W_SCALE = 4096.0f, X_SCALE = 64.0f, D_UNSCALE = 1.0f / (4096.0f * 64.0f);
constexpr float ACC_LO_SCALE = 256.0f, ACC_LO_UNSCALE = 1.0f / 256.0f;            // ST2_TC_ACCURATE low planes
constexpr float F8_WLO = 16.0f, F8_WHI = 1.0f / 256.0f, F8_XHI = 1.0f / 16.0f, F8_XLO = 256.0f;  // e4m3 correction operands

// Range guard (as in linear_tc.cu, with a flag of its own): the fp16 high planes hold |z'| = 64 |z| and |w'| = 4096 |w| below
// 65504, i.e. |z| < 1023.5 after the prologue and |w| < 16; beyond that (or for NaN) the conv writes inf/NaN.  Every stager
// thread keeps one predicate over the rows it converts and raises the flag once; the weight layout kernel checks the weights.
// st2_range_flag_fetch() reports and clears it.  Not covered: the FAST recipe's e4m3 corrections saturate (silently, to
// +-448) from |z| of about 64 on (DESIGN.md "Precision recipes").
__device__ int g_range_flag = 0;
constexpr float FP16_MAX = 65504.0f;

constexpr int SM_W = 0;
constexpr int SM_ACT = SM_W + W_STAGES * W_STAGE_BYTES;
constexpr int SM_RAW = SM_ACT + 2 * ACT_BUF_BYTES;
constexpr int SM_COEF = SM_RAW + RAW_STAGES * RAW_BYTES;
constexpr int SM_EPI = SM_COEF + 4 * CIN_PAD_MAX * 4;   // per-channel prologue coefficients of the current utterance (4 x 1120 floats)
constexpr int TCT_NC_MAX = 128;                   // output channels of the time-major kernel, max
constexpr int SM_SLOT = SM_EPI + 2 * 4 * TCT_NC_MAX * 4;   // time-major statistics scratch [2 warpgroups][4 warps][128 channels]
// Epilogue transpose slot: SLOT_FLOATS floats per consumer warpgroup, one slice of the tile's outputs as [channel][frame]
// rows (64 channels x 64 frames time-major, 32 channels x 128 frames channel-major; slot_index).  The fragments go in, each
// warp then owns whole channel rows, so that one load or store instruction covers 32 consecutive frames of one channel
// (128 contiguous bytes) instead of 4 or 8 short runs of the wgmma fragment mapping.
constexpr int SLOT_FLOATS = 4096;
constexpr int SM_BAR = SM_SLOT + 2 * SLOT_FLOATS * 4;
constexpr int SM_TOTAL = SM_BAR + 512;
static_assert(RAW_CHUNKS % ST_PER_CH == 0 && NUM_STAGERS % 64 == 0 && NUM_STAGERS % CB == 0, "stager mappings");
static_assert(RAW_CHUNKS * 4 >= RW_MAX + 3 && RAW_PITCH >= RAW_CHUNKS * 4 && (RAW_PITCH * 4) % 128 == 64, "raw window rows");
static_assert(SM_TOTAL <= 232448, "shared memory budget (227 KB per CTA)");

// barrier slots (8 B each) inside SM_BAR
constexpr int B_WFULL = 0, B_WEMPTY = W_STAGES, B_AFULL = 2 * W_STAGES, B_AEMPTY = B_AFULL + 2, B_COUNT = B_AFULL + 4;
static_assert(8 * B_COUNT + 8 <= 512, "barrier area");

// Timing-experiment switches (tools/conv_tc_shapes.py --ablate; results are WRONG when any is set; 0 in production):
//   4 = stagers skip the conversion (stale operands), 16 = no weight copies, 32 = no raw activation copies
__device__ int g_dbg = 0;

using namespace st2::ptx;

struct TileCoord {
  int b, cob, tq;
};
__device__ __forceinline__ TileCoord tile_coord(int tile, int n_tq, int n_cob) {
  TileCoord c;
  c.tq = tile % n_tq;
  const int r = tile / n_tq;
  c.cob = r % n_cob;
  c.b = r / n_cob;
  return c;
}

__device__ __forceinline__ uint32_t h2_bits(__half2 h) { return *reinterpret_cast<uint32_t*>(&h); }

// Warp index broadcast from lane 0, so that ptxas can prove it warp-uniform.  With a plain tid >> 5 it treats the consumer
// branch of the role dispatch as divergent and serializes every wgmma behind a full drain (ptxas C7520), which also
// defeats the one-group-in-flight pipeline of the consumer loops.
__device__ __forceinline__ int warp_uniform(int tid) { return __shfl_sync(0xffffffffu, tid >> 5, 0); }

// ---------------------------------------------------------------------------------------------
// Stager inner work for one frame row (8 channels of one K chunk): AdaIN affine + activation (coefficients carry the
// 2^6 operand scale) + plane split + shared-memory stores.  Templated on activation and recipe: no branches per element.
//   p0 row: 8 fp16 (16 B) at chunk kc.   p1 row: MODE_FAST -> 16 e4m3 bytes at chunk kc: [h(z')/16 | l(z')*256] of the 8 channels
//   (the order of the 32 K elements of the correction MMA is free as long as the weights use the same one: one conflict-free
//   128-bit store per row instead of two 64-bit halves);  otherwise 8 fp16 low-plane values (16 B) at chunk kc.
template <int ACT, int MODE>
__device__ __forceinline__ void stage_row(const float (&x)[8], const float (&pa)[8], const float (&pb)[8], const float (&al)[8],
                                          const float (&ia)[8], float slope, bool inb, uint8_t* p0, uint8_t* p1, int kc, int r,
                                          int RWP, bool& in_range) {
  float v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    float z = fmaf(x[j], pa[j], pb[j]);          // = 64 * (a*x + b)
    if (ACT == ST2_ACT_SNAKE) {
      const float sn = __sinf(al[j] * z);        // al = alpha / 64
      z = fmaf(ia[j], sn * sn, z);               // ia = 64 / alpha
    } else if (ACT == ST2_ACT_LRELU) {
      z = z > 0.f ? z : z * slope;
    }
    v[j] = inb ? z : 0.f;  // zero padding applies AFTER the activation
    in_range = in_range && fabsf(v[j]) < FP16_MAX;   // false for NaN too
  }
  uint32_t hp[4];
  float lo[8];
  __half2 h2[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    h2[q] = __floats2half2_rn(v[2 * q], v[2 * q + 1]);
    hp[q] = h2_bits(h2[q]);
    const float2 hf = __half22float2(h2[q]);
    lo[2 * q] = v[2 * q] - hf.x;
    lo[2 * q + 1] = v[2 * q + 1] - hf.y;
  }
  *reinterpret_cast<uint4*>(p0 + (size_t)(kc * RWP + r) * 16) = make_uint4(hp[0], hp[1], hp[2], hp[3]);
  if (MODE == MODE_FAST) {
    uint32_t h8[2], l8[2];
    const __half2 sc = __floats2half2_rn(F8_XHI, F8_XHI);
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const __half2 a0 = __hmul2(h2[2 * q], sc), a1 = __hmul2(h2[2 * q + 1], sc);
      const uint32_t e0 = __nv_cvt_halfraw2_to_fp8x2(*reinterpret_cast<const __half2_raw*>(&a0), __NV_SATFINITE, __NV_E4M3);
      const uint32_t e1 = __nv_cvt_halfraw2_to_fp8x2(*reinterpret_cast<const __half2_raw*>(&a1), __NV_SATFINITE, __NV_E4M3);
      h8[q] = e0 | (e1 << 16);
      const uint32_t f0 = __nv_cvt_float2_to_fp8x2(make_float2(lo[4 * q] * F8_XLO, lo[4 * q + 1] * F8_XLO), __NV_SATFINITE, __NV_E4M3);
      const uint32_t f1 = __nv_cvt_float2_to_fp8x2(make_float2(lo[4 * q + 2] * F8_XLO, lo[4 * q + 3] * F8_XLO), __NV_SATFINITE, __NV_E4M3);
      l8[q] = f0 | (f1 << 16);
    }
    *reinterpret_cast<uint4*>(p1 + (size_t)(kc * RWP + r) * 16) = make_uint4(h8[0], h8[1], l8[0], l8[1]);
  } else {
    const float ls = (MODE == MODE_ACC) ? ACC_LO_SCALE : 1.0f;
    uint32_t lp[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) lp[q] = h2_bits(__floats2half2_rn(lo[2 * q] * ls, lo[2 * q + 1] * ls));
    *reinterpret_cast<uint4*>(p1 + (size_t)(kc * RWP + r) * 16) = make_uint4(lp[0], lp[1], lp[2], lp[3]);
  }
}

// Weight producer role (one lane of warp 8): one 1-D TMA bulk copy per pipeline stage = up to `tps` consecutive taps of one
// 16-channel block (contiguous in the [cob][cb][tap] layout), `wstep` bytes per (16 channels, tap) step.
__device__ __forceinline__ void weight_producer_role(const uint4* __restrict__ wtc, const uint32_t sbase, const uint32_t bar0,
                                                     const int ncb, const int K, const int wstep, const int tps, const int stage_bytes,
                                                     const int ntiles, const int n_tq, const int n_cob) {
  auto BAR = [&](int i) { return bar0 + 8u * i; };
  const int dbg_p = g_dbg;
  int ws = 0, wph = 0;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const TileCoord tc_ = tile_coord(tile, n_tq, n_cob);
    const uint8_t* src = reinterpret_cast<const uint8_t*>(wtc) + (size_t)tc_.cob * ncb * K * wstep;
    for (int cb = 0; cb < ncb; ++cb) {
      for (int tap0 = 0; tap0 < K; tap0 += tps) {
        const uint32_t bytes = (uint32_t)(min(tps, K - tap0) * wstep);
        mbar_wait(BAR(B_WEMPTY + ws), wph ^ 1);
        if (dbg_p & 16) {
          mbar_arrive(BAR(B_WFULL + ws));                    // timing experiment: no weight traffic
        } else {
          mbar_expect_tx(BAR(B_WFULL + ws), bytes);
          bulk_g2s(sbase + SM_W + ws * stage_bytes, src, bytes, BAR(B_WFULL + ws));
        }
        src += bytes;
        if (++ws == W_STAGES) { ws = 0; wph ^= 1; }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Activation stager role (warps ST0/32 .. ST0/32 + NUM_STAGERS/32 - 1), shared by the channel-major and the time-major kernel: both
// read the staged window through the same K-major no-swizzle layout (one 16-byte row per frame and K chunk).
template <int MODE>
__device__ __forceinline__ void stager_role(const st2_conv_args& a, uint8_t* smem, const uint32_t sbase, const uint32_t bar0,
                                            const int ncb, const int RW, const int ntiles, const int n_tq, const int n_cob,
                                            const int tid, const int warp, const int lane) {
  const int RWP = RW + 2;
  auto BAR = [&](int i) { return bar0 + 8u * i; };
  // ================================================================ activation stagers
  // Raw fp32 frame windows travel HBM -> shared memory with 16-byte cp.async copies (no registers held while in
  // flight): a ring of RAW_STAGES 16-channel blocks keeps ~60 KB per SM outstanding, which is what it takes to cover
  // HBM latency.  Rows of the activation tensor start at any 4-byte phase (odd row lengths), so each channel row
  // copies the 16-byte ALIGNED superset of its window; the phase (0..3 floats) is re-derived by the conversion.
  // Chunks outside the tensor are zero-filled (src-size 0), the chunk that crosses the end of the tensor is
  // trimmed; nothing before the 16-byte aligned start of the tensor's allocation is ever touched.
  const int st = tid - ST0;  // 0..NUM_STAGERS-1
  const int Lin_ = a.Lin, pre_act_ = a.pre_act, Cin_ = a.Cin;
  const float slope_ = a.pre_slope;
  const bool has_affine = a.pre_a != nullptr, is_snake = pre_act_ == ST2_ACT_SNAKE;
  float* coef = reinterpret_cast<float*>(smem + SM_COEF);
  const int cin_pad = ncb * CB;
  const int my_tiles = (ntiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  const int total_blocks = my_tiles * ncb;
  const unsigned long long xaddr4 = (unsigned long long)(uintptr_t)a.x >> 2;
  const long long tensor_end = (long long)(a.B - 1) * a.x_bstride + (long long)Cin_ * Lin_;  // floats from a.x
  const float* x_al = reinterpret_cast<const float*>((uintptr_t)a.x & ~(uintptr_t)15);
  // issue mapping: thread -> one channel of the block and every ST_PER_CH-th 16-byte chunk of its row
  const int ich = st / ST_PER_CH, iq0 = st - ich * ST_PER_CH;
  // producer-side state (runs RAW_STAGES-1 blocks ahead of the conversion); issue() is called for g = 0, 1, 2, ... in order,
  // so (tile, channel block, ring slot) advance by counters instead of divisions
  int i_tl = 0, i_cb = 0, i_slot = 0, i_g0 = 0;
  bool i_inter = false;
  long long i_boff = 0;
  const int dbg_i = g_dbg;
  auto issue = [&](int g) {
    if (g < total_blocks && !(dbg_i & 32)) {
      if (i_cb == 0) {
        const TileCoord tc_ = tile_coord(blockIdx.x + i_tl * gridDim.x, n_tq, n_cob);
        i_boff = (long long)tc_.b * a.x_bstride;
        i_g0 = tc_.tq * TN - a.pad;
        i_inter = (i_g0 >= 0) && (i_g0 + RW <= Lin_);   // the whole window lies inside the rows
      }
      const int c = i_cb * CB + ich;
      const long long e0 = i_boff + (long long)min(c, Cin_ - 1) * Lin_ + i_g0;   // first window element, floats from a.x
      const int shift = (int)(((unsigned)xaddr4 + (unsigned)e0) & 3u);
      const long long w0 = e0 - shift;                                          // aligned window start, floats from a.x
      const float* src0 = a.x + w0;
      const long long end_rel = tensor_end - w0;
      uint32_t dst = sbase + SM_RAW + i_slot * RAW_BYTES + (uint32_t)(ich * RAW_PITCH + iq0 * 4) * 4;
      if (i_inter && c < Cin_ && end_rel >= (long long)(RW + 8)) {
        // interior window of an existing channel, every chunk entirely inside the tensor: only the chunk count matters
        const int qhi = (RW + shift + 3) >> 2;
        const float* src = src0 + 4 * iq0;
#pragma unroll
        for (int i = 0; i < RAW_CHUNKS / ST_PER_CH; ++i) {
          const bool ok = (iq0 + ST_PER_CH * i) < qhi;
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst + i * ST_PER_CH * 16), "l"(ok ? src + 4 * ST_PER_CH * i : x_al),
                       "r"(ok ? 16 : 0) : "memory");
        }
      } else {
        const int rlo = max(0, -i_g0), rhi = min(RW, Lin_ - i_g0);              // rows [rlo, rhi) are inside the tensor
        int qlo = 0, qhi = 0;
        if (c < Cin_ && rhi > rlo) { qlo = (rlo + shift) >> 2; qhi = (rhi + shift + 3) >> 2; }
#pragma unroll
        for (int i = 0; i < RAW_CHUNKS / ST_PER_CH; ++i) {
          const int q = iq0 + ST_PER_CH * i;
          const bool ok = (q >= qlo) && (q < qhi);
          const long long rem = end_rel - 4ll * q;
          const int nbytes = ok ? (rem >= 4 ? 16 : (int)rem * 4) : 0;
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(ok ? src0 + 4 * q : x_al), "r"(nbytes) : "memory");
          dst += ST_PER_CH * 16;
        }
      }
      if (++i_cb == ncb) { i_cb = 0; ++i_tl; }
      if (++i_slot == RAW_STAGES) i_slot = 0;
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  for (int g = 0; g < RAW_STAGES - 1; ++g) issue(g);
  int as = 0, aph = 0;
  int c_tile = -1, c_g0 = 0, c_b = 0, last_b = -1;
  long long c_boff = 0;
  // conversion mapping: warp parity -> K chunk, (warp / 2, lane) -> ROWS_PER_PASS rows per pass: every shared-memory access of
  // a warp touches consecutive words / consecutive 16-byte rows
  const int sw = warp - ST0 / 32;
  const int dbg_st = g_dbg;
  const int kc = sw & 1, rg = (sw >> 1) * 32 + lane;
  constexpr int NRC = (RW_MAX + ROWS_PER_PASS - 1) / ROWS_PER_PASS;
  const float xs_ = X_SCALE;
  int cb = 0, c_slot = 0;
  bool in_range = true;   // range guard: every operand this thread converted is below FP16_MAX
  unsigned c_row0 = 0;   // low 32 bits of the element index of (tile's utterance, channel 0, first window frame): only its 4-byte phase is used
  for (int g = 0; g < total_blocks; ++g) {
    if (cb == 0) {
      ++c_tile;
      const TileCoord tc_ = tile_coord(blockIdx.x + c_tile * gridDim.x, n_tq, n_cob);
      c_b = tc_.b;
      c_boff = (long long)tc_.b * a.x_bstride;
      c_g0 = tc_.tq * TN - a.pad;
      c_row0 = (unsigned)xaddr4 + (unsigned)c_boff + (unsigned)c_g0;
    }
    asm volatile("cp.async.wait_group %0;" ::"n"(RAW_STAGES - 2) : "memory");
    asm volatile("bar.sync 1, %0;" ::"n"(NUM_STAGERS));  // block g landed for everybody; block g-1 fully converted
    issue(g + RAW_STAGES - 1);                             // reuses the slot of block g-1
    if (c_b != last_b) {
      // per-channel prologue coefficients of this utterance, with the 2^6 operand scale folded in: z' = 64 z = (64a) x + 64b;
      // snake(z) * 64 = z' + (64/alpha) sin^2((alpha/64) z'); LeakyReLU is positively homogeneous
      for (int c = st; c < cin_pad; c += NUM_STAGERS) {
        float pa = 0.f, pb = 0.f, al = 1.f;  // padded channels stage exact zeros
        if (c < Cin_) {
          pa = 1.f;
          if (has_affine) { pa = a.pre_a[c_b * Cin_ + c]; pb = a.pre_b[c_b * Cin_ + c]; }
          if (is_snake) al = a.pre_alpha[c];
        }
        coef[c] = pa * xs_; coef[CIN_PAD_MAX + c] = pb * xs_; coef[2 * CIN_PAD_MAX + c] = al * (1.0f / X_SCALE);
        coef[3 * CIN_PAD_MAX + c] = xs_ / al;
      }
      asm volatile("bar.sync 2, %0;" ::"n"(NUM_STAGERS));
      last_b = c_b;
    }
    const int c0 = cb * CB + kc * 8;
    float pa[8], pb[8], al[8], ia[8];
    int sh[8];
    {
      const int sh0 = (int)((c_row0 + (unsigned)c0 * (unsigned)Lin_) & 3u), lin3 = Lin_ & 3;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        pa[j] = coef[c0 + j]; pb[j] = coef[CIN_PAD_MAX + c0 + j]; al[j] = coef[2 * CIN_PAD_MAX + c0 + j];
        ia[j] = coef[3 * CIN_PAD_MAX + c0 + j];
        sh[j] = ((sh0 + j * lin3) & 3) + j * RAW_PITCH;   // 4-byte phase of channel c0+j's row start (padded channels: any)
      }
    }
    const float* raw = reinterpret_cast<const float*>(smem + SM_RAW + c_slot * RAW_BYTES) + (kc * 8) * RAW_PITCH;
    mbar_wait(BAR(B_AEMPTY + as), aph ^ 1);
    uint8_t* p0 = smem + SM_ACT + as * ACT_BUF_BYTES;
    uint8_t* p1 = p0 + ACT_PLANE_BYTES;
#pragma unroll
    for (int i = 0; i < NRC; ++i) {
      const int r = rg + ROWS_PER_PASS * i;
      if (r < RW && !(dbg_st & 4)) {
        const int gt = c_g0 + r;
        const bool inb = (gt >= 0) && (gt < Lin_);
        float xv[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) xv[j] = raw[sh[j] + r];
        if (pre_act_ == ST2_ACT_SNAKE) stage_row<ST2_ACT_SNAKE, MODE>(xv, pa, pb, al, ia, slope_, inb, p0, p1, kc, r, RWP, in_range);
        else if (pre_act_ == ST2_ACT_LRELU) stage_row<ST2_ACT_LRELU, MODE>(xv, pa, pb, al, ia, slope_, inb, p0, p1, kc, r, RWP, in_range);
        else stage_row<ST2_ACT_NONE, MODE>(xv, pa, pb, al, ia, slope_, inb, p0, p1, kc, r, RWP, in_range);
      }
    }
    fence_proxy_async();  // generic-proxy smem writes -> visible to the tensor core (async proxy)
    mbar_arrive(BAR(B_AFULL + as));
    if (++as == 2) { as = 0; aph ^= 1; }
    if (++cb == ncb) cb = 0;
    if (++c_slot == RAW_STAGES) c_slot = 0;
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  if (!in_range) atomicExch(&g_range_flag, 1);
}

// Release bookkeeping of the consumer warpgroups: the MMAs of one weight stage are committed as one wgmma group and at most
// one group stays in flight, so a stage (and, after the last stage of a channel block, the activation buffer) is handed
// back to its producer when the NEXT group has been issued and the wait leaves one pending.
struct Pending {
  int ws, as;   // weight stage of the group; activation buffer freed with it (-1: none)
};
__device__ __forceinline__ void release(const uint32_t bar0, const Pending& p, const bool leader) {
  if (leader && p.ws >= 0) {
    mbar_arrive(bar0 + 8u * (B_WEMPTY + p.ws));
    if (p.as >= 0) mbar_arrive(bar0 + 8u * (B_AEMPTY + p.as));
  }
}

// ---------------------------------------------------------------------------------------------
// Pipeline skeleton of both kernels: barriers, producer roles and the consumer K-loop.  The kernels differ only in the
// MMAs of one tap, the taps per weight stage and their epilogues.
__device__ __forceinline__ void init_barriers(const uint32_t bar0) {
  if (threadIdx.x == 0) {
    for (int i = 0; i < W_STAGES; ++i) { mbar_init(bar0 + 8u * (B_WFULL + i), 1); mbar_init(bar0 + 8u * (B_WEMPTY + i), 2); }
    for (int i = 0; i < 2; ++i) {
      mbar_init(bar0 + 8u * (B_AFULL + i), NUM_STAGERS);
      mbar_init(bar0 + 8u * (B_AEMPTY + i), 2);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
}

// Warpgroups 2-3: give registers back, then run the weight producer (warp 8, one lane) or an activation stager.
template <int MODE>
__device__ __forceinline__ void producer_roles(const st2_conv_args& a, const uint4* __restrict__ wtc, uint8_t* smem, const int ncb,
                                               const int RW, const int wstep, const int tps, const int stage_bytes, const int ntiles,
                                               const int n_tq, const int n_cob, const int tid, const int warp, const int lane) {
  const uint32_t sbase = smem_u32(smem), bar0 = sbase + SM_BAR;
  reg_dealloc<REG_AUX>();
  if (warp == NUM_CONS / 32) {
    if (lane == 0) weight_producer_role(wtc, sbase, bar0, ncb, a.K, wstep, tps, stage_bytes, ntiles, n_tq, n_cob);
  } else if (warp < (ST0 + NUM_STAGERS) / 32) {
    stager_role<MODE>(a, smem, sbase, bar0, ncb, RW, ntiles, n_tq, n_cob, tid, warp, lane);
  }
}

// Ring positions of a consumer warpgroup and its wgmma group still in flight, carried from tile to tile.
struct ConsumerRing {
  int ws = 0, wph = 0, as = 0, aph = 0;
  Pending pend{-1, -1};
};

// Consumer K-loop of one tile: per 16-channel block wait for the staged window, then per weight stage of up to `tps` taps
// wait for the weights and issue the stage's MMAs as one wgmma group; the previous group's stage is released once the wait
// leaves this one pending.  mma(w_addr, x_addr, acc) issues one tap: its weights at w_addr (+ w_off in the stage, wstep
// bytes per tap), its window at x_addr (+ x_off in the buffer, one dilation per tap).  TPS > 0 unrolls a compile-time tps.
// Returns with every MMA complete and every stage released; the caller fences its accumulators (wg_fence_regs).
template <int TPS, class Mma>
__device__ __forceinline__ void consumer_k_loop(ConsumerRing& r, const uint32_t sbase, const bool leader, const int ncb, const int K,
                                                const int tps, const int stage_bytes, const int wstep, const uint32_t w_off,
                                                const uint32_t x_off, const uint32_t dil16, Mma&& mma) {
  const uint32_t bar0 = sbase + SM_BAR;
  uint32_t acc = 0;
  for (int cb = 0; cb < ncb; ++cb) {
    mbar_wait(bar0 + 8u * (B_AFULL + r.as), r.aph);
    uint32_t x_addr = sbase + SM_ACT + r.as * ACT_BUF_BYTES + x_off;
    for (int tap0 = 0; tap0 < K; tap0 += tps) {
      mbar_wait(bar0 + 8u * (B_WFULL + r.ws), r.wph);
      wg_fence();
      uint32_t w_addr = sbase + SM_W + r.ws * stage_bytes + w_off;
      const int nt = min(tps, K - tap0);
      auto tap = [&] {
        mma(w_addr, x_addr, acc);
        acc = 1;
        w_addr += wstep;
        x_addr += dil16;
      };
      if constexpr (TPS > 0) {
#pragma unroll
        for (int t = 0; t < TPS; ++t)
          if (t < nt) tap();
      } else {
        for (int t = 0; t < nt; ++t) tap();
      }
      wg_commit();
      wg_wait<1>();
      release(bar0, r.pend, leader);
      r.pend.ws = r.ws;
      r.pend.as = (tap0 + tps >= K) ? r.as : -1;
      if (++r.ws == W_STAGES) { r.ws = 0; r.wph ^= 1; }
    }
    if (++r.as == 2) { r.as = 0; r.aph ^= 1; }
  }
  wg_wait<0>();
  release(bar0, r.pend, leader);
  r.pend.ws = -1;
}

// Output value of one element: bias, residual, divisor, MRF accumulation and output activation, in the order of the SIMT
// kernel.  res_v = the residual, y_old = the y value the MRF accumulation adds to (each read only when its mode is on).
__device__ __forceinline__ float epi_combine(const st2_conv_args& a, float v, float bias, float res_v, float y_old) {
  float val = v + bias;
  if (a.res) val += res_v;
  if (a.out_div != 1.0f) val = __fdiv_rn(val, a.out_div);
  if (a.accum_mode == 1) val = y_old + val;
  else if (a.accum_mode == 2) val = __fdiv_rn(y_old + val, a.accum_div);
  if (a.out_act == ST2_ACT_TANH) val = tanhf(val);
  return val;
}

// The epilogues read the residual and MRF operands of a whole slice BEFORE they store any of it.  The compiler may not move
// a load above a store through a pointer that could alias it, so loading each element's operands just before its store
// pays one full memory latency per element (the consumer warps have nothing else to issue meanwhile).  An element's
// operands are only ever read by the thread that writes it, so the values are the same.
__device__ __forceinline__ void epi_load(const st2_conv_args& a, const float* rrow, const float* yp, int oidx, bool ok, float& res_v,
                                         float& y_old) {
  res_v = (rrow && ok) ? rrow[oidx >> a.res_shift] : 0.f;
  y_old = (a.accum_mode != 0 && ok) ? yp[oidx] : 0.f;
}

// Float index of (channel row r, frame fr) in a warpgroup's slot of rows `pitch` (64 or 128) frames long.  The XOR keeps both
// views free of bank conflicts: a fragment-order access (one register of 32 lanes: g = lane / 4 picks bits 0-2 of the frame
// or the channel, t4 = lane % 4 bits 1-2 of the other) lands on 32 distinct banks, and a row access (one channel, frames
// l + 32 m) only permutes the frames inside their aligned group of 32.  tests/test_cpu_epilogue_slot.py restates it.
__device__ __forceinline__ int slot_index(int r, int fr, int pitch) { return r * pitch + (fr ^ ((r & 1) | ((r & 6) << 2))); }

// Consumer warpgroup barrier around the slot (named barrier 3 + wg, 128 threads).
__device__ __forceinline__ void wg_bar(uint32_t id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

// Row phase of the epilogue for one warp: slot rows r0 .. r0 + nr - 1 (output channels co0 + r), lane l handling frames
// l + 32 m of each, in batches of RB rows (nr is a multiple of RB).  Every residual / MRF operand of a batch is loaded first
// (epi_load), then each value is combined, stored to y at frame t0 + fr when it exists (channel < Cout, fr < nfr) and
// written back to the slot (0 where it does not) for the statistics.  The slot holds the folded accumulators, still scaled
// by 2^18.  The batch loop stays rolled: compact code (the epilogue runs once per tile, mostly from a cold instruction
// cache), and one batch's operands are what the consumer's 128 registers hold next to the accumulators.
template <int RB, int FPL>
__device__ __forceinline__ void epi_rows(const st2_conv_args& a, float* xs, int pitch, int r0, int nr, int co0, int b, int t0, int nfr,
                                         int lane) {
  // row pointers advance by one row per channel; a row at or beyond Cout is never dereferenced (every access is under cok)
  const long long ylen = a.y_len, rlen = a.res ? a.res_len : 0;   // no residual: rrow stays null
  float* yrow = a.y + (long long)b * a.y_bstride + (long long)(co0 + r0) * ylen;
  const float* rrow = a.res ? a.res + (long long)b * a.res_bstride + (long long)(co0 + r0) * rlen : nullptr;
#pragma unroll 1
  for (int k0 = 0; k0 < nr; k0 += RB) {
    float res_v[RB][FPL], y_old[RB][FPL], bias[RB];
#pragma unroll
    for (int k = 0; k < RB; ++k) {
      const int co = co0 + r0 + k0 + k;
      const bool cok = co < a.Cout;
      bias[k] = (a.bias && cok) ? __ldg(a.bias + co) : 0.f;
#pragma unroll
      for (int m = 0; m < FPL; ++m) {
        const int fr = lane + 32 * m;
        epi_load(a, rrow, yrow, t0 + fr, cok && fr < nfr, res_v[k][m], y_old[k][m]);
      }
      yrow += ylen;
      rrow += rlen;
    }
    yrow -= RB * ylen;
#pragma unroll
    for (int k = 0; k < RB; ++k) {
      const int r = r0 + k0 + k, sw = (r & 1) | ((r & 6) << 2);   // slot_index's swizzle of row r
      const bool cok = co0 + r < a.Cout;
      float* xr = xs + r * pitch;
#pragma unroll
      for (int m = 0; m < FPL; ++m) {
        const int fr = lane + 32 * m;
        float val = 0.f;
        if (cok && fr < nfr) {
          val = epi_combine(a, xr[fr ^ sw] * D_UNSCALE, bias[k], res_v[k][m], y_old[k][m]);
          yrow[t0 + fr] = val;
        }
        xr[fr ^ sw] = val;
      }
      yrow += ylen;
    }
  }
}

template <int MODE>
__global__ void __launch_bounds__(THREADS, 1)
conv1d_tc_kernel(const st2_conv_args a, const uint4* __restrict__ wtc, const int ncb, const int RW, const int ntiles,
                 const int n_tq, const int n_cob) {
  // RW = window rows (TN + (K-1)*dil, rounded up to 8); RWP = chunk pitch in rows
  const int RWP = RW + 2;
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, warp = warp_uniform(tid), lane = tid & 31;
  const uint32_t sbase = smem_u32(smem);
  init_barriers(sbase + SM_BAR);

  if (warp < NUM_CONS / 32) {
    // ================================================================ consumers: wgmma (warpgroup wg = channels 64 wg ..) + epilogue
    reg_alloc<REG_CONS>();
    const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t4 = lane & 3;
    const bool leader = (tid & 127) == 0;
    const uint32_t lbo_a = TM * 16, lbo_b = (uint32_t)RWP * 16;
    ConsumerRing ring;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      const TileCoord tc_ = tile_coord(tile, n_tq, n_cob);
      float d0[64], d1[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) { d0[i] = 0.f; d1[i] = 0.f; }
      consumer_k_loop<TPS>(ring, sbase, leader, ncb, a.K, TPS, W_STAGE_BYTES, W_STEP_BYTES, wg * 64 * 16, 0, (uint32_t)a.dil * 16u,
                           [&](uint32_t a_addr, uint32_t b_addr, uint32_t acc) {
        const uint64_t da0 = make_desc(a_addr, lbo_a, 128), da1 = make_desc(a_addr + W_PLANE_BYTES, lbo_a, 128);
        const uint64_t db0 = make_desc(b_addr, lbo_b, 128), db1 = make_desc(b_addr + ACT_PLANE_BYTES, lbo_b, 128);
        if (MODE == MODE_FAST) {
          wgmma_f16_n128(d0, da0, db0, acc);
          wgmma_e4m3_n128(d1, da1, db1, acc);     // both corrections in one e4m3 K=32 MMA, own accumulator
        } else if (MODE == MODE_ACC) {
          wgmma_f16_n128(d0, da0, db0, acc);
          wgmma_f16_n128(d1, da0, db1, acc);
          wgmma_f16_n128(d1, da1, db0, 1u);
        } else {
          wgmma_f16_n128(d0, da0, db0, acc);
          wgmma_f16_n128(d0, da0, db1, 1u);
          wgmma_f16_n128(d0, da1, db0, 1u);
        }
      });
      wg_fence_regs(d0);
      if (MODE != MODE_X3) wg_fence_regs(d1);
      // fold the correction accumulator into d0 (d1 is dead from here on)
#pragma unroll
      for (int r = 0; r < 64; ++r) {
        float v = d0[r];
        if (MODE == MODE_ACC) v = fmaf(d1[r], ACC_LO_UNSCALE, v);
        if (MODE == MODE_FAST) v += d1[r];
        d0[r] = v;
      }

      // ---- epilogue: row = output channel, column = frame.  Each 64-frame half h of the tile (fragment columns j = 8 h ..
      // 8 h + 7) is one slice through the warpgroup's slot and one statistics partial: fragment float 4 (8 h + j) + 2 i + c
      // is channel w * 16 + g + 8 i, frame 8 j + 2 t4 + c of the half.  Each warp computes 16 whole channel rows (epi_rows),
      // the values come back into the fragments, and the half's statistics follow.  The second half of a tail tile can lie
      // entirely beyond Lq: no partial then.
      float* xs = reinterpret_cast<float*>(smem + SM_SLOT) + wg * SLOT_FLOATS;
      const uint32_t bar_id = 3 + wg;
#pragma unroll
      for (int h = 0; h < TN / TP; ++h) {
        const int t0 = tc_.tq * TN + h * TP;
        wg_bar(bar_id);   // the previous half's (or tile's) readers are done
#pragma unroll
        for (int q = 0; q < 32; ++q) xs[slot_index(w * 16 + g + 8 * ((q >> 1) & 1), 8 * (q >> 2) + 2 * t4 + (q & 1), TP)] = d0[32 * h + q];
        wg_bar(bar_id);
        epi_rows<8, TP / 32>(a, xs, TP, w * 16, 16, tc_.cob * TM + wg * 64, tc_.b, t0, a.Lq - t0, lane);
        wg_bar(bar_id);
#pragma unroll
        for (int q = 0; q < 32; ++q) d0[32 * h + q] = xs[slot_index(w * 16 + g + 8 * ((q >> 1) & 1), 8 * (q >> 2) + 2 * t4 + (q & 1), TP)];
        const int ncols = min(TP, a.Lq - t0);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int co = tc_.cob * TM + wg * 64 + w * 16 + g + 8 * i;
          const bool cok = co < a.Cout;
          float s = 0.f, n = 0.f;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              if (cok && 8 * j + 2 * t4 + c < ncols) {
                s += d0[4 * (8 * h + j) + 2 * i + c];
                n += 1.f;
              }
            }
          }
          if (a.stats && ncols > 0) {
            // two-pass (count, mean, M2) of the row over the half's frames: the four lanes t4 of a quad share the row
            s += __shfl_xor_sync(0xffffffffu, s, 1);
            s += __shfl_xor_sync(0xffffffffu, s, 2);
            n += __shfl_xor_sync(0xffffffffu, n, 1);
            n += __shfl_xor_sync(0xffffffffu, n, 2);
            const float mean = n > 0.f ? s / n : 0.f;
            float m2 = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
#pragma unroll
              for (int c = 0; c < 2; ++c) {
                const int col = 8 * j + 2 * t4 + c;
                const float dv = d0[4 * (8 * h + j) + 2 * i + c] - mean;
                if (col < ncols) m2 = fmaf(dv, dv, m2);
              }
            }
            m2 += __shfl_xor_sync(0xffffffffu, m2, 1);
            m2 += __shfl_xor_sync(0xffffffffu, m2, 2);
            if (t4 == 0 && cok) {
              const int part = tc_.tq * (TN / TP) + h;
              float* sp = a.stats + (((long long)tc_.b * a.Cout + co) * a.stats_nparts + a.stats_part_offset + part) * 3;
              sp[0] = n; sp[1] = mean; sp[2] = m2;
            }
          }
        }
      }
    }
  } else {
    producer_roles<MODE>(a, wtc, smem, ncb, RW, W_STEP_BYTES, TPS, W_STAGE_BYTES, ntiles, n_tq, n_cob, tid, warp, lane);
  }
}

// =============================================================================================
// TIME-MAJOR variant for narrow layers (Cout <= 128; HiFi-GAN C = 64 / 32 stages, conv_post): the operand roles are
// swapped --
//     D[t (M = 64 frames per warpgroup, 128 per tile), co (N = NC)] = sum_tap sum_ci z[ci, t + tap*dil - pad] * W_tap[co, ci]
// The staged activation window is the A operand (same K-major 16-byte-row layout, a tap is still a descriptor shift), the
// weights are the B operand with only NC = Cout rounded up to 32 (16 for Cout <= 16) rows: no tensor-pipe time and no weight
// traffic is spent on absent output channels.  The two consumer warpgroups take one half of the tile's frames each (warpgroup
// 1's A descriptor starts 64 rows further into the staged window) and all NC channels; both read the whole weight stage.
// The InstanceNorm partial of a channel over a warpgroup's 64 frames is reduced over the warp's 16 frames with shuffles and
// over the four warps through shared memory (two passes: mean, then M2).  FAST recipe only.
__host__ __device__ __forceinline__ int tmajor_nc(int Cout) { return Cout <= 16 ? 16 : ((Cout + 31) & ~31); }

constexpr int T_WSTAGE = 16384;                           // bytes per weight stage: 16 taps (NC = 16) .. 2 taps (NC = 128)
static_assert(T_WSTAGE <= W_STAGE_BYTES, "time-major stages live in the SM_W ring");

template <int NC>   // output channels (weight rows) = wgmma N
__device__ __forceinline__ void tct_mma(float (&d)[NC / 2], float (&e)[NC / 2], uint64_t a0, uint64_t b0, uint64_t a1, uint64_t b1,
                                        uint32_t acc) {
  if constexpr (NC == 16) { wgmma_f16_n16(d, a0, b0, acc); wgmma_e4m3_n16(e, a1, b1, acc); }
  else if constexpr (NC == 32) { wgmma_f16_n32(d, a0, b0, acc); wgmma_e4m3_n32(e, a1, b1, acc); }
  else if constexpr (NC == 64) { wgmma_f16_n64(d, a0, b0, acc); wgmma_e4m3_n64(e, a1, b1, acc); }
  else if constexpr (NC == 96) { wgmma_f16_n96(d, a0, b0, acc); wgmma_e4m3_n96(e, a1, b1, acc); }
  else { static_assert(NC == 128, "time-major N"); wgmma_f16_n128(d, a0, b0, acc); wgmma_e4m3_n128(e, a1, b1, acc); }
}

template <int NH>   // NC / 2
__global__ void __launch_bounds__(THREADS, 1)
conv1d_tct_kernel(const st2_conv_args a, const uint4* __restrict__ wtc, const int ncb, const int RW, const int ntiles, const int n_tq) {
  constexpr int MODE = MODE_FAST;
  constexpr int NC = 2 * NH;
  constexpr int NJ = NC / 8;
  static_assert(NC <= TCT_NC_MAX, "statistics scratch");
  const int RWP = RW + 2;
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, warp = warp_uniform(tid), lane = tid & 31;
  const uint32_t sbase = smem_u32(smem);
  init_barriers(sbase + SM_BAR);
  const int wstep = 64 * NC;                      // bytes of one (16 channels, tap) step: 2 planes x 2 chunks x NC rows x 16 B
  const int tps = T_WSTAGE / wstep;               // taps per weight stage: 1 (NC = 128, 96) .. 8 (NC = 16)

  if (warp < NUM_CONS / 32) {
    reg_alloc<REG_CONS>();
    const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t4 = lane & 3;
    const bool leader = (tid & 127) == 0;
    const uint32_t lbo_x = (uint32_t)RWP * 16, lbo_w = (uint32_t)NC * 16;
    float* red = reinterpret_cast<float*>(smem + SM_EPI) + wg * 4 * TCT_NC_MAX;   // [4 warps][TCT_NC_MAX channels]
    float* xs = reinterpret_cast<float*>(smem + SM_SLOT) + wg * SLOT_FLOATS;
    const uint32_t bar_id = 3 + wg;
    // fragment float 4 j + q (frame w * 16 + g + 8 (q >> 1) of channel 8 j + 2 t4 + (q & 1)) sits at slot float
    // fofs[q] + 8 TP (j - c0 / 8) of the slice starting at channel c0: the swizzle of a row does not depend on j
    int fofs[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) fofs[q] = slot_index(2 * t4 + (q & 1), w * 16 + g + 4 * (q & 2), TP);
    ConsumerRing ring;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      const int tq = tile % n_tq, b = tile / n_tq;
      float d[NC / 2], e[NC / 2];   // fp16 main products / e4m3 correction products (e4m3 wgmma accumulates at reduced precision)
#pragma unroll
      for (int i = 0; i < NC / 2; ++i) { d[i] = 0.f; e[i] = 0.f; }
      // warpgroup wg: frames TP wg .. of the tile
      consumer_k_loop<0>(ring, sbase, leader, ncb, a.K, tps, T_WSTAGE, wstep, 0, wg * TP * 16, (uint32_t)a.dil * 16u,
                         [&](uint32_t w_addr, uint32_t x_addr, uint32_t acc) {
        tct_mma<NC>(d, e, make_desc(x_addr, lbo_x, 128), make_desc(w_addr, lbo_w, 128), make_desc(x_addr + ACT_PLANE_BYTES, lbo_x, 128),
                    make_desc(w_addr + 2 * NC * 16, lbo_w, 128), acc);
      });
      wg_fence_regs(d);
      wg_fence_regs(e);
#pragma unroll
      for (int i = 0; i < NC / 2; ++i) d[i] += e[i];

      // ---- epilogue: row = frame, column = output channel.  The warpgroup's 64 frames are one statistics partial; the
      // second warpgroup of a tail tile can lie entirely beyond Lq (ncols <= 0): it then writes nothing.
      const int t0 = tq * TN + wg * TP;
      const int ncols = min(TP, a.Lq - t0);
      // Output values through the warpgroup's slot in slices of up to 64 channels: fragment float 4 j + 2 i + c is frame
      // w * 16 + g + 8 i of channel 8 j + 2 t4 + c.  Each warp computes a quarter of the slice's channel rows (epi_rows); the
      // values come back into the fragments for the statistics.
      constexpr int SC = NC < 64 ? NC : 64;
#pragma unroll 1
      for (int c0 = 0; c0 < NC; c0 += SC) {
        wg_bar(bar_id);   // the previous slice's (or tile's) readers are done
#pragma unroll
        for (int j = 0; j < NJ; ++j)
          if (8 * j >= c0 && 8 * j < c0 + SC) {
#pragma unroll
            for (int q = 0; q < 4; ++q) xs[fofs[q] - TP * c0 + 8 * TP * j] = d[4 * j + q];
          }
        wg_bar(bar_id);
        const int nr = min(SC, NC - c0) / 4;
        epi_rows<(SC < 32 ? SC / 4 : 8), TP / 32>(a, xs, TP, w * nr, nr, c0, b, t0, ncols, lane);
        wg_bar(bar_id);
#pragma unroll
        for (int j = 0; j < NJ; ++j)
          if (8 * j >= c0 && 8 * j < c0 + SC) {
#pragma unroll
            for (int q = 0; q < 4; ++q) d[4 * j + q] = xs[fofs[q] - TP * c0 + 8 * TP * j];
          }
      }
      // per-thread sums of each channel over its two frames, in the order the values were produced
      float s[NJ * 2];
#pragma unroll
      for (int j = 0; j < NJ; ++j)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const bool cok = 8 * j + 2 * t4 + c < a.Cout;
          float ss = 0.f;
#pragma unroll
          for (int i = 0; i < 2; ++i)
            if (cok && w * 16 + g + 8 * i < ncols) ss += d[4 * j + 2 * i + c];
          s[2 * j + c] = ss;
        }
      if (a.stats && ncols > 0) {
        // pass 1: sums over the 16 frames of the warp (lanes with equal t4), then over the warpgroup's four warps
#pragma unroll
        for (int k = 0; k < 2 * NJ; ++k) {
#pragma unroll
          for (int o = 4; o < 32; o <<= 1) s[k] += __shfl_xor_sync(0xffffffffu, s[k], o);
        }
        asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");   // the previous tile's readers are done
        if (g == 0) {
#pragma unroll
          for (int j = 0; j < NJ; ++j)
#pragma unroll
            for (int c = 0; c < 2; ++c) red[w * TCT_NC_MAX + 8 * j + 2 * t4 + c] = s[2 * j + c];
        }
        asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
        float mean[2 * NJ], cnt[2 * NJ];
#pragma unroll
        for (int j = 0; j < NJ; ++j)
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int ch = 8 * j + 2 * t4 + c;
            const float tot = red[ch] + red[TCT_NC_MAX + ch] + red[2 * TCT_NC_MAX + ch] + red[3 * TCT_NC_MAX + ch];
            // count of the partial = valid frames (the same for every existing channel)
            cnt[2 * j + c] = (float)max(0, ncols);
            mean[2 * j + c] = ncols > 0 ? tot / (float)ncols : 0.f;
          }
        // pass 2: M2 about the tile mean
        float q[2 * NJ];
#pragma unroll
        for (int j = 0; j < NJ; ++j)
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            float m2 = 0.f;
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              const int fr = w * 16 + g + 8 * i;
              const float dv = d[4 * j + 2 * i + c] - mean[2 * j + c];
              if (fr < ncols) m2 = fmaf(dv, dv, m2);
            }
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) m2 += __shfl_xor_sync(0xffffffffu, m2, o);
            q[2 * j + c] = m2;
          }
        asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
        if (g == 0) {
#pragma unroll
          for (int j = 0; j < NJ; ++j)
#pragma unroll
            for (int c = 0; c < 2; ++c) red[w * TCT_NC_MAX + 8 * j + 2 * t4 + c] = q[2 * j + c];
        }
        asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
        if (w == 0 && g == 0) {
          const int part = tq * (TN / TP) + wg;
#pragma unroll
          for (int j = 0; j < NJ; ++j)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              const int co = 8 * j + 2 * t4 + c;
              if (co < a.Cout) {
                float* gp = a.stats + (((long long)b * a.Cout + co) * a.stats_nparts + a.stats_part_offset + part) * 3;
                gp[0] = cnt[2 * j + c];
                gp[1] = mean[2 * j + c];
                gp[2] = red[co] + red[TCT_NC_MAX + co] + red[2 * TCT_NC_MAX + co] + red[3 * TCT_NC_MAX + co];
              }
            }
        }
      }
    }
  } else {
    producer_roles<MODE>(a, wtc, smem, ncb, RW, wstep, tps, T_WSTAGE, ntiles, n_tq, 1, tid, warp, lane);
  }
}

// One element of a weight stage block [plane 2][chunk 2][rows][16 B] (rows = 128, or NC for the time-major layout): byte index -> value.
//   plane 0: fp16 high plane of w' = w * 2^12, chunk = channels 8*kc .. 8*kc+7 (2 bytes each).
//   plane 1, ST2_TC_FAST: e4m3 bytes; chunk c = [l(w') * 2^4 | h(w') * 2^-8] of channels 8c .. 8c+7 (the order stage_row uses).
//   plane 1, otherwise:   fp16 low plane l(w') (* 2^8 for ST2_TC_ACCURATE).
__device__ __forceinline__ void weight_stage_store(uint8_t* blk, int byte_in_stage, int mode, const float* wrow16 /* 16 channel values of this row */,
                                                   int rows) {
  const int plane_bytes = KCB * rows * 16;
  const int plane = byte_in_stage / plane_bytes;
  const int r = byte_in_stage % plane_bytes;
  const int chunk = r / (rows * 16), within = r % 16;
  if (plane == 0 || mode != MODE_FAST) {
    if (within & 1) return;       // handled by the even byte
    const float wv = wrow16[chunk * 8 + within / 2] * W_SCALE;
    const __half h = __float2half_rn(wv);
    __half o = h;
    if (plane == 1) o = __float2half_rn((wv - __half2float(h)) * (mode == MODE_ACC ? ACC_LO_SCALE : 1.0f));
    *reinterpret_cast<__half*>(blk + byte_in_stage) = o;
  } else {
    // chunk c, byte b: channel 8c + (b & 7); bytes 0-7 meet h(z') (-> l(w') * 2^4), bytes 8-15 meet l(z') (-> h(w') * 2^-8)
    const float wv = wrow16[chunk * 8 + (within & 7)] * W_SCALE;
    const float hf = __half2float(__float2half_rn(wv));
    const float val = (within < 8) ? (wv - hf) * F8_WLO : hf * F8_WHI;
    blk[byte_in_stage] = (uint8_t)__nv_cvt_float_to_fp8(val, __NV_SATFINITE, __NV_E4M3);
  }
}

// Range guard of the weights: w' = w * 2^12 must fit the fp16 high plane (NaN fails the compare too).
__device__ __forceinline__ void weight_range_note(const float (&wr)[16]) {
  bool ok = true;
#pragma unroll
  for (int j = 0; j < 16; ++j) ok = ok && fabsf(wr[j] * W_SCALE) < FP16_MAX;
  if (!ok) atomicExch(&g_range_flag, 1);
}

// Row `col` of output-channel block `cob` -> output channel (or -1): rows are the channels of the block in order (the
// time-major layout has one block of NC rows).
__device__ __forceinline__ int weight_row_channel(int Cout, int cob, int col, bool tmajor) {
  const int co = tmajor ? col : cob * TM + col;
  return co < Cout ? co : -1;
}

// fp32 weights -> S phases of step blocks [n_cob][ncb][J] x (64 * rows) bytes, phase_bytes apart (the taps of one 16-channel
// block are contiguous).  Tap kp of phase ph reads source tap k = k0 + (ph + P) % S + kp * k_step of element (co, ci) at
// w[co * co_stride + ci * ci_stride + k]; k >= K reads zero.  A conv is S = 1, k0 = 0, k_step = 1; a ConvTranspose1d phase
// (a J-tap stride-1 conv, see conv.cu) reads its taps backwards, k0 = (J - 1) S, k_step = -S.
__global__ void weight_layout_kernel(const float* __restrict__ w, uint8_t* __restrict__ out, int Cout, int Cin, int K, long long co_stride,
                                     long long ci_stride, int S, int P, int J, int k0, int k_step, long long phase_bytes, int n_cob, int ncb,
                                     int mode, int rows, int tmajor) {
  // one thread per (phase, stage, plane, chunk, row): writes the 16 bytes of that row
  const long long total = (long long)S * J * n_cob * ncb * 2 * KCB * rows;
  const int step_bytes = 2 * KCB * rows * 16;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long r = i;
    const int col = (int)(r % rows); r /= rows;
    const int chunk = (int)(r % KCB); r /= KCB;
    const int plane = (int)(r % 2); r /= 2;
    const int cb = (int)(r % ncb); r /= ncb;
    const int cob = (int)(r % n_cob); r /= n_cob;
    const int kp = (int)(r % J);
    const int ph = (int)(r / J);
    const int co = weight_row_channel(Cout, cob, col, tmajor != 0);
    const int k = k0 + (ph + P) % S + kp * k_step;
    float wr[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int ci = cb * CB + j;
      wr[j] = (co >= 0 && ci < Cin && k < K) ? w[co * co_stride + ci * ci_stride + k] : 0.f;
    }
    weight_range_note(wr);
    uint8_t* blk = out + ph * phase_bytes + (((long long)cob * ncb + cb) * J + kp) * step_bytes;
    const int base = plane * (KCB * rows * 16) + (chunk * rows + col) * 16;
#pragma unroll
    for (int b = 0; b < 16; ++b) weight_stage_store(blk, base + b, mode, wr, rows);
  }
}

// ---------------------------------------------------------------------------------------------
// Polyphase ConvTranspose1d, second half: the S phase convolutions write PHASE-MAJOR rows tmp[r][b][co][q] (coalesced
// epilogue stores); this kernel interleaves them into y[b][co][q*S + r (+1)], adds the residual, applies the
// ReflectionPad1d((1,0)) duplicate (istftnet.py:365-366: y[0] = y[2], i.e. the unpadded sample 1 = phase 1, q = 0) and
// produces the InstanceNorm statistics of the result: per-thread Welford in fp64, fixed-order Chan merge -> one
// (count, mean, M2) record per row.  Memory-bound: reads tmp + res, writes y.
__global__ void __launch_bounds__(256) convT_interleave_kernel(const float* __restrict__ tmp, long long phase_stride, const float* __restrict__ res,
                                                               long long res_bstride, int res_len, float* __restrict__ y, long long y_bstride,
                                                               int y_len, int C, int Lin, int S, int reflect, float* __restrict__ stats) {
  const int co = blockIdx.x, b = blockIdx.y;
  const float* trow = tmp + ((long long)b * C + co) * Lin;
  const float* rrow = res ? res + (long long)b * res_bstride + (long long)co * res_len : nullptr;
  float* yrow = y + (long long)b * y_bstride + (long long)co * y_len;
  const int Lout = Lin * S + reflect;
  double n = 0.0, mean = 0.0, m2 = 0.0;
  for (int o = threadIdx.x; o < Lout; o += blockDim.x) {
    int u = o - reflect;            // index in the unpadded transposed-conv output
    if (u < 0) u = 1;               // reflection of the left edge
    const int q = u / S, r = u - q * S;
    float v = trow[(long long)r * phase_stride + q];
    if (rrow) v += rrow[o];
    yrow[o] = v;
    n += 1.0;
    const double d = (double)v - mean;
    mean += d / n;
    m2 += d * ((double)v - mean);
  }
  if (!stats) return;
  // merge: lanes, then warps (fixed order)
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const double nb = __shfl_down_sync(0xffffffffu, n, off), mb = __shfl_down_sync(0xffffffffu, mean, off),
                 qb = __shfl_down_sync(0xffffffffu, m2, off);
    const double nn = n + nb;
    if (nn > 0.0) {
      const double dl = mb - mean;
      mean += dl * (nb / nn);
      m2 += qb + dl * dl * (n * nb / nn);
      n = nn;
    }
  }
  __shared__ double sn[8], sm[8], sq[8];
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { sn[w] = n; sm[w] = mean; sq[w] = m2; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double N = sn[0], M = sm[0], Q = sq[0];
    for (int i = 1; i < (int)(blockDim.x >> 5); ++i) {
      const double nn = N + sn[i];
      if (nn > 0.0) {
        const double dl = sm[i] - M;
        M += dl * (sn[i] / nn);
        Q += sq[i] + dl * dl * (N * sn[i] / nn);
        N = nn;
      }
    }
    float* sp = stats + ((long long)b * C + co) * 3;
    sp[0] = (float)N; sp[1] = (float)M; sp[2] = (float)Q;
  }
}

constexpr int TMAJOR = ST2_TC_TMAJOR;   // flag bit of `mode`: time-major weight layout + kernel

// bytes of the weight blocks of one stride-1 convolution in the layout `mode` asks for
static long long weight_bytes_mode(int Cout, int Cin, int K, int mode) {
  const int ncb = cdiv(Cin, CB);
  if (mode & TMAJOR) return (long long)K * ncb * 64 * tmajor_nc(Cout);
  return (long long)K * cdiv(Cout, TM) * ncb * W_STEP_BYTES;
}

// Layout of S phases of J taps (see weight_layout_kernel), each phase weight_bytes_mode(Cout, Cin, J, mode) bytes.
static void weight_layout(const float* w, void* out, int Cout, int Cin, int K, long long co_stride, long long ci_stride, int S, int P,
                          int J, int k0, int k_step, int mode, cudaStream_t st) {
  const bool tm = (mode & TMAJOR) != 0;
  const int n_cob = tm ? 1 : cdiv(Cout, TM), ncb = cdiv(Cin, CB), rows = tm ? tmajor_nc(Cout) : TM;
  weight_layout_kernel<<<1024, 256, 0, st>>>(w, (uint8_t*)out, Cout, Cin, K, co_stride, ci_stride, S, P, J, k0, k_step,
                                             weight_bytes_mode(Cout, Cin, J, mode), n_cob, ncb, mode & ~TMAJOR, rows, tm ? 1 : 0);
  ++g_launches;
}

static int launch_tc(const st2_conv_args& a, const void* wtc, int mode, int max_ctas, cudaStream_t st) {
  const bool tmajor = (mode & TMAJOR) != 0;
  const int n_tq = cdiv(a.Lq, TN), n_cob = tmajor ? 1 : cdiv(a.Cout, TM), ncb = cdiv(a.Cin, CB);
  const int rw = (TN + (a.K - 1) * a.dil + 7) & ~7;
  const int ntiles = a.B * n_cob * n_tq;
  static PerDevice once;   // cudaFuncSetAttribute is per device
  if (once.first()) {
    const int dev = once.dev();
    cudaDeviceGetAttribute(&once.value[dev], cudaDevAttrMultiProcessorCount, dev);
    cudaFuncSetAttribute(conv1d_tc_kernel<MODE_FAST>, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_TOTAL);
    cudaFuncSetAttribute(conv1d_tc_kernel<MODE_ACC>, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_TOTAL);
    cudaFuncSetAttribute(conv1d_tc_kernel<MODE_X3>, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_TOTAL);
    cudaFuncSetAttribute(conv1d_tct_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_TOTAL);
    cudaFuncSetAttribute(conv1d_tct_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_TOTAL);
    cudaFuncSetAttribute(conv1d_tct_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_TOTAL);
    cudaFuncSetAttribute(conv1d_tct_kernel<48>, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_TOTAL);
    cudaFuncSetAttribute(conv1d_tct_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_TOTAL);
  }
  const int num_sms = once.value[once.dev()];
  int grid = ntiles < num_sms ? ntiles : num_sms;
  if (max_ctas > 0 && grid > max_ctas) grid = max_ctas;
  if (tmajor) {
    const int nh = tmajor_nc(a.Cout) / 2;
    if (nh == 8) conv1d_tct_kernel<8><<<grid, THREADS, SM_TOTAL, st>>>(a, (const uint4*)wtc, ncb, rw, ntiles, n_tq);
    else if (nh == 16) conv1d_tct_kernel<16><<<grid, THREADS, SM_TOTAL, st>>>(a, (const uint4*)wtc, ncb, rw, ntiles, n_tq);
    else if (nh == 32) conv1d_tct_kernel<32><<<grid, THREADS, SM_TOTAL, st>>>(a, (const uint4*)wtc, ncb, rw, ntiles, n_tq);
    else if (nh == 48) conv1d_tct_kernel<48><<<grid, THREADS, SM_TOTAL, st>>>(a, (const uint4*)wtc, ncb, rw, ntiles, n_tq);
    else conv1d_tct_kernel<64><<<grid, THREADS, SM_TOTAL, st>>>(a, (const uint4*)wtc, ncb, rw, ntiles, n_tq);
  }
  else if (mode == MODE_FAST) conv1d_tc_kernel<MODE_FAST><<<grid, THREADS, SM_TOTAL, st>>>(a, (const uint4*)wtc, ncb, rw, ntiles, n_tq, n_cob);
  else if (mode == MODE_ACC) conv1d_tc_kernel<MODE_ACC><<<grid, THREADS, SM_TOTAL, st>>>(a, (const uint4*)wtc, ncb, rw, ntiles, n_tq, n_cob);
  else conv1d_tc_kernel<MODE_X3><<<grid, THREADS, SM_TOTAL, st>>>(a, (const uint4*)wtc, ncb, rw, ntiles, n_tq, n_cob);
  ++g_launches;
  return 0;
}

}  // namespace tc

cudaError_t conv_tc_range_flag_fetch(int* flag) {
  int v = 0, zero = 0;
  cudaError_t e = cudaMemcpyFromSymbol(&v, tc::g_range_flag, sizeof(int));   // synchronises with the device
  if (e == cudaSuccess && v) e = cudaMemcpyToSymbol(tc::g_range_flag, &zero, sizeof(int));
  *flag = v;
  return e;
}

}  // namespace st2

using namespace st2;

extern "C" {

long long st2_conv_tc_weight_bytes(int Cout, int Cin, int K) {
  const int n_cob = cdiv(Cout, tc::TM), ncb = cdiv(Cin, tc::CB);
  return (long long)K * n_cob * ncb * tc::W_STEP_BYTES;   // upper bound for every layout (the time-major one is smaller)
}

// recipes 0..2; the time-major flag only with the FAST recipe and Cout <= 128 (one accumulator pair per tile)
static bool tc_mode_ok(int mode, int Cout) {
  const int base = mode & ~tc::TMAJOR;
  if (!(base == ST2_TC_FAST || base == ST2_TC_ACCURATE || base == ST2_TC_F16X3)) return false;
  if (mode & tc::TMAJOR) return base == ST2_TC_FAST && Cout <= 128;
  return true;
}

int st2_conv_tc_weight_layout(const float* w, void* out, int Cout, int Cin, int K, int mode, void* stream) {
  ST2_REQUIRE(w && out && Cout > 0 && Cin > 0 && K > 0 && tc_mode_ok(mode, Cout), "st2_conv_tc_weight_layout", "bad args");
  // w [Cout, Cin, K]: one phase, taps in order
  tc::weight_layout(w, out, Cout, Cin, K, (long long)Cin * K, K, 1, 0, K, 0, 1, mode, (cudaStream_t)stream);
  ST2_CHECK_LAUNCH("st2_conv_tc_weight_layout");
  return 0;
}

int st2_conv_tc_supported(int Cin, int Cout, int K, int stride, int dil) {
  const int rw = (tc::TN + (K - 1) * dil + 7) & ~7;
  return stride == 1 && rw <= tc::RW_MAX && cdiv(Cin, tc::CB) * tc::CB <= tc::CIN_PAD_MAX;
}

int st2_conv1d_tc(const st2_conv_args* a, const void* wtc, int mode, int max_ctas, void* stream) {
  ST2_REQUIRE(a && a->x && wtc && a->y && tc_mode_ok(mode, a->Cout), "st2_conv1d_tc", "null pointer / bad mode");
  ST2_REQUIRE(st2_conv_tc_supported(a->Cin, a->Cout, a->K, a->stride, a->dil), "st2_conv1d_tc", "unsupported shape");
  ST2_REQUIRE(a->pre_act != ST2_ACT_SNAKE || a->pre_alpha, "st2_conv1d_tc", "snake prologue needs alpha");
  ST2_REQUIRE(a->y_tstride == 1 && a->y_toffset == 0, "st2_conv1d_tc", "output positions must be contiguous (y_tstride 1, y_toffset 0)");
  ST2_REQUIRE(a->dup_q0_to < 0, "st2_conv1d_tc", "no reflection duplicate (dup_q0_to < 0)");
  const int nparts = cdiv(a->Lq, tc::TP);
  ST2_REQUIRE(!a->stats || a->stats_nparts >= a->stats_part_offset + nparts, "st2_conv1d_tc", "stats buffer too small (one partial per 64 columns)");
  tc::launch_tc(*a, wtc, mode, max_ctas, (cudaStream_t)stream);
  ST2_CHECK_LAUNCH("st2_conv1d_tc");
  return 0;
}

int st2_debug_set_flags(int flags) {
  cudaError_t e = cudaMemcpyToSymbol(tc::g_dbg, &flags, sizeof(flags));
  if (e != cudaSuccess) { set_error("st2_debug_set_flags", e); return (int)e; }
  return 0;
}

long long st2_convT_tc_weight_bytes(int Cin, int Cout, int K, int S) {
  const int J = (K + S - 1) / S;
  return (long long)S * st2_conv_tc_weight_bytes(Cout, Cin, J);
}

int st2_convT_tc_weight_layout(const float* w, void* out, int Cin, int Cout, int K, int S, int P, int mode, void* stream) {
  ST2_REQUIRE(w && out && Cout > 0 && Cin > 0 && K > 0 && S > 0 && tc_mode_ok(mode, Cout), "st2_convT_tc_weight_layout", "bad args");
  const int J = (K + S - 1) / S;
  // w [Cin, Cout, K]: phase ph = J taps read backwards from (J - 1) S + (ph + P) % S
  tc::weight_layout(w, out, Cout, Cin, K, K, (long long)Cout * K, S, P, J, (J - 1) * S, -S, mode, (cudaStream_t)stream);
  ST2_CHECK_LAUNCH("st2_convT_tc_weight_layout");
  return 0;
}

/* Every phase writes contiguous rows into `tmp` ([S][B][Cout][Lin] floats), one memory-bound pass interleaves, adds the
 * residual and produces ONE statistics record per row (stats [B,Cout,1,3]). */
int st2_conv_transpose1d_tc2(const st2_conv_args* a0, const void* wtc, int mode, int K, int S, int P, int reflect_left1, float* tmp,
                             void* stream) {
  ST2_REQUIRE(a0 && a0->x && wtc && a0->y && tmp && tc_mode_ok(mode, a0->Cout), "st2_conv_transpose1d_tc2", "null pointer / bad mode");
  ST2_REQUIRE(K > 0 && S > 0 && P >= 0, "st2_conv_transpose1d_tc2", "bad shape");
  const int J = (K + S - 1) / S;
  ST2_REQUIRE(st2_conv_tc_supported(a0->Cin, a0->Cout, J, 1, 1), "st2_conv_transpose1d_tc2", "unsupported shape");
  ST2_REQUIRE(!a0->stats || a0->stats_nparts == 1, "st2_conv_transpose1d_tc2", "stats must have exactly one partial per row");
  const long long phase_bytes = tc::weight_bytes_mode(a0->Cout, a0->Cin, J, mode);
  const long long phase_stride = (long long)a0->B * a0->Cout * a0->Lin;
  for (int r = 0; r < S; ++r) {
    st2_conv_args a = *a0;
    const int cr = (r + P) / S;
    a.K = J;
    a.stride = 1;
    a.dil = 1;
    a.pad = (J - 1) - cr;
    a.Lq = a0->Lin;
    a.y = tmp + (long long)r * phase_stride;
    a.y_bstride = (long long)a0->Cout * a0->Lin;
    a.y_tstride = 1;
    a.y_toffset = 0;
    a.y_len = a0->Lin;
    a.res = nullptr;
    a.stats = nullptr;
    a.accum_mode = 0;
    a.out_div = 1.0f;
    a.dup_q0_to = -1;
    tc::launch_tc(a, (const uint8_t*)wtc + (size_t)r * phase_bytes, mode, 0, (cudaStream_t)stream);
  }
  const int y_len = a0->Lin * S + (reflect_left1 ? 1 : 0);
  tc::convT_interleave_kernel<<<dim3(a0->Cout, a0->B), 256, 0, (cudaStream_t)stream>>>(
      tmp, phase_stride, a0->res, a0->res_bstride, a0->res_len, a0->y, a0->y_bstride, y_len, a0->Cout, a0->Lin, S, reflect_left1 ? 1 : 0,
      a0->stats);
  ++g_launches;
  ST2_CHECK_LAUNCH("st2_conv_transpose1d_tc2");
  return 0;
}

}  // extern "C"
