// wgmma flash attention for the spatial attentions of the denoising UNet (sm_90a).
//
//   O[b, q, h, :] = softmax_k( Q[b, q, h, :] . K[b / kv_div, k, h, :] * hd^-0.5 ) @ V[b / kv_div, k, h, :]
//
// covers attn1 (self-attention, kv_div = 1; reference modules/mutual_self_attention.py:176-186) and attn1_5
// (reference attention: K/V projected from the ReferenceNet bank, one bank per CFG half shared by the f frames
// of the window, kv_div = f; :202-219) -- both diffusers AttnProcessor2_0 / F.scaled_dot_product_attention
// without mask (SURVEY.md Appendix B.2).
//
// Per 64-key step, for the 64 query rows of one warpgroup:
//   TMA   : K_j, V_j tiles -> smem ring (3-D view (8, rows, C/8) of the [rows, C] token matrix, so a head slice
//           lands as [hd/8][rows][8] = the no-swizzle core-matrix layout; hd = 40 is zero-padded to 48 in smem
//           only, never in HBM)
//   wgmma : S_j = Q K_j^T  (m64n64k16, both operands K-major from shared memory, fp32 in registers)
//   online softmax in registers (the four lanes of a quad share a row), P_j rounded to bf16 straight into the A
//           fragment of the next MMA (the accumulator layout of m64n16 is the A layout of m64k16)
//   wgmma : O += P_j V_j  (A = P from registers, B = V tile MN-major from shared memory)
// Epilogue: O / l -> bf16 -> out[row, h*hd : (h+1)*hd].
//
// Two main loops compute this, with the same key order, the same accumulation order per row and the same rounding
// points (P -> bf16, O in fp32, O / l -> bf16), so their outputs are bit-identical:
//   flash_attn_pipe_kernel  : one producer warp + NCONS consumer warpgroups (64 NCONS query rows per CTA) around a
//                             full / empty mbarrier ring; each warpgroup issues S_{j+1} and O += P_j V_j together and
//                             runs the softmax of S_{j+1} under the latter (at hd <= 56 with S_{j+2} also in flight,
//                             two S register sets).  Serves hd <= 56, 80, 160.
//   flash_attn_wgmma_kernel : one CTA = one warpgroup = 64 query rows, each step a serial chain.  Serves the wider
//                             heads, and every head dim under VX_FA_V1=1 (the A/B reference).
#include "vx_host.h"
#include "vx_ptx.cuh"

namespace vx {

constexpr int kFaRows = 64;        // query rows per CTA = keys per step
constexpr int kFaThreads = 128;

struct FaArgs {
  int Nq, Nk, hd, kv_div, stages;
  float scale_log2;
  __nv_bfloat16* out;
  long long ldo;
};

// fragment of an m64nN accumulator (per thread): element 4 g + 2 h + e sits at row 16 warp + lane / 4 + 8 h,
// column 8 g + 2 (lane % 4) + e
template <int HDP>
__global__ void __launch_bounds__(kFaThreads)
flash_attn_wgmma_kernel(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                        const __grid_constant__ CUtensorMap mapV, const FaArgs p) {
  constexpr int kTile = kFaRows * HDP * 2;   // bytes of one Q / K / V tile ([HDP/8][64][8])
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + kTile;                   // stages x kTile
  uint8_t* sV = sK + p.stages * kTile;        // stages x kTile
  uint64_t* q_full = reinterpret_cast<uint64_t*>(sV + p.stages * kTile);
  uint64_t* kv_full = q_full + 1;             // [stages]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q_tile = blockIdx.x, head = blockIdx.y, bq = blockIdx.z;
  const int T = (p.Nk + kFaRows - 1) / kFaRows;
  if (HDP > p.hd) {
    // the padding chunk of Q / K / V (hd 40 -> 48) must read as exact zeros; TMA only ever writes chunks < hd / 8
    uint4* z = reinterpret_cast<uint4*>(sQ);
    for (int i = threadIdx.x; i < (1 + 2 * p.stages) * kTile / 16; i += blockDim.x) z[i] = make_uint4(0, 0, 0, 0);
  }
  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < p.stages; ++s) mbar_init(&kv_full[s], 1);
    fence_barrier_init();
  }
  fence_proxy_async_smem();  // generic-proxy zero fill visible to TMA / tensor core (async proxy)
  __syncthreads();
  pdl_wait();   // shared-memory fill and barrier init overlapped the previous grid's tail

  const int col_chunk = head * p.hd / 8;
  const int kv_row0 = (bq / p.kv_div) * p.Nk;
  auto load_kv = [&](int j) {
    const int st = j % p.stages;
    mbar_expect_tx(&kv_full[st], 2 * kFaRows * p.hd * 2);
    tma_load_3d(sK + st * kTile, &mapK, &kv_full[st], 0, kv_row0 + j * kFaRows, col_chunk);
    tma_load_3d(sV + st * kTile, &mapV, &kv_full[st], 0, kv_row0 + j * kFaRows, col_chunk);
  };
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&mapQ);
    tma_prefetch_desc(&mapK);
    tma_prefetch_desc(&mapV);
    mbar_expect_tx(q_full, kFaRows * p.hd * 2);
    tma_load_3d(sQ, &mapQ, q_full, 0, bq * p.Nq + q_tile * kFaRows, col_chunk);
    for (int j = 0; j < p.stages && j < T; ++j) load_kv(j);
  }

  // Q / K: K-major, no swizzle: LBO = 64 rows x 16 B between the 8-wide head-dim chunks, SBO = 128 B between 8-row
  // groups; +2 chunks (+2048 B = +128 in the address field) per 16 head dims.
  // V: MN-major (head dim contiguous): LBO = 128 B between 8-key groups, SBO = 64 x 16 B between 8-wide head-dim chunks;
  // +256 B (= +16) per 16 keys.
  const uint64_t dq = make_smem_desc(smem_u32(sQ), kFaRows * 16, 128, SWZ_NONE);
  const float c = p.scale_log2;
  float o[HDP / 2];
#pragma unroll
  for (int i = 0; i < HDP / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  const int cq = (lane & 3) * 2;
  mbar_wait(q_full, 0);
  for (int j = 0; j < T; ++j) {
    const int st = j % p.stages;
    mbar_wait(&kv_full[st], (uint32_t)((j / p.stages) & 1));
    float s[32];
    const uint64_t dk = make_smem_desc(smem_u32(sK + st * kTile), kFaRows * 16, 128, SWZ_NONE);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < HDP / 16; ++k) Wgmma<64>::ss<0, 0>(s, dq + (uint64_t)(k * 128), dk + (uint64_t)(k * 128), k);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    if ((j + 1) * kFaRows > p.Nk) {   // keys past Nk (the last, partial step) do not exist
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (j * kFaRows + (i >> 2) * 8 + cq + (i & 1) >= p.Nk) s[i] = -INFINITY;
    }
    float alpha[2], mc[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int g = 0; g < 8; ++g) mx = fmaxf(mx, fmaxf(s[4 * g + 2 * h], s[4 * g + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[h], mx);
      alpha[h] = m_run[h] == -INFINITY ? 0.f : exp2f((m_run[h] - m_new) * c);
      m_run[h] = m_new;
      mc[h] = m_new * c;
      l[h] *= alpha[h];
    }
#pragma unroll
    for (int i = 0; i < HDP / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
    uint32_t pa[4][4];
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int h = (i >> 1) & 1;
      const float e0 = exp2f(fmaf(s[i], c, -mc[h])), e1 = exp2f(fmaf(s[i + 1], c, -mc[h]));
      l[h] += e0 + e1;
      pa[i >> 3][(i >> 1) & 3] = pack_bf16(e0, e1);
    }
    const uint64_t dv = make_smem_desc(smem_u32(sV + st * kTile), 128, kFaRows * 16, SWZ_NONE);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kFaRows / 16; ++k) Wgmma<HDP>::template rs<1>(o, pa[k], dv + (uint64_t)(k * 16), 1);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    __syncthreads();   // every warp's MMAs on stage st have completed: refill it
    if (threadIdx.x == 0 && j + p.stages < T) load_kv(j + p.stages);
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float lt = l[h];
    lt += __shfl_xor_sync(0xffffffffu, lt, 1);
    lt += __shfl_xor_sync(0xffffffffu, lt, 2);
    const float inv = 1.f / lt;
    const int qrow = q_tile * kFaRows + warp * 16 + (lane >> 2) + 8 * h;
    if (qrow < p.Nq) {
      __nv_bfloat16* op = p.out + ((long long)bq * p.Nq + qrow) * p.ldo + head * p.hd;
#pragma unroll
      for (int g = 0; g < HDP / 8; ++g)
        if (g * 8 + cq < p.hd)
          *reinterpret_cast<uint32_t*>(op + g * 8 + cq) = pack_bf16(o[4 * g + 2 * h] * inv, o[4 * g + 2 * h + 1] * inv);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Pipelined loop.  Warpgroup 0 is the producer: its warp 0 issues every TMA, and the warpgroup hands its registers to the
// consumers.  Warpgroups 1 .. NCONS are the consumers, 64 query rows each, sharing every K / V stage.
//
// Ring: kv_full[s] (one arrival + transaction bytes) completes when K_j and V_j have landed in stage s = j % stages;
// kv_empty[s] (lane 0 of every consumer warp = 4 NCONS arrivals) completes when every warp's O += P_j V_j has completed.
// For use n = j / stages of a stage the consumers wait for kv_full parity n & 1, and the producer refills for use n >= 1
// behind kv_empty parity (n - 1) & 1.  Neither side gets two phases ahead: fill n + 1 needs release n, which needs fill n.
// A warpgroup whose rows all lie past Nq still consumes and releases every stage; only its stores are suppressed.
//
// MMA schedule of a consumer warpgroup, commit groups in issue order:
//   prologue     [S_0]                         wait<0>   softmax(S_0) -> l, P_0
//   j < T - 1    [S_{j+1}]  [O += P_j V_j]     wait<1>   S_{j+1} complete, O += P_j V_j may still run:
//                                                        softmax(S_{j+1}) in place -> alpha, l   (under the P V MMA)
//                                              wait<0>   O += P_j V_j complete: release stage j, O *= alpha, pack P_{j+1}
//   j = T - 1    [O += P_j V_j]                wait<0>   release stage j
// No MMA is in flight when S_{j+1} issues (the previous iteration ended in wait<0>), so it is never queued behind an
// incomplete MMA on the same registers.  P_j (register A operand) and O are untouched between the issue of O += P_j V_j
// and its wait<0>; S is untouched between the issue of S_{j+1} and wait<1>.  wgmma_fence_regs behind each wait keeps the
// compiler from moving those accesses up, the wgmma_fence in front of each issue orders the thread's own register
// writes (P, O *= alpha) before the MMAs.
//
// The arithmetic is that of flash_attn_wgmma_kernel, operation for operation, spelled with the non-contracting intrinsics
// (there the compiler contracts l * alpha + (e0 + e1) of the first pair into one FMA; here that is written out).  Two
// deliberate differences, neither visible in a result: exponentials are the bare ex2.approx.ftz (identical for every value
// >= 2^-126; smaller ones, which vanish against l >= 1 and O in fp32, flush to zero), and O += P V runs at N = hd rather
// than the padded width (m64n40k16 for hd 40), so V needs no padding chunk.
//
// Configuration per head width and consumer count.  A consumer thread holds O (HD / 2 floats), S (32 per register set)
// and P (16 words):
//   hd <= 56, three consumers : one CTA per SM, 24 / 160 registers (of the 128 x 4 that 512 threads launch with), two S
//                               register sets (below)
//   hd 80 / 160, two          : one CTA per SM, 24 / 232 (of 168 x 3), one S set
//   one consumer (Nq <= 64)   : two CTAs per SM, 24 / 232 (of 128 x 2), one S set
// and the ring is the deepest, up to 4 stages, that leaves room for that many CTAs.  Other widths take the serial loop.
constexpr bool fa_pipe_hd(int hd) { return hd % 8 == 0 && (hd <= 56 || hd == 80 || hd == 160); }
constexpr int fa_pipe_ncons(int hd, int Nq) { return Nq <= kFaRows ? 1 : hd <= 56 ? 3 : 2; }
constexpr int fa_pipe_ctas(int ncons) { return ncons == 1 ? 2 : 1; }
constexpr int fa_pipe_consumer_regs(int ncons) {
  // what the launch allocates per thread (65536 / (CTAs x threads), in steps of 8), pooled over the warpgroups, less
  // the producer's 24, shared among the consumers; setmaxnreg takes at most 232 (in steps of 8)
  const int pool = 65536 / (fa_pipe_ctas(ncons) * 128 * (ncons + 1)) / 8 * 8 * (ncons + 1);
  const int r = (pool - 24) / ncons / 8 * 8;
  return r < 232 ? r : 232;
}
constexpr int fa_pipe_stages(int hd, int ncons) {
  const int tile = kFaRows * ((hd + 15) / 16 * 16) * 2;
  const int per_cta = 228 * 1024 / fa_pipe_ctas(ncons) - 1024 - 256;   // less the per-CTA reserve and barriers
  const int s = (per_cta - ncons * tile) / (2 * tile);
  return s < 4 ? s : 4;
}
static_assert(fa_pipe_stages(160, 1) >= 2 && fa_pipe_stages(160, 2) == 4 && fa_pipe_stages(56, 3) == 4, "ring depth");

template <int HD, int NCONS>
__global__ void __launch_bounds__(128 * (NCONS + 1), fa_pipe_ctas(NCONS))
flash_attn_pipe_kernel(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                       const __grid_constant__ CUtensorMap mapV, const FaArgs p) {
  constexpr int HDP = (HD + 15) / 16 * 16;   // Q / K tile width: the K dimension of S = Q K^T in steps of 16
  constexpr int kTile = kFaRows * HDP * 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
  uint8_t* sQ = smem;                         // NCONS x kTile, one tile per consumer warpgroup
  uint8_t* sK = sQ + NCONS * kTile;           // stages x kTile
  uint8_t* sV = sK + p.stages * kTile;        // stages x kTile
  uint64_t* q_full = reinterpret_cast<uint64_t*>(sV + p.stages * kTile);
  uint64_t* kv_full = q_full + 1;             // [stages]
  uint64_t* kv_empty = kv_full + p.stages;    // [stages]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q_tile = blockIdx.x, head = blockIdx.y, bq = blockIdx.z;
  const int T = (p.Nk + kFaRows - 1) / kFaRows;
  if (HDP > HD) {
    // the padding chunk of Q / K must read as exact zeros; TMA only ever writes chunks < hd / 8
    uint4* z = reinterpret_cast<uint4*>(sQ);
    for (int i = threadIdx.x; i < (NCONS + 2 * p.stages) * kTile / 16; i += blockDim.x) z[i] = make_uint4(0, 0, 0, 0);
  }
  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&kv_full[s], 1);
      mbar_init(&kv_empty[s], 4 * NCONS);
    }
    fence_barrier_init();
  }
  fence_proxy_async_smem();  // generic-proxy zero fill visible to TMA / tensor core (async proxy)
  __syncthreads();
  pdl_wait();   // shared-memory fill and barrier init overlapped the previous grid's tail

  const int col_chunk = head * HD / 8;
  if (warp < 4) {
    // ------------------------------------------------------------------ producer (one lane)
    setmaxnreg_dec<24>();
    if (warp == 0 && lane == 0) {
      tma_prefetch_desc(&mapQ);
      tma_prefetch_desc(&mapK);
      tma_prefetch_desc(&mapV);
      mbar_expect_tx(q_full, NCONS * kFaRows * HD * 2);
      for (int w = 0; w < NCONS; ++w)
        tma_load_3d(sQ + w * kTile, &mapQ, q_full, 0, bq * p.Nq + (q_tile * NCONS + w) * kFaRows, col_chunk);
      const int kv_row0 = (bq / p.kv_div) * p.Nk;
      int st = 0;
      uint32_t phase = 0;
      for (int j = 0; j < T; ++j) {
        if (j >= p.stages) mbar_wait(&kv_empty[st], phase ^ 1);
        mbar_expect_tx(&kv_full[st], 2 * kFaRows * HD * 2);
        tma_load_3d(sK + st * kTile, &mapK, &kv_full[st], 0, kv_row0 + j * kFaRows, col_chunk);
        tma_load_3d(sV + st * kTile, &mapV, &kv_full[st], 0, kv_row0 + j * kFaRows, col_chunk);
        if (++st == p.stages) {
          st = 0;
          phase ^= 1;
        }
      }
    }
    return;
  }
  // -------------------------------------------------------------------- consumers
  setmaxnreg_inc<fa_pipe_consumer_regs(NCONS)>();
  const int wg = (warp >> 2) - 1;
  // Q / K: K-major, no swizzle: LBO = 64 rows x 16 B between the 8-wide head-dim chunks, SBO = 128 B between 8-row
  // groups; +2 chunks (+2048 B = +128 in the address field) per 16 head dims.
  // V: MN-major (head dim contiguous): LBO = 128 B between 8-key groups, SBO = 64 x 16 B between 8-wide head-dim chunks;
  // +256 B (= +16) per 16 keys.
  const uint64_t dq = make_smem_desc(smem_u32(sQ + wg * kTile), kFaRows * 16, 128, SWZ_NONE);
  const float c = p.scale_log2;
  const int cq = (lane & 3) * 2;
  float o[HD / 2], s[32];
  uint32_t pa[4][4];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f}, alpha[2];

  auto issue_s = [&](float (&s)[32], int st) {   // S = Q K^T against stage st, one commit group
    const uint64_t dk = make_smem_desc(smem_u32(sK + st * kTile), kFaRows * 16, 128, SWZ_NONE);
#pragma unroll
    for (int k = 0; k < HDP / 16; ++k) Wgmma<64>::ss<0, 0>(s, dq + (uint64_t)(k * 128), dk + (uint64_t)(k * 128), k);
    wgmma_commit();
  };
  auto softmax = [&](float (&s)[32], int j) {    // scores of step j in s -> alpha, m_run, l; s becomes the unrounded P
    if ((j + 1) * kFaRows > p.Nk) {   // keys past Nk (the last, partial step) do not exist
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (j * kFaRows + (i >> 2) * 8 + cq + (i & 1) >= p.Nk) s[i] = -INFINITY;
    }
    float mc[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int g = 0; g < 8; ++g) mx = fmaxf(mx, fmaxf(s[4 * g + 2 * h], s[4 * g + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[h], mx);   // finite: every step holds at least one real key
      alpha[h] = ex2_ftz(__fmul_rn(__fsub_rn(m_run[h], m_new), c));   // first step: ex2(-inf) = 0
      m_run[h] = m_new;
      mc[h] = __fmul_rn(m_new, c);
    }
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int h = (i >> 1) & 1;
      s[i] = ex2_ftz(__fmaf_rn(s[i], c, -mc[h]));
      s[i + 1] = ex2_ftz(__fmaf_rn(s[i + 1], c, -mc[h]));
      const float e = __fadd_rn(s[i], s[i + 1]);
      l[h] = i < 4 ? __fmaf_rn(l[h], alpha[h], e) : __fadd_rn(l[h], e);
    }
  };
  auto pack = [&](const float (&s)[32]) {   // P -> bf16, straight into the A fragments of O += P V
#pragma unroll
    for (int i = 0; i < 32; i += 2) pa[i >> 3][(i >> 1) & 3] = pack_bf16(s[i], s[i + 1]);
  };

  auto issue_pv = [&](int st) {  // O += P V against stage st, one commit group
    const uint64_t dv = make_smem_desc(smem_u32(sV + st * kTile), 128, kFaRows * 16, SWZ_NONE);
#pragma unroll
    for (int k = 0; k < kFaRows / 16; ++k) Wgmma<HD>::template rs<1>(o, pa[k], dv + (uint64_t)(k * 16), 1);
    wgmma_commit();
  };
  auto pv_done = [&](int st) {   // behind wait<0>: O and P are the thread's again, the stage goes back to the producer
    wgmma_fence_regs(o);
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_fence_regs(pa[k]);
    if (lane == 0) mbar_arrive(&kv_empty[st]);
  };
  auto rescale = [&]() {
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) o[i] = __fmul_rn(o[i], alpha[(i >> 1) & 1]);
  };
  mbar_wait(q_full, 0);
  int st = 0;
  uint32_t phase = 0;
  if constexpr (NCONS == 3) {
    // Two S register sets: S_{j+2} is issued behind O += P_j V_j and runs under the softmax of S_{j+1}, so no step waits
    // for its own S = Q K^T.  Commit groups in issue order:
    //   prologue   [S_0] [S_1]                 wait<1>  softmax(S_0) -> P_0
    //   step j     [O += P_j V_j] [S_{j+2}]    wait<2>  S_{j+1} complete: softmax(S_{j+1})
    //                                          wait<1>  O += P_j V_j complete: release stage j, O *= alpha, pack P_{j+1}
    // and without S_{j+2} (j = T - 2) wait<1> / wait<0>.  The set S_{j+2} lands in held S_j, dead once P_j is packed.
    float s2[32];
    int ist = 0;              // stage / phase of the next S to issue
    uint32_t iph = 0;
    auto next_s = [&](float (&sx)[32]) {
      mbar_wait(&kv_full[ist], iph);
      wgmma_fence();
      issue_s(sx, ist);
      if (++ist == p.stages) {
        ist = 0;
        iph ^= 1;
      }
    };
    // Every path through the loop reaches each wait with the same groups in flight (ptxas serialises every wgmma of the
    // kernel when it cannot prove that): one consumer step per tail shape, T = 1 apart.
    auto step = [&](float (&cur)[32], float (&nxt)[32], int j) {   // P_j in pa, S_{j+1} in flight into cur
      wgmma_fence();
      issue_pv(st);
      next_s(nxt);
      wgmma_wait<2>();
      wgmma_fence_regs(cur);
      softmax(cur, j + 1);
      wgmma_wait<1>();
      pv_done(st);
      rescale();
      pack(cur);
      if (++st == p.stages) st = 0;
    };
    auto last = [&](float (&cur)[32], int j) {   // j = T - 2: no S_{j+2}
      wgmma_fence();
      issue_pv(st);
      wgmma_wait<1>();
      wgmma_fence_regs(cur);
      softmax(cur, j + 1);
      wgmma_wait<0>();
      pv_done(st);
      rescale();
      pack(cur);
      if (++st == p.stages) st = 0;
    };
    next_s(s);
    if (T == 1) {
      wgmma_wait<0>();
      wgmma_fence_regs(s);
      softmax(s, 0);
      pack(s);
    } else {
      next_s(s2);
      wgmma_wait<1>();
      wgmma_fence_regs(s);
      softmax(s, 0);
      pack(s);
      for (int j = 0;; j += 2) {   // S_{j+1} in flight into s2
        if (j + 2 >= T) {
          last(s2, j);
          break;
        }
        step(s2, s, j);
        if (j + 3 >= T) {
          last(s, j + 1);
          break;
        }
        step(s, s2, j + 1);
      }
    }
  } else {
  mbar_wait(&kv_full[0], 0);
  wgmma_fence();
  issue_s(s, 0);
  wgmma_wait<0>();
  wgmma_fence_regs(s);
  softmax(s, 0);
  pack(s);
  for (int j = 0; j + 1 < T; ++j) {
    int st1 = st + 1;
    uint32_t phase1 = phase;
    if (st1 == p.stages) {
      st1 = 0;
      phase1 ^= 1;
    }
    mbar_wait(&kv_full[st1], phase1);
    wgmma_fence();
    issue_s(s, st1);
    issue_pv(st);
    wgmma_wait<1>();
    wgmma_fence_regs(s);
    softmax(s, j + 1);
    wgmma_wait<0>();
    pv_done(st);
    rescale();
    pack(s);
    st = st1;
    phase = phase1;
  }
  }
  wgmma_fence();
  issue_pv(st);   // the last step has no successor to overlap
  wgmma_wait<0>();
  pv_done(st);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float lt = l[h];
    lt += __shfl_xor_sync(0xffffffffu, lt, 1);
    lt += __shfl_xor_sync(0xffffffffu, lt, 2);
    const float inv = 1.f / lt;
    const int qrow = (q_tile * NCONS + wg) * kFaRows + (warp & 3) * 16 + (lane >> 2) + 8 * h;
    if (qrow < p.Nq) {   // per row: a tile may run past the frame, into the next frame's rows
      __nv_bfloat16* op = p.out + ((long long)bq * p.Nq + qrow) * p.ldo + head * HD;
#pragma unroll
      for (int g = 0; g < HD / 8; ++g)
        *reinterpret_cast<uint32_t*>(op + g * 8 + cq) = pack_bf16(o[4 * g + 2 * h] * inv, o[4 * g + 2 * h + 1] * inv);
    }
  }
}

template <auto Kernel>
static cudaError_t launch_fa(dim3 grid, int threads, size_t smem, cudaStream_t st, const CUtensorMap& mQ,
                             const CUtensorMap& mK, const CUtensorMap& mV, const FaArgs& a) {
  static bool configured = false;
  if (!configured) {
    const cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  return launch_k(Kernel, grid, dim3(threads), smem, st, mQ, mK, mV, a);
}

// Fallback for key counts the tensor-core tiling cannot express (Nk < 16 or Nk % 16 != 0, e.g. the 2x2 / 12x12
// maps of reduced test resolutions): one warp per (batch, head, query), exact softmax, CUDA cores.
struct GaArgs {
  const __nv_bfloat16* q; long long ldq;
  const __nv_bfloat16* k; long long ldk;
  const __nv_bfloat16* v; long long ldv;
  __nv_bfloat16* out; long long ldo;
  int Bq, Nq, Nk, heads, hd, kv_div;
  float scale;
};

__global__ void __launch_bounds__(128) generic_attn_kernel(const GaArgs p) {
  pdl_enter();
  extern __shared__ float sc_all[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* sc = sc_all + warp * p.Nk;
  const long long item = (long long)blockIdx.x * 4 + warp;
  const long long total = (long long)p.Bq * p.heads * p.Nq;
  if (item >= total) return;
  const int qi = (int)(item % p.Nq);
  const int head = (int)((item / p.Nq) % p.heads);
  const int b = (int)(item / ((long long)p.Nq * p.heads));
  const __nv_bfloat16* qp = p.q + ((long long)b * p.Nq + qi) * p.ldq + head * p.hd;
  const long long kv0 = (long long)(b / p.kv_div) * p.Nk;
  float mx = -INFINITY;
  for (int j = lane; j < p.Nk; j += 32) {
    const __nv_bfloat16* kp = p.k + (kv0 + j) * p.ldk + head * p.hd;
    float acc = 0.f;
    for (int c = 0; c < p.hd; c += 2) {
      const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(qp + c));
      const float2 bb = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(kp + c));
      acc += a.x * bb.x + a.y * bb.y;
    }
    acc *= p.scale;
    sc[j] = acc;
    mx = fmaxf(mx, acc);
  }
  for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
  for (int j = lane; j < p.Nk; j += 32) {
    const float e = __expf(sc[j] - mx);
    sc[j] = e;
    sum += e;
  }
  for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  __syncwarp();
  const float inv = 1.f / sum;
  for (int c = lane * 2; c < p.hd; c += 64) {
    float o0 = 0.f, o1 = 0.f;
    for (int j = 0; j < p.Nk; ++j) {
      const float2 vv = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p.v + (kv0 + j) * p.ldv + head * p.hd + c));
      o0 += sc[j] * vv.x;
      o1 += sc[j] * vv.y;
    }
    *reinterpret_cast<__nv_bfloat162*>(p.out + ((long long)b * p.Nq + qi) * p.ldo + head * p.hd + c) =
        __floats2bfloat162_rn(o0 * inv, o1 * inv);
  }
}

}  // namespace vx

using namespace vx;

// VX_FA_V1: every head dim on flash_attn_wgmma_kernel (A/B switch, read once; the tools and tests that time or compare the
// two loops in one process re-read it through vx_flash_reload_env).
static bool& fa_v1() {
  static bool v = getenv("VX_FA_V1") != nullptr;
  return v;
}
extern "C" void vx_flash_reload_env() { fa_v1() = getenv("VX_FA_V1") != nullptr; }

// q: [Bq*Nq, ldq], k/v: [Bkv*Nk, ldk] / [.., ldv] (bf16, heads*hd columns used), out: [Bq*Nq, ldo].
// kv batch of query batch b is b / kv_div.
extern "C" int vx_flash_attention(const void* q, long long ldq, const void* k, long long ldk, const void* v,
                                  long long ldv, void* out, long long ldo, int Bq, int Nq, int Bkv, int Nk, int heads,
                                  int hd, int kv_div, void* stream) {
  VX_REQUIRE(hd % 8 == 0 && hd <= 256, "vx_flash_attention: hd=%d unsupported", hd);
  VX_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0, "vx_flash_attention: ld must be %%8");
  VX_REQUIRE(kv_div >= 1 && (Bq + kv_div - 1) / kv_div <= Bkv, "vx_flash_attention: kv_div=%d Bq=%d Bkv=%d", kv_div, Bq, Bkv);
  if (Nk < 16 || Nk % 16 != 0) {
    VX_REQUIRE(Nk * 4 * 4 <= 48 * 1024, "vx_flash_attention: Nk=%d not a multiple of 16 and too long for the fallback", Nk);
    GaArgs g{(const __nv_bfloat16*)q, ldq, (const __nv_bfloat16*)k, ldk, (const __nv_bfloat16*)v, ldv,
             (__nv_bfloat16*)out, ldo, Bq, Nq, Nk, heads, hd, kv_div, 1.0f / sqrtf((float)hd)};
    const long long items = (long long)Bq * heads * Nq;
    launch_k(generic_attn_kernel, dim3((unsigned)((items + 3) / 4)), dim3(128), (size_t)Nk * 4 * 4, (cudaStream_t)stream, g);
    VX_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
  const int hdp = (hd + 15) / 16 * 16;
  const bool pipe = fa_pipe_hd(hd) && !fa_v1();
  // query rows per CTA: 64 per consumer warpgroup (fa_pipe_ncons)
  const int ncons = pipe ? fa_pipe_ncons(hd, Nq) : 1;
  // K / V ring depth of the serial loop: two stages for the wide heads keep two CTAs per SM resident, three otherwise
  const int stages = pipe ? fa_pipe_stages(hd, ncons) : hdp > 96 ? 2 : 3;
  const size_t smem = (size_t)(ncons + 2 * stages) * kFaRows * hdp * 2 + 128 + 128;
  CUtensorMap mQ, mK, mV;
  const void* ptrs[3] = {q, k, v};
  const long long lds[3] = {ldq, ldk, ldv};
  const long long rows[3] = {(long long)Bq * Nq, (long long)Bkv * Nk, (long long)Bkv * Nk};
  CUtensorMap* maps[3] = {&mQ, &mK, &mV};
  for (int i = 0; i < 3; ++i) {
    uint64_t dims[3] = {8, (uint64_t)rows[i], (uint64_t)lds[i] / 8};
    uint64_t str[2] = {(uint64_t)lds[i] * 2, 16};
    uint32_t box[3] = {8, (uint32_t)kFaRows, (uint32_t)hd / 8};
    if (make_tmap_bf16(maps[i], ptrs[i], 3, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE)) return 1;
  }
  FaArgs a{};
  a.Nq = Nq; a.Nk = Nk; a.hd = hd; a.kv_div = kv_div; a.stages = stages;
  a.scale_log2 = 1.4426950408889634f / sqrtf((float)hd);
  a.out = (__nv_bfloat16*)out; a.ldo = ldo;
  const dim3 grid((Nq + ncons * kFaRows - 1) / (ncons * kFaRows), heads, Bq);
  if (pipe) {
    const cudaStream_t cs = (cudaStream_t)stream;
    cudaError_t e;
    switch (hd) {
#define VX_FA_CASE(H)                                                                                       \
    case H:                                                                                                 \
      if (ncons == fa_pipe_ncons(H, kFaRows + 1))                                                           \
        e = launch_fa<flash_attn_pipe_kernel<H, fa_pipe_ncons(H, kFaRows + 1)>>(grid, 128 * (ncons + 1), smem, cs, mQ, \
                                                                             mK, mV, a);                 \
      else e = launch_fa<flash_attn_pipe_kernel<H, 1>>(grid, 256, smem, cs, mQ, mK, mV, a);                    \
      break;
      VX_FA_CASE(8) VX_FA_CASE(16) VX_FA_CASE(24) VX_FA_CASE(32) VX_FA_CASE(40) VX_FA_CASE(48) VX_FA_CASE(56)
      VX_FA_CASE(80) VX_FA_CASE(160)
#undef VX_FA_CASE
      default: return fail("vx_flash_attention: hd=%d unsupported", hd);
    }
    VX_CHECK_CUDA(e);
    VX_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
  switch (hdp) {
#define VX_FA_CASE(H) \
    case H: VX_CHECK_CUDA(launch_fa<flash_attn_wgmma_kernel<H>>(grid, kFaThreads, smem, (cudaStream_t)stream, mQ, mK, mV, a)); break;
    VX_FA_CASE(16) VX_FA_CASE(32) VX_FA_CASE(48) VX_FA_CASE(64) VX_FA_CASE(80) VX_FA_CASE(96) VX_FA_CASE(112) VX_FA_CASE(128)
    VX_FA_CASE(144) VX_FA_CASE(160) VX_FA_CASE(176) VX_FA_CASE(192) VX_FA_CASE(208) VX_FA_CASE(224) VX_FA_CASE(240)
    VX_FA_CASE(256)
#undef VX_FA_CASE
    default: return fail("vx_flash_attention: hd=%d unsupported", hd);
  }
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}
