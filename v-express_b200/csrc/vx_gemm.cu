// wgmma GEMM / implicit-GEMM convolution for sm_90a (persistent, warp-specialised).
//
//   out[m, n] = (sum_k A[m, k] * W[n, k] + bias[n] + bias2[m / bias2_div, n]) * scale + residual[m, n]
//   GEGLU mode: W rows are packed per tile as (value | gate); out[m, j] = (v + bias_v) * gelu_erf(g + bias_g)
//
// A is bf16 row-major (K contiguous), W is bf16 [N, K] (K contiguous): both operands are K-major, so every
// 64-wide K block of a 128-row tile is one TMA box that lands in shared memory in the canonical 128B-swizzled
// K-major layout wgmma consumes.  Accumulation is fp32 in registers.
//
// Three producers share the same MMA + epilogue:
//   * plain GEMM, optionally split-K over two sources (A | A2) -- the `torch.cat([h, skip])` of the up blocks
//     (reference modules/unet_3d_blocks.py:694,831) folded into the K loop;
//   * 3x3 convolution, stride 1, pad 1, NHWC: K = 9 taps x Cin; for tap (dy,dx) the A box is the same pixel
//     rectangle shifted by (dy-1, dx-1) through a 4-D tensor map (C, W, H, N) whose out-of-bounds reads are
//     zero-filled by the TMA unit = the zero padding of nn.Conv2d (reference modules/resnet.py:9-17).
//
// One persistent CTA per SM walks output tiles (n fastest, so concurrently running CTAs share the A rows in L2).
// Roles (384 threads = three warpgroups): warp 0 = TMA producer, warp 1 = TMA store + residual prefetch;
// warpgroups 1 and 2 = MMA + epilogue.  Two consumer schedules:
//   * cooperative: both warpgroups take 64 rows of every 128-row tile (wgmma m64nBNk16, BN <= 256);
//   * ping-pong (PP, BN <= 160; plain GEMM and every convolution producer, not the LayerNorm / row-sum variants): warpgroup
//     w owns the whole 128 x BN tile of every item it = w mod 2 of the CTA (two m64nBNk16 per K step).  An order barrier
//     hands the tensor pipe over at mainloop boundaries, so one warpgroup's epilogue runs under the other's MMAs instead of
//     stalling the pipe.
//   wgmma -> bias/scale (+ residual read from a TMA-prefetched, 64B-swizzled smem tile) -> bf16 -> same smem
//   tile -> TMA store (coalesced, clipped at the M/N edges by the tensor map).  While the consumers run their
// epilogue, the producer already fills the ring with the next tile's operands.  Both schedules add the same products in
// the same K order and round at the same points: their outputs are bit-identical.
// setmaxnreg moves registers from the producer warpgroup (40 per thread) to the consumers (232): room for 2 x 80 fp32
// accumulators per thread at ping-pong BN 160.
//
// e4m3 operands (TIn = __nv_fp8_e4m3, vx_gemm_fp8; plain producer, linear / GEGLU epilogues, both schedules): a 128-element
// e4m3 K block is the same 128-byte swizzled row as a 64-element bf16 block, so stages, TMA boxes (UINT8 maps),
// descriptors and shared-memory budget keep their byte geometry; each stage is four m64nBNk32 e4m3 steps instead of four
// m64nBNk16 bf16 steps.  The epilogue multiplies the fp32 accumulator by a_scale[m] * w_scale[n] (per-row activation
// scale, per-output-channel weight scale) before bias / GEGLU / scale / residual.  One accumulator runs over the whole K,
// as for bf16: the tensor cores add e4m3 products with fewer bits than fp32 (about 14; measured on H100: 2^-14.4 of
// sum |a_k w_k| at K = 64, 2^-11.3 at K = 1280), which is far below the 2^-4 rounding of the e4m3 operands themselves
// (tests/test_fp8_gpu.py states the accumulator model its bound assumes; DESIGN section 3 why there is no promotion).
#include <cuda_fp8.h>
#include "vx_host.h"
#include "vx_ptx.cuh"

namespace vx {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;                            // bf16 elements per K block (128 bytes; 128 e4m3 elements)
constexpr int kThreads = 384;
constexpr int kEpiThreads = 256;
constexpr int kPPMaxBN = 160;  // ping-pong: 2 x BN / 2 accumulators per thread; BN 192 spills at the consumers' 232 registers
constexpr int kPanelCols = 32;                         // staging panel: 32 bf16 = 64 B rows, 64B swizzle
constexpr int kPanelBytes = kBlockM * kPanelCols * 2;  // 8 KB
constexpr int kSmemCap = 227 * 1024;
constexpr int kSmemReserve = 2048;                     // 1024-B alignment slack + barriers

struct GemmArgs {
  int M, N;        // N = number of accumulator columns overall (2x the output width in GEGLU mode)
  int kblocks1;    // 64-wide K blocks taken from A (per tap for conv)
  int kblocks2;    // ... then from A2 (plain mode only)
  int taps;        // 1 = plain GEMM, 9 = 3x3 conv, 4 = nearest-2x upsample folded into the 3x3 conv (see `ups`)
  int rr;          // 3x3 conv "row reuse": one A box of hbox + 2 image rows per (dx, channel block) feeds the three dy taps
  int a_bytes;     // bytes of one A stage tile (128 rows x 128 B, or (hbox + 2) * W rows x 128 B with rr)
  int ups;         // 1: output parity classes (py, px) of conv3x3(upsample2x(x)) as four 2x2 convolutions on x (vx_upconv3x3_bf16)
  int block_n;     // wgmma N (the kernel's BN)
  int pp;          // host only: 1 = ping-pong instantiation (pick_block_n), 0 = cooperative
  int stages;
  int nbuf;        // staging tiles (2 when shared memory allows: TMA store/residual latency fully hidden)
  int rows_valid;  // output rows covered by one tile (128 for plain; wbox*hbox*nbox for conv)
  int W, H;        // conv OUTPUT image size (= input size at stride 1)
  int cstride;     // conv stride (1 | 2): tap (dy, dx) of output pixel (y, x) reads input pixel (cstride * y + dy, cstride * x + dx)
  int cpad;        // conv padding on the low side (1: nn.Conv2d(padding=1); 0: F.pad(x, (0, 1, 0, 1)) + padding 0)
  int tiles_m, tiles_n;
  int geglu;
  int has_residual;
  int out_f32;     // 1: `out` is float* written directly (attention scores feeding an fp32 softmax)
  const float* bias;
  const float* bias2;
  int bias2_div;
  float scale;
  float* out32;
  long long ldc;
  // LayerNorm folded into the epilogue (LNF instantiations only): out = rstd[m] * (acc - mean[m] * colsum[n]) + bias[n]
  // with W pre-multiplied by gamma, colsum[n] = sum_k W'[n,k], bias[n] = sum_k beta[k] W[n,k] + b[n]
  const float* ln_stats;    // [M][2] = (mean, rstd) of the un-normalised rows of A (null with `ares`)
  const float* ln_colsum;   // [N]
  // A-resident LayerNorm GEMM (LNF instantiations, K <= 512): a CTA keeps the K blocks of ONE 128-row tile of A in shared
  // memory while it walks ALL column tiles of that row tile (only W streams through the TMA ring); the consumer threads
  // compute the row statistics from the resident tile -- no statistics pass, no LayerNorm pass, 1/tiles_n of the A traffic.
  int ares;
  int ares_bytes;           // kblocks1 x 16 KB
  // LayerNorm statistics handed from the producer GEMM to the consumer GEMM (no statistics pass over the activations):
  //   producer (linear epilogue): rs_out[(tile_n * 2 + half) * rs_stride + m] = (sum, sum of squares) of the bf16-ROUNDED
  //     outputs of row m in one half of the column tile -- 2 * tiles_n partials per row;
  //   consumer (LNF instantiations): mean / rstd of row m from ln_nparts such partials, summed in slot order
  //     (deterministic), variance = E[x^2] - mean^2 in fp32, eps = ln_eps, channel count 1 / ln_invK.
  float2* rs_out;
  long long rs_stride;
  const float2* ln_parts;
  long long ln_pstride;
  int ln_nparts;
  float ln_invK;
  float ln_eps;
  // e4m3 instantiations: out = acc * a_scale[m] * w_scale[n] before the rest of the epilogue (null for bf16)
  const float* a_scale;   // [M]
  const float* w_scale;   // [N] (GEGLU: in the packed value|gate column order of W)
};

__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_5d(const CUtensorMap* m, const void* src, int c0, int c1, int c2, int c3, int c4) {
  asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// erf-GELU with erf from Abramowitz & Stegun 7.1.28 (|error| < 3e-7, i.e. exact at bf16 precision):
// erf(x) = 1 - (1 + a1 x + ... + a6 x^6)^-16 for x >= 0.  ~13 FMA-pipe instructions + one MUFU.RCP instead of
// libdevice erff (the GEGLU epilogue is erf-bound: 128 x 128 erf evaluations per tile).
__device__ __forceinline__ float gelu_erf(float g) {
  const float x = fabsf(g) * 0.70710678118654752f;
  float pl = fmaf(x, 0.0000430638f, 0.0002765672f);
  pl = fmaf(x, pl, 0.0001520143f);
  pl = fmaf(x, pl, 0.0092705272f);
  pl = fmaf(x, pl, 0.0422820123f);
  pl = fmaf(x, pl, 0.0705230784f);
  pl = fmaf(x, pl, 1.0f);
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(pl));
  r *= r; r *= r; r *= r; r *= r;          // ^16
  const float erf_abs = 1.0f - r;
  return 0.5f * g * (1.0f + copysignf(erf_abs, g));
}

// sum over the four lanes of a quad (the lanes that hold one accumulator row)
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  return v;
}

// staging tile: panel (col / 32) of 128 rows x 64 B, 64B swizzle: byte offset o = row * 64 + (col % 32) * 2 is stored at
// o ^ (((o >> 7) & 3) << 4)
__device__ __forceinline__ uint32_t* staging_word(uint8_t* buf, int row, int col) {
  uint32_t o = (uint32_t)(row * 64 + (col & 31) * 2);
  o ^= ((o >> 7) & 3u) << 4;
  return reinterpret_cast<uint32_t*>(buf + (col >> 5) * kPanelBytes + o);
}

// One 32-byte K step of both K-major operands (m64nBNk16 bf16 or m64nBNk32 e4m3) from shared memory.
template <int BN, typename TIn>
__device__ __forceinline__ void mma_step(float (&d)[BN / 2], uint64_t da, uint64_t db, int scale_d) {
  if constexpr (sizeof(TIn) == 1) WgmmaE4m3<BN>::ss(d, da, db, scale_d);
  else Wgmma<BN>::template ss<0, 0>(d, da, db, scale_d);
}

// wgmma accumulator fragment of m64nBN (per thread): element 4 * g + 2 * h + e sits at row 16 * warp + lane / 4 + 8 * h,
// column 8 * g + 2 * (lane % 4) + e of the warpgroup's 64 x BN block.  Ping-pong: acc[mh] is the block of rows
// [64 mh, 64 mh + 64) of the tile.  TIn: operand type (__nv_bfloat16, or __nv_fp8_e4m3 with the scaled epilogue).
template <int BN, bool LNF, bool PP, typename TIn>
__global__ void __launch_bounds__(kThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapA2,
                  const __grid_constant__ CUtensorMap mapB, const __grid_constant__ CUtensorMap mapR,
                  const __grid_constant__ CUtensorMap mapC, const GemmArgs p) {
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment required by the 128B swizzle atom
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr bool F8 = sizeof(TIn) == 1;
  static_assert(!(F8 && LNF), "e4m3: plain producer only");
  constexpr int KE = kBlockK * 2 / (int)sizeof(TIn);   // elements per 128-byte K block (TMA coordinates)
  const int a_bytes = p.a_bytes;
  constexpr int b_bytes = BN * kBlockK * 2;
  const int nbt = p.rr ? 3 : 1;                         // W tiles per stage (rr: the three dy taps of one dx)
  const int stage_bytes = a_bytes + nbt * b_bytes;
  uint8_t* ring = smem;                         // TMA ring (behind the resident A tile in `ares` mode)
  if constexpr (LNF) ring += p.ares ? p.ares_bytes : 0;
  uint8_t* sC = ring + p.stages * stage_bytes;  // staging: out_cols / 32 panels of 8 KB
  const int out_cols = p.geglu ? BN / 2 : BN;
  const int npanels = out_cols / kPanelCols;
  const int buf_bytes = npanels * kPanelBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sC + (p.out_f32 ? 0 : p.nbuf * buf_bytes));
  uint64_t* empty_bar = full_bar + p.stages;
  uint64_t* c_ready = empty_bar + p.stages;    // [2] staging tile b free (+ residual landed)
  uint64_t* staged = c_ready + 2;              // [2] staging tile b fully written by the epilogue threads
  uint64_t* a_land = staged + 2;               // [8] `ares`: K block of the resident tile landed
  uint64_t* a_empty = a_land + 8;              // [8] `ares`: K block released (last column tile of the row tile done)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int total_kb = p.rr ? 3 * p.kblocks1 : p.taps * p.kblocks1 + p.kblocks2;   // ring stages per output tile
  const int tiles_per_par = p.tiles_m * p.tiles_n;
  const int num_tiles = tiles_per_par * (p.ups ? 4 : 1);   // ups: (parity, row tile, column tile), parity slowest
  // the it-th output tile of this CTA as a flat (row tile, column tile) index, or -1 past the end.  Default: tiles strided
  // over the grid, n fastest.  `ares`: row tiles strided over the grid, each walked through all its column tiles.
  auto item_at = [&](int it) -> int {
    if constexpr (LNF) {
      if (p.ares) {
        const int g = (int)blockIdx.x + (it / p.tiles_n) * (int)gridDim.x;
        return g < p.tiles_m ? g * p.tiles_n + it % p.tiles_n : -1;
      }
    }
    const int t = (int)blockIdx.x + it * (int)gridDim.x;
    return t < num_tiles ? t : -1;
  };

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&mapA);
    tma_prefetch_desc(&mapB);
    if (p.kblocks2) tma_prefetch_desc(&mapA2);
    if (!p.out_f32) tma_prefetch_desc(&mapC);
    if (p.has_residual || p.ups) tma_prefetch_desc(&mapR);
    // ping-pong: a stage / staging tile is consumed by one warpgroup only
    constexpr int consumers = PP ? kEpiThreads / 2 : kEpiThreads;
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], consumers / 32);   // lane 0 of every consumer warp, once its MMAs on the stage completed
    }
    for (int s = 0; s < 2; ++s) {
      mbar_init(&c_ready[s], 1);
      mbar_init(&staged[s], consumers);
    }
    for (int s = 0; s < 8; ++s) {
      mbar_init(&a_land[s], 1);
      mbar_init(&a_empty[s], kEpiThreads / 32);
    }
    fence_barrier_init();
  }
  __syncthreads();
  // barrier init and the tensor-map prefetch overlapped the previous grid's tail; from here on every role touches global memory
  pdl_wait();

  // setmaxnreg is .sync.aligned per warpgroup: each one sits at the top of its warpgroup's branch, so that ptxas can give the
  // consumer code after it the raised budget (issued before the role branches, it is dropped: C7507).
  if (warp < 4) {
    setmaxnreg_dec<40>();   // producer / store warpgroup, idle warps 2 and 3 included: few registers
    if (warp == 0) {
      // ---------------------------------------------------------- TMA producer
      // The whole warp runs the loop in lock-step so that tile / coordinate / barrier values stay warp-uniform; only the
      // elected lane issues.
      const bool leader = elect_one();
      int stage = 0;
      uint32_t phase = 0;
      for (int it = 0, t = item_at(0); t >= 0; t = item_at(++it)) {
        const int par = t / tiles_per_par, tt = t - par * tiles_per_par;
        const int tile_n = tt % p.tiles_n, tile_m = tt / p.tiles_n;
        int n0 = 0, y0 = 0, x0 = 0;
        const long long m0 = (long long)tile_m * p.rows_valid;
        if (p.taps != 1) {
          const long long hw = (long long)p.H * p.W;
          n0 = (int)(m0 / hw);
          const int rem = (int)(m0 % hw);
          y0 = rem / p.W;
          x0 = rem % p.W;
        }
        const uint32_t tx_bytes = (uint32_t)((p.rr ? a_bytes : p.rows_valid * kBlockK * 2) + nbt * b_bytes);
        const int b_row = par * p.N + tile_n * BN;
        if constexpr (LNF) {
          if (p.ares && tile_n == 0) {
            // resident A: every K block of this row tile is loaded once, in front of the first column tile, into its own
            // slot -- all of them before any W stage, since the consumers take the row statistics before their first MMA
            for (int kb = 0; kb < p.kblocks1; ++kb) {
              mbar_wait(&a_empty[kb], (uint32_t)(((it / p.tiles_n) & 1) ^ 1));
              if (leader) {
                mbar_expect_tx(&a_land[kb], (uint32_t)(kBlockM * kBlockK * 2));
                tma_load_2d(smem + kb * (kBlockM * kBlockK * 2), &mapA, &a_land[kb], kb * kBlockK, (int)m0);
              }
            }
            __syncwarp();
          }
        }
        for (int kb = 0; kb < total_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = ring + stage * stage_bytes;
          uint8_t* sb = sa + a_bytes;
          const int tap = p.taps != 1 ? kb / p.kblocks1 : 0;     // rr: tap = dx index (0..2)
          const int cb = kb - tap * p.kblocks1;
          if constexpr (LNF) {
            if (p.ares) {
              if (leader) {
                mbar_expect_tx(&full_bar[stage], (uint32_t)b_bytes);
                tma_load_2d(ring + stage * stage_bytes, &mapB, &full_bar[stage], kb * kBlockK, b_row);
              }
              __syncwarp();
              if (++stage == p.stages) {
                stage = 0;
                phase ^= 1;
              }
              continue;
            }
          }
          if (leader) {
            mbar_expect_tx(&full_bar[stage], tx_bytes);
            if (p.rr) {
              // A: image rows y0 - 1 .. y0 + hbox of the column window shifted by dx (zero-filled outside the image =
              // padding); W: the three taps (dy, dx), dy = 0..2, of this channel block
              tma_load_4d(sa, &mapA, &full_bar[stage], cb * kBlockK, x0 + tap - 1, y0 - 1, n0);
  #pragma unroll
              for (int dyi = 0; dyi < 3; ++dyi)
                tma_load_2d(sb + dyi * b_bytes, &mapB, &full_bar[stage], ((dyi * 3 + tap) * p.kblocks1 + cb) * kBlockK, b_row);
            } else {
              // 3x3: taps (dy, dx) in {-1, 0, 1}^2.  Folded upsample: output pixel (2i + py, 2j + px) reads the 2x2 input
              // neighbourhood rows i + py - 1 + {0, 1}, columns j + px - 1 + {0, 1} (weights pre-summed per parity on the host).
              const int dy = p.ups ? (tap >> 1) + (par >> 1) - 1 : tap / 3 - p.cpad;
              const int dx = p.ups ? (tap & 1) + (par & 1) - 1 : tap % 3 - p.cpad;
              if (p.taps != 1) {
                tma_load_4d(sa, &mapA, &full_bar[stage], cb * kBlockK, x0 * p.cstride + dx, y0 * p.cstride + dy, n0);
              } else if (kb < p.kblocks1) {
                tma_load_2d(sa, &mapA, &full_bar[stage], kb * KE, (int)m0);
              } else {
                tma_load_2d(sa, &mapA2, &full_bar[stage], (kb - p.kblocks1) * KE, (int)m0);
              }
              tma_load_2d(sb, &mapB, &full_bar[stage], kb * KE, b_row);
            }
          }
          __syncwarp();
          if (++stage == p.stages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    } else if (warp == 1) {
      // ---------------------------------------------------------- TMA store + residual prefetch (one lane)
      if (lane == 0 && !p.out_f32) {
        const uint32_t res_bytes = (uint32_t)(p.rows_valid * out_cols * 2);
        auto arm = [&](int t, int b) {  // make staging tile b usable for output tile t
          if (p.has_residual) {   // (never with ups: the upsampler convs have no residual)
            const int tn_ = t % p.tiles_n, tm_ = t / p.tiles_n;
            mbar_expect_tx(&c_ready[b], res_bytes);
            for (int pn = 0; pn < npanels; ++pn)
              tma_load_2d(sC + b * buf_bytes + pn * kPanelBytes, &mapR, &c_ready[b], tn_ * out_cols + pn * kPanelCols,
                          tm_ * p.rows_valid);
          } else {
            mbar_arrive(&c_ready[b]);
          }
        };
        for (int b = 0; b < p.nbuf; ++b)
          if (item_at(b) >= 0) arm(item_at(b), b);
        for (int it = 0, t = item_at(0); t >= 0; t = item_at(++it)) {
          const int b = it % p.nbuf;
          const int par = t / tiles_per_par, tt = t - par * tiles_per_par;
          const int tile_n = tt % p.tiles_n, tile_m = tt / p.tiles_n;
          mbar_wait(&staged[b], (uint32_t)((it / p.nbuf) & 1));
          if (p.ups) {
            // rows of the tile = low-resolution pixels (n, i, j); they land on (n, 2i + py, 2j + px): 5-D map (c, j, i, n, py)
            // per px (mapC: px = 0, mapR: px = 1)
            const long long m0 = (long long)tile_m * p.rows_valid, hw = (long long)p.H * p.W;
            const int n0 = (int)(m0 / hw), rem = (int)(m0 % hw);
            const CUtensorMap* mo = (par & 1) ? &mapR : &mapC;
            if (m0 < p.M)
              for (int pn = 0; pn < npanels; ++pn)
                tma_store_5d(mo, sC + b * buf_bytes + pn * kPanelBytes, tile_n * out_cols + pn * kPanelCols, rem % p.W,
                             rem / p.W, n0, par >> 1);
          } else {
            for (int pn = 0; pn < npanels; ++pn)
              tma_store_2d(&mapC, sC + b * buf_bytes + pn * kPanelBytes, tile_n * out_cols + pn * kPanelCols,
                           tile_m * p.rows_valid);
          }
          tma_store_commit();
          const int tnext = item_at(it + p.nbuf);
          if (tnext >= 0) {
            tma_store_wait_read();  // the store has finished reading tile b
            arm(tnext, b);
          }
        }
        tma_store_wait_all();
      }
    }
  } else {
    setmaxnreg_inc<232>();   // consumer warpgroups: the registers the producer warpgroup gave up
    // -------------------------------------------------------------- MMA + epilogue (warpgroups 1, 2)
    static_assert(!(PP && LNF) && (!PP || BN <= kPPMaxBN), "ping-pong: plain epilogues, BN <= 160");
    constexpr int MH = PP ? 2 : 1;                  // 64-row accumulator blocks per warpgroup
    const int wg = (threadIdx.x >> 7) - 1;          // cooperative: rows [64 wg, 64 wg + 64) of the tile; PP: items wg mod 2
    const int wrow = (PP ? 0 : wg * 64) + (warp & 3) * 16 + (lane >> 2);   // + 8 h (+ 64 mh): the rows of this thread
    const int cq = (lane & 3) * 2;                  // + 8 g: the column pair of this thread in column group g
    float acc[MH][BN / 2];
#pragma unroll
    for (int mh = 0; mh < MH; ++mh)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[mh][i] = 0.f;
    float ln_mean[2] = {0.f, 0.f}, ln_rstd[2] = {1.f, 1.f};
    // PP order barrier (named barriers 1, 2; 128 threads arrive, 128 wait): warpgroup w waits on 1 + w before the mainloop
    // of each item but its first and, once its MMAs are issued, lets the other warpgroup go if the CTA has a next item.
    // Every arrive is matched by exactly one wait.
    for (int it = PP ? wg : 0, t = item_at(it); t >= 0; it += PP ? 2 : 1, t = item_at(it)) {
      // ring position of the item's first K block: the producer fills the ring in item order, total_kb stages per item
      const long long g0 = (long long)it * total_kb;
      int stage = (int)(g0 % p.stages);
      uint32_t phase = (uint32_t)((g0 / p.stages) & 1);
      if constexpr (PP) {
        if (it > 0) asm volatile("bar.sync %0, 256;" ::"r"(1 + wg) : "memory");
      }
      const int tt = t % tiles_per_par;
      const int tile_n = tt % p.tiles_n, tile_m = tt / p.tiles_n;
      bool a_last = false;   // ares: last column tile of the row tile -> its MMAs release the resident K blocks
      if constexpr (LNF) {
        if (p.ares) {
          a_last = tile_n == p.tiles_n - 1;
          if (tile_n == 0) {
            // row statistics of the new row tile from the resident K blocks (128B-swizzled K-major: row r of K block kb = 128
            // bytes at kb * 16 KB + r * 128, its eight 16-byte chunks permuted -- sums do not care).  The four lanes of a quad
            // share the thread's two rows and take two chunks each.  Two passes: the textbook variance, not E[x^2] - mean^2.
            const uint32_t a_phase = (uint32_t)((it / p.tiles_n) & 1);
            float s[2] = {0.f, 0.f};
            for (int kb = 0; kb < p.kblocks1; ++kb) {
              mbar_wait(&a_land[kb], a_phase);
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const uint8_t* rowp = smem + kb * (kBlockM * kBlockK * 2) + (wrow + 8 * h) * 128;
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                  const uint4 q = *reinterpret_cast<const uint4*>(rowp + ((lane & 3) + 4 * j) * 16);
                  const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
                  for (int i = 0; i < 4; ++i) {
                    const float2 f2 = unpack_bf16(w[i]);
                    s[h] += f2.x + f2.y;
                  }
                }
              }
            }
            const float invK = 1.0f / (float)(p.kblocks1 * kBlockK);
#pragma unroll
            for (int h = 0; h < 2; ++h) ln_mean[h] = quad_sum(s[h]) * invK;
            float q2[2] = {0.f, 0.f};
            for (int kb = 0; kb < p.kblocks1; ++kb) {
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const uint8_t* rowp = smem + kb * (kBlockM * kBlockK * 2) + (wrow + 8 * h) * 128;
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                  const uint4 q = *reinterpret_cast<const uint4*>(rowp + ((lane & 3) + 4 * j) * 16);
                  const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
                  for (int i = 0; i < 4; ++i) {
                    const float2 f2 = unpack_bf16(w[i]);
                    const float d0 = f2.x - ln_mean[h], d1 = f2.y - ln_mean[h];
                    q2[h] = fmaf(d0, d0, q2[h]);
                    q2[h] = fmaf(d1, d1, q2[h]);
                  }
                }
              }
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) ln_rstd[h] = rsqrtf(quad_sum(q2[h]) * invK + p.ln_eps);
          }
        }
      }
      // ------------------------------------------------------------ main loop: one ring stage per 64-wide K block
      int prev = -1;
      for (int kb = 0; kb < total_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        uint32_t sa = smem_u32(ring + stage * stage_bytes);
        const uint32_t sb = sa + (uint32_t)a_bytes;
        if constexpr (LNF) {
          if (p.ares) sa = smem_u32(smem + kb * (kBlockM * kBlockK * 2));
        }
        if constexpr (!PP) sa += (uint32_t)(wg * 64 * 128);
        wgmma_fence();
        if (p.rr) {
          // tap dy reads the 128 tile rows that start dy image rows (W x 128 B, a multiple of the 1024-B swizzle atom)
          // into the A box, against its own W tile
#pragma unroll
          for (int dyi = 0; dyi < 3; ++dyi) {
            const uint64_t db = make_smem_desc(sb + (uint32_t)(dyi * b_bytes), 16, 1024, SWZ_128B);
#pragma unroll
            for (int k = 0; k < kBlockK / 16; ++k)   // +32 bytes per K step = +2 in the (addr >> 4) field
#pragma unroll
              for (int mh = 0; mh < MH; ++mh) {
                const uint64_t da = make_smem_desc(sa + (uint32_t)(dyi * p.W * 128 + mh * 64 * 128), 16, 1024, SWZ_128B);
                mma_step<BN, TIn>(acc[mh], da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), (kb | dyi | k) != 0);
              }
          }
        } else {
          const uint64_t db = make_smem_desc(sb, 16, 1024, SWZ_128B);
#pragma unroll
          for (int k = 0; k < kBlockK / 16; ++k)   // four 32-byte K steps: k16 bf16 or k32 e4m3
#pragma unroll
            for (int mh = 0; mh < MH; ++mh) {   // PP: rows 64 mh.. of the A tile, 64 x 128 B further on
              const uint64_t da = make_smem_desc(sa + (uint32_t)(mh * 64 * 128), 16, 1024, SWZ_128B);
              mma_step<BN, TIn>(acc[mh], da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), (kb | k) != 0);
            }
        }
        wgmma_commit();
        wgmma_wait<1>();                              // the MMAs of the previous stage have completed: release it
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == p.stages) {
          stage = 0;
          phase ^= 1;
        }
      }
      if constexpr (PP) {   // MMAs issued: the other warpgroup's mainloop queues behind them while this one finishes
        if (item_at(it + 1) >= 0) asm volatile("bar.arrive %0, 256;" ::"r"(1 + (wg ^ 1)) : "memory");
      }
      wgmma_wait<0>();
#pragma unroll
      for (int mh = 0; mh < MH; ++mh) wgmma_fence_regs(acc[mh]);
      if (lane == 0) {
        mbar_arrive(&empty_bar[prev]);
        if constexpr (LNF) {
          if (a_last)
            for (int kb = 0; kb < p.kblocks1; ++kb) mbar_arrive(&a_empty[kb]);
        }
      }

      // ------------------------------------------------------------ epilogue
      const int sb = it % p.nbuf;
      if (!p.out_f32) mbar_wait(&c_ready[sb], (uint32_t)((it / p.nbuf) & 1));
      uint8_t* buf = sC + sb * buf_bytes;
      const int nbase = tile_n * BN;  // accumulator column base (bias index)
#pragma unroll
      for (int mh = 0; mh < MH; ++mh) {   // PP: the two 64-row blocks one after the other (fewer live registers)
        const int rbase = wrow + 64 * mh;
        float (&ac)[BN / 2] = acc[mh];
        long long m[2];
        bool row_ok[2];
        const float* b2[2];
        float as[2] = {1.f, 1.f};   // e4m3: activation scale of the thread's two rows
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = rbase + 8 * h;
          m[h] = (long long)tile_m * p.rows_valid + r;
          row_ok[h] = r < p.rows_valid && m[h] < p.M;
          b2[h] = p.bias2 ? p.bias2 + (row_ok[h] ? (m[h] / p.bias2_div) : 0) * (long long)p.N : nullptr;
          if constexpr (F8) as[h] = row_ok[h] ? __ldg(p.a_scale + m[h]) : 0.f;
          if constexpr (LNF) {
            if (p.ares) {
            } else if (p.ln_parts) {
              if (row_ok[h]) {
                float s1 = 0.f, s2 = 0.f;
                for (int j = 0; j < p.ln_nparts; ++j) {
                  const float2 v = __ldg(p.ln_parts + (long long)j * p.ln_pstride + m[h]);
                  s1 += v.x;
                  s2 += v.y;
                }
                ln_mean[h] = s1 * p.ln_invK;
                ln_rstd[h] = rsqrtf(fmaxf(fmaf(-ln_mean[h], ln_mean[h], s2 * p.ln_invK), 0.f) + p.ln_eps);
              }
            } else if (row_ok[h]) {
              const float2 st = *reinterpret_cast<const float2*>(p.ln_stats + 2 * m[h]);
              ln_mean[h] = st.x;
              ln_rstd[h] = st.y;
            }
          }
        }
        if (p.geglu) {
          constexpr int G2 = BN / 16;   // value column groups; the gate of group g is group g + G2
#pragma unroll
          for (int g = 0; g < G2; ++g) {
            const int nl = g * 8 + cq;
            const int nv = nbase + nl, ng = nbase + BN / 2 + nl;
            const float2 bv = p.bias ? *reinterpret_cast<const float2*>(p.bias + nv) : make_float2(0.f, 0.f);
            const float2 bg = p.bias ? *reinterpret_cast<const float2*>(p.bias + ng) : make_float2(0.f, 0.f);
            float2 sv = make_float2(0.f, 0.f), sg = make_float2(0.f, 0.f);
            if constexpr (LNF) {
              sv = *reinterpret_cast<const float2*>(p.ln_colsum + nv);
              sg = *reinterpret_cast<const float2*>(p.ln_colsum + ng);
            }
            float2 wv = make_float2(1.f, 1.f), wg2 = make_float2(1.f, 1.f);
            if constexpr (F8) {
              wv = __ldg(reinterpret_cast<const float2*>(p.w_scale + nv));
              wg2 = __ldg(reinterpret_cast<const float2*>(p.w_scale + ng));
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float v0 = ac[4 * g + 2 * h], v1 = ac[4 * g + 2 * h + 1];
              float g0 = ac[4 * (g + G2) + 2 * h], g1 = ac[4 * (g + G2) + 2 * h + 1];
              if constexpr (F8) {
                v0 *= as[h] * wv.x;
                v1 *= as[h] * wv.y;
                g0 *= as[h] * wg2.x;
                g1 *= as[h] * wg2.y;
              }
              if constexpr (LNF) {
                v0 = ln_rstd[h] * (v0 - ln_mean[h] * sv.x);
                v1 = ln_rstd[h] * (v1 - ln_mean[h] * sv.y);
                g0 = ln_rstd[h] * (g0 - ln_mean[h] * sg.x);
                g1 = ln_rstd[h] * (g1 - ln_mean[h] * sg.y);
              }
              const float f0 = (v0 + bv.x) * gelu_erf(g0 + bg.x), f1 = (v1 + bv.y) * gelu_erf(g1 + bg.y);
              *staging_word(buf, rbase + 8 * h, nl) = pack_bf16(f0, f1);
            }
          }
        } else {
          float rs_sum[2][2] = {{0.f, 0.f}, {0.f, 0.f}}, rs_sq[2][2] = {{0.f, 0.f}, {0.f, 0.f}};   // [row][column half]
#pragma unroll
          for (int g = 0; g < BN / 8; ++g) {
            const int nl = g * 8 + cq;
            const int n = nbase + nl;
            const float2 bv = p.bias ? *reinterpret_cast<const float2*>(p.bias + n) : make_float2(0.f, 0.f);
            float2 cs = make_float2(0.f, 0.f);
            if constexpr (LNF) cs = *reinterpret_cast<const float2*>(p.ln_colsum + n);
            float2 ws = make_float2(1.f, 1.f);
            if constexpr (F8) ws = __ldg(reinterpret_cast<const float2*>(p.w_scale + n));
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float f0 = ac[4 * g + 2 * h], f1 = ac[4 * g + 2 * h + 1];
              if constexpr (F8) {
                f0 *= as[h] * ws.x;
                f1 *= as[h] * ws.y;
              }
              if constexpr (LNF) {
                f0 = ln_rstd[h] * (f0 - ln_mean[h] * cs.x);
                f1 = ln_rstd[h] * (f1 - ln_mean[h] * cs.y);
              }
              f0 += bv.x;
              f1 += bv.y;
              if (b2[h]) {
                const float2 t2 = *reinterpret_cast<const float2*>(b2[h] + n);
                f0 += t2.x;
                f1 += t2.y;
              }
              f0 *= p.scale;
              f1 *= p.scale;
              if (p.out_f32) {
                if (row_ok[h]) *reinterpret_cast<float2*>(p.out32 + m[h] * p.ldc + n) = make_float2(f0, f1);
                continue;
              }
              uint32_t* sp = staging_word(buf, rbase + 8 * h, nl);
              if (p.has_residual) {
                const float2 r2 = unpack_bf16(*sp);
                f0 += r2.x;
                f1 += r2.y;
              }
              const uint32_t pk = pack_bf16(f0, f1);
              *sp = pk;
              if (!PP && p.rs_out) {
                const float2 t2 = unpack_bf16(pk);
                const int half = nl >= BN / 2;
                rs_sum[h][half] += t2.x + t2.y;
                rs_sq[h][half] = fmaf(t2.x, t2.x, fmaf(t2.y, t2.y, rs_sq[h][half]));
              }
            }
          }
          if (!PP && p.rs_out) {
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int half = 0; half < 2; ++half) {
                const float s1 = quad_sum(rs_sum[h][half]), s2 = quad_sum(rs_sq[h][half]);
                if ((lane & 3) == 0 && row_ok[h]) p.rs_out[(long long)(tile_n * 2 + half) * p.rs_stride + m[h]] = make_float2(s1, s2);
              }
          }
        }
      }
      if (!p.out_f32) {
        fence_proxy_async_smem();     // staging writes -> visible to the TMA store (async proxy)
        mbar_arrive(&staged[sb]);
      }
    }
  }
}

// A/B switches (bring-up only) are read ONCE per process: the launch path never touches the environment
// (the sweep tools re-read them through vx_gemm_reload_env).
struct GemmEnv {
  int stages, nbuf, bn, verbose, conv_rr, pp;
  static int geti(const char* name, int dflt) {
    const char* s = getenv(name);
    return s ? atoi(s) : dflt;
  }
  GemmEnv() {
    stages = geti("VX_GEMM_STAGES", 0);
    nbuf = geti("VX_GEMM_NBUF", 0);
    bn = geti("VX_GEMM_BN", 0);
    verbose = geti("VX_GEMM_VERBOSE", 0);
    conv_rr = geti("VX_CONV_RR", 1);
    pp = geti("VX_GEMM_PP", -1);   // -1: schedule from the shape; 0: cooperative; 1: ping-pong wherever the kernel has it
  }
};
static GemmEnv& gemm_env() {
  static GemmEnv e;
  return e;
}

// column-tile widths the kernel is instantiated for
static bool bn_supported(int bn) {
  switch (bn) {
    case 16: case 32: case 64: case 96: case 128: case 160: case 192: case 256: return true;
    default: return false;
  }
}

// column-tile widths the ping-pong schedule is instantiated for
static bool pp_bn_supported(int bn) { return bn == 32 || bn == 64 || bn == 96 || bn == 128 || bn == 160; }

// Same-tile speed-up of the ping-pong schedule over the cooperative one on a CTA that walks two tiles or more (the
// epilogue and the tile-boundary drain of one warpgroup run under the other's MMAs), and the longest K loop (in 64-wide
// blocks) it pays on: beyond K = 1280 one warpgroup's mainloop, which waits on its own MMAs every stage, feeds the tensor
// pipe worse than two cooperative ones and the hidden epilogue no longer makes up for it.  Row-reuse convolutions are
// exempt (their ping-pong ring is deeper than the cooperative one).  Measured with tools/gemm_ab.py (DESIGN section 9).
constexpr double kPPGain = 1.12;
constexpr int kPPMaxKBlocks = 20;

// Pick the schedule and the wgmma N (only `fixed_bn` if it is set).  Among the supported widths (multiples of `gran` that
// divide N) and both schedules, minimise waves(tiles) x tile cost, waves = tiles per CTA of the persistent grid.
//   Cooperative tile: cycles per K block x K blocks + epilogue, cycles per 128 x bn x 64 block = max(MMA 4 bn,
//   shared-memory operand feed 128 + 2 bn at 128 B/clk: A once, W once per consumer warpgroup) + issue overhead.
//   Ping-pong (where `pp_ok`, bn <= pp_max_bn and, unless `pp_any_k`, total_kb <= kPPMaxKBlocks): the same tile cost /
//   kPPGain when a CTA gets two tiles or more.  With one tile per CTA (small M) there is no second tile to overlap and one
//   warpgroup would idle: the cooperative schedule.
// Ties go to the wider tile, then to the cooperative schedule.
// VX_GEMM_PP=0: cooperative only (the widths are the cost model's); 1: ping-pong at the widest width that divides N.
static int pick_block_n(long long tiles_m, int N, int gran, int total_kb, int fixed_bn = 0, bool pp_ok = false,
                        int* pp = nullptr, int pp_max_bn = kPPMaxBN, bool pp_any_k = false) {
  const int mode = gemm_env().pp;
  auto fits = [&](int bn) { return N % bn == 0 && bn % gran == 0 && bn_supported(bn) && (fixed_bn <= 0 || bn == fixed_bn); };
  if (pp) *pp = 0;
  pp_ok = pp_ok && pp && mode != 0;
  if (pp_ok && mode == 1) {
    for (int bn = kPPMaxBN; bn >= 32; bn -= 32)
      if (fits(bn) && pp_bn_supported(bn) && bn <= pp_max_bn) {
        *pp = 1;
        return bn;
      }
  }
  if (!pp_any_k && total_kb > kPPMaxKBlocks) pp_ok = false;
  const int sms = device_sms();
  int best = 0, best_pp = 0;
  double best_cost = 1e30;
  for (int bn = 256; bn >= gran; bn -= gran) {
    if (!fits(bn)) continue;
    const long long items = tiles_m * (N / bn);
    const long long waves = (items + sms - 1) / sms;
    const double cyc = (4.0 * bn > 128.0 + 2.0 * bn) ? 4.0 * bn : 128.0 + 2.0 * bn;
    const double cost = (double)waves * (total_kb * (cyc + 40.0) + 4.0 * bn);
    if (cost < best_cost * 0.999) {
      best_cost = cost;
      best = bn;
      best_pp = 0;
    }
    if (pp_ok && pp_bn_supported(bn) && bn <= pp_max_bn && waves >= 2 && cost / kPPGain < best_cost * 0.999) {
      best_cost = cost / kPPGain;
      best = bn;
      best_pp = 1;
    }
  }
  if (pp) *pp = best_pp;
  return best;
}

template <int BN, bool LNF, bool PP, typename TIn>
static cudaError_t launch_bn(const CUtensorMap& mA, const CUtensorMap& mA2, const CUtensorMap& mB, const CUtensorMap& mR,
                             const CUtensorMap& mC, const GemmArgs& a, int grid, size_t smem, cudaStream_t st) {
  static bool configured = false;
  if (!configured) {
    const cudaError_t e = cudaFuncSetAttribute(gemm_wgmma_kernel<BN, LNF, PP, TIn>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               kSmemCap);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  return launch_k((gemm_wgmma_kernel<BN, LNF, PP, TIn>), dim3(grid), dim3(kThreads), smem, st, mA, mA2, mB, mR, mC, a);
}

template <bool LNF>
static cudaError_t launch_lnf(const CUtensorMap& mA, const CUtensorMap& mA2, const CUtensorMap& mB, const CUtensorMap& mR,
                              const CUtensorMap& mC, const GemmArgs& a, int grid, size_t smem, cudaStream_t st) {
  using T = __nv_bfloat16;
  if constexpr (!LNF) {
    if (a.pp) {
      switch (a.block_n) {
        case 32: return launch_bn<32, false, true, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
        case 64: return launch_bn<64, false, true, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
        case 96: return launch_bn<96, false, true, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
        case 128: return launch_bn<128, false, true, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
        case 160: return launch_bn<160, false, true, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
        default: return cudaErrorInvalidValue;
      }
    }
  }
  switch (a.block_n) {
    case 16: return launch_bn<16, LNF, false, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
    case 32: return launch_bn<32, LNF, false, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
    case 64: return launch_bn<64, LNF, false, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
    case 96: return launch_bn<96, LNF, false, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
    case 128: return launch_bn<128, LNF, false, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
    case 160: return launch_bn<160, LNF, false, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
    case 192: return launch_bn<192, LNF, false, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
    case 256: return launch_bn<256, LNF, false, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
    default: return cudaErrorInvalidValue;
  }
}

// e4m3 operands (vx_gemm_fp8): the plain producer at the widths of bf16 output tiles (BN 16 is the fp32-output width)
static cudaError_t launch_f8(const CUtensorMap& mA, const CUtensorMap& mA2, const CUtensorMap& mB, const CUtensorMap& mR,
                             const CUtensorMap& mC, const GemmArgs& a, int grid, size_t smem, cudaStream_t st) {
  using T = __nv_fp8_e4m3;
  if (a.pp) {
    switch (a.block_n) {
      case 32: return launch_bn<32, false, true, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
      case 64: return launch_bn<64, false, true, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
      case 96: return launch_bn<96, false, true, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
      case 128: return launch_bn<128, false, true, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
      case 160: return launch_bn<160, false, true, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
      default: return cudaErrorInvalidValue;
    }
  }
  switch (a.block_n) {
    case 32: return launch_bn<32, false, false, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
    case 64: return launch_bn<64, false, false, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
    case 96: return launch_bn<96, false, false, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
    case 128: return launch_bn<128, false, false, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
    case 160: return launch_bn<160, false, false, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
    case 192: return launch_bn<192, false, false, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
    case 256: return launch_bn<256, false, false, T>(mA, mA2, mB, mR, mC, a, grid, smem, st);
    default: return cudaErrorInvalidValue;
  }
}

static int launch(const CUtensorMap& mA, const CUtensorMap& mA2, const CUtensorMap& mB, const CUtensorMap& mR,
                  const CUtensorMap& mC, GemmArgs& a, cudaStream_t st) {
  VX_REQUIRE(bn_supported(a.block_n), "vx_gemm: block_n=%d is not one of 16, 32, 64, 96, 128, 160, 192, 256", a.block_n);
  if (a.ares) a.a_bytes = 0;   // A lives in its own resident slots, the ring stages hold W only
  else if (a.a_bytes <= 0) a.a_bytes = kBlockM * kBlockK * 2;
  const int stage_bytes = a.a_bytes + (a.rr ? 3 : 1) * a.block_n * kBlockK * 2;
  const int out_cols = a.geglu ? a.block_n / 2 : a.block_n;
  const int buf_bytes = a.out_f32 ? 0 : out_cols / kPanelCols * kPanelBytes;
  const int total_kb = a.rr ? 3 * a.kblocks1 : a.taps * a.kblocks1 + a.kblocks2;
  const size_t cap = (size_t)kSmemCap - kSmemReserve - (a.ares ? (size_t)a.ares_bytes : 0);
  // deep TMA rings only pay off for long K loops; short K loops need the second staging tile instead
  int want_stages = gemm_env().stages;
  if (want_stages <= 0) want_stages = total_kb < 6 ? (total_kb < 3 ? 3 : total_kb) : 6;
  int nbuf = (!a.out_f32 && (size_t)3 * stage_bytes + 2 * buf_bytes <= cap) ? 2 : 1;
  if (a.rr) {
    // a row-reuse stage is 3 taps deep (12 MMAs per warpgroup): three stages when they fit beside ONE staging tile, else
    // two beside two.  Ping-pong: three stages beside two staging tiles (conv3x3_entry checked that they fit)
    nbuf = (a.pp || (size_t)3 * stage_bytes + buf_bytes > cap) ? 2 : 1;
    want_stages = nbuf == 1 || a.pp ? 3 : 2;
    if (!a.pp && (size_t)want_stages * stage_bytes + (size_t)nbuf * buf_bytes > cap) nbuf = 1;
  }
  if (a.ares) {   // every column tile of a row tile streams the whole W panel: a deep ring, two staging tiles when they fit
    nbuf = ((size_t)4 * stage_bytes + 2 * (size_t)buf_bytes <= cap) ? 2 : 1;
    want_stages = 8;
  }
  const int force_nbuf = gemm_env().nbuf;
  if (force_nbuf == 1 || (force_nbuf == 2 && (size_t)2 * stage_bytes + 2 * buf_bytes <= cap)) nbuf = force_nbuf;
  int stages = want_stages;
  while (stages > 2 && (size_t)stages * stage_bytes + (size_t)nbuf * buf_bytes > cap) --stages;
  a.stages = stages;
  a.nbuf = nbuf;
  // ping-pong: warpgroup b owns staging tile b (a shared tile would let one warpgroup run a phase ahead of the other)
  if (a.pp && !a.out_f32 && nbuf != 2) a.pp = 0;
  const size_t smem = (size_t)stages * stage_bytes + (size_t)nbuf * buf_bytes + kSmemReserve + (a.ares ? (size_t)a.ares_bytes : 0);
  VX_REQUIRE(smem <= (size_t)kSmemCap, "vx_gemm: %zu bytes of shared memory needed (bn=%d, K blocks=%d)", smem, a.block_n,
             a.kblocks1);
  if (gemm_env().verbose)
    fprintf(stderr, "[vx_gemm] M=%d N=%d kb=%d taps=%d bn=%d pp=%d rr=%d stages=%d nbuf=%d tiles=%dx%d%s\n", a.M, a.N,
            total_kb, a.taps, a.block_n, a.pp, a.rr, stages, nbuf, a.tiles_m, a.tiles_n, a.a_scale ? " e4m3" : "");
  const int npar = a.ups ? 4 : 1;
  const bool lnf = a.ln_stats != nullptr || a.ln_parts != nullptr || a.ares;
  VX_REQUIRE(!a.pp || (!lnf && !a.rs_out && pp_bn_supported(a.block_n)), "vx_gemm: no ping-pong kernel for bn=%d", a.block_n);
  const long long tiles = a.ares ? a.tiles_m : (long long)a.tiles_m * a.tiles_n * npar;
  const int grid = tiles < device_sms() ? (int)tiles : device_sms();
  VX_REQUIRE(!a.a_scale || (!lnf && !a.rs_out && a.taps == 1 && !a.kblocks2 && !a.out_f32 && a.block_n >= 32),
             "vx_gemm_fp8: plain producer, linear / GEGLU bf16 epilogue, block_n >= 32 only");
  if (lnf) VX_CHECK_CUDA((launch_lnf<true>(mA, mA2, mB, mR, mC, a, grid, smem, st)));
  else if (a.a_scale) VX_CHECK_CUDA((launch_f8(mA, mA2, mB, mR, mC, a, grid, smem, st)));
  else VX_CHECK_CUDA((launch_lnf<false>(mA, mA2, mB, mR, mC, a, grid, smem, st)));
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

static int make_out_maps(CUtensorMap* mR, CUtensorMap* mC, const void* residual, long long ldr, void* out,
                         long long ldc, long long M, int out_N, int rows_valid) {
  uint64_t dims[2] = {(uint64_t)out_N, (uint64_t)M};
  uint32_t box[2] = {kPanelCols, (uint32_t)rows_valid};
  {
    uint64_t str[1] = {(uint64_t)ldc * 2};
    if (make_tmap_bf16(mC, out, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_64B)) return 1;
  }
  if (residual) {
    uint64_t str[1] = {(uint64_t)ldr * 2};
    if (make_tmap_bf16(mR, residual, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_64B)) return 1;
  } else {
    *mR = *mC;
  }
  return 0;
}

}  // namespace vx

using namespace vx;

extern "C" void vx_gemm_reload_env() { gemm_env() = GemmEnv(); }   // sweep-tool hook (csrc/vx_bringup.h), not product ABI

// LayerNorm statistics hand-over between two GEMMs (GemmArgs::rs_out / ln_parts)
struct RowStatsIO {
  float* out;            // producer: [2 * tiles_n][stride] float2 partial (sum, sum of squares) per row, or null
  long long out_stride;  // >= M
  int out_cap;           // slots the caller allocated
  int* nparts_out;       // producer: receives 2 * tiles_n
  const float* parts;    // consumer: partials of the rows of A, or null
  long long parts_stride;
  int nparts;
};

// epilogue: 0 = linear (bias, bias2, scale, residual); 1 = GEGLU (W / bias packed per tile as value|gate halves,
// see vx_geglu_pack_rows; out has N/2 columns)
static int gemm_entry(const void* A, long long lda, int K1, const void* A2, long long lda2, int K2, const void* Wt,
                      long long ldw, int M, int N, const float* bias, const float* bias2, int bias2_div, float scale,
                      const void* residual, long long ldr, void* out, long long ldc, int out_f32, int block_n,
                      const float* ln_stats, const float* ln_colsum, void* stream, float ln_eps = 0.f,
                      const RowStatsIO* rs = nullptr, const float* a_scale = nullptr, const float* w_scale = nullptr) {
  const int geglu = out_f32 == 2 ? 1 : 0;  // out_f32: 0 bf16, 1 fp32, 2 bf16 + GEGLU epilogue
  const bool ares = ln_colsum && !ln_stats && !(rs && rs->parts);   // LayerNorm GEMM with in-kernel statistics (A tile resident)
  // operand element size: 2 (bf16), or 1 (e4m3 with per-row / per-column scales): K blocks of kKE elements = 128 bytes
  const bool f8 = a_scale != nullptr;
  const int esz = f8 ? 1 : 2, kKE = kBlockK * 2 / esz;
  const CUtensorMapDataType tdt = f8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  if (geglu) out_f32 = 0;
  VX_REQUIRE(M > 0 && N > 0 && K1 > 0, "vx_gemm_bf16: bad shape M=%d N=%d K1=%d", M, N, K1);
  const int gran = geglu ? 64 : (out_f32 ? 16 : 32);
  VX_REQUIRE(N % gran == 0, "vx_gemm_bf16: N=%d must be a multiple of %d", N, gran);
  VX_REQUIRE(K1 % (16 / esz) == 0 && K2 % 8 == 0 && lda % (16 / esz) == 0 && ldw % (16 / esz) == 0 && ldc % 8 == 0,
             "vx_gemm: K/ld must be multiples of 16 bytes (TMA strides), ldc of 8 elements");
  VX_REQUIRE(!f8 || (w_scale && K2 == 0 && !out_f32 && !ln_colsum && !ln_stats && !rs),
             "vx_gemm_fp8: w_scale missing, or an operand mode the e4m3 GEMM does not have");
  VX_REQUIRE(K2 == 0 || (K1 % kBlockK == 0 && lda2 % 8 == 0), "vx_gemm_bf16: split-K needs K1 %% 64 == 0");
  VX_REQUIRE(!residual || (ldr % 8 == 0 && !out_f32 && !geglu), "vx_gemm_bf16: residual needs bf16 linear epilogue, ldr %%8");
  VX_REQUIRE(!geglu || (!bias2 && scale == 1.0f), "vx_gemm_bf16: GEGLU epilogue takes only the packed bias");
  const int tiles_m = (M + kBlockM - 1) / kBlockM;
  const int total_kb = (K1 + kKE - 1) / kKE + (K2 + kBlockK - 1) / kBlockK;
  if (block_n <= 0) block_n = gemm_env().bn;
  if (ares) {
    VX_REQUIRE(K2 == 0 && K1 % kBlockK == 0 && K1 <= 8 * kBlockK && !out_f32,
               "vx_gemm_ln_bf16: K=%d must be a multiple of 64, <= 512 (the row tile stays in shared memory)", K1);
    const size_t cap = (size_t)kSmemCap - kSmemReserve - (size_t)(K1 / kBlockK) * kBlockM * kBlockK * 2;
    auto fits = [&](int bn, int nbuf, int stages) {   // `stages` ring stages + nbuf staging tiles
      const size_t b = (size_t)bn * kBlockK * 2, buf = (size_t)((geglu ? bn / 2 : bn) / kPanelCols) * kPanelBytes;
      return stages * b + nbuf * buf <= cap;
    };
    if (geglu) {
      // the weights are packed per column tile (vx_geglu_pack_rows): the tile width is fixed, the ring gets shallower instead
      VX_REQUIRE(block_n > 0 && N % block_n == 0 && bn_supported(block_n) && fits(block_n, 1, 2),
                 "vx_gemm_ln_bf16: GEGLU column tile %d does not fit beside the resident K=%d tile", block_n, K1);
    } else if (block_n <= 0 || N % block_n || block_n % gran || !bn_supported(block_n) || !fits(block_n, 1, 4)) {
      block_n = 0;
      for (int nbuf = 2; nbuf >= 1 && !block_n; --nbuf)   // widest column tile that keeps both staging tiles, else one
        for (int bn = 256; bn >= gran; bn -= gran)
          if (N % bn == 0 && bn_supported(bn) && fits(bn, nbuf, 4)) {
            block_n = bn;
            break;
          }
    }
    VX_REQUIRE(block_n > 0, "vx_gemm_ln_bf16: no column tile of N=%d fits beside the resident K=%d tile", N, K1);
  }
  // ping-pong covers the plain producer with the linear / GEGLU / fp32 epilogues (not the LayerNorm or row-sum variants)
  const bool pp_ok = !ln_colsum && !(rs && rs->out);
  int pp = 0;
  if (!ares) {
    const int fixed = block_n;
    block_n = pick_block_n(tiles_m, N, gran, total_kb, fixed, pp_ok, &pp);
    if (!block_n) block_n = fixed;   // not a width the picker knows: rejected below
  }
  VX_REQUIRE(block_n >= gran && block_n % gran == 0 && block_n <= 256 && N % block_n == 0,
             "vx_gemm_bf16: block_n=%d invalid for N=%d", block_n, N);
  CUtensorMap mA, mA2, mB, mR, mC;
  {
    uint64_t dims[2] = {(uint64_t)K1, (uint64_t)M};
    uint64_t str[1] = {(uint64_t)lda * esz};
    uint32_t box[2] = {(uint32_t)kKE, kBlockM};
    if (make_tmap_bf16(&mA, A, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, nullptr, tdt)) return 1;
  }
  if (K2 > 0) {
    uint64_t dims[2] = {(uint64_t)K2, (uint64_t)M};
    uint64_t str[1] = {(uint64_t)lda2 * 2};
    uint32_t box[2] = {kBlockK, kBlockM};
    if (make_tmap_bf16(&mA2, A2, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B)) return 1;
  } else {
    mA2 = mA;
  }
  {
    uint64_t dims[2] = {(uint64_t)(K1 + K2), (uint64_t)N};
    uint64_t str[1] = {(uint64_t)ldw * esz};
    uint32_t box[2] = {(uint32_t)kKE, (uint32_t)block_n};
    if (make_tmap_bf16(&mB, Wt, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, nullptr, tdt)) return 1;
  }
  if (!out_f32) {
    if (make_out_maps(&mR, &mC, residual, ldr, out, ldc, M, geglu ? N / 2 : N, kBlockM)) return 1;
  } else {
    mR = mA;
    mC = mA;
  }
  GemmArgs a{};
  a.M = M; a.N = N;
  a.kblocks1 = (K1 + kKE - 1) / kKE;
  a.kblocks2 = (K2 + kBlockK - 1) / kBlockK;
  a.taps = 1;
  a.a_scale = a_scale;
  a.w_scale = w_scale;
  a.block_n = block_n;
  a.pp = pp;
  a.rows_valid = kBlockM;
  a.W = a.H = 1;
  a.tiles_m = tiles_m;
  a.tiles_n = N / block_n;
  a.geglu = geglu;
  a.has_residual = residual ? 1 : 0;
  a.out_f32 = out_f32;
  a.bias = bias; a.bias2 = bias2; a.bias2_div = bias2_div > 0 ? bias2_div : 1; a.scale = scale;
  a.out32 = (float*)out; a.ldc = ldc;
  a.ln_stats = ln_stats; a.ln_colsum = ln_colsum;
  a.ares = ares ? 1 : 0;
  a.ares_bytes = ares ? a.kblocks1 * kBlockM * kBlockK * 2 : 0;
  a.ln_eps = ln_eps;
  if (rs && rs->out) {
    VX_REQUIRE(!out_f32 && !geglu && rs->out_stride >= M, "vx_gemm_rowsums_bf16: linear bf16 epilogue only, stride >= M");
    VX_REQUIRE(2 * a.tiles_n <= rs->out_cap, "vx_gemm_rowsums_bf16: %d partial slots needed, %d allocated", 2 * a.tiles_n, rs->out_cap);
    a.rs_out = reinterpret_cast<float2*>(rs->out);
    a.rs_stride = rs->out_stride;
    if (rs->nparts_out) *rs->nparts_out = 2 * a.tiles_n;
  }
  if (rs && rs->parts) {
    VX_REQUIRE(ln_colsum && K2 == 0 && rs->nparts > 0 && rs->parts_stride >= M, "vx_gemm_lnparts_bf16: bad statistics operands");
    a.ln_parts = reinterpret_cast<const float2*>(rs->parts);
    a.ln_pstride = rs->parts_stride;
    a.ln_nparts = rs->nparts;
    a.ln_invK = 1.0f / (float)K1;
  }
  return launch(mA, mA2, mB, mR, mC, a, (cudaStream_t)stream);
}

extern "C" int vx_gemm_bf16(const void* A, long long lda, int K1, const void* A2, long long lda2, int K2,
                            const void* Wt, long long ldw, int M, int N, const float* bias, const float* bias2,
                            int bias2_div, float scale, const void* residual, long long ldr, void* out,
                            long long ldc, int out_f32, int block_n, void* stream) {
  return gemm_entry(A, lda, K1, A2, lda2, K2, Wt, ldw, M, N, bias, bias2, bias2_div, scale, residual, ldr, out, ldc,
                    out_f32, block_n, nullptr, nullptr, stream);
}

// e4m3 operands with per-row / per-output-channel scales: out = epilogue(sum_k A[m,k] W[n,k] * a_scale[m] * w_scale[n]),
// the epilogue (bias, bias2, scale, residual; or GEGLU with W, w_scale and bias packed as for vx_gemm_bf16) as in
// vx_gemm_bf16.  A [M, K] and W [N, K] hold float8_e4m3fn codes, K-major; K, lda, ldw multiples of 16.
extern "C" int vx_gemm_fp8(const void* A, long long lda, const float* a_scale, int K, const void* Wt, long long ldw,
                           const float* w_scale, int M, int N, const float* bias, const float* bias2, int bias2_div,
                           float scale, const void* residual, long long ldr, void* out, long long ldc, int geglu,
                           int block_n, void* stream) {
  VX_REQUIRE(a_scale && w_scale, "vx_gemm_fp8: a_scale / w_scale missing (M=%d N=%d)", M, N);
  return gemm_entry(A, lda, K, nullptr, 0, 0, Wt, ldw, M, N, bias, bias2, bias2_div, scale, residual, ldr, out, ldc,
                    geglu ? 2 : 0, block_n, nullptr, nullptr, stream, 0.f, nullptr, a_scale, w_scale);
}

// LayerNorm folded into the GEMM: A holds the UN-normalised rows, Wt = W * gamma (per input channel),
// out = rstd[m] * (A @ Wt^T - mean[m] * colsum) + bias (+ bias2, scale, residual, GEGLU as in vx_gemm_bf16) with
// stats[m] = (mean, rstd) from vx_row_stats, colsum[n] = sum_k Wt[n,k], bias[n] = sum_k beta[k] W[n,k] + b[n].
extern "C" int vx_gemm_lnfold_bf16(const void* A, long long lda, int K, const void* Wt, long long ldw, int M, int N,
                                   const float* stats, const float* colsum, const float* bias, const float* bias2,
                                   int bias2_div, float scale, const void* residual, long long ldr, void* out,
                                   long long ldc, int geglu, int block_n, void* stream) {
  VX_REQUIRE(stats && colsum, "vx_gemm_lnfold_bf16: stats / colsum missing (M=%d)", M);
  return gemm_entry(A, lda, K, nullptr, 0, 0, Wt, ldw, M, N, bias, bias2, bias2_div, scale, residual, ldr, out, ldc,
                    geglu ? 2 : 0, block_n, stats, colsum, stream);
}

// Producer side of the LayerNorm hand-over: vx_gemm_bf16's linear epilogue (bias, bias2, scale, residual; bf16 out) that also
// writes, per output row, 2 * ceil(N / block_n) partial (sum, sum of squares) pairs of the ROUNDED outputs:
// row_parts[slot * parts_stride + m] as float2, slot < *nparts.  The consumer GEMM (vx_gemm_lnparts_bf16) turns them into
// mean / rstd, so LayerNorm(out) needs neither a normalisation pass nor a statistics pass over `out`.
extern "C" int vx_gemm_rowsums_bf16(const void* A, long long lda, int K1, const void* A2, long long lda2, int K2,
                                    const void* Wt, long long ldw, int M, int N, const float* bias, const float* bias2,
                                    int bias2_div, float scale, const void* residual, long long ldr, void* out,
                                    long long ldc, int block_n, float* row_parts, long long parts_stride, int parts_cap,
                                    int* nparts, void* stream) {
  VX_REQUIRE(row_parts && nparts, "vx_gemm_rowsums_bf16: row_parts / nparts missing (M=%d)", M);
  RowStatsIO rs{row_parts, parts_stride, parts_cap, nparts, nullptr, 0, 0};
  return gemm_entry(A, lda, K1, A2, lda2, K2, Wt, ldw, M, N, bias, bias2, bias2_div, scale, residual, ldr, out, ldc, 0,
                    block_n, nullptr, nullptr, stream, 0.f, &rs);
}

// Consumer side: vx_gemm_lnfold_bf16 with the row statistics taken from a producer's partial sums instead of a
// vx_row_stats array: mean = sum / K, variance = sum of squares / K - mean^2 (fp32), rstd = rsqrt(variance + eps).
extern "C" int vx_gemm_lnparts_bf16(const void* A, long long lda, int K, const void* Wt, long long ldw, int M, int N,
                                    const float* row_parts, long long parts_stride, int nparts, float eps,
                                    const float* colsum, const float* bias, const float* bias2, int bias2_div, float scale,
                                    const void* residual, long long ldr, void* out, long long ldc, int geglu, int block_n,
                                    void* stream) {
  VX_REQUIRE(row_parts && colsum, "vx_gemm_lnparts_bf16: row_parts / colsum missing (M=%d)", M);
  RowStatsIO rs{nullptr, 0, 0, nullptr, row_parts, parts_stride, nparts};
  return gemm_entry(A, lda, K, nullptr, 0, 0, Wt, ldw, M, N, bias, bias2, bias2_div, scale, residual, ldr, out, ldc,
                    geglu ? 2 : 0, block_n, nullptr, colsum, stream, eps, &rs);
}

// LayerNorm -> Linear in ONE kernel: A holds the un-normalised rows (K <= 512), Wt / colsum / bias are the folded parameters
// of vx_gemm_lnfold_bf16; the row statistics are computed inside the kernel from the shared-memory resident row tile
// (two-pass mean / variance, eps as in nn.LayerNorm), so neither LayerNorm(A) nor a statistics array ever exists in HBM.
extern "C" int vx_gemm_ln_bf16(const void* A, long long lda, int K, const void* Wt, long long ldw, int M, int N,
                               const float* colsum, const float* bias, float eps, const float* bias2, int bias2_div,
                               float scale, const void* residual, long long ldr, void* out, long long ldc, int geglu,
                               int block_n, void* stream) {
  VX_REQUIRE(colsum, "vx_gemm_ln_bf16: colsum missing (M=%d)", M);
  return gemm_entry(A, lda, K, nullptr, 0, 0, Wt, ldw, M, N, bias, bias2, bias2_div, scale, residual, ldr, out, ldc,
                    geglu ? 2 : 0, block_n, nullptr, colsum, stream, eps);
}

// X: NHWC bf16 [NB, Hin, Win, C];  Wt: [Cout, 9*C] with K index = (ky*3+kx)*C + c;  out: [NB*H*W, ldc], H x W the output
// size.  stride 2: the A boxes are fetched through a tensor map with traversal stride 2 along x and y (the box covers
// 2 * wbox x 2 * hbox input pixels, every second one lands in shared memory), so the tile of output pixels (y, x) gets
// input pixels (2y + dy, 2x + dx) for tap (dy, dx) without any gathered copy of the input (no im2col tensor).
static int conv3x3_entry(const void* X, int NB, int Hin, int Win, int C, const void* Wt, int Cout, const float* bias,
                         const float* bias2, int bias2_div, float scale, const void* residual, long long ldr, void* out,
                         long long ldc, int block_n, int stride, int pad_lo, void* stream) {
  VX_REQUIRE(C % kBlockK == 0 && Cout % 32 == 0, "vx_conv3x3_bf16: C=%d must be %%64, Cout=%d %%32", C, Cout);
  VX_REQUIRE(ldc % 8 == 0 && (!residual || ldr % 8 == 0), "vx_conv3x3_bf16: ld must be %%8");
  VX_REQUIRE(stride == 1 || (stride == 2 && Hin % 2 == 0 && Win % 2 == 0), "vx_conv3x3: stride %d on %dx%d unsupported", stride,
             Hin, Win);
  VX_REQUIRE(pad_lo == 1 || (pad_lo == 0 && stride == 2), "vx_conv3x3: pad_lo=%d only with stride 2", pad_lo);
  const int H = Hin / stride, W = Win / stride;   // 3x3, pad 1 (or (0,1,0,1)), even sizes: H_out = H_in / stride
  // pixel rectangle of <= 128 output rows that is contiguous in NHWC row order
  int wbox, hbox = 1, nbox = 1;
  if (W >= kBlockM) {
    wbox = kBlockM;                 // widest divisor of W that fits a tile (192 -> 96 at the 768x768 VAE level)
    while (W % wbox) --wbox;
  } else {
    wbox = W;
    hbox = kBlockM / W;
    if (hbox > H) {
      hbox = H;
      nbox = kBlockM / (W * H);
      if (nbox > NB) nbox = NB;
      if (nbox < 1) nbox = 1;
      while (NB % nbox) --nbox;
    } else {
      while (H % hbox) --hbox;
    }
  }
  const int rows_valid = wbox * hbox * nbox;
  const long long M = (long long)NB * H * W;
  VX_REQUIRE(M % rows_valid == 0, "vx_conv3x3_bf16: NB*H*W=%lld not tileable by %d", M, rows_valid);
  const long long tiles_m = M / rows_valid;
  const int total_kb = 9 * (C / kBlockK);
  // Row reuse: when a tile is hbox >= 2 whole image rows of one frame, ONE box of hbox + 2 rows per (dx, channel block)
  // serves the three dy taps (each tap's 128 rows start dy image rows further down, a multiple of the swizzle atom):
  // 3 (hbox + 2) / (9 hbox) of the A traffic.  It needs two ring stages beside one staging tile; ping-pong takes it with
  // three stages beside two staging tiles (one per warpgroup: with two stages it lost to the cooperative schedule at every
  // shape measured).  Its K order (dx, channel block, dy) differs from tap by tap (dy, dx, channel block), so the producer
  // is chosen at the cooperative schedule's width, and ping-pong is only taken at widths where the same producer fits: the
  // result does not depend on the schedule.
  bool rr = gemm_env().conv_rr && stride == 1 && nbox == 1 && wbox == W && hbox >= 2 && rows_valid == kBlockM && (W * 128) % 1024 == 0;
  auto rr_fits = [&](int bn, int stages, int nbuf) {
    const size_t st = (size_t)(hbox + 2) * W * kBlockK * 2 + (size_t)3 * bn * kBlockK * 2;
    return stages * st + (size_t)nbuf * (bn / kPanelCols) * kPanelBytes <= (size_t)kSmemCap - kSmemReserve;
  };
  if (block_n <= 0) block_n = gemm_env().bn;
  int pp = 0;
  {
    const int fixed = block_n;
    const int coop_bn = pick_block_n(tiles_m, Cout, 32, total_kb, fixed);
    rr = rr && coop_bn > 0 && rr_fits(coop_bn, 2, 1);
    int pp_max_bn = kPPMaxBN;
    while (rr && pp_max_bn > 0 && !rr_fits(pp_max_bn, 3, 2)) pp_max_bn -= 32;
    block_n = pick_block_n(tiles_m, Cout, 32, total_kb, fixed, true, &pp, pp_max_bn, rr);
    if (!block_n) block_n = fixed;   // not a width the picker knows: rejected below
  }
  VX_REQUIRE(block_n % 32 == 0 && block_n >= 32 && block_n <= 256 && Cout % block_n == 0,
             "vx_conv3x3_bf16: block_n=%d invalid for Cout=%d", block_n, Cout);
  CUtensorMap mA, mB, mR, mC;
  {
    uint64_t dims[4] = {(uint64_t)C, (uint64_t)Win, (uint64_t)Hin, (uint64_t)NB};
    uint64_t str[3] = {(uint64_t)C * 2, (uint64_t)Win * C * 2, (uint64_t)Hin * Win * C * 2};
    uint32_t box[4] = {kBlockK, (uint32_t)(wbox * stride), (uint32_t)((rr ? hbox + 2 : hbox) * stride), (uint32_t)nbox};
    uint32_t est[4] = {1, (uint32_t)stride, (uint32_t)stride, 1};
    if (make_tmap_bf16(&mA, X, 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, est)) return 1;
  }
  {
    uint64_t dims[2] = {(uint64_t)9 * C, (uint64_t)Cout};
    uint64_t str[1] = {(uint64_t)9 * C * 2};
    uint32_t box[2] = {kBlockK, (uint32_t)block_n};
    if (make_tmap_bf16(&mB, Wt, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B)) return 1;
  }
  if (make_out_maps(&mR, &mC, residual, ldr, out, ldc, M, Cout, rows_valid)) return 1;
  GemmArgs a{};
  a.M = (int)M; a.N = Cout;
  a.kblocks1 = C / kBlockK;
  a.kblocks2 = 0;
  a.taps = 9;
  a.rr = rr ? 1 : 0;
  a.a_bytes = rr ? (hbox + 2) * W * kBlockK * 2 : kBlockM * kBlockK * 2;
  a.block_n = block_n;
  a.pp = pp;
  a.rows_valid = rows_valid;
  a.W = W; a.H = H;
  a.cstride = stride; a.cpad = pad_lo;
  a.tiles_m = (int)tiles_m;
  a.tiles_n = Cout / block_n;
  a.geglu = 0;
  a.has_residual = residual ? 1 : 0;
  a.out_f32 = 0;
  a.bias = bias; a.bias2 = bias2; a.bias2_div = bias2_div > 0 ? bias2_div : 1; a.scale = scale;
  a.out32 = (float*)out; a.ldc = ldc;
  return launch(mA, mA, mB, mR, mC, a, (cudaStream_t)stream);
}

extern "C" int vx_conv3x3_bf16(const void* X, int NB, int H, int W, int C, const void* Wt, int Cout,
                               const float* bias, const float* bias2, int bias2_div, float scale,
                               const void* residual, long long ldr, void* out, long long ldc, int block_n,
                               void* stream) {
  return conv3x3_entry(X, NB, H, W, C, Wt, Cout, bias, bias2, bias2_div, scale, residual, ldr, out, ldc, block_n, 1, 1, stream);
}

// 3x3 convolution with stride 2 on an even-sized NHWC image -> [NB * (H/2) * (W/2), ldc].  pad_lo = 1: nn.Conv2d(padding=1)
// (Downsample3D / Downsample2D of the UNets, reference modules/resnet.py:93-120); pad_lo = 0: F.pad(x, (0, 1, 0, 1)) + padding 0
// (diffusers Downsample2D(padding=0) of the VAE encoder).  Out-of-image taps are zero-filled by the TMA unit.
extern "C" int vx_conv3x3s2_bf16(const void* X, int NB, int H, int W, int C, const void* Wt, int Cout, const float* bias,
                                 int pad_lo, void* out, long long ldc, int block_n, void* stream) {
  return conv3x3_entry(X, NB, H, W, C, Wt, Cout, bias, nullptr, 1, 1.0f, nullptr, 0, out, ldc, block_n, 2, pad_lo, stream);
}

// conv3x3(nearest_upsample_2x(X)) without the upsampled tensor (reference modules/resnet.py:53-90 Upsample3D,
// diffusers Upsample2D in the VAE decoder): output pixel (2i + py, 2j + px) only ever sees the 2x2 input neighbourhood
// rows {i + py - 1, i + py}, columns {j + px - 1, j + px}, so each of the four output parity classes is a 2x2 convolution of
// X with the 3x3 weights summed over the taps that land on the same input pixel (host: vexpress_b200.ops.pack_upconv_weight)
// -- 4/9 of the FLOPs, and the 4x tensor is never written or read.
// X: NHWC bf16 [NB, H, W, C];  Wt: [4 * Cout, 4 * C] = parity-major (py, px) blocks, K index = (a * 2 + b) * C + c;
// out: [NB * 2H * 2W, ldc] (NHWC of the upsampled image).
extern "C" int vx_upconv3x3_bf16(const void* X, int NB, int H, int W, int C, const void* Wt, int Cout, const float* bias,
                                 void* out, long long ldc, int block_n, void* stream) {
  VX_REQUIRE(C % kBlockK == 0 && Cout % 32 == 0, "vx_upconv3x3_bf16: C=%d must be %%64, Cout=%d %%32", C, Cout);
  VX_REQUIRE(ldc % 8 == 0, "vx_upconv3x3_bf16: ldc must be %%8");
  int wbox, hbox = 1, nbox = 1;
  if (W >= kBlockM) {
    wbox = kBlockM;                 // widest divisor of W that fits a tile (192 -> 96 at the 768x768 VAE level)
    while (W % wbox) --wbox;
  } else {
    wbox = W;
    hbox = kBlockM / W;
    if (hbox > H) {
      hbox = H;
      nbox = kBlockM / (W * H);
      if (nbox > NB) nbox = NB;
      if (nbox < 1) nbox = 1;
      while (NB % nbox) --nbox;
    } else {
      while (H % hbox) --hbox;
    }
  }
  const int rows_valid = wbox * hbox * nbox;
  const long long M = (long long)NB * H * W;
  VX_REQUIRE(M % rows_valid == 0, "vx_upconv3x3_bf16: NB*H*W=%lld not tileable by %d", M, rows_valid);
  const long long tiles_m = M / rows_valid;
  const int total_kb = 4 * (C / kBlockK);
  if (block_n <= 0) block_n = gemm_env().bn;
  int pp = 0;
  {
    const int fixed = block_n;
    block_n = pick_block_n(tiles_m * 4, Cout, 32, total_kb, fixed, true, &pp);
    if (!block_n) block_n = fixed;
  }
  VX_REQUIRE(block_n % 32 == 0 && block_n >= 32 && block_n <= 256 && Cout % block_n == 0,
             "vx_upconv3x3_bf16: block_n=%d invalid for Cout=%d", block_n, Cout);
  CUtensorMap mA, mB, mC0, mC1;
  {
    uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)NB};
    uint64_t str[3] = {(uint64_t)C * 2, (uint64_t)W * C * 2, (uint64_t)H * W * C * 2};
    uint32_t box[4] = {kBlockK, (uint32_t)wbox, (uint32_t)hbox, (uint32_t)nbox};
    if (make_tmap_bf16(&mA, X, 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B)) return 1;
  }
  {
    uint64_t dims[2] = {(uint64_t)4 * C, (uint64_t)4 * Cout};
    uint64_t str[1] = {(uint64_t)4 * C * 2};
    uint32_t box[2] = {kBlockK, (uint32_t)block_n};
    if (make_tmap_bf16(&mB, Wt, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B)) return 1;
  }
  for (int px = 0; px < 2; ++px) {
    // (c, j, i, n, py) view of the [NB, 2H, 2W, ldc] output for one column parity
    uint64_t dims[5] = {(uint64_t)Cout, (uint64_t)W, (uint64_t)H, (uint64_t)NB, 2};
    uint64_t str[4] = {(uint64_t)2 * ldc * 2, (uint64_t)2 * (2 * W) * ldc * 2, (uint64_t)(2 * H) * (2 * W) * ldc * 2,
                       (uint64_t)(2 * W) * ldc * 2};
    uint32_t box[5] = {kPanelCols, (uint32_t)wbox, (uint32_t)hbox, (uint32_t)nbox, 1};
    if (make_tmap_bf16(px ? &mC1 : &mC0, (const __nv_bfloat16*)out + (long long)px * ldc, 5, dims, str, box,
                       CU_TENSOR_MAP_SWIZZLE_64B))
      return 1;
  }
  GemmArgs a{};
  a.M = (int)M; a.N = Cout;
  a.kblocks1 = C / kBlockK;
  a.kblocks2 = 0;
  a.taps = 4;
  a.ups = 1;
  a.cstride = 1; a.cpad = 1;
  a.block_n = block_n;
  a.pp = pp;
  a.rows_valid = rows_valid;
  a.W = W; a.H = H;
  a.tiles_m = (int)tiles_m;
  a.tiles_n = Cout / block_n;
  a.geglu = 0;
  a.has_residual = 0;
  a.out_f32 = 0;
  a.bias = bias; a.bias2 = nullptr; a.bias2_div = 1; a.scale = 1.0f;
  a.out32 = (float*)out; a.ldc = ldc;
  return launch(mA, mA, mB, mC1, mC0, a, (cudaStream_t)stream);
}
