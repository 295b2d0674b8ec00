// HBM-bound normalisation / activation kernels on channels-last bf16 token matrices [rows, C]:
//   * GroupNorm (per frame, 32 groups) as a deterministic two-kernel pair: partial statistics per
//     (frame, pixel chunk, group), then finalise (Chan merge in fixed order) + apply (+ optional SiLU).
//     Reads may come from TWO sources (x1 | x2 channel-concatenated): the `torch.cat([h, skip], 1)` of the
//     up blocks (reference modules/unet_3d_blocks.py:694,831) is never materialised on its own.
//     Reference: InflatedGroupNorm modules/resnet.py:20-28, ResnetBlock3D.forward :220-221,235-241,
//     Transformer3DModel.forward modules/transformer_3d.py:124, TemporalTransformer3DModel modules/motion_module.py:156.
//   * LayerNorm over C (eps 1e-5) with the optional sinusoidal positional-encoding add of the temporal
//     attention (reference modules/motion_module.py:244,262-277,365-366; attention.py:329-333).  The e4m3 form
//     (vx_layernorm_fp8) writes float8_e4m3fn codes of the fp32 result and one scale per row, amax(|row|) / 448.
//   * GEGLU gate: out = h * gelu_erf(gate) (diffusers FeedForward/GEGLU, SURVEY.md Appendix B.3).
// All loads/stores are 16-byte vectors, threads walk the contiguous channel dimension.
#include "vx_host.h"
#include "vx_ptx.cuh"

namespace vx {

__device__ __forceinline__ void load8(const __nv_bfloat16* p, float (&f)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = unpack_bf16(w[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ void store8(__nv_bfloat16* p, const float (&f)[8]) {
  *reinterpret_cast<uint4*>(p) =
      make_uint4(pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]), pack_bf16(f[4], f[5]), pack_bf16(f[6], f[7]));
}
// two e4m3 codes (round to nearest even, saturated to +-448): a in the low byte, b in the high byte
__device__ __forceinline__ uint32_t pack_e4m3x2(float a, float b) {
  uint16_t d;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(d) : "f"(b), "f"(a));
  return d;
}
// f[j] * inv as eight e4m3 codes (8 bytes)
__device__ __forceinline__ void store8_e4m3(uint8_t* p, const float (&f)[8], float inv) {
  const uint32_t lo = pack_e4m3x2(f[0] * inv, f[1] * inv) | pack_e4m3x2(f[2] * inv, f[3] * inv) << 16;
  const uint32_t hi = pack_e4m3x2(f[4] * inv, f[5] * inv) | pack_e4m3x2(f[6] * inv, f[7] * inv) << 16;
  *reinterpret_cast<uint2*>(p) = make_uint2(lo, hi);
}
// e4m3 row scale from the row's amax: codes are value / scale, the largest one 448 (the e4m3 maximum); an all-zero row gets 1
__device__ __forceinline__ float e4m3_row_scale(float amax) { return amax > 0.f ? amax / 448.f : 1.f; }

// ------------------------------------------------------------------ GroupNorm statistics
// grid (S, NB); block = V*R threads (V = C/8 vectors per pixel, R pixel rows in flight).
// partial[(n*S + s)*G + g] = {count, mean, M2}
struct GnStatsArgs {
  const __nv_bfloat16* x1; long long ld1; int C1;
  const __nv_bfloat16* x2; long long ld2; int C2;
  int HW, G, S, R;
  float* partial;
};

// The statistics are sums of x - pivot, pivot = the bf16 value at pixel 0 of the group's first channel in frame n: the
// same value for every chunk, CTA and kernel, so partials (whose means are relative to it) merge as before.  Without the
// shift, fp32 sums of x and x^2 cancel in M2 = sum x^2 - mean sum x once a group's mean is large against its spread (the
// relative variance error grows as (mean / std)^2); with it, x - pivot is exact in fp32 and of the size of the spread.
__device__ __forceinline__ float gn_pivot(const __nv_bfloat16* x1, long long ld1, int C1, const __nv_bfloat16* x2,
                                          long long ld2, int HW, int n, int g, int cpg) {
  const int c = g * cpg;
  return __bfloat162float(c < C1 ? x1[(long long)n * HW * ld1 + c] : x2[(long long)n * HW * ld2 + (c - C1)]);
}

__device__ __forceinline__ void gn_stats_body(const GnStatsArgs& p, float* sm, const int n, const int s) {
  // sm: [R][C] sums, [R][C] sumsq
  const int C = p.C1 + p.C2;
  const int V = C / 8;
  const int cpg = C / p.G;
  const int v = threadIdx.x % V, r = threadIdx.x / V;
  const int chunk = (p.HW + p.S - 1) / p.S;
  const int p0 = s * chunk;
  const int p1 = min(p.HW, p0 + chunk);
  float sum[8], sq[8], piv[8];
  const int c0 = v * 8;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    sum[i] = sq[i] = 0.f;
    piv[i] = gn_pivot(p.x1, p.ld1, p.C1, p.x2, p.ld2, p.HW, n, (c0 + i) / cpg, cpg);   // independent loads, L1 hits
  }
  const bool second = c0 >= p.C1;
  const __nv_bfloat16* base = second ? p.x2 + (long long)n * p.HW * p.ld2 + (c0 - p.C1)
                                     : p.x1 + (long long)n * p.HW * p.ld1 + c0;
  const long long ld = second ? p.ld2 : p.ld1;
#pragma unroll 8
  for (int px = p0 + r; px < p1; px += p.R) {
    float f[8];
    load8(base + px * ld, f);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float d = f[i] - piv[i];
      sum[i] += d;
      sq[i] += d * d;
    }
  }
  float* ssum = sm;
  float* ssq = sm + p.R * C;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    ssum[r * C + c0 + i] = sum[i];
    ssq[r * C + c0 + i] = sq[i];
  }
  __syncthreads();
  for (int g = threadIdx.x; g < p.G; g += blockDim.x) {   // mean relative to the group's pivot
    float a = 0.f, b = 0.f;
    for (int rr = 0; rr < p.R; ++rr)
      for (int c = g * cpg; c < (g + 1) * cpg; ++c) {
        a += ssum[rr * C + c];
        b += ssq[rr * C + c];
      }
    const float cnt = (float)(p1 - p0) * cpg;
    const float mean = cnt > 0 ? a / cnt : 0.f;
    const float m2 = cnt > 0 ? fmaxf(b - a * mean, 0.f) : 0.f;
    float* o = p.partial + ((long long)(n * p.S + s) * p.G + g) * 3;
    o[0] = cnt;
    o[1] = mean;
    o[2] = m2;
  }
}

__global__ void gn_stats_kernel(const GnStatsArgs p) {
  pdl_enter();
  extern __shared__ float sm[];
  gn_stats_body(p, sm, blockIdx.y, blockIdx.x);
}

// ------------------------------------------------------------------ GroupNorm finalise + apply (+SiLU)
struct GnApplyArgs {
  const __nv_bfloat16* x1; long long ld1; int C1;
  const __nv_bfloat16* x2; long long ld2; int C2;
  int HW, G, S;
  const float* partial;
  const float* gamma; const float* beta;
  float eps; int silu;
  __nv_bfloat16* out; long long ldo;
  int chunk;  // pixels per CTA
};

// SiLU as y sigmoid(y), sigmoid(y) = 0.5 + 0.5 tanh(y / 2): one MUFU op per element.  tanh.approx is within a relative
// 2^-11 of tanh, so sigmoid is within 2^-12 absolute: on the negative tail (y < -4) that is more than the bf16 rounding of
// silu(y).  __fdividef(y, 1 + __expf(-y)) is accurate to a few 2^-23 there but took up to 1.38x the kernel time (1.28x
// summed over the VAE decoder's shapes) on an H100 SXM at 700 W (tools/norm_ab_h100.txt).
__device__ __forceinline__ float gn_silu(float y) {
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.5f * y));
  return y * fmaf(0.5f, t, 0.5f);
}

// `depart` (fused kernel only): called by every thread once the partial statistics of the frame have been merged, i.e.
// when this CTA no longer depends on its peers.
template <typename Depart>
__device__ __forceinline__ void gn_apply_body(const GnApplyArgs& p, float* sm, const int n, const int chunk_idx, Depart depart) {
  // sm: scale[C], shift[C], mean[G], rstd[G]
  const int C = p.C1 + p.C2;
  float* scale = sm;
  float* shift = sm + C;
  float* gmean = sm + 2 * C;
  float* grstd = gmean + p.G;
  const int cpg = C / p.G;
  // the pivot of group threadIdx.x (the partial means are relative to it, gn_stats_body), in flight during the merge
  const float gpiv = (int)threadIdx.x < p.G ? gn_pivot(p.x1, p.ld1, p.C1, p.x2, p.ld2, p.HW, n, threadIdx.x, cpg) : 0.f;
  {
    // Chan et al. parallel-variance merge of the S partials of every group: one warp per group, lane s holds partial
    // s (and s + 32), then a fixed shuffle-down tree -- the same order in every CTA and every run (deterministic).
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nfull = blockDim.x >> 5;
    if (warp < nfull) {
      for (int g = warp; g < p.G; g += nfull) {
        float cnt = 0.f, mean = 0.f, m2 = 0.f;
        for (int s = lane; s < p.S; s += 32) {
          const float* q = p.partial + ((long long)(n * p.S + s) * p.G + g) * 3;
          const float cb = __ldcg(q), mb = __ldcg(q + 1), qb = __ldcg(q + 2);   // written by other CTAs: bypass L1
          if (cb > 0.f) {
            const float tot = cnt + cb, delta = mb - mean;
            mean += delta * (cb / tot);
            m2 += qb + delta * delta * (cnt * cb / tot);
            cnt = tot;
          }
        }
#pragma unroll
        for (int off = 16; off; off >>= 1) {
          const float cb = __shfl_down_sync(0xffffffffu, cnt, off);
          const float mb = __shfl_down_sync(0xffffffffu, mean, off);
          const float qb = __shfl_down_sync(0xffffffffu, m2, off);
          if (cb > 0.f) {
            const float tot = cnt + cb, delta = mb - mean;
            mean += delta * (cb / tot);
            m2 += qb + delta * delta * (cnt * cb / tot);
            cnt = tot;
          }
        }
        if (lane == 0) {
          gmean[g] = mean;
          grstd[g] = rsqrtf(m2 / cnt + p.eps);
        }
      }
    }
  }
  __syncthreads();
  depart();
  for (int g = threadIdx.x; g < p.G; g += blockDim.x)
    gmean[g] += g == (int)threadIdx.x ? gpiv : gn_pivot(p.x1, p.ld1, p.C1, p.x2, p.ld2, p.HW, n, g, cpg);
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int g = c / cpg;
    const float sc = grstd[g] * p.gamma[c];
    scale[c] = sc;
    shift[c] = p.beta[c] - gmean[g] * sc;
  }
  __syncthreads();
  const int V = C / 8;
  const int p0 = chunk_idx * p.chunk;
  const int p1 = min(p.HW, p0 + p.chunk);
  // thread = (channel vector v, pixel lane r): scale/shift of its 8 channels live in registers
  const int R = blockDim.x / V;
  const int v = threadIdx.x % V, r = threadIdx.x / V;
  if (r >= R) return;
  const int c0 = v * 8;
  float sc[8], sh[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    sc[i] = scale[c0 + i];
    sh[i] = shift[c0 + i];
  }
  const bool second = c0 >= p.C1;
  const __nv_bfloat16* src = second ? p.x2 + (long long)n * p.HW * p.ld2 + (c0 - p.C1)
                                    : p.x1 + (long long)n * p.HW * p.ld1 + c0;
  const long long lds = second ? p.ld2 : p.ld1;
  __nv_bfloat16* dst = p.out + (long long)n * p.HW * p.ldo + c0;
  // back to front: in the one-launch kernel the tail of the chunk is what the statistics pass read last, i.e. what the L2
  // still holds; the output goes out with evict-first stores so that it does not push the input out.  The loads of U pixels
  // are issued before the first store: the compiler may not hoist a load above a store through possibly aliasing pointers,
  // so a plain unrolled loop keeps ONE 16-byte load in flight per thread (ncu r02_gn_fused: 37 % of the DRAM peak).
  auto emit = [&](const uint4& raw, int px) {
    const uint32_t w4[4] = {raw.x, raw.y, raw.z, raw.w};
    float f[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 t = unpack_bf16(w4[i]);
      f[2 * i] = t.x;
      f[2 * i + 1] = t.y;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float y = fmaf(f[i], sc[i], sh[i]);
      f[i] = p.silu ? gn_silu(y) : y;
    }
    __stcs(reinterpret_cast<uint4*>(dst + (long long)px * p.ldo),
           make_uint4(pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]), pack_bf16(f[4], f[5]), pack_bf16(f[6], f[7])));
  };
  constexpr int U = 6;
  int px = p1 - 1 - r;
  for (; px - (U - 1) * R >= p0; px -= U * R) {
    uint4 raw[U];
#pragma unroll
    for (int u = 0; u < U; ++u) raw[u] = *reinterpret_cast<const uint4*>(src + (long long)(px - u * R) * lds);
#pragma unroll
    for (int u = 0; u < U; ++u) emit(raw[u], px - u * R);
  }
  for (; px >= p0; px -= R) emit(*reinterpret_cast<const uint4*>(src + (long long)px * lds), px);
}

__global__ void gn_apply_kernel(const GnApplyArgs p) {
  pdl_enter();
  extern __shared__ float sm[];
  gn_apply_body(p, sm, blockIdx.y, blockIdx.x, [] {});
}

// ------------------------------------------------------------------ GroupNorm in ONE launch
// Statistics and apply of the two-kernel pair above fused behind a per-frame rendezvous: grid (S, NB), every CTA writes
// the partial statistics of its pixel chunk, arrives on the frame's counter, waits until all S chunks of the frame have
// arrived, merges the S partials (same fixed order as gn_apply_kernel: bit-identical results) and normalises the SAME
// chunk it has just read -- at the UNet's sizes (<= 84 MB per tensor) that second read is served by the 126 MB L2 instead
// of HBM, and one launch latency disappears.  The host only launches it when all NB * S CTAs are co-resident (occupancy
// query), which is what makes the spin-wait safe.  counters: int[2 * NB] = {arrived, departed} per frame, zero before the
// first launch; the last CTA to leave a frame resets both, so the buffer is reusable launch after launch (and under CUDA
// graph replay) without a memset.
struct GnFusedArgs {
  GnStatsArgs st;
  GnApplyArgs ap;
  int* counters;
};

__global__ void gn_fused_kernel(const GnFusedArgs p) {
  pdl_enter();
  extern __shared__ float sm[];
  const int n = blockIdx.y, s = blockIdx.x;
  gn_stats_body(p.st, sm, n, s);
  int* arrived = p.counters + 2 * n;
  int* departed = arrived + 1;
  __threadfence();                      // partial statistics visible device-wide before the arrival
  __syncthreads();
  if (threadIdx.x == 0) {
    atomicAdd(arrived, 1);
    while (*reinterpret_cast<volatile int*>(arrived) < p.st.S) __nanosleep(64);
    __threadfence();
  }
  __syncthreads();
  gn_apply_body(p.ap, sm, n, s, [&] {
    if (threadIdx.x == 0) {
      if (atomicAdd(departed, 1) == p.st.S - 1) {   // every CTA of the frame has read the counter: safe to recycle
        *reinterpret_cast<volatile int*>(arrived) = 0;
        *reinterpret_cast<volatile int*>(departed) = 0;
        __threadfence();
      }
    }
  });
}

// ------------------------------------------------------------------ GroupNorm with the frame resident in a cluster
// Small frames (the 8x8 and 16x16 levels of the UNet: 64 / 256 pixels x <= 2560 channels) fit the shared memory of a
// thread-block cluster: grid (CL, NB), cluster (CL, 1, 1), CTA r of frame n keeps pixels [r * P, (r + 1) * P) as raw bf16 in
// shared memory.  ONE pass over HBM: load the chunk (statistics on the fly) -> per-CTA partial (count, mean, M2) per group
// in shared memory -> cluster barrier -> every CTA reads all CL partials through distributed shared memory and merges them
// in rank order (Chan et al., deterministic) -> normalise (+SiLU) its chunk out of shared memory -> store.  No global
// partials, no counters, no spin wait, no second read; same per-chunk / merge arithmetic as gn_stats_body + gn_apply_body.
struct GnClusterArgs {
  const __nv_bfloat16* x1; long long ld1; int C1;
  const __nv_bfloat16* x2; long long ld2; int C2;
  int HW, G, P, R;          // P pixels per CTA (HW = CL * P), R pixel lanes (blockDim.x = (C / 8) * R)
  const float* gamma; const float* beta;
  float eps; int silu;
  __nv_bfloat16* out; long long ldo;
};

__device__ __forceinline__ uint32_t gn_cluster_rank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void gn_cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ float gn_ld_dsmem(const float* local, uint32_t rank) {   // the same offset in CTA `rank`'s shared memory
  uint32_t ra;
  float v;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(smem_u32(local)), "r"(rank));
  asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(ra) : "memory");
  return v;
}

// At most 640 threads (R = 640 / V pixel lanes, C <= GN_MAX_C) and <= 48 registers, i.e. two CTAs per SM: at the 54
// registers the pivots take without the cap, the 8x8 level (32 frames, clusters of four) took 1.5x the time.
__global__ void __launch_bounds__(640, 2) gn_cluster_kernel(const GnClusterArgs p) {
  pdl_enter();
  extern __shared__ __align__(16) uint8_t gn_smem[];
  const int C = p.C1 + p.C2, V = C / 8, G = p.G, cpg = C / G, R = p.R, P = p.P;
  uint4* tile = reinterpret_cast<uint4*>(gn_smem);                      // [P][V] raw bf16 vectors
  float* ssum = reinterpret_cast<float*>(tile + (size_t)P * V);         // [R][C]
  float* ssq = ssum + (size_t)R * C;                                    // [R][C]
  float* part = ssq + (size_t)R * C;                                    // [G][3]: read by the peers
  float* gmean = part + 3 * G;                                          // [G]
  float* grstd = gmean + G;                                             // [G]
  float* scale = grstd + G;                                             // [C]
  float* shift = scale + C;                                             // [C]
  const int n = blockIdx.y;
  const uint32_t rank = gn_cluster_rank(), CL = gridDim.x;
  const int p0 = (int)rank * P;
  const int v = threadIdx.x % V, r = threadIdx.x / V;
  const int c0 = v * 8;
  const bool second = c0 >= p.C1;
  const __nv_bfloat16* base = second ? p.x2 + (long long)n * p.HW * p.ld2 + (c0 - p.C1)
                                     : p.x1 + (long long)n * p.HW * p.ld1 + c0;
  const long long ld = second ? p.ld2 : p.ld1;
  float sum[8], sq[8], piv[8];   // sums of x - pivot (gn_stats_body)
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    sum[i] = sq[i] = 0.f;
    piv[i] = gn_pivot(p.x1, p.ld1, p.C1, p.x2, p.ld2, p.HW, n, (c0 + i) / cpg, cpg);
  }
  constexpr int U = 4;   // global loads in flight per thread
  int px = r;
  for (; px + (U - 1) * R < P; px += U * R) {
    uint4 raw[U];
#pragma unroll
    for (int u = 0; u < U; ++u) raw[u] = *reinterpret_cast<const uint4*>(base + (long long)(p0 + px + u * R) * ld);
#pragma unroll
    for (int u = 0; u < U; ++u) {
      tile[(size_t)(px + u * R) * V + v] = raw[u];
      const uint32_t w4[4] = {raw[u].x, raw[u].y, raw[u].z, raw[u].w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 t = unpack_bf16(w4[i]);
        const float d0 = t.x - piv[2 * i], d1 = t.y - piv[2 * i + 1];
        sum[2 * i] += d0; sq[2 * i] = fmaf(d0, d0, sq[2 * i]);
        sum[2 * i + 1] += d1; sq[2 * i + 1] = fmaf(d1, d1, sq[2 * i + 1]);
      }
    }
  }
  for (; px < P; px += R) {
    const uint4 raw = *reinterpret_cast<const uint4*>(base + (long long)(p0 + px) * ld);
    tile[(size_t)px * V + v] = raw;
    const uint32_t w4[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 t = unpack_bf16(w4[i]);
      const float d0 = t.x - piv[2 * i], d1 = t.y - piv[2 * i + 1];
      sum[2 * i] += d0; sq[2 * i] = fmaf(d0, d0, sq[2 * i]);
      sum[2 * i + 1] += d1; sq[2 * i + 1] = fmaf(d1, d1, sq[2 * i + 1]);
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    ssum[(size_t)r * C + c0 + i] = sum[i];
    ssq[(size_t)r * C + c0 + i] = sq[i];
  }
  __syncthreads();
  for (int g = threadIdx.x; g < G; g += blockDim.x) {   // this CTA's partial of group g (as gn_stats_body)
    float a = 0.f, b = 0.f;
    for (int rr = 0; rr < R; ++rr)
      for (int c = g * cpg; c < (g + 1) * cpg; ++c) {
        a += ssum[(size_t)rr * C + c];
        b += ssq[(size_t)rr * C + c];
      }
    const float cnt = (float)P * cpg;
    const float mean = a / cnt;
    part[3 * g] = cnt;
    part[3 * g + 1] = mean;
    part[3 * g + 2] = fmaxf(b - a * mean, 0.f);
  }
  gn_cluster_sync();                                    // every CTA's partials are written and visible cluster-wide
  for (int g = threadIdx.x; g < G; g += blockDim.x) {   // merge the CL partials in rank order (same in every CTA)
    float cnt = 0.f, mean = 0.f, m2 = 0.f;
    for (uint32_t k = 0; k < CL; ++k) {
      const float cb = gn_ld_dsmem(part + 3 * g, k), mb = gn_ld_dsmem(part + 3 * g + 1, k), qb = gn_ld_dsmem(part + 3 * g + 2, k);
      const float tot = cnt + cb, delta = mb - mean;
      mean += delta * (cb / tot);
      m2 += qb + delta * delta * (cnt * cb / tot);
      cnt = tot;
    }
    gmean[g] = gn_pivot(p.x1, p.ld1, p.C1, p.x2, p.ld2, p.HW, n, g, cpg) + mean;   // one load per group, in parallel
    grstd[g] = rsqrtf(m2 / cnt + p.eps);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int g = c / cpg;
    const float sc = grstd[g] * p.gamma[c];
    scale[c] = sc;
    shift[c] = p.beta[c] - gmean[g] * sc;
  }
  __syncthreads();
  float sc[8], sh[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    sc[i] = scale[c0 + i];
    sh[i] = shift[c0 + i];
  }
  __nv_bfloat16* dst = p.out + (long long)n * p.HW * p.ldo + c0;
  for (int q = r; q < P; q += R) {
    const uint4 raw = tile[(size_t)q * V + v];
    const uint32_t w4[4] = {raw.x, raw.y, raw.z, raw.w};
    float f[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 t = unpack_bf16(w4[i]);
      f[2 * i] = t.x;
      f[2 * i + 1] = t.y;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float y = fmaf(f[i], sc[i], sh[i]);
      f[i] = p.silu ? gn_silu(y) : y;
    }
    store8(dst + (long long)(p0 + q) * p.ldo, f);
  }
  gn_cluster_sync();                                    // nobody leaves while a peer may still read its partials
}

// ------------------------------------------------------------------ LayerNorm (+PE)
// One warp per row; the row lives in registers (C <= 2048), exact two-pass mean/variance like torch.
// TOut = uint8_t: e4m3 codes of the fp32 result and row_scale[row] (vx_layernorm_fp8).
template <int MAXV, typename TOut>
__global__ void layernorm_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, int rows, int C,
                                 const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                 const float* __restrict__ pe, int pe_rows_per_frame, int pe_frames,
                                 TOut* __restrict__ out, long long ldo, float* __restrict__ row_scale) {
  constexpr bool F8 = sizeof(TOut) == 1;
  pdl_enter();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const int V = C / 8;
  float f[MAXV][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int v = lane + i * 32;
    if (v < V) {
      load8(x + (long long)warp * ldx + v * 8, f[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += f[i][j];
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int v = lane + i * 32;
    if (v < V) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = f[i][j] - mean;
        q += d * d;
      }
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / C + eps);
  const float* perow = nullptr;
  if (pe) perow = pe + (long long)((warp / pe_rows_per_frame) % pe_frames) * C;
  auto norm8 = [&](int i, int v, float (&y)[8]) {
    const float4 g0 = *reinterpret_cast<const float4*>(gamma + v * 8), g1 = *reinterpret_cast<const float4*>(gamma + v * 8 + 4);
    const float4 b0 = *reinterpret_cast<const float4*>(beta + v * 8), b1 = *reinterpret_cast<const float4*>(beta + v * 8 + 4);
    const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
    const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
    for (int j = 0; j < 8; ++j) y[j] = (f[i][j] - mean) * rstd * gg[j] + bb[j];
    if (perow) {
      const float4 p0 = *reinterpret_cast<const float4*>(perow + v * 8), p1 = *reinterpret_cast<const float4*>(perow + v * 8 + 4);
      y[0] += p0.x; y[1] += p0.y; y[2] += p0.z; y[3] += p0.w; y[4] += p1.x; y[5] += p1.y; y[6] += p1.z; y[7] += p1.w;
    }
  };
  float inv = 1.f;
  if constexpr (F8) {   // amax pass over the normalised row; the write pass recomputes the same fp32 values
    float amax = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int v = lane + i * 32;
      if (v < V) {
        float y[8];
        norm8(i, v, y);
#pragma unroll
        for (int j = 0; j < 8; ++j) amax = fmaxf(amax, fabsf(y[j]));
      }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    const float sc = e4m3_row_scale(amax);
    inv = 1.0f / sc;
    if (lane == 0) row_scale[warp] = sc;
  }
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int v = lane + i * 32;
    if (v < V) {
      float y[8];
      norm8(i, v, y);
      if constexpr (F8) store8_e4m3(out + (long long)warp * ldo + v * 8, y, inv);
      else store8(out + (long long)warp * ldo + v * 8, y);
    }
  }
}

// ------------------------------------------------------------------ GEGLU gate
__global__ void geglu_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, long long rows, int inner,
                             __nv_bfloat16* __restrict__ out, long long ldo) {
  pdl_enter();
  const int V = inner / 8;
  const long long total = rows * V;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long r = idx / V;
    const int c0 = (int)(idx % V) * 8;
    float h[8], g[8];
    load8(x + r * ldx + c0, h);
    load8(x + r * ldx + inner + c0, g);
#pragma unroll
    for (int i = 0; i < 8; ++i) h[i] *= 0.5f * g[i] * (1.f + erff(g[i] * 0.70710678118654752f));  // stand-alone GEGLU (unfused path)
    store8(out + r * ldo + c0, h);
  }
}

// ------------------------------------------------------------------ row softmax (fp32 scores -> bf16 probs)
// one CTA per row; used by the single-head hd=512 attention of the VAE decoder mid block
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ x, long long ldx, int n,
                                                           __nv_bfloat16* __restrict__ out, long long ldo) {
  pdl_enter();
  __shared__ float red[8];
  const float* row = x + (long long)blockIdx.x * ldx;
  float mx = -INFINITY;
  for (int i = threadIdx.x * 4; i < n; i += 1024) {
    const float4 v = *reinterpret_cast<const float4*>(row + i);
    mx = fmaxf(fmaxf(mx, fmaxf(v.x, v.y)), fmaxf(v.z, v.w));
  }
  for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
  for (int i = 1; i < 8; ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int i = threadIdx.x * 4; i < n; i += 1024) {
    const float4 v = *reinterpret_cast<const float4*>(row + i);
    sum += __expf(v.x - mx) + __expf(v.y - mx) + __expf(v.z - mx) + __expf(v.w - mx);
  }
  for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  sum = 0.f;
  for (int i = 0; i < 8; ++i) sum += red[i];
  const float inv = 1.f / sum;
  __nv_bfloat16* orow = out + (long long)blockIdx.x * ldo;
  for (int i = threadIdx.x * 4; i < n; i += 1024) {
    const float4 v = *reinterpret_cast<const float4*>(row + i);
    *reinterpret_cast<uint2*>(orow + i) = make_uint2(pack_bf16(__expf(v.x - mx) * inv, __expf(v.y - mx) * inv),
                                                     pack_bf16(__expf(v.z - mx) * inv, __expf(v.w - mx) * inv));
  }
}


// ---- LayerNorm for C = 40 * LPR (320 / 640 / 1280, the three transformer widths): LPR lanes per row and exactly
// five 16-byte vectors per lane (no idle lanes, 128-byte coalesced segments), 32 / LPR rows per warp pass.  gamma and
// beta live in registers for the whole grid-stride loop: the per-row version above spends four parameter loads per
// data load on them.
// TOut = uint8_t: e4m3 codes of the fp32 result and row_scale[row] (vx_layernorm_fp8).
template <int LPR, int MINB, typename TOut>
__global__ void __launch_bounds__(256, MINB) layernorm5_kernel(const __nv_bfloat16* __restrict__ x, long long ldx,
                                                            long long rows, const float* __restrict__ gamma,
                                                            const float* __restrict__ beta, float eps,
                                                            const float* __restrict__ pe, int pe_rows_per_frame,
                                                            int pe_frames, TOut* __restrict__ out, long long ldo,
                                                            float* __restrict__ row_scale) {
  constexpr bool F8 = sizeof(TOut) == 1;
  pdl_enter();
  constexpr int RPW = 32 / LPR;
  constexpr int C = LPR * 40;
  // gamma / beta live in shared memory (2.5 - 10 KB): in registers they cost 80 registers per thread, i.e. ONE resident
  // block per SM and 40 KB of loads in flight -- the kernel then sits at 40 % of the HBM peak on latency (ncu r02_ln5:
  // 195 registers, 11.8 % warps active).  Two blocks per SM double the bytes in flight.
  __shared__ __align__(16) float sg[C], sb[C];
  for (int c = threadIdx.x; c < C; c += 256) {
    sg[c] = gamma[c];
    sb[c] = beta[c];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int sub = lane / LPR, l = lane % LPR;
  const long long nwarps = (long long)gridDim.x * 8;
  const long long ngroups = (rows + RPW - 1) / RPW;
  // two row sets per iteration (rows r and r + RPW): twice the bytes in flight for the same parameter registers
  const long long npairs = (ngroups + 1) / 2;
  for (long long grp = (long long)blockIdx.x * 8 + (threadIdx.x >> 5); grp < npairs; grp += nwarps) {
    long long row[2];
    bool ok[2];
    uint4 u[2][5];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      row[r] = (grp * 2 + r) * RPW + sub;
      ok[r] = row[r] < rows;
      const __nv_bfloat16* xp = x + (ok[r] ? row[r] : 0) * ldx + l * 8;
#pragma unroll
      for (int i = 0; i < 5; ++i) u[r][i] = *reinterpret_cast<const uint4*>(xp + i * LPR * 8);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < 5; ++i) {
        const uint32_t w4[4] = {u[r][i].x, u[r][i].y, u[r][i].z, u[r][i].w};
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float2 v = unpack_bf16(w4[t]);
          s += v.x + v.y;
        }
      }
#pragma unroll
      for (int o = LPR / 2; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      const float mean = s * (1.0f / C);
      float q = 0.f;
#pragma unroll
      for (int i = 0; i < 5; ++i) {
        const uint32_t w4[4] = {u[r][i].x, u[r][i].y, u[r][i].z, u[r][i].w};
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float2 v = unpack_bf16(w4[t]);
          const float d0 = v.x - mean, d1 = v.y - mean;
          q = fmaf(d0, d0, q);
          q = fmaf(d1, d1, q);
        }
      }
#pragma unroll
      for (int o = LPR / 2; o; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
      const float rstd = rsqrtf(q * (1.0f / C) + eps);
      const float* perow = pe ? pe + (long long)((row[r] / pe_rows_per_frame) % pe_frames) * C + l * 8 : nullptr;
      TOut* op = out + (ok[r] ? row[r] : 0) * ldo + l * 8;
      auto norm8 = [&](int i, float (&y)[8]) {
        const uint32_t w4[4] = {u[r][i].x, u[r][i].y, u[r][i].z, u[r][i].w};
        int c = (l + i * LPR) * 8;
        asm volatile("" : "+r"(c));     // opaque to the optimiser: or it hoists all 80 parameter loads out of the row loop again
        const float4 g0 = *reinterpret_cast<const float4*>(sg + c), g1 = *reinterpret_cast<const float4*>(sg + c + 4);
        const float4 b0 = *reinterpret_cast<const float4*>(sb + c), b1 = *reinterpret_cast<const float4*>(sb + c + 4);
        const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
        const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float2 v = unpack_bf16(w4[t]);
          y[2 * t] = (v.x - mean) * rstd * gg[2 * t] + bb[2 * t];
          y[2 * t + 1] = (v.y - mean) * rstd * gg[2 * t + 1] + bb[2 * t + 1];
        }
        if (perow) {
          const float4 p0 = *reinterpret_cast<const float4*>(perow + i * LPR * 8);
          const float4 p1 = *reinterpret_cast<const float4*>(perow + i * LPR * 8 + 4);
          y[0] += p0.x; y[1] += p0.y; y[2] += p0.z; y[3] += p0.w; y[4] += p1.x; y[5] += p1.y; y[6] += p1.z; y[7] += p1.w;
        }
      };
      if constexpr (F8) {   // the lane's 40 normalised values stay in registers until the row's amax is known
        float y[5][8];
        float amax = 0.f;
#pragma unroll
        for (int i = 0; i < 5; ++i) {
          norm8(i, y[i]);
#pragma unroll
          for (int j = 0; j < 8; ++j) amax = fmaxf(amax, fabsf(y[i][j]));
        }
#pragma unroll
        for (int o = LPR / 2; o; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
        const float sc = e4m3_row_scale(amax);
        const float inv = 1.0f / sc;
        if (ok[r]) {
#pragma unroll
          for (int i = 0; i < 5; ++i) store8_e4m3(op + i * LPR * 8, y[i], inv);
          if (l == 0) row_scale[row[r]] = sc;
        }
      } else {
#pragma unroll
        for (int i = 0; i < 5; ++i) {
          float y[8];
          norm8(i, y);
          if (ok[r]) store8(op + i * LPR * 8, y);
        }
      }
    }
  }
}


// ---- LayerNorm statistics only: stats[row] = (mean, rstd) with torch's two-pass variance, for the GEMM that applies the
// normalisation in its epilogue (vx_gemm_lnfold_bf16).  C = 40 * LPR uses LPR lanes per row (five 16-byte vectors per
// lane); any other C (multiple of 8, <= 2048) one warp per row.
template <int LPR>
__global__ void __launch_bounds__(256) row_stats5_kernel(const __nv_bfloat16* __restrict__ x, long long ldx,
                                                         long long rows, float eps, float* __restrict__ stats) {
  pdl_enter();
  constexpr int RPW = 32 / LPR;
  constexpr int C = LPR * 40;
  const int lane = threadIdx.x & 31;
  const int sub = lane / LPR, l = lane % LPR;
  const long long nwarps = (long long)gridDim.x * 8;
  const long long ngroups = (rows + RPW - 1) / RPW;
  for (long long grp = (long long)blockIdx.x * 8 + (threadIdx.x >> 5); grp < ngroups; grp += nwarps) {
    const long long row = grp * RPW + sub;
    const bool ok = row < rows;
    const __nv_bfloat16* xp = x + (ok ? row : 0) * ldx + l * 8;
    uint4 u[5];
#pragma unroll
    for (int i = 0; i < 5; ++i) u[i] = *reinterpret_cast<const uint4*>(xp + i * LPR * 8);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      const uint32_t w4[4] = {u[i].x, u[i].y, u[i].z, u[i].w};
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float2 v = unpack_bf16(w4[t]);
        s += v.x + v.y;
      }
    }
#pragma unroll
    for (int o = LPR / 2; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s * (1.0f / C);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      const uint32_t w4[4] = {u[i].x, u[i].y, u[i].z, u[i].w};
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float2 v = unpack_bf16(w4[t]);
        const float d0 = v.x - mean, d1 = v.y - mean;
        q = fmaf(d0, d0, q);
        q = fmaf(d1, d1, q);
      }
    }
#pragma unroll
    for (int o = LPR / 2; o; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    if (ok && l == 0) *reinterpret_cast<float2*>(stats + 2 * row) = make_float2(mean, rsqrtf(q * (1.0f / C) + eps));
  }
}

template <int MAXV>
__global__ void row_stats_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, long long rows, int C, float eps,
                                 float* __restrict__ stats) {
  pdl_enter();
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const int V = C / 8;
  float f[MAXV][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int v = lane + i * 32;
    if (v < V) {
      load8(x + warp * ldx + v * 8, f[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += f[i][j];
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int v = lane + i * 32;
    if (v < V) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = f[i][j] - mean;
        q += d * d;
      }
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  if (lane == 0) *reinterpret_cast<float2*>(stats + 2 * warp) = make_float2(mean, rsqrtf(q / C + eps));
}

}  // namespace vx

using namespace vx;

// Every kernel in this file moves 16-byte vectors (8 bf16 / 4 fp32 values) and never checks the address: the entry points
// reject pointers and leading dimensions that would make one of them misaligned, before any CUDA call.
static bool al16(const void* p) { return ((uintptr_t)p & 15) == 0; }

extern "C" int vx_softmax_rows(const float* x, long long ldx, long long rows, int n, void* out, long long ldo,
                               void* stream) {
  VX_REQUIRE(al16(x) && al16(out) && ldx % 4 == 0 && ldo % 4 == 0,
             "vx_softmax_rows: x / out must be 16-byte aligned and ldx=%lld, ldo=%lld multiples of 4", ldx, ldo);
  VX_REQUIRE(n % 4 == 0, "vx_softmax_rows: n=%d must be a multiple of 4", n);
  launch_k(softmax_rows_kernel, dim3((unsigned)rows), dim3(256), 0, (cudaStream_t)stream, x, ldx, n, (__nv_bfloat16*)out, ldo);
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

static int gn_block(int C, int* R) {
  const int V = C / 8;
  int r = 256 / V;
  if (r < 1) r = 1;
  while (V * r > 1024) --r;
  *R = r;
  return V * r;
}

extern "C" int vx_groupnorm_stats_ws_floats(int NB, int G, int S) { return NB * S * G * 3; }

// Widest [x1 | x2]: the apply and one-launch kernels run C / 8 threads for C >= 2048, and at their ~80 registers a
// 1024-thread block (C = 8192) does not fit the register file.  The model's widest GroupNorm is 2560.
constexpr int GN_MAX_C = 4096;

// [x1 | x2] (x2 only when C2 > 0) and out (when given) 16-byte aligned, leading dimensions multiples of 8
static bool gn_layout_ok(const void* x1, long long ld1, const void* x2, long long ld2, int C2, const void* out, long long ldo) {
  return al16(x1) && ld1 % 8 == 0 && (C2 == 0 || (al16(x2) && ld2 % 8 == 0)) && al16(out) && ldo % 8 == 0;
}
#define GN_REQUIRE_LAYOUT(name, out, ldo)                                                                          \
  VX_REQUIRE(gn_layout_ok(x1, ld1, x2, ld2, C2, out, ldo),                                                          \
             "%s: x1 / x2 / out must be 16-byte aligned with leading dimensions multiples of 8 (ld1=%lld ld2=%lld ldo=%lld)", \
             name, ld1, ld2, (long long)(ldo))

// x = [x1 | x2] per row (x2 may be null, C2 = 0); rows = NB*HW; partial: float[NB*S*G*3] workspace.
extern "C" int vx_groupnorm_stats(const void* x1, long long ld1, int C1, const void* x2, long long ld2, int C2,
                                  int NB, int HW, int G, int S, float* partial, void* stream) {
  GN_REQUIRE_LAYOUT("vx_groupnorm_stats", nullptr, 0);
  const int C = C1 + C2;
  VX_REQUIRE(C1 % 8 == 0 && C2 % 8 == 0 && C % G == 0 && S >= 1, "vx_groupnorm_stats: bad C1=%d C2=%d G=%d", C1, C2, G);
  VX_REQUIRE(C <= GN_MAX_C, "vx_groupnorm_stats: C=%d too wide (at most %d)", C, GN_MAX_C);
  GnStatsArgs a{(const __nv_bfloat16*)x1, ld1, C1, (const __nv_bfloat16*)x2, ld2, C2, HW, G, S, 0, partial};
  const int threads = gn_block(C, &a.R);
  const size_t smem = (size_t)2 * a.R * C * sizeof(float);
  VX_REQUIRE(smem <= 200 * 1024, "vx_groupnorm_stats: smem %zu too large", smem);
  if (smem > 48 * 1024)
    VX_CHECK_CUDA(cudaFuncSetAttribute(gn_stats_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  launch_k(gn_stats_kernel, dim3(S, NB), dim3(threads), smem, (cudaStream_t)stream, a);
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int vx_groupnorm_apply(const void* x1, long long ld1, int C1, const void* x2, long long ld2, int C2,
                                  int NB, int HW, int G, int S, const float* partial, const float* gamma,
                                  const float* beta, float eps, int silu, void* out, long long ldo, void* stream) {
  GN_REQUIRE_LAYOUT("vx_groupnorm_apply", out, ldo);
  const int C = C1 + C2;
  VX_REQUIRE(C1 % 8 == 0 && C2 % 8 == 0 && C % G == 0, "vx_groupnorm_apply: bad C1=%d C2=%d G=%d", C1, C2, G);
  VX_REQUIRE(C <= GN_MAX_C, "vx_groupnorm_apply: C=%d too wide (at most %d)", C, GN_MAX_C);
  GnApplyArgs a{(const __nv_bfloat16*)x1, ld1, C1, (const __nv_bfloat16*)x2, ld2, C2, HW, G, S, partial, gamma, beta,
                eps, silu, (__nv_bfloat16*)out, ldo, 0};
  VX_REQUIRE(S >= 1, "vx_groupnorm_apply: S=%d", S);
  // same partition as the statistics pass: S chunks per frame, sized by the caller so that NB * S CTAs fill the
  // SMs evenly in one wave (a fixed 64 KB chunk left a 10 % second wave at the 64x64 level)
  int chunk = (HW + S - 1) / S;
  if (chunk < 1) chunk = 1;
  a.chunk = chunk;
  const size_t smem = (size_t)(2 * C + 2 * G) * sizeof(float);
  int Rr;
  const int threads = gn_block(C, &Rr);
  launch_k(gn_apply_kernel, dim3((HW + chunk - 1) / chunk, NB), dim3(threads), smem, (cudaStream_t)stream, a);
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// CTAs of the GroupNorm kernels that are resident at once on the whole device for C channels (occupancy query): the host
// sizes S with it so that NB * S CTAs form exactly one wave -- required by the rendezvous of the fused kernel, and what
// keeps the two-kernel pair free of a ragged second wave.
extern "C" int vx_groupnorm_capacity(int C) {
  int R = 1;
  const int threads = gn_block(C, &R);
  size_t smem = (size_t)2 * R * C * sizeof(float);
  if (smem > 200 * 1024) return 0;
  if (smem > 48 * 1024) cudaFuncSetAttribute(gn_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  int per_sm = 0, dev = 0, sms = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gn_fused_kernel, threads, smem) != cudaSuccess) return 0;
  int per_sm2 = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm2, gn_apply_kernel, threads, (size_t)(2 * C + 64) * sizeof(float)) ==
          cudaSuccess && per_sm2 < per_sm)
    per_sm = per_sm2;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return per_sm * sms;
}

// One-launch GroupNorm.  Returns 2 (and launches nothing) when the NB * S CTAs cannot all be resident at once -- the
// caller then uses the two-kernel pair.  counters: int[2 * NB], zero-initialised once by the caller.
extern "C" int vx_groupnorm_fused(const void* x1, long long ld1, int C1, const void* x2, long long ld2, int C2, int NB,
                                  int HW, int G, int S, float* partial, int* counters, const float* gamma,
                                  const float* beta, float eps, int silu, void* out, long long ldo, void* stream) {
  GN_REQUIRE_LAYOUT("vx_groupnorm_fused", out, ldo);
  const int C = C1 + C2;
  VX_REQUIRE(C1 % 8 == 0 && C2 % 8 == 0 && C % G == 0 && S >= 1, "vx_groupnorm_fused: bad C1=%d C2=%d G=%d", C1, C2, G);
  VX_REQUIRE(C <= GN_MAX_C && counters, "vx_groupnorm_fused: C=%d too wide (at most %d) / no counters", C, GN_MAX_C);
  GnFusedArgs a{};
  a.st = GnStatsArgs{(const __nv_bfloat16*)x1, ld1, C1, (const __nv_bfloat16*)x2, ld2, C2, HW, G, S, 0, partial};
  const int threads = gn_block(C, &a.st.R);
  int chunk = (HW + S - 1) / S;
  if (chunk < 1) chunk = 1;
  a.ap = GnApplyArgs{(const __nv_bfloat16*)x1, ld1, C1, (const __nv_bfloat16*)x2, ld2, C2, HW, G, S, partial, gamma, beta,
                     eps, silu, (__nv_bfloat16*)out, ldo, chunk};
  a.counters = counters;
  size_t smem = (size_t)2 * a.st.R * C * sizeof(float);
  const size_t smem_apply = (size_t)(2 * C + 2 * G) * sizeof(float);
  if (smem_apply > smem) smem = smem_apply;
  if (smem > 200 * 1024) return 2;
  static size_t configured = 48 * 1024;
  if (smem > configured) {
    VX_CHECK_CUDA(cudaFuncSetAttribute(gn_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    configured = 200 * 1024;
  }
  int per_sm = 0, dev = 0, sms = 0;
  VX_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gn_fused_kernel, threads, smem));
  VX_CHECK_CUDA(cudaGetDevice(&dev));
  VX_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  if ((long long)NB * S > (long long)per_sm * sms) return 2;   // a rendezvous needs every CTA resident
  launch_k(gn_fused_kernel, dim3(S, NB), dim3(threads), smem, (cudaStream_t)stream, a);
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// GroupNorm of small frames with the frame resident in the shared memory of a thread-block cluster (gn_cluster_kernel).
// Returns 2 (and launches nothing) when the frame does not fit a cluster of <= 8 CTAs -- the caller then takes the
// one-launch rendezvous kernel or the two-kernel pair.
extern "C" int vx_groupnorm_cluster(const void* x1, long long ld1, int C1, const void* x2, long long ld2, int C2, int NB,
                                    int HW, int G, const float* gamma, const float* beta, float eps, int silu, void* out,
                                    long long ldo, void* stream) {
  GN_REQUIRE_LAYOUT("vx_groupnorm_cluster", out, ldo);
  const int C = C1 + C2;
  VX_REQUIRE(C1 % 8 == 0 && C2 % 8 == 0 && C % G == 0, "vx_groupnorm_cluster: bad C1=%d C2=%d G=%d", C1, C2, G);
  VX_REQUIRE(C <= GN_MAX_C, "vx_groupnorm_cluster: C=%d too wide (at most %d)", C, GN_MAX_C);
  const int V = C / 8;
  int R = 640 / V;                       // ~640 threads: 4 pixel lanes at C = 1280, 2 at C = 2560
  if (R < 1) R = 1;
  while (V * R > 1024) --R;
  const int threads = V * R;
  const size_t fixed = ((size_t)2 * R * C + 5 * (size_t)G + 2 * (size_t)C) * sizeof(float);
  int CL = 0;
  for (int cl = 1; cl <= 8; cl *= 2) {
    if (HW % cl) break;
    const size_t need = (size_t)(HW / cl) * C * 2 + fixed;
    if (need <= (size_t)200 * 1024) {
      CL = cl;
      break;
    }
  }
  // One wave only: with more clusters than the device holds at once (the 16x16 level needs 8 CTAs x 32 frames at one CTA per
  // SM) the second wave costs more than the rendezvous kernel's second (L2) read.
  if (!CL || (long long)NB * CL > device_sms()) return 2;
  // more, smaller chunks while the whole grid still is one wave: every SM pulls its chunk at its own (latency-bound) rate
  while (CL * 2 <= 8 && (long long)NB * CL * 2 <= device_sms() && HW % (CL * 2) == 0 && HW / (CL * 2) >= R) CL *= 2;
  GnClusterArgs a{(const __nv_bfloat16*)x1, ld1, C1, (const __nv_bfloat16*)x2, ld2, C2, HW, G, HW / CL, R, gamma, beta, eps, silu,
                  (__nv_bfloat16*)out, ldo};
  const size_t smem = (size_t)(HW / CL) * C * 2 + fixed;
  static bool configured = false;
  if (!configured) {
    VX_CHECK_CUDA(cudaFuncSetAttribute(gn_cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    configured = true;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(CL, NB);
  cfg.blockDim = dim3(threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CL;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 2 : 1;
  VX_CHECK_CUDA(cudaLaunchKernelEx(&cfg, gn_cluster_kernel, a));
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// VX_LN_V1: every C on the one-warp-per-row layernorm_kernel (A/B switch, read once; tests that compare the two kernels in
// one process re-read it through vx_norm_reload_env).
static bool& ln_v1() {
  static bool v = getenv("VX_LN_V1") != nullptr;
  return v;
}
extern "C" void vx_norm_reload_env() { ln_v1() = getenv("VX_LN_V1") != nullptr; }

// pe: optional float [pe_frames, C]; row r uses pe[(r / rows_per_frame) % pe_frames].  TOut = uint8_t: e4m3 codes + row_scale.
template <typename TOut>
static int layernorm_entry(const void* x, long long ldx, long long rows, int C, const float* gamma, const float* beta,
                           float eps, const float* pe, int rows_per_frame, int pe_frames, void* out, long long ldo,
                           float* row_scale, void* stream) {
  constexpr bool F8 = sizeof(TOut) == 1;
  const char* name = F8 ? "vx_layernorm_fp8" : "vx_layernorm";
  // x: 16-byte rows; gamma / beta / pe: float4 loads; out: 16-byte (bf16) or 8-byte (e4m3) stores
  VX_REQUIRE(al16(x) && ldx % 8 == 0 && ((uintptr_t)out & (F8 ? 7 : 15)) == 0 && ldo % 8 == 0 && al16(gamma) && al16(beta) &&
                 al16(pe),
             "%s: x / gamma / beta / pe must be 16-byte aligned, out %d-byte aligned, ldx=%lld and ldo=%lld multiples of 8",
             name, F8 ? 8 : 16, ldx, ldo);
  VX_REQUIRE(C % 8 == 0 && C <= 2048, "%s: C=%d unsupported", name, C);
  VX_REQUIRE(!F8 || row_scale, "vx_layernorm_fp8: row_scale missing");
  const int threads = 256;
  const long long blocks = (rows * 32 + threads - 1) / threads;
  const int V = C / 8;
  auto st = (cudaStream_t)stream;
  if (pe && (rows_per_frame <= 0 || pe_frames <= 0)) return fail("%s: bad pe args", name);
  // The positional-encoding variant (temporal attention norms) takes the same kernel since its parameters moved to shared
  // memory: 63.5 -> ~41 us at the 320-wide level (the one-warp-per-row kernel used to be as fast).  VX_LN_PE5=0: old choice.
  static const bool ln_pe5 = !(getenv("VX_LN_PE5") && atoi(getenv("VX_LN_PE5")) == 0);
  if ((C == 320 || C == 640 || C == 1280) && (!pe || ln_pe5) && !ln_v1()) {
    const int lpr = C / 40;
    const long long groups = (rows + 32 / lpr - 1) / (32 / lpr);
    long long nb = ((groups + 1) / 2 + 7) / 8;
    static const int minb_env = getenv("VX_LN_BLOCKS") ? atoi(getenv("VX_LN_BLOCKS")) : 3;   // read once (A/B switch)
    // e4m3: the lane's 40 normalised values wait in registers for the row amax -- two blocks per SM (three spill)
    const int minb = F8 ? 2 : minb_env;
    if (nb > device_sms() * minb * 2) nb = device_sms() * minb * 2;   // `minb` 256-thread blocks are resident per SM; two waves balance the tail
    if (nb < 1) nb = 1;
#define LN5_LAUNCH(LPR)                                                                                               \
  do {                                                                                                               \
    if (minb == 2) {                                                                                                 \
      launch_k((layernorm5_kernel<LPR, 2, TOut>), dim3((unsigned)nb), dim3(256), 0, st, (const __nv_bfloat16*)x, ldx, rows, gamma, beta, \
               eps, pe, rows_per_frame, pe_frames, (TOut*)out, ldo, row_scale);                                      \
    } else if constexpr (!F8) {                                                                                      \
      launch_k((layernorm5_kernel<LPR, 3, TOut>), dim3((unsigned)nb), dim3(256), 0, st, (const __nv_bfloat16*)x, ldx, rows, gamma, beta, \
               eps, pe, rows_per_frame, pe_frames, (TOut*)out, ldo, row_scale);                                      \
    }                                                                                                                \
  } while (0)
    if (lpr == 8) LN5_LAUNCH(8);
    else if (lpr == 16) LN5_LAUNCH(16);
    else LN5_LAUNCH(32);
#undef LN5_LAUNCH
    VX_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
#define LN_LAUNCH(MV)                                                                                            \
  launch_k(layernorm_kernel<MV, TOut>, dim3((unsigned)blocks), dim3(threads), 0, st, (const __nv_bfloat16*)x, ldx, (int)rows, C, \
           gamma, beta, eps, pe, rows_per_frame, pe_frames, (TOut*)out, ldo, row_scale)
  if (V <= 32) LN_LAUNCH(1);
  else if (V <= 64) LN_LAUNCH(2);
  else if (V <= 96) LN_LAUNCH(3);
  else if (V <= 160) LN_LAUNCH(5);
  else LN_LAUNCH(8);
#undef LN_LAUNCH
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int vx_layernorm(const void* x, long long ldx, long long rows, int C, const float* gamma,
                            const float* beta, float eps, const float* pe, int rows_per_frame, int pe_frames,
                            void* out, long long ldo, void* stream) {
  return layernorm_entry<__nv_bfloat16>(x, ldx, rows, C, gamma, beta, eps, pe, rows_per_frame, pe_frames, out, ldo, nullptr,
                                        stream);
}

// LayerNorm (+ pe) -> float8_e4m3fn codes out[row, c] = sat_rn(y / row_scale[row]) of the fp32 result y (no bf16 rounding
// on the way), row_scale[row] = amax_c |y| / 448 (1 for an all-zero row): the A operand of vx_gemm_fp8.
extern "C" int vx_layernorm_fp8(const void* x, long long ldx, long long rows, int C, const float* gamma,
                                const float* beta, float eps, const float* pe, int rows_per_frame, int pe_frames,
                                void* out, long long ldo, float* row_scale, void* stream) {
  return layernorm_entry<uint8_t>(x, ldx, rows, C, gamma, beta, eps, pe, rows_per_frame, pe_frames, out, ldo, row_scale,
                                  stream);
}

// x: [rows, 2*inner] = (h | gate) -> out [rows, inner]
extern "C" int vx_geglu(const void* x, long long ldx, long long rows, int inner, void* out, long long ldo,
                        void* stream) {
  VX_REQUIRE(al16(x) && al16(out) && ldx % 8 == 0 && ldo % 8 == 0,
             "vx_geglu: x / out must be 16-byte aligned and ldx=%lld, ldo=%lld multiples of 8", ldx, ldo);
  VX_REQUIRE(inner % 8 == 0, "vx_geglu: inner=%d", inner);
  const long long total = rows * (inner / 8);
  long long blocks = (total + 255) / 256;
  if (blocks > device_sms() * 16) blocks = device_sms() * 16;
  launch_k(geglu_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, (const __nv_bfloat16*)x, ldx, rows, inner,
                                                                  (__nv_bfloat16*)out, ldo);
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}


// stats: float[rows][2] = (mean, rstd) of every row of x (LayerNorm statistics, eps inside the rsqrt like torch)
extern "C" int vx_row_stats(const void* x, long long ldx, long long rows, int C, float eps, float* stats, void* stream) {
  VX_REQUIRE(al16(x) && ldx % 8 == 0 && ((uintptr_t)stats & 7) == 0,
             "vx_row_stats: x must be 16-byte aligned with ldx=%lld a multiple of 8, stats 8-byte aligned", ldx);
  VX_REQUIRE(C % 8 == 0 && C <= 2048, "vx_row_stats: C=%d unsupported", C);
  auto st = (cudaStream_t)stream;
  if (C == 320 || C == 640 || C == 1280) {
    const int lpr = C / 40;
    const long long groups = (rows + 32 / lpr - 1) / (32 / lpr);
    long long nb = (groups + 7) / 8;
    if (nb > device_sms() * 8) nb = device_sms() * 8;
    if (nb < 1) nb = 1;
    if (lpr == 8) launch_k(row_stats5_kernel<8>, dim3((unsigned)nb), dim3(256), 0, st, (const __nv_bfloat16*)x, ldx, rows, eps, stats);
    else if (lpr == 16) launch_k(row_stats5_kernel<16>, dim3((unsigned)nb), dim3(256), 0, st, (const __nv_bfloat16*)x, ldx, rows, eps, stats);
    else launch_k(row_stats5_kernel<32>, dim3((unsigned)nb), dim3(256), 0, st, (const __nv_bfloat16*)x, ldx, rows, eps, stats);
  } else {
    const long long blocks = (rows * 32 + 255) / 256;
    const int V = C / 8;
    if (V <= 32) launch_k(row_stats_kernel<1>, dim3((unsigned)blocks), dim3(256), 0, st, (const __nv_bfloat16*)x, ldx, rows, C, eps, stats);
    else if (V <= 64) launch_k(row_stats_kernel<2>, dim3((unsigned)blocks), dim3(256), 0, st, (const __nv_bfloat16*)x, ldx, rows, C, eps, stats);
    else if (V <= 96) launch_k(row_stats_kernel<3>, dim3((unsigned)blocks), dim3(256), 0, st, (const __nv_bfloat16*)x, ldx, rows, C, eps, stats);
    else if (V <= 160) launch_k(row_stats_kernel<5>, dim3((unsigned)blocks), dim3(256), 0, st, (const __nv_bfloat16*)x, ldx, rows, C, eps, stats);
    else launch_k(row_stats_kernel<8>, dim3((unsigned)blocks), dim3(256), 0, st, (const __nv_bfloat16*)x, ldx, rows, C, eps, stats);
  }
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}
