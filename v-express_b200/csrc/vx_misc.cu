// Small kernels around the GEMM/conv/attention core (all HBM- or latency-bound, CUDA cores):
//   * conv_in  : 3x3 conv from Cin<=8 planar (n,c,h,w)/(b,c,f,h,w) input to NHWC bf16, + bias + kps_features
//                (reference modules/unet_3d.py:485-487; also the VAE decoder conv_in).
//   * conv_out : 3x3 conv from NHWC bf16 to Cout<=4 planar output (reference modules/unet_3d.py:573; VAE conv_out
//                with the (x/2+0.5).clamp(0,1) of pipelines/v_express_pipeline.py:160 fused).
//   * im2col for the stride-2 Downsample3D conv (modules/resnet.py:93-120), nearest-2x Upsample3D (:53-82).
//   * skinny linear for the time embedding MLP and the 22 time_emb_proj (modules/unet_3d.py:464-470,
//     modules/resnet.py:225-228): rows <= 8, one warp per output feature.
//   * CFG + /count + overlap accumulation and the DDIM update (pipelines/v_express_pipeline.py:548-572).
#include "vx_host.h"
#include "vx_ptx.cuh"

namespace vx {

// ------------------------------------------------------------------ conv_in
// in: planar, element (img n, ch c, y, x) at in[n*sn + c*sc + y*W + x]  (bf16)
// wt: fp32 [Cin*9][Cout] (transposed conv weight) ; out NHWC [n*H*W + y*W + x][Cout]
// addend (optional): NHWC bf16 rows indexed by add_row[n] (frame gather) or n when add_row == null
struct ConvInArgs {
  const __nv_bfloat16* in; long long sn, sc;
  int NB, H, W, Cin, Cout;
  const float* wt; const float* bias;
  const __nv_bfloat16* addend; const int* add_frame; long long add_ld;
  float pre_scale; const float* pre_w; const float* pre_b;  // optional per-pixel 1x1 pre-transform
  __nv_bfloat16* out; long long ldo;
};

__device__ __forceinline__ float rbf16(float v) { return __bfloat162float(__float2bfloat16(v)); }

template <int CIN>
__global__ void __launch_bounds__(256) conv_in_kernel(const ConvInArgs p) {
  pdl_enter();
  // Every thread owns 8 output channels of 4 horizontally adjacent pixels, so each weight read from shared memory
  // feeds 4 FMAs (one pixel per thread left the kernel bound by shared-memory bandwidth, 1 LDS word per FMA).
  // Weights sit in two planes [K][Cout/2] (channels 8v..8v+3 | 8v+4..8v+7 of vector v) so that consecutive lanes
  // read consecutive 16-byte words.  p.w is pre-transposed on the host side of the ABI ([Cin*9][Cout]).
  extern __shared__ float sw[];
  constexpr int K = CIN * 9;
  const int half = p.Cout / 2;
  for (int i = threadIdx.x; i < K * p.Cout; i += blockDim.x) {
    const int k = i / p.Cout, c = i % p.Cout;
    sw[((c & 4) ? K * half : 0) + k * half + (c >> 3) * 4 + (c & 3)] = p.wt[i];
  }
  __syncthreads();
  const int vecs = p.Cout / 8;
  const int WQ = (p.W + 3) / 4;
  const long long total = (long long)p.NB * p.H * WQ * vecs;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(idx % vecs);
    const long long quad = idx / vecs;
    const int x0 = (int)(quad % WQ) * 4;
    const int y = (int)((quad / WQ) % p.H);
    const int n = (int)(quad / ((long long)WQ * p.H));
    float acc[4][8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float bv = p.bias ? p.bias[cv * 8 + i] : 0.f;
#pragma unroll
      for (int px = 0; px < 4; ++px) acc[px][i] = bv;
    }
#pragma unroll
    for (int dy = 0; dy < 3; ++dy) {
      const int yy = y + dy - 1;
      if (yy < 0 || yy >= p.H) continue;
      float vin[6][CIN];   // columns x0-1 .. x0+4 of input row yy; zero outside the image (conv padding)
#pragma unroll
      for (int cx = 0; cx < 6; ++cx) {
        const int xx = x0 + cx - 1;
        const bool valid = xx >= 0 && xx < p.W;
#pragma unroll
        for (int c = 0; c < CIN; ++c)
          vin[cx][c] = valid ? __bfloat162float(p.in[n * p.sn + c * p.sc + yy * p.W + xx]) : 0.f;
        if (p.pre_w && valid) {
          float tmp[CIN];
#pragma unroll
          for (int c = 0; c < CIN; ++c) tmp[c] = rbf16(p.pre_scale * vin[cx][c]);
#pragma unroll
          for (int c = 0; c < CIN; ++c) {
            float a = p.pre_b ? p.pre_b[c] : 0.f;
#pragma unroll
            for (int k = 0; k < CIN; ++k) a += p.pre_w[c * CIN + k] * tmp[k];
            vin[cx][c] = rbf16(a);
          }
        }
      }
#pragma unroll
      for (int dx = 0; dx < 3; ++dx) {
#pragma unroll
        for (int c = 0; c < CIN; ++c) {
          const int k = c * 9 + dy * 3 + dx;
          const float4 w0 = *reinterpret_cast<const float4*>(sw + k * half + cv * 4);
          const float4 w1 = *reinterpret_cast<const float4*>(sw + K * half + k * half + cv * 4);
          const float wr[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
          for (int px = 0; px < 4; ++px) {
            const float v = vin[px + dx][c];
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[px][i] += v * wr[i];
          }
        }
      }
    }
#pragma unroll
    for (int px = 0; px < 4; ++px) {
      const int x = x0 + px;
      if (x >= p.W) continue;
      const long long pix = ((long long)n * p.H + y) * p.W + x;
      if (p.addend) {
        const long long arow = (p.add_frame ? (long long)p.add_frame[n] : (long long)n) * p.H * p.W + (long long)y * p.W + x;
        const uint4 u = *reinterpret_cast<const uint4*>(p.addend + arow * p.add_ld + cv * 8);
        const uint32_t ww[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 t = unpack_bf16(ww[i]);
          acc[px][2 * i] += t.x;
          acc[px][2 * i + 1] += t.y;
        }
      }
      *reinterpret_cast<uint4*>(p.out + pix * p.ldo + cv * 8) =
          make_uint4(pack_bf16(acc[px][0], acc[px][1]), pack_bf16(acc[px][2], acc[px][3]),
                     pack_bf16(acc[px][4], acc[px][5]), pack_bf16(acc[px][6], acc[px][7]));
    }
  }
}

// ------------------------------------------------------------------ conv_out
// x NHWC bf16 [NB*H*W, C] (already normalised + SiLU) ; w fp32 [Cout][9][C] ; one warp per output pixel.
// out planar: element (n, co, y, x) at out[n*sn + co*sc + y*W + x]; out_f32 selects fp32 vs bf16 storage;
// post = 1 applies (v/2 + 0.5).clamp(0,1).
struct ConvOutArgs {
  const __nv_bfloat16* x; long long ldx;
  int NB, H, W, C, Cout;
  const float* w; const float* bias;
  void* out; long long sn, sc; int out_f32, post;
};

__global__ void conv_out_kernel(const ConvOutArgs p) {
  pdl_enter();
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long npix = (long long)p.NB * p.H * p.W;
  if (warp >= npix) return;
  const int x = (int)(warp % p.W);
  const int y = (int)((warp / p.W) % p.H);
  const long long n = warp / ((long long)p.W * p.H);
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  const int vecs = p.C / 8;
  for (int t = 0; t < 9; ++t) {
    const int yy = y + t / 3 - 1, xx = x + t % 3 - 1;
    if (yy < 0 || yy >= p.H || xx < 0 || xx >= p.W) continue;
    const __nv_bfloat16* row = p.x + ((n * p.H + yy) * p.W + xx) * p.ldx;
    for (int v = lane; v < vecs; v += 32) {
      const uint4 u = *reinterpret_cast<const uint4*>(row + v * 8);
      const uint32_t ww[4] = {u.x, u.y, u.z, u.w};
      float f[8];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 tt = unpack_bf16(ww[i]);
        f[2 * i] = tt.x;
        f[2 * i + 1] = tt.y;
      }
      for (int co = 0; co < p.Cout; ++co) {
        const float* wr = p.w + ((long long)co * 9 + t) * p.C + v * 8;
        const float4 w0 = *reinterpret_cast<const float4*>(wr);
        const float4 w1 = *reinterpret_cast<const float4*>(wr + 4);
        acc[co] += f[0] * w0.x + f[1] * w0.y + f[2] * w0.z + f[3] * w0.w + f[4] * w1.x + f[5] * w1.y + f[6] * w1.z +
                   f[7] * w1.w;
      }
    }
  }
#pragma unroll
  for (int co = 0; co < 4; ++co)
#pragma unroll
    for (int o = 16; o; o >>= 1) acc[co] += __shfl_xor_sync(0xffffffffu, acc[co], o);
  if (lane < p.Cout) {
    float v = acc[0];
    if (lane == 1) v = acc[1];
    if (lane == 2) v = acc[2];
    if (lane == 3) v = acc[3];
    v += p.bias ? p.bias[lane] : 0.f;
    if (p.post) v = fminf(fmaxf(v * 0.5f + 0.5f, 0.f), 1.f);
    const long long off = n * p.sn + lane * p.sc + (long long)y * p.W + x;
    if (p.out_f32) reinterpret_cast<float*>(p.out)[off] = v;
    else reinterpret_cast<__nv_bfloat16*>(p.out)[off] = __float2bfloat16(v);
  }
}

// ------------------------------------------------------------------ NHWC (first Cout <= 8 channels) -> planar
// Tail of the tensor-core conv_out path: the 3x3 conv runs on the wgmma kernel with Cout zero-padded to 32;
// this extracts the real channels into (n, co, y, x) planes (+ optional (v/2+0.5).clamp(0,1), fp32 or bf16).
__global__ void extract_planar_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, long long npix, int HW,
                                      int Cout, void* __restrict__ out, long long sn, long long sc, int out_f32,
                                      int post) {
  pdl_enter();
  for (long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x; pix < npix;
       pix += (long long)gridDim.x * blockDim.x) {
    const uint4 u = *reinterpret_cast<const uint4*>(x + pix * ldx);
    const uint32_t w4[4] = {u.x, u.y, u.z, u.w};
    float f[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 t = unpack_bf16(w4[i]);
      f[2 * i] = t.x;
      f[2 * i + 1] = t.y;
    }
    const long long n = pix / HW, r = pix % HW;
#pragma unroll
    for (int co = 0; co < 8; ++co) {
      if (co < Cout) {
        float v = f[co];
        if (post) v = fminf(fmaxf(v * 0.5f + 0.5f, 0.f), 1.f);
        const long long off = n * sn + co * sc + r;
        if (out_f32) reinterpret_cast<float*>(out)[off] = v;
        else reinterpret_cast<__nv_bfloat16*>(out)[off] = __float2bfloat16(v);
      }
    }
  }
}

// ------------------------------------------------------------------ im2col (3x3, stride 2, pad 1), NHWC
__global__ void im2col_s2_kernel(const __nv_bfloat16* __restrict__ x, int NB, int H, int W, int C,
                                 __nv_bfloat16* __restrict__ out) {
  pdl_enter();
  const int Ho = H / 2, Wo = W / 2, V = C / 8;
  const long long total = (long long)NB * Ho * Wo * 9 * V;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(idx % V);
    const int t = (int)((idx / V) % 9);
    const long long opix = idx / ((long long)V * 9);
    const int ox = (int)(opix % Wo), oy = (int)((opix / Wo) % Ho);
    const long long n = opix / ((long long)Wo * Ho);
    const int yy = oy * 2 + t / 3 - 1, xx = ox * 2 + t % 3 - 1;
    uint4 val = make_uint4(0, 0, 0, 0);
    if (yy >= 0 && yy < H && xx >= 0 && xx < W)
      val = *reinterpret_cast<const uint4*>(x + ((n * H + yy) * W + xx) * C + v * 8);
    *reinterpret_cast<uint4*>(out + opix * 9 * C + (long long)t * C + v * 8) = val;
  }
}

// ------------------------------------------------------------------ nearest 2x upsample, NHWC
__global__ void upsample2x_kernel(const __nv_bfloat16* __restrict__ x, int NB, int H, int W, int C,
                                  __nv_bfloat16* __restrict__ out) {
  pdl_enter();
  const int V = C / 8;
  const long long total = (long long)NB * 2 * H * 2 * W * V;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(idx % V);
    const long long opix = idx / V;
    const int ox = (int)(opix % (2 * W)), oy = (int)((opix / (2 * W)) % (2 * H));
    const long long n = opix / ((long long)4 * W * H);
    *reinterpret_cast<uint4*>(out + opix * C + v * 8) =
        *reinterpret_cast<const uint4*>(x + ((n * H + oy / 2) * W + ox / 2) * C + v * 8);
  }
}

// ------------------------------------------------------------------ skinny linear (rows <= 8)
// y[r, n] = act_out( sum_k act_in(x[r,k]) * W[n,k] + b[n] );  act: 0 none, 1 SiLU.  x,y fp32; W bf16.
__global__ void skinny_linear_kernel(const float* __restrict__ x, int rows, int K, const __nv_bfloat16* __restrict__ w,
                                     const float* __restrict__ bias, int N, int act_in, int act_out,
                                     float* __restrict__ y) {
  pdl_enter();
  const int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (n >= N) return;
  float acc[8];
#pragma unroll
  for (int r = 0; r < 8; ++r) acc[r] = 0.f;
  for (int k = lane * 8; k < K; k += 256) {
    float wv[8];
    const uint4 u = *reinterpret_cast<const uint4*>(w + (long long)n * K + k);
    const uint32_t ww[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 t = unpack_bf16(ww[i]);
      wv[2 * i] = t.x;
      wv[2 * i + 1] = t.y;
    }
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      if (r < rows) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          float xv = x[r * K + k + i];
          if (act_in) xv = xv / (1.f + __expf(-xv));
          acc[r] += xv * wv[i];
        }
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 8; ++r)
#pragma unroll
    for (int o = 16; o; o >>= 1) acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], o);
  if (lane == 0) {
    for (int r = 0; r < rows; ++r) {
      float v = acc[r] + (bias ? bias[n] : 0.f);
      if (act_out) v = v / (1.f + __expf(-v));
      y[(long long)r * N + n] = v;
    }
  }
}

// Timesteps(dim, flip_sin_to_cos=True, shift 0): out[r] = [cos(t*f_i) | sin(t*f_i)], rounded through bf16 like the
// reference's cast to the model dtype (modules/unet_3d.py:469).
__global__ void timestep_embed_kernel(const float* __restrict__ t, int rows, int dim, float* __restrict__ out) {
  pdl_enter();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int half = dim / 2;
  if (idx >= rows * half) return;
  const int r = idx / half, i = idx % half;
  const float freq = expf(-logf(10000.f) * (float)i / (float)half);
  const float a = t[r] * freq;
  out[r * dim + i] = __bfloat162float(__float2bfloat16(cosf(a)));
  out[r * dim + half + i] = __bfloat162float(__float2bfloat16(sinf(a)));
}

// ------------------------------------------------------------------ CFG + /count + overlap accumulate
// noise: frame-major planar bf16 ((b f), 4, h, w) from the UNet's conv_out; local frame i -> global frame win[i]:
//   acc[:, win[i]] += bf16( bf16(u + g*(c-u)) / count[win[i]] )     (same rounding points as the reference's
//   model-dtype arithmetic, pipelines/v_express_pipeline.py:548-560)
struct CfgArgs {
  const __nv_bfloat16* noise; int f, hw, L, do_cfg;
  const int* win; const int* count; float g;
  float* acc;  // fp32 (4, L, hw) accumulator holding bf16-representable partial sums
};

__device__ __forceinline__ float rbf(float v) { return __bfloat162float(__float2bfloat16(v)); }

__global__ void cfg_overlap_kernel(const CfgArgs p) {
  pdl_enter();
  const long long total = (long long)4 * p.f * p.hw;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int px = (int)(idx % p.hw);
    const int i = (int)((idx / p.hw) % p.f);
    const int c = (int)(idx / ((long long)p.hw * p.f));
    const long long off = ((long long)i * 4 + c) * p.hw + px;
    const int fr = p.win[i];
    if (fr < 0) continue;            // slot discarded by the reference's bookkeeping (pipelines/context.py overlap_plan)
    float v;
    if (p.do_cfg) {
      const float u = __bfloat162float(p.noise[off]);
      const float cd = __bfloat162float(p.noise[(long long)4 * p.f * p.hw + off]);
      v = rbf(u + rbf(p.g * rbf(cd - u)));
    } else {
      v = __bfloat162float(p.noise[off]);
    }
    v = rbf(v / (float)p.count[fr]);
    float* a = p.acc + ((long long)c * p.L + fr) * p.hw + px;
    *a = rbf(*a + v);
  }
}

// The same for n samples in one launch: noise ((b n f), 4, h, w) laid out [uncond s0..s(n-1) | cond s0..s(n-1)], each
// block f frames; acc fp32 (n, 4, L, hw).  Every element goes through exactly the rounding points of cfg_overlap_kernel,
// so sample s of an n-sample window accumulates the same bits as a one-sample window would.
struct CfgNArgs {
  const __nv_bfloat16* noise; int n, f, hw, L, do_cfg;
  const int* win; const int* count; float g;
  float* acc;
};

__global__ void cfg_overlap_n_kernel(const CfgNArgs p) {
  pdl_enter();
  const long long per = (long long)4 * p.f * p.hw;   // one sample's block of the noise
  const long long total = per * p.n;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int px = (int)(idx % p.hw);
    const int i = (int)((idx / p.hw) % p.f);
    const int c = (int)((idx / ((long long)p.hw * p.f)) % 4);
    const int s = (int)(idx / per);
    const int fr = p.win[i];
    if (fr < 0) continue;
    const long long off = (long long)s * per + ((long long)i * 4 + c) * p.hw + px;
    float v;
    if (p.do_cfg) {
      const float u = __bfloat162float(p.noise[off]);
      const float cd = __bfloat162float(p.noise[(long long)p.n * per + off]);
      v = rbf(u + rbf(p.g * rbf(cd - u)));
    } else {
      v = __bfloat162float(p.noise[off]);
    }
    v = rbf(v / (float)p.count[fr]);
    float* a = p.acc + (((long long)s * 4 + c) * p.L + fr) * p.hw + px;
    *a = rbf(*a + v);
  }
}

// DDIM v-prediction step on all frames (eta = 0), bf16 rounding after every tensor op like the reference
// (diffusers DDIMScheduler.step with fp32 scalar coefficients on model-dtype tensors, SURVEY.md B.5).
__device__ __forceinline__ __nv_bfloat16 ddim_update(float x, float acc, float sa, float sb, float sap, float sbp) {
  const float v = rbf(acc);   // no-op on one GPU; after the fp32 all-reduce of two bf16 partial sums = their bf16 sum
  const float x0 = rbf(rbf(sa * x) - rbf(sb * v));
  const float eps = rbf(rbf(sa * v) + rbf(sb * x));
  const float dir = rbf(sbp * eps);
  return __float2bfloat16(rbf(sap * x0) + dir);
}

__global__ void ddim_step_kernel(__nv_bfloat16* __restrict__ latents, const float* __restrict__ acc, long long n,
                                 float sa, float sb, float sap, float sbp) {
  pdl_enter();
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n;
       idx += (long long)gridDim.x * blockDim.x)
    latents[idx] = ddim_update(__bfloat162float(latents[idx]), acc[idx], sa, sb, sap, sbp);
}

// Stochastic DDIM (eta > 0): the same update with c_dir = sqrt(1 - a_prev - sigma^2) in place of sqrt(1 - a_prev),
// then diffusers' `prev_sample + std_dev_t * variance_noise` on model-dtype tensors: bf16(sigma * noise), then the bf16
// add.  noise is the fp32 image of the draw (exact for bf16 / fp16 / fp32 draws), laid out like latents.
__global__ void ddim_step_eta_kernel(__nv_bfloat16* __restrict__ latents, const float* __restrict__ acc,
                                     const float* __restrict__ noise, long long n, float sa, float sb, float sap,
                                     float c_dir, float sigma) {
  pdl_enter();
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n;
       idx += (long long)gridDim.x * blockDim.x) {
    const float prev = __bfloat162float(ddim_update(__bfloat162float(latents[idx]), acc[idx], sa, sb, sap, c_dir));
    latents[idx] = __float2bfloat16(prev + rbf(sigma * noise[idx]));
  }
}

// The same update on the k frames listed in `frames` of latents / acc (ns, L, hw) -- ns = n samples x 4 channels --
// zeroing those acc entries for the next step's sums.  The wavefront schedule of VExpressPipeline.stream finalises a
// frame's step as soon as its last window has contributed, so frames are at different steps and acc is cleared per frame.
__global__ void ddim_step_frames_kernel(__nv_bfloat16* __restrict__ latents, float* __restrict__ acc, int ns, int L,
                                        int hw, const int* __restrict__ frames, int k, float sa, float sb, float sap,
                                        float sbp) {
  pdl_enter();
  const long long total = (long long)ns * k * hw;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int px = (int)(idx % hw);
    const int j = (int)((idx / hw) % k);
    const long long sc = idx / ((long long)hw * k);
    const long long off = (sc * L + frames[j]) * hw + px;
    latents[off] = ddim_update(__bfloat162float(latents[off]), acc[off], sa, sb, sap, sbp);
    acc[off] = 0.f;
  }
}

// DPM-Solver++ (diffusers DPMSolverMultistepScheduler, algorithm_type "dpmsolver++", solver_type "midpoint",
// v-prediction) with the rounding points of the library's eager arithmetic on bf16 CUDA tensors: convert_model_output
// runs on the bf16 sample, so the x0 prediction m0 and the history are bf16; step then upcasts the sample to fp32, so
// ratio * x stays fp32 while every fp32-scalar x bf16-tensor product rounds to bf16; prev_sample is cast back to bf16.
// The fp32 products and differences are spelled with _rn intrinsics so that no FMA contraction changes them.
struct DpmCoeffs {
  float alpha_s, sigma_s, ratio, c0, inv_r0, c0h;  // c0 = alpha_t (e^-h - 1), c0h = 0.5 c0; inv_r0 / c0h: order 2 only
  int order;
};

__device__ __forceinline__ void dpmpp_update(__nv_bfloat16* lat, float acc, __nv_bfloat16* hist, const DpmCoeffs& c) {
  const float x = __bfloat162float(*lat);
  const float m0 = rbf(rbf(c.alpha_s * x) - rbf(c.sigma_s * rbf(acc)));
  float xt = __fsub_rn(__fmul_rn(c.ratio, x), rbf(c.c0 * m0));
  if (c.order == 2) {
    const float d1 = rbf(c.inv_r0 * rbf(m0 - __bfloat162float(*hist)));
    xt = __fsub_rn(xt, rbf(c.c0h * d1));
  }
  *hist = __float2bfloat16(m0);
  *lat = __float2bfloat16(xt);
}

__global__ void dpmpp_step_kernel(__nv_bfloat16* __restrict__ latents, const float* __restrict__ acc,
                                  __nv_bfloat16* __restrict__ x0_prev, long long n, DpmCoeffs c) {
  pdl_enter();
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n;
       idx += (long long)gridDim.x * blockDim.x)
    dpmpp_update(latents + idx, acc[idx], x0_prev + idx, c);
}

// The same update on the k frames listed in `frames`, zeroing those acc entries (the wavefront of
// VExpressPipeline.stream, as ddim_step_frames_kernel).
__global__ void dpmpp_step_frames_kernel(__nv_bfloat16* __restrict__ latents, float* __restrict__ acc,
                                         __nv_bfloat16* __restrict__ x0_prev, int ns, int L, int hw,
                                         const int* __restrict__ frames, int k, DpmCoeffs c) {
  pdl_enter();
  const long long total = (long long)ns * k * hw;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int px = (int)(idx % hw);
    const int j = (int)((idx / hw) % k);
    const long long sc = idx / ((long long)hw * k);
    const long long off = (sc * L + frames[j]) * hw + px;
    dpmpp_update(latents + off, acc[off], x0_prev + off, c);
    acc[off] = 0.f;
  }
}

}  // namespace vx

using namespace vx;

extern "C" int vx_conv_in(const void* in, long long sn, long long sc, int NB, int H, int W, int Cin, int Cout,
                          const float* w, const float* bias, const void* addend, const int* add_frame,
                          long long add_ld, float pre_scale, const float* pre_w, const float* pre_b, void* out,
                          long long ldo, void* stream) {
  VX_REQUIRE(Cout % 8 == 0 && Cin == 4 && Cin * 9 * Cout * 4 <= 200 * 1024, "vx_conv_in: Cin=%d (must be 4) Cout=%d unsupported", Cin, Cout);
  ConvInArgs a{(const __nv_bfloat16*)in, sn, sc, NB, H, W, Cin, Cout, w, bias, (const __nv_bfloat16*)addend, add_frame,
               add_ld, pre_scale, pre_w, pre_b, (__nv_bfloat16*)out, ldo};
  const size_t smem = (size_t)Cin * 9 * Cout * 4;
  static bool cfg = false;
  if (!cfg) {
    VX_CHECK_CUDA(cudaFuncSetAttribute(conv_in_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    cfg = true;
  }
  const long long total = (long long)NB * H * ((W + 3) / 4) * (Cout / 8);
  long long blocks = (total + 255) / 256;
  if (blocks > device_sms() * 4) blocks = device_sms() * 4;
  launch_k(conv_in_kernel<4>, dim3((unsigned)blocks), dim3(256), smem, (cudaStream_t)stream, a);
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int vx_conv_out(const void* x, long long ldx, int NB, int H, int W, int C, int Cout, const float* w,
                           const float* bias, void* out, long long sn, long long sc, int out_f32, int post,
                           void* stream) {
  VX_REQUIRE(C % 8 == 0 && Cout >= 1 && Cout <= 4, "vx_conv_out: C=%d Cout=%d unsupported", C, Cout);
  ConvOutArgs a{(const __nv_bfloat16*)x, ldx, NB, H, W, C, Cout, w, bias, out, sn, sc, out_f32, post};
  const long long npix = (long long)NB * H * W;
  launch_k(conv_out_kernel, dim3((unsigned)((npix * 32 + 255) / 256)), dim3(256), 0, (cudaStream_t)stream, a);
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int vx_extract_planar(const void* x, long long ldx, int NB, int HW, int Cout, void* out, long long sn,
                                 long long sc, int out_f32, int post, void* stream) {
  VX_REQUIRE(Cout >= 1 && Cout <= 8 && ldx % 8 == 0, "vx_extract_planar: Cout=%d ldx=%lld", Cout, ldx);
  const long long npix = (long long)NB * HW;
  long long blocks = (npix + 255) / 256;
  if (blocks > device_sms() * 16) blocks = device_sms() * 16;
  launch_k(extract_planar_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, (const __nv_bfloat16*)x, ldx, npix, HW, Cout,
                                                                          out, sn, sc, out_f32, post);
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int vx_im2col_s2(const void* x, int NB, int H, int W, int C, void* out, void* stream) {
  VX_REQUIRE(C % 8 == 0 && H % 2 == 0 && W % 2 == 0, "vx_im2col_s2: bad shape");
  const long long total = (long long)NB * (H / 2) * (W / 2) * 9 * (C / 8);
  long long blocks = (total + 255) / 256;
  if (blocks > device_sms() * 16) blocks = device_sms() * 16;
  launch_k(im2col_s2_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, (const __nv_bfloat16*)x, NB, H, W, C,
                                                                      (__nv_bfloat16*)out);
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int vx_upsample2x(const void* x, int NB, int H, int W, int C, void* out, void* stream) {
  VX_REQUIRE(C % 8 == 0, "vx_upsample2x: C=%d", C);
  const long long total = (long long)NB * 4 * H * W * (C / 8);
  long long blocks = (total + 255) / 256;
  if (blocks > device_sms() * 16) blocks = device_sms() * 16;
  launch_k(upsample2x_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, (const __nv_bfloat16*)x, NB, H, W, C,
                                                                       (__nv_bfloat16*)out);
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int vx_skinny_linear(const float* x, int rows, int K, const void* w, const float* bias, int N, int act_in,
                                int act_out, float* y, void* stream) {
  VX_REQUIRE(rows >= 1 && rows <= 8 && K % 8 == 0, "vx_skinny_linear: rows=%d K=%d", rows, K);
  launch_k(skinny_linear_kernel, dim3((N * 32 + 255) / 256), dim3(256), 0, (cudaStream_t)stream, x, rows, K, (const __nv_bfloat16*)w, bias,
                                                                              N, act_in, act_out, y);
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int vx_timestep_embed(const float* t, int rows, int dim, float* out, void* stream) {
  const int n = rows * (dim / 2);
  launch_k(timestep_embed_kernel, dim3((n + 127) / 128), dim3(128), 0, (cudaStream_t)stream, t, rows, dim, out);
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int vx_cfg_overlap_accumulate(const void* noise, int f, int hw, int L, int do_cfg, const int* win,
                                         const int* count, float guidance, float* acc, void* stream) {
  CfgArgs a{(const __nv_bfloat16*)noise, f, hw, L, do_cfg, win, count, guidance, acc};
  const long long total = (long long)4 * f * hw;
  launch_k(cfg_overlap_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, (cudaStream_t)stream, a);
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int vx_cfg_overlap_accumulate_n(const void* noise, int n, int f, int hw, int L, int do_cfg, const int* win,
                                           const int* count, float guidance, float* acc, void* stream) {
  VX_REQUIRE(n >= 1 && f >= 1 && hw >= 1 && L >= 1, "vx_cfg_overlap_accumulate_n: n=%d f=%d hw=%d L=%d", n, f, hw, L);
  CfgNArgs a{(const __nv_bfloat16*)noise, n, f, hw, L, do_cfg, win, count, guidance, acc};
  const long long total = (long long)n * 4 * f * hw;
  long long blocks = (total + 255) / 256;
  if (blocks > device_sms() * 16) blocks = device_sms() * 16;
  launch_k(cfg_overlap_n_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, a);
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int vx_ddim_step(void* latents, const float* acc, long long n, float sqrt_a, float sqrt_1ma,
                            float sqrt_aprev, float sqrt_1maprev, void* stream) {
  long long blocks = (n + 255) / 256;
  if (blocks > device_sms() * 8) blocks = device_sms() * 8;
  launch_k(ddim_step_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, (__nv_bfloat16*)latents, acc, n, sqrt_a,
                                                                      sqrt_1ma, sqrt_aprev, sqrt_1maprev);
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int vx_ddim_step_eta(void* latents, const float* acc, const float* noise, long long n, float sqrt_a,
                                float sqrt_1ma, float sqrt_aprev, float c_dir, float sigma, void* stream) {
  VX_REQUIRE(n >= 1 && latents && acc && noise, "vx_ddim_step_eta: n=%lld", n);
  long long blocks = (n + 255) / 256;
  if (blocks > device_sms() * 8) blocks = device_sms() * 8;
  launch_k(ddim_step_eta_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, (__nv_bfloat16*)latents, acc,
           noise, n, sqrt_a, sqrt_1ma, sqrt_aprev, c_dir, sigma);
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int vx_ddim_step_frames(void* latents, float* acc, int ns, int L, int hw, const int* frames, int k, float sqrt_a,
                                   float sqrt_1ma, float sqrt_aprev, float sqrt_1maprev, void* stream) {
  VX_REQUIRE(ns >= 1 && L >= 1 && hw >= 1 && k >= 1 && k <= L && frames, "vx_ddim_step_frames: ns=%d L=%d hw=%d k=%d", ns, L,
             hw, k);
  const long long total = (long long)ns * k * hw;
  long long blocks = (total + 255) / 256;
  if (blocks > device_sms() * 8) blocks = device_sms() * 8;
  launch_k(ddim_step_frames_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, (__nv_bfloat16*)latents, acc, ns,
           L, hw, frames, k, sqrt_a, sqrt_1ma, sqrt_aprev, sqrt_1maprev);
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int vx_dpmpp_step(void* latents, const float* acc, void* x0_prev, long long n, float alpha_s, float sigma_s,
                             float ratio, float c0, float inv_r0, float c0h, int order, void* stream) {
  VX_REQUIRE(n >= 1 && latents && acc && x0_prev && (order == 1 || order == 2), "vx_dpmpp_step: n=%lld order=%d", n,
             order);
  long long blocks = (n + 255) / 256;
  if (blocks > device_sms() * 8) blocks = device_sms() * 8;
  launch_k(dpmpp_step_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, (__nv_bfloat16*)latents, acc,
           (__nv_bfloat16*)x0_prev, n, DpmCoeffs{alpha_s, sigma_s, ratio, c0, inv_r0, c0h, order});
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int vx_dpmpp_step_frames(void* latents, float* acc, void* x0_prev, int ns, int L, int hw, const int* frames,
                                    int k, float alpha_s, float sigma_s, float ratio, float c0, float inv_r0, float c0h,
                                    int order, void* stream) {
  VX_REQUIRE(ns >= 1 && L >= 1 && hw >= 1 && k >= 1 && k <= L && frames && latents && acc && x0_prev &&
                 (order == 1 || order == 2),
             "vx_dpmpp_step_frames: ns=%d L=%d hw=%d k=%d order=%d", ns, L, hw, k, order);
  const long long total = (long long)ns * k * hw;
  long long blocks = (total + 255) / 256;
  if (blocks > device_sms() * 8) blocks = device_sms() * 8;
  launch_k(dpmpp_step_frames_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, (__nv_bfloat16*)latents,
           acc, (__nv_bfloat16*)x0_prev, ns, L, hw, frames, k, DpmCoeffs{alpha_s, sigma_s, ratio, c0, inv_r0, c0h, order});
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}
