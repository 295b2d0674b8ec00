// Post-processing of the decoded video (SURVEY.md 8(f) row f3; reference pipelines/utils.py:46-63, 70-73):
//   3x3x3 median over (t, y, x) with reflect padding on all three axes, then (v * 255) truncated to uint8 in
//   (t, y, x, c) order -- the frames `save_video` hands to the encoder.  The reference materialises a 27x unfolded
//   tensor per frame and moves every frame device <-> CPU; here one thread owns one output pixel (all channels),
//   gathers the 27 neighbours through L1 and selects the median with a pruned Batcher odd-even merge network held in
//   registers (selection, so the result is bit-exact).  Compute-light and HBM-light: 4 B read + 1 B written per value.
//   The same kernel filters a run of frames of a video decoded chunk by chunk (vx_median3d_range_u8, for
//   VExpressPipeline.stream): the buffer carries one halo frame on each side and time reflects at the video's ends.
// Checked on the GPU: the median / uint8 path bit-exact against the oracle and the golden (tests/test_zz_post_gpu.py),
// im2col3x3 bit-exact as a gather and within an fp64 bound for its SiLU (tests/test_prologue_bounds_gpu.py).
#include "vx_host.h"
#include "vx_ptx.cuh"

namespace vx {

__device__ __forceinline__ void cswap(float& a, float& b) {
  const float lo = fminf(a, b), hi = fmaxf(a, b);
  a = lo;
  b = hi;
}

// Median of 27 registers: Batcher's odd-even merge network for 32 inputs with the comparators that touch the five
// +inf padding wires removed (156 left) and then pruned to those the 14th-smallest output depends on (126), emitted
// as straight-line code so that the values never leave the register file (a loop-nest formulation ended up in local
// memory).  Checked against sorted() on 20k random / tie-heavy inputs when it was generated.
__device__ __forceinline__ float median27(float (&v)[27]) {
#define CS(a, b) cswap(v[a], v[b]);
  CS(0,1) CS(2,3) CS(4,5) CS(6,7) CS(8,9) CS(10,11) CS(12,13) CS(14,15) CS(16,17) CS(18,19)
  CS(20,21) CS(22,23) CS(24,25) CS(0,2) CS(1,3) CS(4,6) CS(5,7) CS(8,10) CS(9,11) CS(12,14)
  CS(13,15) CS(16,18) CS(17,19) CS(20,22) CS(21,23) CS(24,26) CS(1,2) CS(5,6) CS(9,10) CS(13,14)
  CS(17,18) CS(21,22) CS(25,26) CS(0,4) CS(1,5) CS(2,6) CS(3,7) CS(8,12) CS(9,13) CS(10,14)
  CS(11,15) CS(16,20) CS(17,21) CS(18,22) CS(19,23) CS(2,4) CS(3,5) CS(10,12) CS(11,13) CS(18,20)
  CS(19,21) CS(1,2) CS(3,4) CS(5,6) CS(9,10) CS(11,12) CS(13,14) CS(17,18) CS(19,20) CS(21,22)
  CS(25,26) CS(0,8) CS(1,9) CS(2,10) CS(3,11) CS(4,12) CS(5,13) CS(6,14) CS(7,15) CS(16,24)
  CS(17,25) CS(18,26) CS(4,8) CS(5,9) CS(6,10) CS(7,11) CS(20,24) CS(21,25) CS(22,26) CS(2,4)
  CS(3,5) CS(6,8) CS(7,9) CS(10,12) CS(11,13) CS(18,20) CS(19,21) CS(22,24) CS(23,25) CS(1,2)
  CS(3,4) CS(5,6) CS(7,8) CS(9,10) CS(11,12) CS(13,14) CS(17,18) CS(19,20) CS(21,22) CS(23,24)
  CS(25,26) CS(0,16) CS(1,17) CS(2,18) CS(3,19) CS(4,20) CS(5,21) CS(6,22) CS(7,23) CS(8,24)
  CS(9,25) CS(10,26) CS(8,16) CS(9,17) CS(10,18) CS(11,19) CS(12,20) CS(13,21) CS(14,22) CS(7,11)
  CS(12,16) CS(13,17) CS(14,18) CS(11,13) CS(14,16) CS(13,14)
#undef CS
  return v[13];
}

__device__ __forceinline__ int reflect(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * (n - 1) - i : i); }

// video: [C][nbuf][H][W] fp32 holding frames [buf0, buf0 + nbuf) of a T-frame video; the kernel filters the `nown` frames
// from own0 on (time reflected at the video's ends 0 and T - 1, not at the buffer's).  filtered (optional): [C][nown][H][W];
// frames (optional): [nown][H][W][C] uint8.  The whole video is buf0 = own0 = 0, nbuf = nown = T.
__global__ void __launch_bounds__(256) median3d_kernel(const float* __restrict__ video, int C, int nbuf, int buf0, int own0,
                                                       int nown, int T, int H, int W, float* __restrict__ filtered,
                                                       unsigned char* __restrict__ frames) {
  pdl_enter();
  const long long npix = (long long)nown * H * W;
  const long long plane = (long long)H * W;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < npix;
       idx += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(idx % W);
    const int y = (int)((idx / W) % H);
    const int t = own0 + (int)(idx / plane);
    int tt[3], yy[3], xx[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      tt[d] = reflect(t + d - 1, T) - buf0;
      yy[d] = reflect(y + d - 1, H);
      xx[d] = reflect(x + d - 1, W);
    }
    for (int c = 0; c < C; ++c) {
      const float* base = video + (long long)c * nbuf * plane;
      float v[27];
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b)
#pragma unroll
          for (int d = 0; d < 3; ++d) v[(a * 3 + b) * 3 + d] = __ldg(base + (long long)tt[a] * plane + (long long)yy[b] * W + xx[d]);
      const float m = median27(v);                 // 14th smallest of 27
      if (filtered) filtered[(long long)c * nown * plane + idx] = m;
      if (frames) frames[idx * C + c] = (unsigned char)(m * 255.0f);   // truncation, like numpy astype(uint8)
    }
  }
}

// ------------------------------------------------------------------ im2col (3x3, stride 1 or 2, pad 1), NHWC, with
// an optional SiLU on the gathered input: the conv stacks of the conditioning prologue (VKpsGuider, SURVEY 8f-f2;
// reference modules/v_kps_guider.py:35-45) are conv -> SiLU chains with 16..256 channels, too narrow for the
// implicit-GEMM conv (C % 64); they run as im2col(SiLU(x)) + tensor-core GEMM instead.  K order = (tap, channel), the
// order of pack_conv3x3_weight.  Same structure as im2col_s2_kernel (vx_misc.cu).
__global__ void im2col3x3_kernel(const __nv_bfloat16* __restrict__ x, int NB, int H, int W, int C, int stride, int silu,
                                 int pad_lo, __nv_bfloat16* __restrict__ out) {
  pdl_enter();
  // pad_lo = 1: pad 1 on every side (nn.Conv2d(padding=1)); pad_lo = 0: pad (0, 1, 0, 1) -- right/bottom only, the
  // diffusers Downsample2D(padding=0) of the VAE encoder -- same output size for even H, W at stride 2
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1, V = C / 8;
  const long long total = (long long)NB * Ho * Wo * 9 * V;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(idx % V);
    const int t = (int)((idx / V) % 9);
    const long long opix = idx / ((long long)V * 9);
    const int ox = (int)(opix % Wo), oy = (int)((opix / Wo) % Ho);
    const long long n = opix / ((long long)Wo * Ho);
    const int yy = oy * stride + t / 3 - pad_lo, xx = ox * stride + t % 3 - pad_lo;
    uint4 val = make_uint4(0, 0, 0, 0);
    if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
      val = *reinterpret_cast<const uint4*>(x + ((n * H + yy) * W + xx) * C + v * 8);
      if (silu) {
        uint32_t w4[4] = {val.x, val.y, val.z, val.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = unpack_bf16(w4[i]);
          w4[i] = pack_bf16(f.x / (1.f + __expf(-f.x)), f.y / (1.f + __expf(-f.y)));
        }
        val = make_uint4(w4[0], w4[1], w4[2], w4[3]);
      }
    }
    *reinterpret_cast<uint4*>(out + opix * 9 * C + (long long)t * C + v * 8) = val;
  }
}

}  // namespace vx

using namespace vx;

extern "C" int vx_im2col3x3(const void* x, int NB, int H, int W, int C, int stride, int silu, int pad_lo, void* out,
                            void* stream) {
  VX_REQUIRE(C % 8 == 0 && (stride == 1 || stride == 2), "vx_im2col3x3: C=%d stride=%d", C, stride);
  VX_REQUIRE(pad_lo == 1 || (pad_lo == 0 && stride == 2 && H % 2 == 0 && W % 2 == 0), "vx_im2col3x3: pad_lo=%d needs stride 2, even H/W", pad_lo);
  const long long total = (long long)NB * ((H - 1) / stride + 1) * ((W - 1) / stride + 1) * 9 * (C / 8);
  long long blocks = (total + 255) / 256;
  if (blocks > device_sms() * 16) blocks = device_sms() * 16;
  launch_k(im2col3x3_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, (const __nv_bfloat16*)x, NB, H, W, C, stride, silu,
                                                                      pad_lo, (__nv_bfloat16*)out);
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int vx_median3d_u8(const float* video, int C, int T, int H, int W, float* filtered, unsigned char* frames,
                              void* stream) {
  VX_REQUIRE(C >= 1 && T >= 2 && H >= 2 && W >= 2, "vx_median3d_u8: reflect padding needs T, H, W >= 2 (got %d %d %d)", T, H, W);
  VX_REQUIRE(filtered || frames, "vx_median3d_u8: no output requested (C=%d)", C);
  const long long npix = (long long)T * H * W;
  long long blocks = (npix + 255) / 256;
  if (blocks > device_sms() * 16) blocks = device_sms() * 16;
  launch_k(median3d_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, video, C, T, 0, 0, T, T, H, W, filtered,
           frames);
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int vx_median3d_range_u8(const float* buf, int C, int nbuf, int buf_start, int own_start, int own_count, int T,
                                    int H, int W, unsigned char* frames, void* stream) {
  VX_REQUIRE(C >= 1 && T >= 2 && H >= 2 && W >= 2, "vx_median3d_range_u8: reflect padding needs T, H, W >= 2 (got %d %d %d)",
             T, H, W);
  VX_REQUIRE(own_start >= 0 && own_count >= 1 && own_start + own_count <= T && frames,
             "vx_median3d_range_u8: frames [%d, %d) outside the video of %d", own_start, own_start + own_count, T);
  // every temporal neighbour of an owned frame (reflected at the video's ends) must be in the buffer
  const int need_lo = own_start > 0 ? own_start - 1 : 0;
  const int need_hi = own_start + own_count < T ? own_start + own_count + 1 : T;
  VX_REQUIRE(buf_start >= 0 && buf_start <= need_lo && buf_start + nbuf >= need_hi && buf_start + nbuf <= T,
             "vx_median3d_range_u8: buffer [%d, %d) must cover frames [%d, %d)", buf_start, buf_start + nbuf, need_lo, need_hi);
  const long long npix = (long long)own_count * H * W;
  long long blocks = (npix + 255) / 256;
  if (blocks > device_sms() * 16) blocks = device_sms() * 16;
  launch_k(median3d_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, buf, C, nbuf, buf_start, own_start,
           own_count, T, H, W, (float*)nullptr, frames);
  VX_CHECK_CUDA(cudaGetLastError());
  return 0;
}
