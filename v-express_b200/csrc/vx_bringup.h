/* Bring-up probes: NOT part of the product ABI (include/vxb200.h).  They exist so that tests/test_probe_gpu.py can pin the
 * wgmma shared-memory descriptor conventions and the TMA box layouts the kernels rely on; also
 * vx_flash_reload_env, the sweep tools' hook to re-read the A/B switches. */
#ifndef VX_BRINGUP_H
#define VX_BRINGUP_H
#ifdef __cplusplus
extern "C" {
#endif
int vx_probe_umma(const void* a_img, int a_bytes, const void* b_img, int b_bytes, unsigned lboA, unsigned sboA,
                  unsigned layA, unsigned lboB, unsigned sboB, unsigned layB, int a_mn, int b_mn, int N, int ksteps,
                  int a_step, int b_step, float* out, void* stream);
int vx_probe_tma(const void* base, int rank, const unsigned long long* dims, const unsigned long long* strides_bytes,
                 const unsigned* box, int swizzle, const int* coords, int nbytes, void* out, void* stream);

void vx_flash_reload_env(void);
void vx_gemm_reload_env(void);
void vx_norm_reload_env(void);
void vx_pdl_set(int on);   /* programmatic dependent launch on / off (default: VX_PDL, read once) */
int vx_pdl_get(void);
#ifdef __cplusplus
}
#endif
#endif
