// C-ABI surface shared bits: last-error string, version, GEMM entry point (see include/espnet_b200.h).
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "gemm.h"

#ifndef ESPB_PDL_DEFAULT
#define ESPB_PDL_DEFAULT 1
#endif

static thread_local char g_err[512] = "";

void espb_set_error(const char* msg) {
  strncpy(g_err, msg ? msg : "", sizeof(g_err) - 1);
  g_err[sizeof(g_err) - 1] = 0;
}

namespace espb {
// ESPB_PDL=1 / 0 overrides the default; read once.
bool pdl_enabled() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("ESPB_PDL"); v = e ? (e[0] == '1') : ESPB_PDL_DEFAULT; }
  return v == 1;
}
}  // namespace espb

extern "C" {

const char* espb_last_error(void) { return g_err; }
int espb_abi_version(void) { return 7; }   // 7: espb_ctc_extend_state_f32 (streaming beam search); 3: espb_flash_attn_f32; 4: LM fusion helpers; 5: hop / window generality of the frontend entry points; 6: contextual-block (streaming encoder) helpers

int espb_device_sm(int* major, int* minor) {
  int dev = 0;
  cudaDeviceProp prop;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess) {
    espb_set_error("no CUDA device");
    return ESPB_ERR_CUDA;
  }
  *major = prop.major; *minor = prop.minor;
  return ESPB_OK;
}

// use_tc = 1: wgmma 3xTF32 kernel, 2: the same with chunked fp32 promotion (TMA needs 16-byte aligned strides/bases); 0: SIMT fp32 kernel.
int espb_gemm_f32(const EspbGemmDesc* d, int use_tc, cudaStream_t stream) {
  if (!d) { espb_set_error("gemm: null descriptor"); return ESPB_ERR_ARG; }
  return use_tc ? espb_gemm_tc_launch(*d, stream, use_tc == 2 ? 2 : 1) : espb_gemm_simt_launch(*d, stream);
}

}  // extern "C"
