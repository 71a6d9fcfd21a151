// cambrian_b200 — the AdamW arithmetic and the host-state pointer checks shared by the optimizer kernels that spell out
// every rounding: adamw_host_kernel (offload.cu, fp32 moments in host memory) and adamw8_kernel (adam8bit.cu, 8-bit
// moments on the device or in host memory).
#pragma once
#include "common.cuh"

namespace cb {

// ---------------------------------------------------------------------------------- the AdamW arithmetic
// Bitwise equal to adamw_kernel (elementwise.cu).  adamw_kernel writes plain expressions and leaves the choice of which
// multiply-add pairs to fuse to the compiler; that choice depends on the surrounding code, so here every rounding is
// spelled out with an _rn intrinsic, as the instructions adamw_kernel compiles to: decay = fma(-lr, wd, 1), m and v each
// one fma over two products, denom = fma(sqrt(v), rsqrt(bc2), eps), and p = p * decay - step_size * (m / denom) with
// three separate roundings for elements 0-6 of each 8-element group but with the last two fused into one fma for element
// 7 (adamw_kernel<1> and <4> alike).  tests/test_offload_gpu.py compares the two kernels bit for bit.
struct AdamwScalars {
  float gs, inv_sqrt_bc2, step_size, decay;
};

// `coef` (optional, device): gradient scale written by clip_coef_kernel; `grad_scale` when null
__device__ __forceinline__ AdamwScalars adamw_scalars(float lr, float wd, float bc1, float bc2, float grad_scale,
                                                      const float* __restrict__ coef) {
  AdamwScalars s;
  s.gs = coef ? __ldg(coef) : grad_scale;
  s.inv_sqrt_bc2 = rsqrtf(bc2), s.step_size = __fdiv_rn(lr, bc1), s.decay = __fmaf_rn(-lr, wd, 1.f);
  return s;
}

// one 8-element group: p, m, v updated in place from the bf16 gradient unpacked into gf
__device__ __forceinline__ void adamw_update8(const float* gf, float* pf, float* mf, float* vf, float b1, float b2,
                                              float eps, const AdamwScalars& s) {
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float gg = __fmul_rn(gf[e], s.gs);
    mf[e] = __fmaf_rn(1.f - b1, gg, __fmul_rn(b1, mf[e]));                   // b1 m + (1 - b1) g
    vf[e] = __fmaf_rn(gg, __fmul_rn(1.f - b2, gg), __fmul_rn(b2, vf[e]));     // b2 v + (1 - b2) g^2
    const float denom = __fmaf_rn(__fsqrt_rn(vf[e]), s.inv_sqrt_bc2, eps);
    const float q = __fdiv_rn(mf[e], denom), pd = __fmul_rn(pf[e], s.decay);
    pf[e] = e == 7 ? __fmaf_rn(-s.step_size, q, pd) : __fsub_rn(pd, __fmul_rn(s.step_size, q));
  }
}

// ------------------------------------------------------------------------------------------ host
static inline const char* memory_kind(cudaMemoryType t) {
  switch (t) {
    case cudaMemoryTypeHost: return "registered host memory";
    case cudaMemoryTypeDevice: return "device memory";
    case cudaMemoryTypeManaged: return "managed memory";
    default: return "unregistered (pageable) host memory";
  }
}

// A failed runtime query leaves its error as the thread's last error: clear it, or the next launch check reports it.
static inline cudaPointerAttributes pointer_attributes(const void* ptr) {
  cudaPointerAttributes a{};
  if (cudaPointerGetAttributes(&a, ptr) != cudaSuccess) {
    (void)cudaGetLastError();
    a.type = cudaMemoryTypeUnregistered;
  }
  return a;
}

// `ptr` .. `ptr + bytes` must be registered, mapped host memory: its device-side address goes to *dev.  `op` prefixes
// the error message.
static inline int host_state_pointer(void* ptr, long long bytes, const char* op, const char* name, void** dev) {
  const char* last = reinterpret_cast<const char*>(ptr) + bytes - 1;
  const cudaPointerAttributes a = pointer_attributes(ptr), b = pointer_attributes(last);
  CB_CHECK_ARG(a.type == cudaMemoryTypeHost && b.type == cudaMemoryTypeHost,
               "%s: %s must be host memory registered with CUDA (cudaHostRegister, mapped), got %s", op, name,
               memory_kind(a.type == cudaMemoryTypeHost ? b.type : a.type));
  void *d0 = nullptr, *d1 = nullptr;
  if (cudaHostGetDevicePointer(&d0, ptr, 0) != cudaSuccess ||
      cudaHostGetDevicePointer(&d1, const_cast<char*>(last), 0) != cudaSuccess) {
    (void)cudaGetLastError();
    return set_error(CB_ERR_INVALID, "%s: %s is registered host memory without a device mapping (register it "
                     "with cudaHostRegisterMapped)", op, name);
  }
  CB_CHECK_ARG(static_cast<char*>(d1) - static_cast<char*>(d0) == bytes - 1,
               "%s: %s spans host registrations that are not contiguous in the device address space", op, name);
  *dev = d0;
  return CB_OK;
}

static inline int device_pointer(const void* ptr, const char* op, const char* name) {
  int cur = 0;
  if (cudaGetDevice(&cur) != cudaSuccess) {
    (void)cudaGetLastError();
    return set_error(CB_ERR_CUDA, "%s: no CUDA device", op);
  }
  const cudaPointerAttributes a = pointer_attributes(ptr);
  CB_CHECK_ARG(a.type == cudaMemoryTypeDevice, "%s: %s must be device memory, got %s", op, name, memory_kind(a.type));
  CB_CHECK_ARG(a.device == cur, "%s: %s is on device %d, the current device is %d", op, name, a.device, cur);
  return CB_OK;
}

// a kernel without (much) shared memory would otherwise leave its SMs configured for a small shared-memory carveout, and
// a GEMM CTA needing ~200 KB could not be placed beside it: the two would serialise instead of sharing the SMs.  One
// attribute call per kernel and device.
template <typename K>
static inline int prefer_max_shared_carveout(K kernel, bool (&done)[64], const char* op) {
  int dev = 0;
  if (cudaGetDevice(&dev) == cudaSuccess && dev >= 0 && dev < 64 && !done[dev]) {
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared) !=
        cudaSuccess)
      return set_error(CB_ERR_CUDA, "%s: cudaFuncSetAttribute: %s", op, cudaGetErrorString(cudaGetLastError()));
    done[dev] = true;
  }
  return CB_OK;
}

}  // namespace cb
