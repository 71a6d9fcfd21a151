// cambrian_b200 — AdamW with the fp32 optimizer state in host memory (TrainEngine(offload_optimizer=True)).
//
// The master weights and both moments (12 of the 16 bytes per trainable parameter) live in host memory registered with
// CUDA and mapped into the device address space; the bf16 gradient and the bf16 compute copy stay on the device.  One
// kernel streams the state over PCIe, updates it with exactly adamw_kernel's arithmetic and writes it back
// in the same pass: no staging copies, no CPU arithmetic.
#include "common.cuh"
#include <algorithm>

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

// 8-element groups whose loads one thread issues before it uses any of them.  A PCIe read takes microseconds, so the
// bytes in flight, not the thread count, set the rate: 2 groups x 96 state bytes per thread.  A third group would need
// 24 more registers than the 72 the launch bounds allow.
constexpr int HOST_GROUPS = 2;
constexpr int HOST_THREADS = 128;

// 128 threads, <= 72 registers (launch bounds: 7 blocks per SM), no shared memory: a block fits next to a resident
// persistent GEMM CTA (the register budget of adamw_launch's background shape, elementwise.cu).
__global__ void __launch_bounds__(HOST_THREADS, 7)
    adamw_host_kernel(float* __restrict__ p, float* __restrict__ m, float* __restrict__ v, const bf16* __restrict__ g,
                      bf16* __restrict__ p16, long long n, float lr, float b1, float b2, float eps, float wd, float bc1,
                      float bc2, float grad_scale, const float* __restrict__ coef) {
  const long long nvec = n >> 3;
  const AdamwScalars s = adamw_scalars(lr, wd, bc1, bc2, grad_scale, coef);
  // a block works on tiles of HOST_GROUPS x 128 consecutive groups; group k of a thread sits k x 128 groups (4 KB of each
  // state array) after its first, a constant offset that needs no address registers of its own
  const long long stride = (long long)gridDim.x * HOST_GROUPS * HOST_THREADS;
  for (long long i0 = (long long)blockIdx.x * HOST_GROUPS * HOST_THREADS + threadIdx.x; i0 < nvec; i0 += stride) {
    float4* pp = reinterpret_cast<float4*>(p) + 2 * i0;
    float4* mp = reinterpret_cast<float4*>(m) + 2 * i0;
    float4* vp = reinterpret_cast<float4*>(v) + 2 * i0;
    float pf[HOST_GROUPS][8], mf[HOST_GROUPS][8], vf[HOST_GROUPS][8];
#pragma unroll
    for (int k = 0; k < HOST_GROUPS; ++k) {          // every PCIe read of this iteration is issued here
      const int o = 2 * k * HOST_THREADS;
      if (i0 + k * HOST_THREADS < nvec) {
        *reinterpret_cast<float4*>(pf[k]) = pp[o]; *reinterpret_cast<float4*>(pf[k] + 4) = pp[o + 1];
        *reinterpret_cast<float4*>(mf[k]) = mp[o]; *reinterpret_cast<float4*>(mf[k] + 4) = mp[o + 1];
        *reinterpret_cast<float4*>(vf[k]) = vp[o]; *reinterpret_cast<float4*>(vf[k] + 4) = vp[o + 1];
      }
    }
#pragma unroll
    for (int k = 0; k < HOST_GROUPS; ++k) {
      const long long i = i0 + k * HOST_THREADS;
      const int o = 2 * k * HOST_THREADS;
      if (i < nvec) {
        float gf[8];
        unpack8(ldg_nc(reinterpret_cast<const uint4*>(g) + i), gf);
        adamw_update8(gf, pf[k], mf[k], vf[k], b1, b2, eps, s);
        pp[o] = *reinterpret_cast<float4*>(pf[k]); pp[o + 1] = *reinterpret_cast<float4*>(pf[k] + 4);
        mp[o] = *reinterpret_cast<float4*>(mf[k]); mp[o + 1] = *reinterpret_cast<float4*>(mf[k] + 4);
        vp[o] = *reinterpret_cast<float4*>(vf[k]); vp[o + 1] = *reinterpret_cast<float4*>(vf[k] + 4);
        reinterpret_cast<uint4*>(p16)[i] = pack8(pf[k]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------ host
static const char* memory_kind(cudaMemoryType t) {
  switch (t) {
    case cudaMemoryTypeHost: return "registered host memory";
    case cudaMemoryTypeDevice: return "device memory";
    case cudaMemoryTypeManaged: return "managed memory";
    default: return "unregistered (pageable) host memory";
  }
}

// A failed runtime query leaves its error as the thread's last error: clear it, or the next launch check reports it.
static cudaPointerAttributes pointer_attributes(const void* ptr) {
  cudaPointerAttributes a{};
  if (cudaPointerGetAttributes(&a, ptr) != cudaSuccess) {
    (void)cudaGetLastError();
    a.type = cudaMemoryTypeUnregistered;
  }
  return a;
}

// `ptr` .. `ptr + bytes` must be registered, mapped host memory: its device-side address goes to *dev
static int host_state_pointer(float* ptr, long long bytes, const char* name, float** dev) {
  const char* last = reinterpret_cast<const char*>(ptr) + bytes - 1;
  const cudaPointerAttributes a = pointer_attributes(ptr), b = pointer_attributes(last);
  CB_CHECK_ARG(a.type == cudaMemoryTypeHost && b.type == cudaMemoryTypeHost,
               "adamw_host: %s must be host memory registered with CUDA (cudaHostRegister, mapped), got %s", name,
               memory_kind(a.type == cudaMemoryTypeHost ? b.type : a.type));
  void *d0 = nullptr, *d1 = nullptr;
  if (cudaHostGetDevicePointer(&d0, ptr, 0) != cudaSuccess ||
      cudaHostGetDevicePointer(&d1, const_cast<char*>(last), 0) != cudaSuccess) {
    (void)cudaGetLastError();
    return set_error(CB_ERR_INVALID, "adamw_host: %s is registered host memory without a device mapping (register it "
                     "with cudaHostRegisterMapped)", name);
  }
  CB_CHECK_ARG(static_cast<char*>(d1) - static_cast<char*>(d0) == bytes - 1,
               "adamw_host: %s spans host registrations that are not contiguous in the device address space", name);
  *dev = static_cast<float*>(d0);
  return CB_OK;
}

static int device_pointer(const void* ptr, const char* name) {
  int cur = 0;
  if (cudaGetDevice(&cur) != cudaSuccess) {
    (void)cudaGetLastError();
    return set_error(CB_ERR_CUDA, "adamw_host: no CUDA device");
  }
  const cudaPointerAttributes a = pointer_attributes(ptr);
  CB_CHECK_ARG(a.type == cudaMemoryTypeDevice, "adamw_host: %s must be device memory, got %s", name, memory_kind(a.type));
  CB_CHECK_ARG(a.device == cur, "adamw_host: %s is on device %d, the current device is %d", name, a.device, cur);
  return CB_OK;
}

// Default grid: the smallest of the sweep that reaches >= 90 % of the plateau (tools/offload_step.py --kernel, 2 GB of
// state, H100 80GB HBM3 SXM at 700 W): ctas 4 / 8 / 16 / 32 / 64 / 132 -> 41.9 / 45.1 / 44.6 / 45.0 / 43.5 / 43.5 GB/s of
// PCIe traffic, against 61.9 GB/s for the copy engines moving the same bytes both ways at once.  Fewer blocks also leave
// more SMs to kernels that cannot share one (the attention backward's dK / dV CTA takes the whole register file).
constexpr int HOST_DEFAULT_CTAS = 4;

int adamw_host_launch(float* p, float* m, float* v, const void* g, void* p16, long long n, float lr, float b1, float b2,
                      float eps, float wd, int step, float grad_scale, const float* clip_coef, int ctas, cudaStream_t st) {
  CB_CHECK_ARG(n >= 0 && n % 8 == 0, "adamw_host: element count must be a non-negative multiple of 8 (got %lld)", n);
  CB_CHECK_ARG(step >= 1, "adamw_host: step must be >= 1");
  CB_CHECK_ARG(ctas >= 0, "adamw_host: ctas must be >= 0 (0 = default), got %d", ctas);
  if (n == 0) return CB_OK;
  const struct { const void* ptr; const char* name; } args[] = {{p, "p"}, {m, "m"}, {v, "v"}, {g, "g"}, {p16, "p16"}};
  for (const auto& a : args) {
    CB_CHECK_ARG(a.ptr != nullptr, "adamw_host: %s is null", a.name);
    CB_CHECK_ARG(reinterpret_cast<uintptr_t>(a.ptr) % 16 == 0, "adamw_host: %s must be 16-byte aligned", a.name);
  }
  // every pointer is checked before anything is launched: a misplaced operand is an error code, not a GPU fault
  float *pd = nullptr, *md = nullptr, *vd = nullptr;
  int rc;
  if ((rc = host_state_pointer(p, 4 * n, "p", &pd)) != CB_OK) return rc;
  if ((rc = host_state_pointer(m, 4 * n, "m", &md)) != CB_OK) return rc;
  if ((rc = host_state_pointer(v, 4 * n, "v", &vd)) != CB_OK) return rc;
  if ((rc = device_pointer(g, "g")) != CB_OK) return rc;
  if ((rc = device_pointer(p16, "p16")) != CB_OK) return rc;
  if (clip_coef && (rc = device_pointer(clip_coef, "clip_coef")) != CB_OK) return rc;
  // a kernel without shared memory would otherwise leave its SMs configured for a small shared-memory carveout, and a
  // GEMM CTA needing ~200 KB could not be placed beside it: the two would serialise instead of sharing the SMs
  static bool carveout_set[64] = {false};
  int dev = 0;
  if (cudaGetDevice(&dev) == cudaSuccess && dev >= 0 && dev < 64 && !carveout_set[dev]) {
    if (cudaFuncSetAttribute(adamw_host_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                             cudaSharedmemCarveoutMaxShared) != cudaSuccess)
      return set_error(CB_ERR_CUDA, "adamw_host: cudaFuncSetAttribute: %s", cudaGetErrorString(cudaGetLastError()));
    carveout_set[dev] = true;
  }
  const float bc1 = 1.f - powf(b1, (float)step), bc2 = 1.f - powf(b2, (float)step);   // as adamw_launch
  const long long nvec = n / 8;
  const long long want = (nvec + HOST_GROUPS * HOST_THREADS - 1) / (HOST_GROUPS * HOST_THREADS);
  const int grid = (int)std::min<long long>(ctas > 0 ? ctas : HOST_DEFAULT_CTAS, want);
  adamw_host_kernel<<<grid, HOST_THREADS, 0, st>>>(pd, md, vd, (const bf16*)g, (bf16*)p16, n, lr, b1, b2, eps, wd, bc1, bc2,
                                                   grad_scale, clip_coef);
  CB_CUDA_LAUNCH_CHECK("adamw_host");
  return CB_OK;
}

}  // namespace cb
