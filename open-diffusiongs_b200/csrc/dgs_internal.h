// dgs_internal.h -- shared host-side helpers of libdgs_b200.so (not part of the public C ABI).
#pragma once
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>

#include "dgs_b200.h"

namespace dgs {

void set_error(const char* fmt, ...);

#define DGS_CUDA_OK(expr)                                                                 \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      ::dgs::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return DGS_ERR_CUDA;                                                                \
    }                                                                                     \
  } while (0)

// number of kernels of THIS library launched so far (dgs_kernel_launch_count)
extern unsigned long long g_kernel_launches;

// after a kernel launch: count it, always check the launch itself; in debug mode also synchronise
#define DGS_LAUNCH_OK(stream, debug)                                   \
  do {                                                                 \
    ::dgs::g_kernel_launches++;                                        \
    DGS_CUDA_OK(cudaGetLastError());                                   \
    if (debug) DGS_CUDA_OK(cudaStreamSynchronize(stream));             \
  } while (0)
#define DGS_POST_LAUNCH()                  \
  do {                                     \
    ::dgs::g_kernel_launches++;            \
    DGS_CUDA_OK(cudaGetLastError());       \
  } while (0)

// Optional per-kernel-family timing (dgs_profile_enable): CUDA events recorded on the launching stream
// around each family's launches; a no-op (one predictable branch) when disabled.
enum ProfFamily {
  PROF_RASTER_PROJECT = 0, PROF_RASTER_SCAN, PROF_RASTER_EMIT, PROF_RASTER_SORT, PROF_RASTER_RANGES,
  PROF_RASTER_BLEND_FWD, PROF_RASTER_BLEND_BWD, PROF_RASTER_GEOM_BWD,
  PROF_DIT_INPUT, PROF_DIT_COND, PROF_DIT_LN, PROF_DIT_GEMM_QKV, PROF_DIT_ATTN, PROF_DIT_GEMM_PROJ,
  PROF_DIT_GEMM_FC1, PROF_DIT_GEMM_FC2, PROF_DIT_HEADS,
  PROF_DIT_BWD_ELEM, PROF_DIT_BWD_WGRAD, PROF_DIT_BWD_DGRAD, PROF_DIT_BWD_ATTN, PROF_N
};
extern bool g_prof_on;
void prof_begin(cudaStream_t st, int family);
void prof_end(cudaStream_t st, int family);
struct ProfScope {
  cudaStream_t st; int fam;
  ProfScope(cudaStream_t s, int f) : st(s), fam(f) { if (g_prof_on) prof_begin(st, fam); }
  ~ProfScope() { if (g_prof_on) prof_end(st, fam); }
};

#define DGS_REQUIRE(cond, ...)             \
  do {                                     \
    if (!(cond)) {                         \
      ::dgs::set_error(__VA_ARGS__);       \
      return DGS_ERR_INVALID_ARGUMENT;     \
    }                                      \
  } while (0)

// Carves typed, 256-byte aligned sub-buffers out of one arena (or just measures, base == nullptr).
struct Carver {
  char* base;
  size_t off = 0;
  explicit Carver(void* b) : base(reinterpret_cast<char*>(b)) {}
  template <typename T>
  T* take(size_t count) {
    off = (off + 255) & ~size_t(255);
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += count * sizeof(T);
    return p;
  }
  size_t bytes() const { return (off + 255) & ~size_t(255); }
};

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// dgs_marching_cubes (mesh.cu) with its messages prefixed by `name`; with a weight array [nx, ny, nz] (else nullptr)
// only the points of weight > 0 are observed, and the mesh keeps to the voxels whose 8 corners are (mesh.cu's header).
int marching_cubes(const char* name, const float* field, const int* weight, int nx, int ny, int nz, float iso,
                   dgs_alloc_fn alloc, void* alloc_user, float** vertices, int** triangles, long long* num_vertices,
                   long long* num_triangles, cudaStream_t st);

// Launch with programmatic dependent launch allowed (DGS_PDL=0 disables it).  ONLY for kernels that execute
// griddepcontrol.wait before their first access to global memory written by earlier kernels.
bool pdl_enabled();
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                     Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

}  // namespace dgs
