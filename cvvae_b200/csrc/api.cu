// Library-wide state of libcvvae_b200 (error string, launch counter, driver entry point) and the
// shared-memory matrix descriptor probe used by the GPU test-suite.
#include <stdarg.h>
#include <string.h>

#include "common.cuh"
#include "ptx.cuh"

namespace cvvae {

static thread_local char g_err[1024] = "";
std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

PFN_encodeTiled get_encode_tiled() {
  static PFN_encodeTiled fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

// One warpgroup: TMA a [rows_total][64] 16-bit matrix and a [N][64] matrix into SWIZZLE_128B shared memory, run a
// 128 x N x 64 product as two 64-row wgmma chains whose A descriptor starts `row_shift` rows (128 B each) into the slab
// and whose 8-row groups are `sbo_rows` rows apart (8 = dense; 16 = every other group, i.e. a tile of 8-position image
// rows cut out of a wider slab).
template <int N>
__global__ void __launch_bounds__(128) probe_kernel(const __grid_constant__ CUtensorMap tmA,
                                                    const __grid_constant__ CUtensorMap tmB, float* out, int rows_total,
                                                    int row_shift, int base_offset_mode, int sbo_rows) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;                  // rows_total * 128 B (<= 48 KB)
  uint8_t* sB = smem + 49152;          // N * 128 B
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + 49152 + 32768);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    ptx::mbar_init(bar, 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    ptx::mbar_expect_tx(bar, static_cast<uint32_t>(rows_total + N) * 128u);
    ptx::tma_load_3d(sA, &tmA, bar, 0, 0, 0);                                   // two boxes of rows_total / 2 rows
    ptx::tma_load_3d(sA + (rows_total / 2) * 128, &tmA, bar, 0, rows_total / 2, 0);
    ptx::tma_load_3d(sB, &tmB, bar, 0, 0, 0);
  }
  ptx::mbar_wait(bar, 0);
  float acc[2][N / 2];
  const uint32_t b0 = ptx::smem_u32(sB);
  ptx::wgmma_fence();
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    const uint32_t a0 = ptx::smem_u32(sA) + static_cast<uint32_t>(row_shift + c * 8 * sbo_rows) * 128u;
    const uint64_t bo = base_offset_mode ? static_cast<uint64_t>((a0 >> 7) & 7u) << 49 : 0ull;
#pragma unroll
    for (int k = 0; k < 4; ++k)
      ptx::Wgmma<CVVAE_F16, N>::run(acc[c], ptx::wgmma_desc_sw128(a0 + k * 32, static_cast<uint32_t>(sbo_rows) * 128u) | bo,
                                    ptx::wgmma_desc_sw128(b0 + k * 32), k > 0);
  }
  ptx::wgmma_commit();
  ptx::wgmma_wait<0>();
#pragma unroll
  for (int c = 0; c < 2; ++c) ptx::fence_regs(acc[c]);
#pragma unroll
  for (int c = 0; c < 2; ++c)
#pragma unroll
    for (int j = 0; j < N / 8; ++j)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = c * 64 + warp * 16 + (lane >> 2) + (i >> 1) * 8;
        const int col = 8 * j + 2 * (lane & 3) + (i & 1);
        out[r * N + col] = acc[c][4 * j + i];
      }
}

}  // namespace cvvae

using namespace cvvae;

extern "C" const char* cvvae_last_error(void) { return g_err; }
extern "C" int cvvae_abi_version(void) { return CVVAE_ABI_VERSION; }
extern "C" int64_t cvvae_launch_count(void) { return g_launches.load(); }

extern "C" int cvvae_probe_umma_shift(const void* a_rows, const void* b_rows, float* out, int32_t n, int32_t row_shift,
                                      int32_t base_offset_mode, int32_t sbo_rows, void* stream_) {
  CVVAE_CHECK_ARG(a_rows && b_rows && out && (n == 64 || n == 128 || n == 256) && row_shift >= 0 && row_shift <= 64 &&
                      sbo_rows >= 8 && sbo_rows <= 16,
                  "cvvae_probe_umma_shift: bad argument");
  PFN_encodeTiled enc = get_encode_tiled();
  CVVAE_CHECK_ARG(enc, "cuTensorMapEncodeTiled entry point not available");
  const int rows_total = 320;   // 15 groups x 16 rows + 8 + shift 64 <= 320
  CUtensorMap tmA, tmB;
  cuuint32_t estr[3] = {1, 1, 1};
  {
    cuuint64_t dims[3] = {64, (cuuint64_t)rows_total, 1};
    cuuint64_t strides[2] = {128, 128ull * rows_total};
    cuuint32_t box[3] = {64, (cuuint32_t)(rows_total / 2), 1};
    CUresult r = enc(&tmA, CU_TENSOR_MAP_DATA_TYPE_UINT16, 3, const_cast<void*>(a_rows), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    CVVAE_CHECK_ARG(r == CUDA_SUCCESS, "probe: tensor map A failed (%d)", (int)r);
  }
  {
    cuuint64_t dims[3] = {64, (cuuint64_t)n, 1};
    cuuint64_t strides[2] = {128, 128ull * n};
    cuuint32_t box[3] = {64, (cuuint32_t)n, 1};
    CUresult r = enc(&tmB, CU_TENSOR_MAP_DATA_TYPE_UINT16, 3, const_cast<void*>(b_rows), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    CVVAE_CHECK_ARG(r == CUDA_SUCCESS, "probe: tensor map B failed (%d)", (int)r);
  }
  const size_t smem = 1024 + 49152 + 32768 + 64;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (n == 64) {
    CVVAE_CUDA(cudaFuncSetAttribute(probe_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    probe_kernel<64><<<1, 128, smem, stream>>>(tmA, tmB, out, rows_total, row_shift, base_offset_mode, sbo_rows);
  } else if (n == 128) {
    CVVAE_CUDA(cudaFuncSetAttribute(probe_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    probe_kernel<128><<<1, 128, smem, stream>>>(tmA, tmB, out, rows_total, row_shift, base_offset_mode, sbo_rows);
  } else {
    CVVAE_CUDA(cudaFuncSetAttribute(probe_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    probe_kernel<256><<<1, 128, smem, stream>>>(tmA, tmB, out, rows_total, row_shift, base_offset_mode, sbo_rows);
  }
  CVVAE_LAUNCH_CHECK();
  return CVVAE_OK;
}
