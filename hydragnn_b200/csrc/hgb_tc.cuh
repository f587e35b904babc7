// Hopper building blocks shared by the tensor-core kernels (hgb_tc.cu, hgb_painn_tc.cu): mbarrier, TMA, wgmma TF32 and the
// shared-memory layout of its K-major SWIZZLE_128B operands, plus the host-side tensor-map encoder.  sm_90a only.
#pragma once
#include <cuda.h>

#include "hgb_common.cuh"

namespace {

// ------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(smem_dst)),
      "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
          smem_u32(smem_dst)),
      "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// ---- wgmma (warpgroup MMA: 4 warps, A and B from shared memory, D in registers) ----
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// warpgroup register reallocation: the producer warpgroup hands registers to the accumulator-holding consumers
template <int R>
__device__ __forceinline__ void regs_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void regs_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;   // 128 x 40 + 256 x 232 <= 64 K registers

// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
template <int N>
__device__ __forceinline__ void fence_regs(float* r) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}

// D[64 x 32 NC] += A[64 x 8] . B[32 NC x 8]^T: one instruction for every output column of a Linear piece, so A is read from shared
// memory once per k-step.  Fragment: d[4i + 2h + e] = D(16 w + lane/4 + 8h, 8i + 2(lane%4) + e), i < 4 NC.
template <int NC>
__device__ __forceinline__ void wgmma_tf32(float* d, uint64_t ad, uint64_t bd);
#define TC_R16_0 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
#define TC_R16_1 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
#define TC_R16_2 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47"
#define TC_R16_3 "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
#define TC_R16_4 "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79"
#define TC_R16_5 "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95"
#define TC_R16_6 "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111"
#define TC_R16_7 "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
#define TC_D16(o)                                                                                                                   \
  "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), "+f"(d[o + 7]),      \
      "+f"(d[o + 8]), "+f"(d[o + 9]), "+f"(d[o + 10]), "+f"(d[o + 11]), "+f"(d[o + 12]), "+f"(d[o + 13]), "+f"(d[o + 14]),       \
      "+f"(d[o + 15])
// AD, BD, SC: the operand numbers of the two descriptors and of the scale-d flag, which follow the 16 NC accumulators
#define TC_WGMMA(NC, SHAPE, AD, BD, SC, REGS, ...)                                                                                  \
  template <>                                                                                                                       \
  __device__ __forceinline__ void wgmma_tf32<NC>(float* d, uint64_t ad, uint64_t bd) {                                             \
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, " SC ", 0;\nwgmma.mma_async.sync.aligned." SHAPE ".f32.tf32.tf32 {" REGS     \
                 "}, " AD ", " BD ", p, 1, 1;\n}"                                                                                  \
                 : __VA_ARGS__                                                                                                      \
                 : "l"(ad), "l"(bd), "r"(1));                                                                                       \
  }
TC_WGMMA(1, "m64n32k8", "%16", "%17", "%18", TC_R16_0, TC_D16(0))
TC_WGMMA(2, "m64n64k8", "%32", "%33", "%34", TC_R16_0 ", " TC_R16_1, TC_D16(0), TC_D16(16))
TC_WGMMA(3, "m64n96k8", "%48", "%49", "%50", TC_R16_0 ", " TC_R16_1 ", " TC_R16_2, TC_D16(0), TC_D16(16), TC_D16(32))
TC_WGMMA(4, "m64n128k8", "%64", "%65", "%66", TC_R16_0 ", " TC_R16_1 ", " TC_R16_2 ", " TC_R16_3, TC_D16(0), TC_D16(16), TC_D16(32),
         TC_D16(48))
TC_WGMMA(5, "m64n160k8", "%80", "%81", "%82", TC_R16_0 ", " TC_R16_1 ", " TC_R16_2 ", " TC_R16_3 ", " TC_R16_4, TC_D16(0), TC_D16(16),
         TC_D16(32), TC_D16(48), TC_D16(64))
TC_WGMMA(6, "m64n192k8", "%96", "%97", "%98", TC_R16_0 ", " TC_R16_1 ", " TC_R16_2 ", " TC_R16_3 ", " TC_R16_4 ", " TC_R16_5, TC_D16(0),
         TC_D16(16), TC_D16(32), TC_D16(48), TC_D16(64), TC_D16(80))
TC_WGMMA(7, "m64n224k8", "%112", "%113", "%114", TC_R16_0 ", " TC_R16_1 ", " TC_R16_2 ", " TC_R16_3 ", " TC_R16_4 ", " TC_R16_5 ", " TC_R16_6,
         TC_D16(0), TC_D16(16), TC_D16(32), TC_D16(48), TC_D16(64), TC_D16(80), TC_D16(96))
TC_WGMMA(8, "m64n256k8", "%128", "%129", "%130", TC_R16_0 ", " TC_R16_1 ", " TC_R16_2 ", " TC_R16_3 ", " TC_R16_4 ", " TC_R16_5 ", " TC_R16_6
         ", " TC_R16_7, TC_D16(0), TC_D16(16), TC_D16(32), TC_D16(48), TC_D16(64), TC_D16(80), TC_D16(96), TC_D16(112))
#undef TC_WGMMA
#undef TC_D16

// TMA store of one box from shared memory, tracked by the issuing thread's bulk async-groups
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* tmap, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(tmap), "r"(smem_u32(smem_src)),
               "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all but the newest N bulk groups of this thread have finished reading their shared-memory source
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// shared-memory matrix descriptor of a K-major operand in the 128-byte swizzle: rows of 32 fp32 (128 B), 8-row groups 1024 B
// apart (SBO); the k-step of 8 tf32 inside the swizzle atom is a 32-byte advance of the start address.  The operand base must be
// 1024-byte aligned (the swizzle phase is taken from the address bits).
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;                 // leading byte offset: unused by swizzled K-major operands
  d |= (uint64_t)(1024 >> 4) << 32;       // stride byte offset
  d |= (uint64_t)1 << 62;                 // SWIZZLE_128B
  return d;
}

// byte offset of element (r, c) of a K-major SWIZZLE_128B operand stored as column blocks of 32 fp32:
// block cb = c/32 is a [rows x 128 B] slab; 8-row groups are 1024 B apart; 16-B chunks are XOR-swizzled by r%8
__device__ __forceinline__ uint32_t kmajor_sw128_off(int r, int c, int rows) {
  const int cb = c >> 5, cc = (c & 31) >> 2, j = c & 3;
  return (uint32_t)cb * rows * 128 + (uint32_t)(r >> 3) * 1024 + (uint32_t)(r & 7) * 128 + (uint32_t)((cc ^ (r & 7)) << 4) + j * 4;
}

constexpr size_t SMEM_MAX = 227 * 1024;          // opt-in dynamic shared memory per block

// ------------------------------------------------------------------------------------------------
// host: tensor maps
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

// fp32 tensor of `rank` dims (dims[0] innermost, strides in bytes of dims 1..), box `box`; elements outside read as zero
int encode_tmap(CUtensorMap* tm, const float* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides, const cuuint32_t* box,
                CUtensorMapSwizzle swz) {
  EncodeTiledFn enc = get_encode();
  if (!enc) { hgb_set_error("tc: cuTensorMapEncodeTiled is not available from the driver"); return HGB_ECUDA; }
  // the encoder needs a current context, and a thread that has made no runtime call yet (the autograd engine's worker, when a
  // backward pass starts with this call) has none: make the device's primary context current, once per thread
  static thread_local bool ctx_current = false;
  if (!ctx_current) {
    int dev = 0;
    ctx_current = cudaGetDevice(&dev) == cudaSuccess && cudaSetDevice(dev) == cudaSuccess;
  }
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, rank, const_cast<float*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { hgb_set_error("tc: cuTensorMapEncodeTiled failed (%d)", (int)r); return HGB_ECUDA; }
  return HGB_OK;
}

// 2-D fp32 row-major tensor [rows, cols] with row stride ld (elements); box = [box_rows x 32 cols]
int make_tmap(CUtensorMap* tm, const float* base, int64_t rows, int64_t cols, int64_t ld, int box_rows, CUtensorMapSwizzle swz) {
  const cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t gstr[1] = {(cuuint64_t)ld * 4};
  const cuuint32_t box[2] = {32, (cuuint32_t)box_rows};
  return encode_tmap(tm, base, 2, gdim, gstr, box, swz);
}

}  // namespace
