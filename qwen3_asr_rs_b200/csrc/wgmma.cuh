// wgmma.cuh -- sm_90a building blocks of the TMA-fed wgmma GEMMs (gemm_tc.cu, score.cu): mbarriers, TMA tile loads,
// shared-memory matrix descriptors of 128B-swizzled K-major tiles, and the m64n128k16 bf16 wgmma.
#pragma once
#include <cuda.h>
#include <cstdint>

namespace asrb {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra.uni WAIT_DONE;\n"
        "bra.uni WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, int c3, int c4, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5, %6}], [%7];"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4), "r"(smem_u32(bar)) : "memory");
}
// wgmma matrix descriptor of a K-major, 128B-swizzled operand tile: rows of 64 bf16 (128 B), 8-row groups 1024 B apart
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3ffff) >> 4);          // start address, 16-byte units
    d |= (uint64_t)1 << 16;                           // leading byte offset (unused for swizzled K-major)
    d |= (uint64_t)(1024 >> 4) << 32;                 // stride byte offset between 8-row groups
    d |= (uint64_t)1 << 62;                           // SWIZZLE_128B
    return d;
}
// D[64][128] (+)= A[64][16] * B[128][16]^T, both K-major in shared memory; scale_d = 0 overwrites D
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma boundary
__device__ __forceinline__ void fence_operand(float& r) { asm volatile("" : "+f"(r)::"memory"); }

// The consumer main loop of one output tile (gemm_tc.cu, score.cu).  Warpgroup `half` (0 / 1) of the consumers multiplies
// its 64 rows of the A tile by the 128-row B tile for num_kb k-blocks: for each block wait for its ring stage, issue
// nplanes x BK / 16 wgmma, release the stage.  The tensor core accumulates CH k-blocks at a time into `acc`; each
// finished chunk is added into `sum` in fp32 round-to-nearest (a tensor core that does not round to nearest biases
// long-K sums; gemm_tc.cu).  `kg` is the CTA's global stage counter, shared with the producer's order.
template <int STAGES, int STAGE_BYTES, int TILE_A_BYTES, int BK, int CH>
__device__ __forceinline__ void consume_k_blocks(uint8_t* smem, uint64_t* full, uint64_t* empty, int half, int lane, int num_kb,
                                                 int nplanes, uint32_t& kg, float (&acc)[64], float (&sum)[64]) {
    for (int kb = 0; kb < num_kb; ++kb, ++kg) {
        const int s = kg % STAGES; const uint32_t par = (kg / STAGES) & 1;
        const bool chunk_first = (kb % CH) == 0;
        mbar_wait(&full[s], par);
        const uint32_t sa = smem_u32(smem + s * STAGE_BYTES);
        const uint64_t bdesc = make_smem_desc(sa + 3 * TILE_A_BYTES);
#pragma unroll
        for (int j = 0; j < 64; ++j) fence_operand(acc[j]);
        wgmma_fence();
#pragma unroll
        for (int p = 0; p < 3; ++p) {
            if (p >= nplanes) break;
            const uint64_t adesc = make_smem_desc(sa + p * TILE_A_BYTES + half * (64 * BK * 2));
#pragma unroll
            for (int k = 0; k < BK / 16; ++k)     // +32 B per K=16 step inside the 128 B swizzle atom
                wgmma_m64n128k16(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), (p == 0 && k == 0) ? !chunk_first : 1u);
        }
        wgmma_commit();
        wgmma_wait_all();
#pragma unroll
        for (int j = 0; j < 64; ++j) fence_operand(acc[j]);
        __syncwarp();
        if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&empty[s])) : "memory");
        if ((kb % CH) == CH - 1 || kb == num_kb - 1) {
#pragma unroll
            for (int j = 0; j < 64; ++j) sum[j] += acc[j];
        }
    }
}

// Columns 32 g .. 32 g + 31 of a warp's 16 accumulator rows into its [16][LD] float slab: in the wgmma layout lane l holds
// rows l / 4 and l / 4 + 8, columns 8 j + 2 (l % 4) + {0, 1}.  Ends with __syncwarp: the slab is readable by any lane.
template <int LD>
__device__ __forceinline__ void stage_slab(float* slab, const float (&sum)[64], int g, int lane) {
    const int r0 = lane >> 2, c0 = 2 * (lane & 3);
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
        const int j = g * 4 + jj;
        *reinterpret_cast<float2*>(slab + r0 * LD + 8 * jj + c0) = make_float2(sum[4 * j], sum[4 * j + 1]);
        *reinterpret_cast<float2*>(slab + (r0 + 8) * LD + 8 * jj + c0) = make_float2(sum[4 * j + 2], sum[4 * j + 3]);
    }
    __syncwarp();
}

}  // namespace tc

// bf16 TMA tensor map with 128B swizzle, encoded once per distinct (base, shape, strides, box) (gemm_tc.cu)
const CUtensorMap& tc_cached_map(const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                                 const cuuint32_t* box);

}  // namespace asrb
