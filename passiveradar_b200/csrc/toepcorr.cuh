// toepcorr.cuh -- lag correlations of the LS normal equations on the Hopper tensor cores (wgmma).
//
// The Gram column c[m] = sum_i conj(ref[i]) ref[i+m] and the right-hand side x[m] = sum_i conj(ref[i])
// srv[i+m] of LS_Filter (reference clutter_removal.py:39,45) are the one step of the hot path that is
// a dense GEMM (north_star: "the Toeplitz normal equations use tensor cores ... that step really is
// a dense cgemm").  Here it is evaluated as a *Toeplitz GEMM* on interleaved real data:
//
//   z = (re0, im0, re1, im1, ...) of a complex64 signal, row a of a block = 128 consecutive floats
//   D[u][v] = sum_a zx[128 a + u] * zs[128 a + v]          u in [0,128), v in [0, 2*(64+nlag))
//   real diagonal delta = v - u collects every pair (x sample, s sample) at complex lag delta/2:
//     delta even : re(C[delta/2])   += D[u][v]                        (re*re + im*im)
//     delta odd  : im(C[(delta+1)/2]) += D[u][v]   for odd  u        (im*re)
//                  im(C[(delta-1)/2]) -= D[u][v]   for even u        (re*im)
//   with C[l] = sum_i x[i] conj(s[i+l]).
//
// A CTA tile is M = 128 rows (u) x N = 128 columns (one "pass" of v); two consumer warpgroups each issue
// wgmma.m64n128k16 (BF16 operands, fp32 accumulators in registers) on 64 of the rows, K = 16 rows a per
// instruction.  fp32 accuracy comes from a three-way BF16 split z = b0 + b1 + b2 (24 significand bits)
// and the six products of order <= 2:
//   D += b0*b0' + b0*b1' + b1*b0' + b0*b2' + b2*b0' + b1*b1'      (dropped terms ~2^-24 relative)
// Operands are MN-major (contiguous along u / v) with the 128-byte swizzle; both wgmma operands come from
// shared memory (transposed-operand form).  The overlapping ("im2col") rows of the s operand are
// materialised by the producers straight from the interleaved BF16 planes -- no expanded matrix ever
// exists in HBM.  Warps 0-7: two consumer warpgroups (MMA + diagonal-sum epilogue); warps 8-11: producers.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace prc {
namespace tc {

constexpr int ROW = 128;            // elements per K-row (= 64 complex samples)
constexpr int KSTEP = 16;           // K-rows per MMA (bf16: K = 16)
constexpr int NPASS = 128;          // columns per pass (wgmma N)
constexpr int STAGES = 4;
constexpr int NPLANE = 3;           // b0, b1, b2
constexpr int A_BYTES = ROW * KSTEP * 2;          // 4 KB per plane
constexpr int B_BYTES = NPASS * KSTEP * 2;        // 4 KB per plane
constexpr int STAGE_BYTES = NPLANE * (A_BYTES + B_BYTES);   // 24 KB
// 128-byte-swizzled MN-major tiles: atom = 8 K-rows x 128 B (64 elements along MN), the 16-byte chunk
// index inside a row is XOR-ed with the row index (Swizzle<3,4,3>); atoms ordered [k-group][mn-group].
constexpr int ATOM_BYTES = 1024;
constexpr int A_SBO = (ROW / 64) * ATOM_BYTES;    // stride between the two 8-row K groups of an A tile
constexpr int B_SBO = (NPASS / 64) * ATOM_BYTES;  // ... of a B tile
constexpr int MN_LBO = ATOM_BYTES;                // stride between 64-element MN groups
constexpr int NUM_MMA_WG = 2, NUM_LOAD_WARPS = 4;
constexpr int THREADS = 32 * (4 * NUM_MMA_WG + NUM_LOAD_WARPS);   // 12 warps
static_assert(STAGES == NUM_LOAD_WARPS, "loader warp w owns pipeline stage w");
constexpr int EPI_PARTS = 4 * NUM_MMA_WG;          // one private set of lag sums per consumer warp
constexpr int TILE_LD = 65;                        // accumulator tile of a warpgroup, column-major, 64 rows + 1 pad
constexpr int TILE_FLOATS = NPASS * TILE_LD;

struct ToepParams {
    const uint16_t* x[NPLANE];       // interleaved BF16 planes of the x operand, zero beyond the signal
    const uint16_t* s[2][NPLANE];    // per problem: s rotated by dmin and circularly extended
    int nk;                 // K-steps (of 16 rows = 1024 complex samples) in the signal
    int nlag;               // complex lags wanted: 0 .. nlag-1
    int npass;              // ceil(2*(64+nlag) / NPASS)
    int ranges;             // LS mode: CTAs per (problem, pass): gridDim.x = 2 * npass * ranges
    int kb;                 // block mode (> 0): K-steps per block; items = nblk * npass, any gridDim.x
    int nblk;
    int HT;                 // row length of the partial buffer (padded lag count)
    float2* partial;        // LS: [problem][pass*ranges + range][HT];  block mode: [blk][pass][HT]
};

// ---- TMA producer (TMA = true) ------------------------------------------------------------------------------
// Tensor maps of the BF16 planes: element (c0, c1) = plane[128 * c1 + c0], i.e. K-row c1 of the Toeplitz
// operand starting at column c0.  Rows are 256 bytes apart but NPASS * npass elements wide: they OVERLAP in
// memory (cuTensorMapEncodeTiled accepts that), which is what materialises the im2col operand without ever
// storing it.  Box = 64 elements x 16 K-rows, SWIZZLE_128B: it lands as 16 rows of 128 bytes with the
// 16-byte chunk index XOR-ed with (row & 7) -- the wgmma operand layout, with the two 8-row K groups of one
// 64-element MN group contiguous (SBO = 1 KB) and MN groups 2 KB apart (LBO).  One elected thread per
// stage instead of four full warps of address arithmetic.
struct ToepMaps {
    CUtensorMap x[NPLANE];
    CUtensorMap s[2][NPLANE];
};
constexpr int TMA_BOX_BYTES = 64 * 2 * KSTEP;     // 2 KB: one 64-element MN group, both 8-row K groups
constexpr int TMA_LBO = TMA_BOX_BYTES;            // stride between MN groups
constexpr int TMA_SBO = ATOM_BYTES;               // stride between the two K groups inside a box
constexpr int MAX_SLOTS = STAGES;
constexpr int OPERAND_BYTES = STAGES * STAGE_BYTES;         // operand area of the dynamic shared memory

// ---------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(smem_u32(dst)), "l"(src));
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// TMA: one thread arms the stage's mbarrier with the byte count, then issues 2-D tiled bulk-tensor copies
// that complete on it.
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* tm, int c0, int c1, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tm)), "r"(c0), "r"(c1), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tm) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tm)) : "memory");
}

// wgmma: fence before the first MMA that reads registers written by ordinary instructions (zeroed
// accumulators, A fragments), commit closes a group, wait<N> leaves at most N groups in flight.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x 128] += A[64 x 16] * B[16 x 128], both operands MN-major in shared memory (fp32 accumulators:
// thread t of the warpgroup holds d[i] at row 16 (t / 32) + (t % 32) / 4 + 8 ((i / 2) % 2), column
// 8 (i / 4) + 2 (t % 4) + i % 2)
__device__ __forceinline__ void wgmma_ss(float (&d)[64], uint64_t da, uint64_t db) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\nwgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 1, 1;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(da), "l"(db), "r"(1));
}

// the same with A from registers (four BF16 pairs per thread, the mma.m16n8k16 A layout per warp) and B
// K-major in shared memory
__device__ __forceinline__ void wgmma_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t db) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %69, 0;\nwgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64, %65, %66, %67}, %68, p, 1, 1, 0;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(1));
}

// shared-memory matrix descriptor, SWIZZLE_128B.  MN-major: LBO = stride between 64-element MN groups,
// SBO = stride between 8-row K groups.  K-major: SBO = stride between 8-row groups, LBO unused.
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    d |= (uint64_t)1 << 62;          // layout type 1 = SWIZZLE_128B, base offset 0 (operands start on 1 KB boundaries)
    return d;
}

struct __align__(16) ToepShared {
    uint64_t full[MAX_SLOTS];
    uint64_t empty[MAX_SLOTS];
};

// One unit of work of a CTA: an accumulation over K-steps [kbeg, kbeg + kcount) for one (problem, pass),
// whose diagonal sums go to partial row `row`.
struct ToepItem {
    int valid, prob, pass, kbeg, kcount;
    long long row;
};

// LS mode (kb == 0): item = blockIdx.x only; (problem, pass, K-range) as in ToepParams.
// Block mode (kb > 0): items blockIdx.x, blockIdx.x + gridDim.x, ... < nblk * npass; item id = blk * npass + pass,
// K-steps [blk * kb, (blk + 1) * kb), row = item id.
__device__ __forceinline__ ToepItem toep_item(const ToepParams& p, int it) {
    ToepItem r;
    if (p.kb == 0) {
        const int per_prob = p.npass * p.ranges;
        const int prob = blockIdx.x / per_prob;
        const int rem = blockIdx.x - prob * per_prob;
        const int pass = rem / p.ranges;
        const int range = rem - pass * p.ranges;
        r.valid = (it == 0);
        r.prob = prob;
        r.pass = pass;
        r.kbeg = (int)(((long long)p.nk * range) / p.ranges);
        r.kcount = (int)(((long long)p.nk * (range + 1)) / p.ranges) - r.kbeg;
        r.row = (long long)prob * per_prob + rem;
    } else {
        const long long id = (long long)blockIdx.x + (long long)it * gridDim.x;
        r.valid = id < (long long)p.nblk * p.npass;
        const int blk = (int)(id / p.npass);
        r.prob = 0;
        r.pass = (int)(id - (long long)blk * p.npass);
        r.kbeg = blk * p.kb;
        r.kcount = p.kb;
        r.row = id;
    }
    return r;
}

// DUAL: the dominant b0*b0' chain and the five 2^-8-smaller cross terms in separate accumulators, so the
// rounding of the long chain is not mixed into the small terms (long K ranges: LS correlations).  !DUAL:
// one accumulator (many short items per CTA: CAF Doppler blocks); the producers run ahead into the next
// item while the consumers sum the diagonals of the current one.
// dynamic shared memory: [stages x {A_b0, A_b1, A_b2, B_b0, B_b1, B_b2}] [2 x accumulator tile] [8 x 2 x HT floats]
template <bool DUAL, bool TMA>
__global__ void __launch_bounds__(THREADS, 1) toepcorr_kernel(const __grid_constant__ ToepParams p, const __grid_constant__ ToepMaps maps) {
    extern __shared__ __align__(1024) uint8_t tsm[];
    __shared__ ToepShared sh;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool is_loader = warp >= 4 * NUM_MMA_WG;

    uint8_t* stage_base = tsm;
    float* tiles = reinterpret_cast<float*>(tsm + OPERAND_BYTES);                    // [2][TILE_FLOATS]
    float* cacc = tiles + NUM_MMA_WG * TILE_FLOATS;                                  // [8][2][HT]

    if (threadIdx.x == 0) {
        for (int s = 0; s < MAX_SLOTS; ++s) { mbar_init(&sh.full[s], 1); mbar_init(&sh.empty[s], NUM_MMA_WG); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int i = threadIdx.x; i < EPI_PARTS * 2 * p.HT; i += blockDim.x) cacc[i] = 0.f;
    __syncthreads();

    if (TMA && is_loader) {
        // ======================= TMA producers: lane 0 of loader warp w owns pipeline stage w.  Per K-step: arm
        // the stage's mbarrier with 24 KB, then 12 bulk-tensor copies (per plane: 2 boxes of the x rows, 2 boxes
        // of the overlapping s rows).
        const int lw = warp - 4 * NUM_MMA_WG;
        if (lane == 0) {
#pragma unroll
            for (int pl = 0; pl < NPLANE; ++pl) { tma_prefetch_desc(&maps.x[pl]); tma_prefetch_desc(&maps.s[0][pl]); tma_prefetch_desc(&maps.s[1][pl]); }
            int g = 0;
            for (int it = 0;; ++it) {
                const ToepItem item = toep_item(p, it);
                if (!item.valid) break;
                for (int t = 0; t < item.kcount; ++t, ++g) {
                    if ((g & (STAGES - 1)) != lw) continue;
                    if (g >= STAGES) mbar_wait(&sh.empty[lw], ((g / STAGES) - 1) & 1);
                    uint8_t* st = stage_base + lw * STAGE_BYTES;
                    const int row0 = (item.kbeg + t) * KSTEP;
                    mbar_expect_tx(&sh.full[lw], STAGE_BYTES);
#pragma unroll
                    for (int pl = 0; pl < NPLANE; ++pl) {
#pragma unroll
                        for (int m = 0; m < ROW / 64; ++m)
                            tma_load_2d(st + pl * A_BYTES + m * TMA_BOX_BYTES, &maps.x[pl], 64 * m, row0, &sh.full[lw]);
#pragma unroll
                        for (int m = 0; m < NPASS / 64; ++m)
                            tma_load_2d(st + NPLANE * A_BYTES + pl * B_BYTES + m * TMA_BOX_BYTES, &maps.s[item.prob][pl],
                                        item.pass * NPASS + 64 * m, row0, &sh.full[lw]);
                    }
                }
            }
        }
    } else if (is_loader) {
        // ======================= loaders: 16-byte cp.async into 128B-swizzled MN-major tiles.
        // Loader warp w owns pipeline stage w: it issues the whole 24 KB stage, waits for ITS copies only,
        // publishes them to the async proxy and arrives.
        const int lw = warp - 4 * NUM_MMA_WG;                    // 0..3 = stage
        const int ch = lane & 7;                                 // 16-byte chunk inside a 128-byte row
        const int r4 = lane >> 3;                                // 0..3: row inside a group of four
        int g = 0;                                               // K-steps issued by the CTA so far
        for (int it = 0;; ++it) {
            const ToepItem item = toep_item(p, it);
            if (!item.valid) break;
            for (int t = 0; t < item.kcount; ++t, ++g) {
                if ((g & (STAGES - 1)) != lw) continue;
                if (g >= STAGES) mbar_wait(&sh.empty[lw], ((g / STAGES) - 1) & 1);
                uint8_t* st = stage_base + lw * STAGE_BYTES;
                const size_t rowbase = (size_t)(item.kbeg + t) * KSTEP;
#pragma unroll
                for (int pl = 0; pl < NPLANE; ++pl) {
                    uint8_t* dstA = st + pl * A_BYTES;
                    uint8_t* dstB = st + NPLANE * A_BYTES + pl * B_BYTES;
#pragma unroll
                    for (int rr = 0; rr < KSTEP; rr += 4) {      // four K-rows per warp instruction
                        const int row = rr + r4;                 // 0..15
                        const int gk = row >> 3, r8 = row & 7;
                        const uint32_t swz = (uint32_t)((ch ^ r8) << 4) + (uint32_t)r8 * 128;
                        const uint16_t* srcA = p.x[pl] + (rowbase + row) * ROW + 8 * ch;
#pragma unroll
                        for (int m = 0; m < ROW / 64; ++m) cp_async16(dstA + gk * A_SBO + m * MN_LBO + swz, srcA + 64 * m);
                        const uint16_t* srcB = p.s[item.prob][pl] + (rowbase + row) * ROW + (size_t)item.pass * NPASS + 8 * ch;
#pragma unroll
                        for (int m = 0; m < NPASS / 64; ++m) cp_async16(dstB + gk * B_SBO + m * MN_LBO + swz, srcB + 64 * m);
                    }
                }
                asm volatile("cp.async.commit_group;" ::: "memory");
                asm volatile("cp.async.wait_group 0;" ::: "memory");
                fence_proxy_async();
                __syncwarp();
                if (lane == 0) mbar_arrive(&sh.full[lw]);
            }
        }
    } else {
        // ======================= consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of every tile
        const int wg = warp >> 2, wq = warp & 3;
        const bool leader = (threadIdx.x & 127) == 0;
        const uint32_t lbo = TMA ? TMA_LBO : MN_LBO;
        const uint32_t sbo_a = TMA ? TMA_SBO : A_SBO, sbo_b = TMA ? TMA_SBO : B_SBO;
        float* tile = tiles + wg * TILE_FLOATS;                  // [column][row], leading dimension TILE_LD
        float* cre = cacc + (warp * 2 + 0) * p.HT;
        float* cim = cacc + (warp * 2 + 1) * p.HT;
        int g = 0;
        for (int it = 0;; ++it) {
            const ToepItem item = toep_item(p, it);
            if (!item.valid) break;
            float acc0[64];
            float acc1[DUAL ? 64 : 1];
#pragma unroll
            for (int i = 0; i < 64; ++i) acc0[i] = 0.f;
            if constexpr (DUAL) {
#pragma unroll
                for (int i = 0; i < 64; ++i) acc1[i] = 0.f;
            }
            for (int t = 0; t < item.kcount; ++t, ++g) {
                const int s = g & (STAGES - 1);
                mbar_wait(&sh.full[s], (g / STAGES) & 1);
                const uint32_t a0 = smem_u32(stage_base + s * STAGE_BYTES) + (uint32_t)wg * lbo;   // MN group wg of A
                const uint32_t b0 = smem_u32(stage_base + s * STAGE_BYTES) + NPLANE * A_BYTES;
                uint64_t da[NPLANE], db[NPLANE];
#pragma unroll
                for (int pl = 0; pl < NPLANE; ++pl) {
                    da[pl] = make_desc_sw128(a0 + pl * A_BYTES, lbo, sbo_a);
                    db[pl] = make_desc_sw128(b0 + pl * B_BYTES, lbo, sbo_b);
                }
                wgmma_fence();
                wgmma_ss(acc0, da[0], db[0]);
                if constexpr (DUAL) {
                    wgmma_ss(acc1, da[0], db[1]);
                    wgmma_ss(acc1, da[1], db[0]);
                    wgmma_ss(acc1, da[0], db[2]);
                    wgmma_ss(acc1, da[2], db[0]);
                    wgmma_ss(acc1, da[1], db[1]);
                } else {
                    wgmma_ss(acc0, da[0], db[1]);
                    wgmma_ss(acc0, da[1], db[0]);
                    wgmma_ss(acc0, da[0], db[2]);
                    wgmma_ss(acc0, da[2], db[0]);
                    wgmma_ss(acc0, da[1], db[1]);
                }
                wgmma_commit();
                if (t > 0) {                                     // the previous K-step's MMAs have read their stage
                    wgmma_wait<1>();
                    if (leader) mbar_arrive(&sh.empty[(g - 1) & (STAGES - 1)]);
                }
            }
            wgmma_wait<0>();
            if (leader) mbar_arrive(&sh.empty[(g - 1) & (STAGES - 1)]);
            // accumulators -> this warpgroup's tile (column-major: the diagonal walk below is conflict-free)
#pragma unroll
            for (int i = 0; i < 64; ++i) {
                const int r = wq * 16 + (lane >> 2) + 8 * ((i >> 1) & 1);
                const int col = (i >> 2) * 8 + 2 * (lane & 3) + (i & 1);
                float v = acc0[i];
                if constexpr (DUAL) v += acc1[i];
                tile[col * TILE_LD + r] = v;
            }
            asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
            // diagonal sums of 32 x 32 sub-tiles: the warp takes two of its warpgroup's eight
#pragma unroll 1
            for (int k = 0; k < 2; ++k) {
                const int idx = wq + 4 * k;
                const int rq = idx >> 2, cq = idx & 3;
                // real diagonal delta = base + dd - 31, dd = jj - l + 31 in [0, 62]; wanted: -1 <= delta <= 2*nlag - 1
                const int base = item.pass * NPASS + cq * 32 - (wg * 64 + rq * 32);
                if (base + 31 < -1 || base - 31 > 2 * p.nlag - 1) continue;      // tile entirely outside the lag band
                const float* sk = tile + cq * 32 * TILE_LD + rq * 32;            // sk[jj * TILE_LD + l] = D[l][jj]
                // For row l this lane needs column jj = dd - 31 + l of exactly one of its two diagonals
                // (dd = lane: valid when l >= 31 - lane; dd = lane + 32: valid when l <= 30 - lane), so one
                // load per row feeds both sums: 32 pipelined loads instead of 64 half-masked ones.
                float se[2] = {0.f, 0.f}, so[2] = {0.f, 0.f};
#pragma unroll
                for (int l = 0; l < 32; ++l) {
                    const float val = sk[((lane + l + 1) & 31) * TILE_LD + l];
                    const bool hi = (l + lane <= 30);            // belongs to dd = lane + 32
                    if (l & 1) { so[1] += hi ? val : 0.f; so[0] += hi ? 0.f : val; }
                    else       { se[1] += hi ? val : 0.f; se[0] += hi ? 0.f : val; }
                }
                // Scatter into this warp's private sums, branch-free.  base is even, so delta = base + dd - 31
                // is even exactly on odd lanes:
                //   odd lane : re[delta/2] += se + so
                //   even lane: im[(delta+1)/2] += so   (odd rows)   then   im[(delta-1)/2] -= se   (even rows)
                // Within a round all target addresses differ (dd and dd + 32 are 16 lags apart).
                {
                    const bool oddl = lane & 1;
                    float* tgt[2];
                    float val[2];
                    bool ok[2];
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int dd = lane + 32 * h;
                        const int delta = base + dd - 31;
                        const int d = oddl ? (delta >> 1) : ((delta + 1) >> 1);
                        ok[h] = dd <= 62 && (oddl ? delta >= 0 : delta + 1 >= 0) && d < p.nlag;
                        tgt[h] = (oddl ? cre : cim) + (ok[h] ? d : 0);
                        val[h] = oddl ? se[h] + so[h] : so[h];
                    }
                    const float c0 = ok[0] ? *tgt[0] : 0.f, c1 = ok[1] ? *tgt[1] : 0.f;
                    if (ok[0]) *tgt[0] = c0 + val[0];
                    if (ok[1]) *tgt[1] = c1 + val[1];
                    __syncwarp();
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int dd = lane + 32 * h;
                        const int delta = base + dd - 31;
                        const int d = (delta - 1) >> 1;
                        ok[h] = !oddl && dd <= 62 && delta - 1 >= 0 && d < p.nlag;
                        tgt[h] = cim + (ok[h] ? d : 0);
                    }
                    const float e0 = ok[0] ? *tgt[0] : 0.f, e1 = ok[1] ? *tgt[1] : 0.f;
                    if (ok[0]) *tgt[0] = e0 - se[0];
                    if (ok[1]) *tgt[1] = e1 - se[1];
                    __syncwarp();
                }
            }
            // combine the eight parts, write the row, clear the sums for the next item
            asm volatile("bar.sync 3, %0;" ::"n"(EPI_PARTS * 32) : "memory");
            float2* out = p.partial + (size_t)item.row * (size_t)p.HT;
            for (int l = threadIdx.x; l < p.HT; l += EPI_PARTS * 32) {
                float re = 0.f, im = 0.f;
#pragma unroll
                for (int w = 0; w < EPI_PARTS; ++w) {
                    re += cacc[(w * 2 + 0) * p.HT + l];
                    im += cacc[(w * 2 + 1) * p.HT + l];
                    cacc[(w * 2 + 0) * p.HT + l] = 0.f;
                    cacc[(w * 2 + 1) * p.HT + l] = 0.f;
                }
                out[l] = make_float2(re, im);
            }
            asm volatile("bar.sync 3, %0;" ::"n"(EPI_PARTS * 32) : "memory");
        }
    }
    __syncthreads();
}

// ---------------------------------------------------------------------------------------------
// split kernel: three interleaved BF16 planes.  plane[2q + c] = component c of sig[(q + dmin) mod n]
// for q < n_valid (else 0): n_valid = n for the x operand (zero tail), = len for the s operand (circular
// extension).  b0 = bf16(z), b1 = bf16(z - b0), b2 = bf16(z - b0 - b1): b0 + b1 + b2 = z to 2^-24.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint16_t bf16_rn_bits(float v) {
    uint32_t u = __float_as_uint(v);
    u += 0x7FFFu + ((u >> 16) & 1u);             // round to nearest even (no NaN/Inf inputs on this path)
    return (uint16_t)(u >> 16);
}
__device__ __forceinline__ float bf16_bits_to_float(uint16_t b) { return __uint_as_float((uint32_t)b << 16); }

__global__ void bf16_split_kernel(const float2* __restrict__ sig, int n, int dmin, uint16_t* __restrict__ p0,
                                  uint16_t* __restrict__ p1, uint16_t* __restrict__ p2, long long len, long long n_valid) {
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= len) return;
    float2 v = make_float2(0.f, 0.f);
    if (q < n_valid) {
        long long i = (q + dmin) % n;
        if (i < 0) i += n;
        v = sig[i];
    }
    const float c[2] = {v.x, v.y};
    uint16_t o[3][2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const uint16_t a0 = bf16_rn_bits(c[k]);
        const float r1 = c[k] - bf16_bits_to_float(a0);
        const uint16_t a1 = bf16_rn_bits(r1);
        const float r2 = r1 - bf16_bits_to_float(a1);
        o[0][k] = a0; o[1][k] = a1; o[2][k] = bf16_rn_bits(r2);
    }
    reinterpret_cast<uint32_t*>(p0)[q] = (uint32_t)o[0][0] | ((uint32_t)o[0][1] << 16);
    reinterpret_cast<uint32_t*>(p1)[q] = (uint32_t)o[1][0] | ((uint32_t)o[1][1] << 16);
    reinterpret_cast<uint32_t*>(p2)[q] = (uint32_t)o[2][0] | ((uint32_t)o[2][1] << 16);
}

// Fused per-frame preparation (one launch, blockIdx.y = signal): BF16 planes of ref (circular
// extension, also the x operand when n is a multiple of 1024) and of srv rotated by -peek; while ref is
// in registers, optionally emit refw = ref * window for the CAF.  Four samples per thread, loads first.
struct PrepParams {
    const float2* sig[2];
    int dmin[2];
    int zero_outside[2];    // 1: samples outside [0, n) are zero (x operand); 0: circular (s operand)
    long long n_valid[2];   // plane entries q >= n_valid are zero (0 = no limit)
    uint16_t* plane[2][3];
    const float* win;       // optional
    float2* refw;           // optional: ref * win for q < n
    int n;
    long long len;
    // optional (signal 0 only): BF16 planes of the CAF x operand, cafx[q + caf_off] = ref[q] * win[q]
    // (zero for indices below caf_off), written for indices < caf_nx
    uint16_t* cafx[3];
    long long caf_off, caf_nx;
};

__device__ __forceinline__ void bf16_split3(float v, uint16_t (&b)[3]) {
    b[0] = bf16_rn_bits(v);
    const float r1 = v - bf16_bits_to_float(b[0]);
    b[1] = bf16_rn_bits(r1);
    b[2] = bf16_rn_bits(r1 - bf16_bits_to_float(b[1]));
}

__global__ void __launch_bounds__(256) tc_prep_kernel(const __grid_constant__ PrepParams p) {
    const int sg = blockIdx.y;
    const long long q0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (q0 >= p.len) return;
    const float2* __restrict__ sig = p.sig[sg];
    long long i0 = (q0 + p.dmin[sg]) % p.n;
    if (i0 < 0) i0 += p.n;
    float2 v[4];
    float w[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        long long i = i0 + k;
        if (i >= p.n) i -= p.n;
        if (i >= p.n) i %= p.n;
        const long long lin = q0 + k + p.dmin[sg];           // un-wrapped sample index
        const bool ok = (q0 + k < p.len) && (!p.zero_outside[sg] || (lin >= 0 && lin < p.n)) &&
                        (p.n_valid[sg] == 0 || q0 + k < p.n_valid[sg]);
        v[k] = ok ? sig[i] : make_float2(0.f, 0.f);
        w[k] = (sg == 0 && p.win && lin >= 0 && lin < p.n) ? p.win[lin] : 1.f;
    }
    uint32_t o[3][4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float c[2] = {v[k].x, v[k].y};
        uint16_t b[3][2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const uint16_t a0 = bf16_rn_bits(c[e]);
            const float r1 = c[e] - bf16_bits_to_float(a0);
            const uint16_t a1 = bf16_rn_bits(r1);
            const float r2 = r1 - bf16_bits_to_float(a1);
            b[0][e] = a0; b[1][e] = a1; b[2][e] = bf16_rn_bits(r2);
        }
#pragma unroll
        for (int pl = 0; pl < 3; ++pl) o[pl][k] = (uint32_t)b[pl][0] | ((uint32_t)b[pl][1] << 16);
    }
    if (q0 + 3 < p.len) {
#pragma unroll
        for (int pl = 0; pl < 3; ++pl)
            reinterpret_cast<uint4*>(p.plane[sg][pl])[q0 / 4] = make_uint4(o[pl][0], o[pl][1], o[pl][2], o[pl][3]);
    } else {
        for (int k = 0; k < 4 && q0 + k < p.len; ++k)
#pragma unroll
            for (int pl = 0; pl < 3; ++pl) reinterpret_cast<uint32_t*>(p.plane[sg][pl])[q0 + k] = o[pl][k];
    }
    // signal 0 may carry a lead-in (dmin < 0): its sample index is lin = q + dmin
    const long long lin0 = q0 + p.dmin[0];
    if (sg == 0 && p.refw) {
        for (int k = 0; k < 4; ++k)
            if (lin0 + k >= 0 && lin0 + k < p.n && q0 + k < p.len) p.refw[lin0 + k] = make_float2(v[k].x * w[k], v[k].y * w[k]);
    }
    if (sg == 0 && p.cafx[0] && lin0 >= 0) {
        uint32_t c[3][4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            uint16_t br[3], bi[3];
            const bool in = lin0 + k < p.n && q0 + k < p.len;
            bf16_split3(in ? v[k].x * w[k] : 0.f, br);
            bf16_split3(in ? v[k].y * w[k] : 0.f, bi);
#pragma unroll
            for (int pl = 0; pl < 3; ++pl) c[pl][k] = (uint32_t)br[pl] | ((uint32_t)bi[pl] << 16);
        }
        const long long t0 = lin0 + p.caf_off;
#pragma unroll
        for (int pl = 0; pl < 3; ++pl) {
            uint32_t* dst = reinterpret_cast<uint32_t*>(p.cafx[pl]);
            if (lin0 + 3 < p.n && t0 + 3 < p.caf_nx) reinterpret_cast<uint4*>(dst)[t0 / 4] = make_uint4(c[pl][0], c[pl][1], c[pl][2], c[pl][3]);
            else for (int k = 0; k < 4; ++k) if (lin0 + k < p.n && t0 + k < p.caf_nx) dst[t0 + k] = c[pl][k];
            if (lin0 < p.caf_off) for (int k = 0; k < 4; ++k) if (lin0 + k < p.caf_off && lin0 + k < p.caf_nx) dst[lin0 + k] = 0u;   // zero lead-in
        }
    }
}

inline size_t toep_smem_bytes(int HT) {
    return (size_t)OPERAND_BYTES + (size_t)NUM_MMA_WG * TILE_FLOATS * sizeof(float) + (size_t)EPI_PARTS * 2 * HT * sizeof(float);
}

}  // namespace tc
}  // namespace prc
