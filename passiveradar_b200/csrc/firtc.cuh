// firtc.cuh -- the clutter FIR  out[i] = srv[i] - sum_k w[k] ref[i + peek - k]  on the Hopper tensor cores (wgmma).
//
// (reference clutter_removal.py:51 `srv - A @ filterTaps`, and np.convolve at :153-155 for the Toeplitz
// variant).  With interleaved real data z = (re0, im0, re1, im1, ...) a block of 64 complex outputs is a
// row vector of 128 reals, and
//
//     clutter[a][u'] = sum_v' Z[a][v'] * Wm[v'][u'],      Z[a][v'] = z[128 a + v' - 2 PRE]
//
// where Wm (KV x 128, KV = 2 (64 + peek + PRE)) is a constant band matrix made of the taps: for output
// (io, ao) and input (iq, bq) the tap index is k = io + peek + PRE - iq and the entry is the (ao, bq)
// element of [[wr, -wi], [wi, wr]].  So the FIR is a plain GEMM, M = row blocks a, N = 128, K = KV, with
// K-major operands: A rows are overlapping windows of the signal planes, B is Wm^T, built once per frame
// by fir_bmat_kernel.  Same BF16x3 split as toepcorr.cuh (six products, fp32 accumulation); the a0*b0
// chain and the five cross terms are accumulated apart.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "toepcorr.cuh"

namespace prc {
namespace tc {

constexpr int FIR_ROWS = 128;                 // row blocks per CTA (two warpgroups of wgmma M = 64)
constexpr int FIR_N = 128;                    // reals per row block (wgmma N)
constexpr int FIR_KATOM = 64;                 // K elements per 128-byte swizzle atom
constexpr int FIR_STAGES = 2;                 // pipeline stages of the taps-matrix (B) tiles
constexpr int FIR_TILE_BYTES = FIR_ROWS * 128;               // one B plane, one K-atom: 16 KB
constexpr int FIR_BSTAGE_BYTES = NPLANE * FIR_TILE_BYTES;    // 48 KB
constexpr int FIR_MAX_ATOMS = 16;             // kvp <= 1024  (M + peek up to ~440 taps)
// The A operand of K-atom kc = 2 j + h is "signal row (m + j), half h": successive atoms are the same
// data shifted by one row.  So the CTA keeps the raw rows [a0, a0 + 128 + j_max] resident (two swizzled
// half-buffers per plane, loaded ONCE); the consumers read the row-shifted operand with ldmatrix into
// registers (wgmma's register-A form) instead of re-reading a 6x Toeplitz-expanded operand from L2.
constexpr int FIR_AROWS = FIR_ROWS + FIR_MAX_ATOMS / 2;      // 136 = 17 groups of 8
constexpr int FIR_AHALF_BYTES = FIR_AROWS * 128;             // 17 KB
constexpr int FIR_A_BYTES = NPLANE * 2 * FIR_AHALF_BYTES;    // 102 KB
constexpr int FIR_MMA_WG = 2, FIR_LOAD_WARPS = 4;
constexpr int FIR_THREADS = 32 * (4 * FIR_MMA_WG + FIR_LOAD_WARPS);
constexpr int FIR_EPI_STRIDE = 132;           // floats per staged row (conflict-free 128-bit stores)

struct FirTcParams {
    const uint16_t* z[NPLANE];    // signal planes (interleaved BF16); row a starts at element 128 a + zoff
    long long zoff;               // 2 * (LEAD - PRE)
    const uint16_t* b[NPLANE];    // Wm^T planes: [128][kvp] row-major
    int kvp;                      // padded K (multiple of 64, <= 64 * FIR_MAX_ATOMS)
    const float2* srv;
    float2* out;
    int n;
    // optional: BF16 planes of the cleaned channel for the tensor-core CAF (see FirParams in kernels.cuh)
    uint16_t* cafs[3];
    long long caf_off, caf_slen;
};

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], uint32_t saddr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(saddr) : "memory");
}

struct __align__(16) FirShared {
    uint64_t full[FIR_STAGES];
    uint64_t empty[FIR_STAGES];
    uint64_t a_ready;
};

// dynamic shared memory: [A: plane x half x 136 rows x 128 B] [B stages: 2 x plane x 128 rows x 128 B];
// the B stages are reused as the epilogue's transpose buffer.  Warps 0-7: two consumer warpgroups
// (rows [64 wg, 64 wg + 64) of the CTA's row blocks); warps 8-11: loaders.
__global__ void __launch_bounds__(FIR_THREADS, 1) firtc_kernel(const __grid_constant__ FirTcParams p) {
    extern __shared__ __align__(1024) uint8_t fsm[];
    __shared__ FirShared sh;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long a0 = (long long)blockIdx.x * FIR_ROWS;            // first row block of this CTA
    const int natoms = p.kvp / FIR_KATOM;
    uint8_t* abase = fsm;
    uint8_t* bbase = fsm + FIR_A_BYTES;

    if (threadIdx.x == 0) {
        for (int s = 0; s < FIR_STAGES; ++s) { mbar_init(&sh.full[s], FIR_LOAD_WARPS / FIR_STAGES); mbar_init(&sh.empty[s], FIR_MMA_WG); }
        mbar_init(&sh.a_ready, FIR_LOAD_WARPS);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp >= 4 * FIR_MMA_WG) {
        // loaders need few registers: hand them to the consumers, whose two 64-register accumulators, A
        // fragments and descriptors would otherwise not leave room for MMAs in flight
        asm volatile("setmaxnreg.dec.sync.aligned.u32 56;");
        const int lw = warp - 4 * FIR_MMA_WG;             // 0..3
        const int ch = lane & 7, r4 = lane >> 3;
        // ---- resident A: raw signal rows a0 .. a0 + arows - 1, both 64-element halves, three planes
        const int arows = FIR_ROWS + (natoms + 1) / 2;
        for (int pl = 0; pl < NPLANE; ++pl) {
            const uint16_t* zr = p.z[pl] + p.zoff + a0 * 128 + 8 * ch;
            for (int rr = 4 * lw; rr < arows; rr += 4 * FIR_LOAD_WARPS) {
                const int row = rr + r4;
                if (row < arows) {
                    const uint32_t off = (uint32_t)(row >> 3) * 1024 + (uint32_t)(row & 7) * 128 + (uint32_t)((ch ^ (row & 7)) << 4);
                    uint8_t* d0 = abase + (pl * 2 + 0) * FIR_AHALF_BYTES + off;
                    cp_async16(d0, zr + (long long)row * 128);
                    cp_async16(d0 + FIR_AHALF_BYTES, zr + (long long)row * 128 + 64);
                }
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncwarp();
        if (lane == 0) mbar_arrive(&sh.a_ready);
        // ---- streamed B: two warps per stage, each copies half of the stage's rows
        const int st = lw & 1;
        const int half = lw >> 1;
        for (int kc = st; kc < natoms; kc += FIR_STAGES) {
            const int use = kc / FIR_STAGES;
            if (use >= 1) mbar_wait(&sh.empty[st], (use - 1) & 1);
            uint8_t* sb = bbase + st * FIR_BSTAGE_BYTES;
#pragma unroll
            for (int pl = 0; pl < NPLANE; ++pl) {
                uint8_t* dB = sb + pl * FIR_TILE_BYTES;
                const uint16_t* zB = p.b[pl] + (long long)FIR_KATOM * kc + 8 * ch;
#pragma unroll 4
                for (int rr = 0; rr < 64; rr += 4) {
                    const int row = 64 * half + rr + r4;              // 0..127
                    const uint32_t off = (uint32_t)(row >> 3) * 1024 + (uint32_t)(row & 7) * 128 + (uint32_t)((ch ^ (row & 7)) << 4);
                    cp_async16(dB + off, zB + (long long)row * p.kvp);
                }
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
            asm volatile("cp.async.wait_group 0;" ::: "memory");
            fence_proxy_async();
            __syncwarp();
            if (lane == 0) mbar_arrive(&sh.full[st]);
        }
    } else {
        // ======================= consumers
        asm volatile("setmaxnreg.inc.sync.aligned.u32 224;");
        const int wg = warp >> 2, wq = warp & 3;
        const bool leader = (threadIdx.x & 127) == 0;
        // ldmatrix.x4 row addresses: lanes 8 q .. 8 q + 7 address matrix q = (rows +8 if q odd, K chunk +1 if q >= 2)
        const int mq = lane >> 3;
        const int arow = wg * 64 + wq * 16 + (lane & 7) + 8 * (mq & 1);
        const int achunk = mq >> 1;
        float accm[64], accs[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) { accm[i] = 0.f; accs[i] = 0.f; }
        mbar_wait(&sh.a_ready, 0);
        for (int kc = 0; kc < natoms; ++kc) {
            const int st = kc & (FIR_STAGES - 1);
            mbar_wait(&sh.full[st], (kc / FIR_STAGES) & 1);
            const int row = arow + (kc >> 1);                  // A of atom kc = signal rows shifted by kc / 2
            const uint32_t sa = smem_u32(abase) + (uint32_t)(kc & 1) * FIR_AHALF_BYTES + (uint32_t)(row >> 3) * 1024 + (uint32_t)(row & 7) * 128;
            const uint32_t sbm = smem_u32(bbase + st * FIR_BSTAGE_BYTES);
#pragma unroll
            for (int kk = 0; kk < FIR_KATOM / 16; ++kk) {
                uint32_t fa[NPLANE][4];
                uint64_t db[NPLANE];
                const uint32_t chunk = (uint32_t)(((2 * kk + achunk) ^ (row & 7)) << 4);
#pragma unroll
                for (int pl = 0; pl < NPLANE; ++pl) {
                    ldmatrix_x4(fa[pl], sa + pl * 2 * FIR_AHALF_BYTES + chunk);
                    db[pl] = make_desc_sw128(sbm + pl * FIR_TILE_BYTES + kk * 32, 16, 1024);
                }
                wgmma_fence();
                wgmma_rs(accm, fa[0], db[0]);
                wgmma_rs(accs, fa[0], db[1]);
                wgmma_rs(accs, fa[1], db[0]);
                wgmma_rs(accs, fa[0], db[2]);
                wgmma_rs(accs, fa[2], db[0]);
                wgmma_rs(accs, fa[1], db[1]);
                wgmma_commit();
            }
            wgmma_wait<0>();
            if (leader) mbar_arrive(&sh.empty[st]);           // this stage's B tiles have been read
        }
        // ======================= epilogue: out = srv - clutter.  Registers -> shared-memory tile (row = row
        // block) -> each warp's 16 rows x 64 samples are contiguous ranges of srv / out, streamed with fully
        // coalesced 128-bit accesses (and 64-bit stores per BF16 plane).
        asm volatile("bar.sync 1, %0;" ::"n"(32 * 4 * FIR_MMA_WG) : "memory");   // every MMA has read its B stage
        float* tile = reinterpret_cast<float*>(bbase);                             // [FIR_ROWS][FIR_EPI_STRIDE]
#pragma unroll
        for (int i = 0; i < 64; i += 2) {
            const int r = wg * 64 + wq * 16 + (lane >> 2) + 8 * ((i >> 1) & 1);
            const int col = (i >> 2) * 8 + 2 * (lane & 3);
            *reinterpret_cast<float2*>(tile + r * FIR_EPI_STRIDE + col) = make_float2(accm[i] + accs[i], accm[i + 1] + accs[i + 1]);
        }
        asm volatile("bar.sync 1, %0;" ::"n"(32 * 4 * FIR_MMA_WG) : "memory");
        const int tw = warp >> 1;                      // 32-row group of the tile
        const int rbase = (warp & 1) * 16;             // this warp's 16 rows of it
        const float* trows = tile + tw * 32 * FIR_EPI_STRIDE;
        const long long ibase = (a0 + tw * 32) * 64 + 2 * lane;        // two samples per lane and row
        constexpr int RB = 8;
        for (int r0 = rbase; r0 < rbase + 16; r0 += RB) {
            float4 sv[RB];
#pragma unroll
            for (int u = 0; u < RB; ++u) {
                const long long i = ibase + (long long)(r0 + u) * 64;
                if (i + 1 < p.n) sv[u] = *reinterpret_cast<const float4*>(p.srv + i);
                else if (i < p.n) { const float2 t = p.srv[i]; sv[u] = make_float4(t.x, t.y, 0.f, 0.f); }
                else sv[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int u = 0; u < RB; ++u) {
                const int r = r0 + u;
                const long long i = ibase + (long long)r * 64;
                if (i >= p.n) continue;
                const float4 cl = *reinterpret_cast<const float4*>(trows + r * FIR_EPI_STRIDE + 4 * lane);
                const float4 ov = make_float4(sv[u].x - cl.x, sv[u].y - cl.y, sv[u].z - cl.z, sv[u].w - cl.w);
                if (i + 1 < p.n) *reinterpret_cast<float4*>(p.out + i) = ov;
                else p.out[i] = make_float2(ov.x, ov.y);
                if (p.cafs[0]) {
                    float c4[4] = {ov.x, ov.y, ov.z, ov.w};
                    uint32_t w0[3], w1[3];
#pragma unroll
                    for (int pl = 0; pl < 3; ++pl) {
                        uint16_t b4[4];
#pragma unroll
                        for (int e = 0; e < 4; ++e) { b4[e] = bf16_rn_bits(c4[e]); c4[e] -= bf16_bits_to_float(b4[e]); }
                        w0[pl] = (uint32_t)b4[0] | ((uint32_t)b4[1] << 16);
                        w1[pl] = (uint32_t)b4[2] | ((uint32_t)b4[3] << 16);
                    }
                    const long long q1 = i + p.caf_off, q2 = i - (p.n - p.caf_off);
                    const bool two = i + 1 < p.n;
#pragma unroll
                    for (int pl = 0; pl < 3; ++pl) {
                        uint32_t* dst = reinterpret_cast<uint32_t*>(p.cafs[pl]);
                        if (two && q1 + 1 < p.caf_slen && !(q1 & 1)) *reinterpret_cast<uint2*>(dst + q1) = make_uint2(w0[pl], w1[pl]);
                        else {
                            if (q1 < p.caf_slen) dst[q1] = w0[pl];
                            if (two && q1 + 1 < p.caf_slen) dst[q1 + 1] = w1[pl];
                        }
                        if (q2 >= 0 && q2 < p.caf_slen) dst[q2] = w0[pl];
                        if (two && q2 + 1 >= 0 && q2 + 1 < p.caf_slen) dst[q2 + 1] = w1[pl];
                    }
                }
            }
        }
    }
    __syncthreads();
}

// Wm^T planes: B[u'][v'] for u' = 2 io + ao, v' = 2 iq + bq:  k = io + shift - iq (shift = peek + PRE);
// 0 <= k < M: (ao,bq) = (0,0): wr, (0,1): -wi, (1,0): wi, (1,1): wr;  else 0.
__global__ void fir_bmat_kernel(const float2* __restrict__ taps, int M, int shift, int kvp,
                                uint16_t* __restrict__ p0, uint16_t* __restrict__ p1, uint16_t* __restrict__ p2) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= FIR_N * kvp) return;
    const int u = idx / kvp, v = idx - u * kvp;
    const int io = u >> 1, ao = u & 1, iq = v >> 1, bq = v & 1;
    const int k = io + shift - iq;
    float val = 0.f;
    if (k >= 0 && k < M) {
        const float2 w = taps[k];
        val = (ao == bq) ? w.x : (ao ? w.y : -w.y);
    }
    uint16_t b[3];
    bf16_split3(val, b);
    p0[idx] = b[0];
    p1[idx] = b[1];
    p2[idx] = b[2];
}

inline size_t firtc_smem_bytes() { return (size_t)FIR_A_BYTES + (size_t)FIR_STAGES * FIR_BSTAGE_BYTES; }

}  // namespace tc
}  // namespace prc
