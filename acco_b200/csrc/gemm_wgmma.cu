// KERNEL B - persistent, warp-specialised wgmma GEMM (Hopper, sm_90a).  One kernel serves every contraction of the training step
//
//        D[M, N] (+)= A[M, K] * B[N, K]^T  (+ bias[N])        bf16 in, fp32 accumulate in registers, bf16 out
//
//   forward   Y  = X  * W^T      A = X  (K-major)    B = W  (K-major)                      ("TN")
//   dgrad     dX = dY * W        A = dY (K-major)    B = W  stored [K, N] -> MN-major      ("NN")
//   wgrad     dW += dY^T * X     A = dY stored [K, M] -> MN-major,  B = X stored [K, N] -> MN-major, split-K,
//                                epilogue = add into the bf16 gradient arena (beta = 1)
//
// and its weight operand can be ALL-GATHERED ON THE FLY: W is a weight matrix living in the flat parameter arena.  After an ACCO
// round the fresh values of a row-block of W exist only on the rank that owns that slice of the arena (the round kernel can skip
// pushing it).  In gather mode this kernel is the *first consumer* of W in the next forward pass and performs the all-gather
// itself, tile by tile, overlapped with the math:
//
//   * the CTA that computes output tile (m 0, n_blk) TMA-loads its B tiles straight from the OWNER's memory over NVLink (tensor
//     map built on the peer-mapped address), feeds them to the tensor cores, and TMA-stores them into the local copy of W and
//     publishes a per-(n_blk, k_blk) ready flag (st.release.gpu);
//   * every other CTA of that column waits on the flag (ld.acquire.gpu, by its single producer thread) and loads the tile from the
//     local copy - L2-resident, whereas peer memory bypasses the local L2, so each remote byte crosses NVLink exactly once;
//   * later kernels (dgrad / wgrad / next micro-batches) simply use the now complete local copy.
//
// Pipeline (one CTA per SM, 3 warpgroups, a CTA computes 128 x BN output tiles in a persistent loop):
//   warpgroup 0 : TMA producer   - one thread: cp.async.bulk.tensor (128B swizzle) into a 4-8 stage smem ring, mbarrier tx counts;
//                                  with a cluster of pm x pn CTAs the CTAs of a row share their A tile and the CTAs of a column
//                                  their B tile: each loads its share and TMA-multicasts it
//   warpgroups 1-2 : consumers   - wgmma.mma_async m64nBNk16 on 64 rows each, accumulators in registers, one wgmma group in flight;
//                                  release a stage to every CTA that wrote into it, then the epilogue (+bias, bf16, global store /
//                                  exact fp32 read-modify-write for beta = 1 / bf16x2 atomic add for split-K partial sums)
//
// Operand layouts in shared memory (wgmma canonical layouts, 128-byte swizzle):
//   K-major  : rows of 64 k (128 B), 8-row swizzle atoms 1024 B apart (SBO); one TMA box {64 k, rows}
//   MN-major : one TMA box {64 mn, 64 k} gives 64 rows (k) of 128 B = 8 KiB per 64-mn chunk;
//              SBO = 1024 B between 8-k groups, LBO = 8192 B between 64-mn chunks; advancing K by 16 = +2048 B
// In both layouts the 64-row half of the A tile that consumer warpgroup w multiplies starts 8 KiB * w into the stage.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include <mutex>
#include <unordered_map>

#include "wgmma.cuh"

namespace acco_gemm {

using namespace acco_tc;

constexpr int BM = 128, BN_MAX = 256, BK = 64;
constexpr int A_BYTES = BM * BK * 2;               // 16 KiB per stage
constexpr int RING_BYTES = 192 * 1024;             // 4 x 48 KiB (BN 256), 6 x 32 KiB (BN 128), 8 x 24 KiB (BN 64)
constexpr int MAX_STAGES = 8;
constexpr int SMEM_BYTES = RING_BYTES + 1024 /*align*/ + 256 /*barriers*/;
constexpr int THREADS = 384;
constexpr int MAX_PEERS = 8;
constexpr int MN_CHUNK_BYTES = 64 * BK * 2;        // one {64 mn, 64 k} box of an MN-major operand

struct Params {
    CUtensorMap map_a;                 // K-major: box {64 k, 128 / pn rows} of A [M, K]; MN-major: box {64 m, 64 k} of A^T [K, M]
    CUtensorMap map_b;                 // K-major: box {64 k, BN / pm rows} of B [N, K]; MN-major: box {64 n, 64 k} of B^T [K, N]
    CUtensorMap map_b_peer[MAX_PEERS]; // gather mode: B on each rank (peer-mapped), box {64 k, BN rows}
    const __nv_bfloat16* bias;         // optional [N]
    const int* tile_owner;             // [num_n] : -1 -> local copy is valid, r -> gather from rank r
    uint32_t* flags;                   // [num_n * num_k * 2] ready epochs
    uint32_t* epoch;                   // device word: last completed gather epoch
    uint32_t* done_ctas;               // device word: CTA completion counter (self resetting)
    __nv_bfloat16* out;                // D, row stride ldd
    long long ldd;
    int M, N, K;
    int splits, kb_per_split;          // split-K: unit = (split, m-block, n-block)
    int reduce;                        // epilogue: 0 = store, 1 = D += (exact fp32 read-modify-write with one K split)
    int atomic;                        // 1: several K splits add into the same tile - bf16x2 atomic adds
    int gather;                        // 0: plain GEMM (tile_owner ignored)
    int stages, stage_bytes;           // smem ring geometry: stages x (16 KiB of A + BN * 128 B of B)
    int pm, pn;                        // cluster = pm x pn CTAs: the pn CTAs of a row share A, the pm CTAs of a column share B
    unsigned long long* dbg;           // optional: CTA 0 writes %globaltimer stamps of its phases (tools/gemm_timeline.py)
};

__device__ __forceinline__ void wait_flag_gpu(const uint32_t* f, uint32_t epoch) {
    uint32_t v;
    unsigned spins = 0;
    unsigned long long t0 = 0;
    do {
        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(f) : "memory");
        if ((++spins & 0xFFFFF) == 0) {       // watchdog: the gathering CTA never published this tile
            unsigned long long now;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
            if (t0 == 0) t0 = now;
            else if (now - t0 > 60ull * 1000000000ull) __trap();
        }
    } while ((int32_t)(v - epoch) < 0);
}

__device__ __forceinline__ void stamp(const Params& P, int slot) {
    if (P.dbg != nullptr && blockIdx.x == 0) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        P.dbg[slot] = t;
    }
}

// work decomposition shared by every role: unit t -> (split, m-block, n-block, k-block range).  A cluster of pm x pn CTAs owns a
// super-tile of pm x pn adjacent tiles; CTA (pi, pj) computes tile (smb * pm + pi, sn * pn + pj).  Tiles beyond the matrix (odd
// counts) are phantom: their loads are zero-filled by TMA and nothing is stored, but the CTA still contributes its share of the
// multicast operand loads.
struct Unit {
    int mb, n_blk, kb0, kb1;
};
__device__ __forceinline__ Unit decode_unit(int t, int tiles, int num_sn, int num_k, int kb_per_split, int pm, int pn, int pi, int pj) {
    Unit u;
    const int s = t / tiles, tile = t - s * tiles;
    const int smb = tile / num_sn;
    u.mb = smb * pm + pi;
    u.n_blk = (tile - smb * num_sn) * pn + pj;
    u.kb0 = s * kb_per_split;
    u.kb1 = min(num_k, u.kb0 + kb_per_split);
    return u;
}

template <int BN, int TA, int TB>
__device__ __forceinline__ void mma_k16(float (&acc)[BN / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
    if constexpr (BN == 256) wgmma_m64n256k16<TA, TB>(acc, da, db, scale_d);
    else if constexpr (BN == 128) wgmma_m64n128k16<TA, TB>(acc, da, db, scale_d);
    else wgmma_m64n64k16<TA, TB>(acc, da, db, scale_d);
}

template <int BN, int A_MN, int B_MN>
__global__ void __launch_bounds__(THREADS, 1) gemm_kernel(const __grid_constant__ Params P) {
    extern __shared__ uint8_t smem_raw[];
    if (threadIdx.x == 0) stamp(P, 0);
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);   // SWIZZLE_128B needs 1024 B alignment
    uint64_t* full_bar = (uint64_t*)(smem + RING_BYTES);      // [MAX_STAGES]  TMA bytes landed
    uint64_t* empty_bar = full_bar + MAX_STAGES;              // [MAX_STAGES]  stage reusable (every consumer that reads it released it)

    constexpr int B_BYTES = BN * BK * 2;
    const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
    const int n_stages = P.stages, stage_bytes = P.stage_bytes;
    const int pm = P.pm, pn = P.pn, cl_size = pm * pn;
    const uint32_t cl_rank = cl_size > 1 ? cluster_ctarank() : 0u;
    const int pi = (int)cl_rank / pn, pj = (int)cl_rank - pi * pn;
    const int unit0 = blockIdx.x / cl_size, unit_stride = gridDim.x / cl_size;
    const int num_n = (P.N + BN - 1) / BN, num_k = (P.K + BK - 1) / BK, num_mb = (P.M + BM - 1) / BM;
    const int num_sn = (num_n + pn - 1) / pn;
    const int tiles = ((num_mb + pm - 1) / pm) * num_sn;
    const int num_units = tiles * P.splits;
    const int kbs = P.kb_per_split;
    // multicast masks (cluster ranks): the CTAs of my row share my A tile, the CTAs of my column my B tile.  The same set (row and
    // column mates, me included) writes into my stages, so each of my consumers releases a stage to all of them.
    uint16_t mask_a = 0, mask_b = 0;
    for (int j = 0; j < pn; ++j) mask_a |= (uint16_t)(1u << (pi * pn + j));
    for (int i = 0; i < pm; ++i) mask_b |= (uint16_t)(1u << (i * pn + pj));
    const uint16_t mask_rel = mask_a | mask_b;

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&P.map_a) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&P.map_b) : "memory");
        for (int s = 0; s < n_stages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 2u * (uint32_t)(pm + pn - 1));   // both consumer warpgroups of every CTA that reads what I (multi)cast
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (cl_size > 1) cluster_sync_all();           // the peers' barriers exist before anyone signals them
    // Programmatic dependent launch: everything above overlaps the tail of the preceding kernel; global memory is touched only after
    // the upstream grid has completed and flushed.
    if (threadIdx.x == 0) stamp(P, 1);
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    if (threadIdx.x == 0) stamp(P, 2);
    const uint32_t epoch = P.gather ? (*(volatile uint32_t*)P.epoch + 1u) : 0u;
    auto flag_ptr = [&](int n_blk, int kb, int half) { return P.flags + ((size_t)n_blk * num_k + kb) * 2 + half; };

    if (wg == 0) {
        // ============================ TMA PRODUCER ============================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (tid == 0) {
            int stage = 0;
            uint32_t phase = 0;
            // my share of the operand tiles: 1/pn of the A tile (multicast to my row), 1/pm of the B tile (to my column)
            const int a_rows = BM / pn, a_off = pj * a_rows;                  // K-major A: rows [a_off, a_off + a_rows)
            const int nach = (BM / 64) / pn, a_ch0 = pj * nach;               // MN-major A: 64-m chunks [a_ch0, a_ch0 + nach)
            const int b_rows = BN / pm, b_off = pi * b_rows;                  // K-major B: rows [b_off, b_off + b_rows)
            const int nbch = (BN / 64) / pm, b_ch0 = pi * nbch;               // MN-major B: 64-n chunks [b_ch0, b_ch0 + nbch)
            const bool mc_a = pn > 1, mc_b = pm > 1;
            for (int t = unit0; t < num_units; t += unit_stride) {
                const Unit u = decode_unit(t, tiles, num_sn, num_k, kbs, pm, pn, pi, pj);
                const int n_blk = u.n_blk;
                const int m0 = u.mb * BM, n0 = n_blk * BN;
                const int owner = P.gather ? P.tile_owner[n_blk] : -1;
                const bool gatherer = owner >= 0 && u.mb == 0;
                const bool waiter = owner >= 0 && u.mb != 0;
                const CUtensorMap* bmap = gatherer ? &P.map_b_peer[owner] : &P.map_b;
                // Flags of one n_blk are released in k order by a single thread, so "last k-block ready" implies "all ready": one
                // acquire per tile in the common case, per-k-block polling only while the gatherer is still streaming.
                bool all_ready = !waiter;
                if (waiter) {
                    uint32_t v0, v1;
                    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v0) : "l"(flag_ptr(n_blk, num_k - 1, 0)) : "memory");
                    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v1) : "l"(flag_ptr(n_blk, num_k - 1, 1)) : "memory");
                    all_ready = (int32_t)(v0 - epoch) >= 0 && (int32_t)(v1 - epoch) >= 0;
                    if (all_ready) asm volatile("fence.proxy.async;" ::: "memory");
                }
                for (int kb = u.kb0; kb < u.kb1; ++kb) {
                    if (!all_ready) {
                        wait_flag_gpu(flag_ptr(n_blk, kb, 0), epoch);
                        wait_flag_gpu(flag_ptr(n_blk, kb, 1), epoch);
                        asm volatile("fence.proxy.async;" ::: "memory");   // generic-proxy observation -> async-proxy (TMA) read
                    }
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    uint8_t* sa = smem + stage * stage_bytes;
                    uint8_t* sb = sa + A_BYTES;
                    mbar_expect_tx(&full_bar[stage], (uint32_t)(A_BYTES + B_BYTES));   // everything landing in MY stage
                    if (A_MN) {
                        for (int c = a_ch0; c < a_ch0 + nach; ++c) {
                            if (mc_a) tma_load_2d_mc(&P.map_a, &full_bar[stage], sa + c * MN_CHUNK_BYTES, m0 + c * 64, kb * BK, mask_a);
                            else tma_load_2d(&P.map_a, &full_bar[stage], sa + c * MN_CHUNK_BYTES, m0 + c * 64, kb * BK);
                        }
                    } else {
                        if (mc_a) tma_load_2d_mc(&P.map_a, &full_bar[stage], sa + a_off * 128, kb * BK, m0 + a_off, mask_a);
                        else tma_load_2d(&P.map_a, &full_bar[stage], sa, kb * BK, m0);
                    }
                    if (B_MN) {
                        for (int c = b_ch0; c < b_ch0 + nbch; ++c) {
                            if (mc_b) tma_load_2d_mc(bmap, &full_bar[stage], sb + c * MN_CHUNK_BYTES, n0 + c * 64, kb * BK, mask_b);
                            else tma_load_2d(bmap, &full_bar[stage], sb + c * MN_CHUNK_BYTES, n0 + c * 64, kb * BK);
                        }
                    } else {
                        if (mc_b) tma_load_2d_mc(bmap, &full_bar[stage], sb + b_off * 128, kb * BK, n0 + b_off, mask_b);
                        else tma_load_2d(bmap, &full_bar[stage], sb, kb * BK, n0);
                    }
                    if (gatherer) {
                        // write the pulled tile through to the local copy of W, then publish it (both halves of the 256-row tile)
                        mbar_wait(&full_bar[stage], phase);
                        fence_async_smem();
                        tma_store_2d(&P.map_b, sb, kb * BK, n0);
                        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");       // writes complete (not just smem read)
                        asm volatile("fence.proxy.async;" ::: "memory");
                        asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(flag_ptr(n_blk, kb, 0)), "r"(epoch) : "memory");
                        asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(flag_ptr(n_blk, kb, 1)), "r"(epoch) : "memory");
                    }
                    if (t == unit0 && kb == u.kb0) stamp(P, 3);
                    if (++stage == n_stages) { stage = 0; phase ^= 1; }
                }
            }
            stamp(P, 9);
        }
    } else {
        // ============================ CONSUMERS (warpgroups 1 and 2: rows [64 cw, 64 cw + 64) of the tile) ============================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        const int cw = wg - 1;
        const int warp = tid >> 5, lane = tid & 31;
        // stage release: thread r of the warpgroup signals CTA r of the cluster when r reads my stages (one arrival per warpgroup)
        const bool releaser = cl_size > 1 ? (tid < 16 && ((mask_rel >> tid) & 1)) : tid == 0;
        constexpr uint32_t a_lbo = A_MN ? (MN_CHUNK_BYTES >> 4) : 1, a_sbo = 1024 >> 4, a_kstep = A_MN ? 2048 : 32;
        constexpr uint32_t b_lbo = B_MN ? (MN_CHUNK_BYTES >> 4) : 1, b_sbo = 1024 >> 4, b_kstep = B_MN ? 2048 : 32;
        auto release = [&](int s) {
            if (!releaser) return;
            if (cl_size > 1) mbar_arrive_cluster_addr(map_to_cta(&empty_bar[s], (uint32_t)tid));
            else mbar_arrive(&empty_bar[s]);
        };
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        int stage = 0;
        uint32_t phase = 0;
        for (int t = unit0; t < num_units; t += unit_stride) {
            const Unit u = decode_unit(t, tiles, num_sn, num_k, kbs, pm, pn, pi, pj);
            int prev = -1;
            for (int kb = u.kb0; kb < u.kb1; ++kb) {
                mbar_wait(&full_bar[stage], phase);
                if (cw == 0 && tid == 0 && t == unit0 && kb == u.kb0) stamp(P, 4);
                const uint32_t a_addr = smem_u32(smem + stage * stage_bytes) + (uint32_t)(cw * 8192);
                const uint32_t b_addr = smem_u32(smem + stage * stage_bytes + A_BYTES);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / 16; ++k) {
                    const uint64_t da = make_smem_desc(a_addr + k * a_kstep, a_lbo, a_sbo);
                    const uint64_t db = make_smem_desc(b_addr + k * b_kstep, b_lbo, b_sbo);
                    mma_k16<BN, A_MN, B_MN>(acc, da, db, (uint32_t)((kb > u.kb0) | (k != 0)));
                }
                wgmma_commit();
                if (prev >= 0) {
                    wgmma_wait<1>();                   // the previous stage's wgmmas have retired: hand it back
                    release(prev);
                }
                prev = stage;
                if (++stage == n_stages) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            reg_fence(acc);
            release(prev);
            // ---------------- epilogue: fragment (row 16 warp + lane/4 (+8), columns 8 j + 2 (lane % 4) (+1)) -> global
            const int row0 = u.mb * BM + cw * 64 + warp * 16 + (lane >> 2);
            const int colb = u.n_blk * BN + 2 * (lane & 3);
            const bool bias_on = P.bias != nullptr && u.kb0 == 0;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int col = colb + 8 * j;
                if (col >= P.N) continue;                              // N % 8 == 0: col < N implies col + 1 < N
                float b0 = 0.f, b1 = 0.f;
                if (bias_on) {
                    const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(P.bias + col));
                    b0 = f.x; b1 = f.y;
                }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int row = row0 + 8 * h;
                    if (row >= P.M) continue;
                    float v0 = acc[4 * j + 2 * h] + b0, v1 = acc[4 * j + 2 * h + 1] + b1;
                    __nv_bfloat16* dst = P.out + (size_t)row * (size_t)P.ldd + col;
                    if (P.atomic) {
                        __nv_bfloat162 hv = __floats2bfloat162_rn(v0, v1);
                        asm volatile("red.global.add.noftz.bf16x2 [%0], %1;" ::"l"(dst), "r"(*reinterpret_cast<uint32_t*>(&hv)) : "memory");
                        continue;
                    }
                    if (P.reduce) {
                        // beta = 1 with a single K split: exact fp32 accumulate (one rounding), nobody else touches this tile
                        const float2 c = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(dst));
                        v0 += c.x; v1 += c.y;
                    }
                    *reinterpret_cast<__nv_bfloat162*>(dst) = __floats2bfloat162_rn(v0, v1);
                }
            }
        }
        if (cw == 0 && tid == 0) stamp(P, 7);
    }

    // ---------------- teardown ----------------
    __syncthreads();
    if (threadIdx.x == 0) stamp(P, 10);
    if (cl_size > 1) cluster_sync_all();           // no CTA may exit while a peer can still multicast into it or signal it
    if (P.gather && threadIdx.x == 0) {
        __threadfence();
        const uint32_t prev = atomicAdd(P.done_ctas, 1u);
        if (prev == gridDim.x - 1) {
            *P.done_ctas = 0;
            __threadfence();
            *P.epoch = epoch;
        }
    }
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                             const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeFn get_encode() {
    static EncodeFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess) fn = (EncodeFn)p;
    });
    return fn;
}

// The driver's tensor-map encoder needs a current context.  A thread that has not made a runtime call yet - PyTorch's autograd worker
// runs the backward GEMMs of the first step - has none: make the runtime's device's primary context current on it.
static bool bind_primary_context() {
    typedef CUresult (*DeviceGetFn)(CUdevice*, int);
    typedef CUresult (*RetainFn)(CUcontext*, CUdevice);
    typedef CUresult (*SetCurrentFn)(CUcontext);
    void *p_get = nullptr, *p_retain = nullptr, *p_set = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuDeviceGet", &p_get, cudaEnableDefault, &q) != cudaSuccess ||
        cudaGetDriverEntryPoint("cuDevicePrimaryCtxRetain", &p_retain, cudaEnableDefault, &q) != cudaSuccess ||
        cudaGetDriverEntryPoint("cuCtxSetCurrent", &p_set, cudaEnableDefault, &q) != cudaSuccess)
        return false;
    int dev = 0;
    CUdevice d;
    CUcontext c = nullptr;
    if (cudaGetDevice(&dev) != cudaSuccess || ((DeviceGetFn)p_get)(&d, dev) != CUDA_SUCCESS) return false;
    return ((RetainFn)p_retain)(&c, d) == CUDA_SUCCESS && ((SetCurrentFn)p_set)(c) == CUDA_SUCCESS;
}

// Tensor maps are pure functions of (base, extents, leading dimension, box): encode once, reuse (the parameter / gradient
// arenas and the CUDA-graph static activations keep their addresses for the whole run).
struct MapKey {
    const void* base;
    uint64_t inner, outer, ld;
    uint32_t box_inner, box_outer;
    int elem_bytes;
    bool operator==(const MapKey& o) const {
        return base == o.base && inner == o.inner && outer == o.outer && ld == o.ld && box_inner == o.box_inner && box_outer == o.box_outer &&
               elem_bytes == o.elem_bytes;
    }
};
struct MapKeyHash {
    size_t operator()(const MapKey& k) const {
        size_t h = (size_t)k.base;
        auto mix = [&h](uint64_t v) { h ^= v + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2); };
        mix(k.inner); mix(k.outer); mix(k.ld); mix(((uint64_t)k.box_inner << 32) | k.box_outer); mix((uint64_t)k.elem_bytes);
        return h;
    }
};
static std::mutex g_map_mu;
static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_maps;
static long long g_map_encodes = 0;

// row-major matrix (bf16: elem_bytes 2, fp32: 4) with `outer` rows of `inner` contiguous elements (row stride `ld` elements),
// box {box_inner, box_outer}, 128-byte swizzle (box_inner * elem_bytes = 128 B)
int make_map_typed(CUtensorMap* m, const void* base, uint64_t inner, uint64_t outer, uint64_t ld, uint32_t box_inner, uint32_t box_outer,
                   int elem_bytes) {
    const MapKey key{base, inner, outer, ld, box_inner, box_outer, elem_bytes};
    {
        std::lock_guard<std::mutex> g(g_map_mu);
        auto it = g_maps.find(key);
        if (it != g_maps.end()) { *m = it->second; return 0; }
    }
    EncodeFn enc = get_encode();
    if (!enc) return -2;
    cuuint64_t dims[2] = {inner, outer};
    cuuint64_t strides[1] = {ld * (uint64_t)elem_bytes};
    cuuint32_t box[2] = {box_inner, box_outer};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(m, elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r == CUDA_ERROR_INVALID_CONTEXT && bind_primary_context()) {
        r = enc(m, elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    }
    if (r != CUDA_SUCCESS) return -3;
    std::lock_guard<std::mutex> g(g_map_mu);
    if (g_maps.size() > 8192) g_maps.clear();      // unbounded address churn (eager mode without the caching allocator): start over
    g_maps.emplace(key, *m);
    ++g_map_encodes;
    return 0;
}
static int make_map(CUtensorMap* m, const void* base, uint64_t inner, uint64_t outer, uint64_t ld, uint32_t box_inner, uint32_t box_outer) {
    return make_map_typed(m, base, inner, outer, ld, box_inner, box_outer, 2);
}

typedef void (*KernelFn)(const Params);
// instantiations: BN in {64, 128, 256} x operand majors (the wgmma transpose flags are immediates)
template <int BN>
static KernelFn kernel_for(int a_mn, int b_mn) {
    if (a_mn) return b_mn ? gemm_kernel<BN, 1, 1> : gemm_kernel<BN, 1, 0>;
    return b_mn ? gemm_kernel<BN, 0, 1> : gemm_kernel<BN, 0, 0>;
}
static KernelFn kernel_for(int bn, int a_mn, int b_mn) {
    if (bn == 256) return kernel_for<256>(a_mn, b_mn);
    if (bn == 128) return kernel_for<128>(a_mn, b_mn);
    return kernel_for<64>(a_mn, b_mn);
}

static int g_pm = 0, g_pn = 0;                     // ACCO_GEMM_CLUSTER="pm,pn": force the cluster shape (0 = heuristic)
static unsigned long long* g_dbg = nullptr;        // device buffer for phase time stamps (acco_gemm_set_debug)
static int g_pdl = 1;                              // ACCO_GEMM_PDL=0: no programmatic dependent launch
static int init_once() {
    static int rc = 0;
    static std::once_flag once;
    std::call_once(once, [] {
        for (int bn : {64, 128, 256})
            for (int a = 0; a < 2; ++a)
                for (int b = 0; b < 2; ++b)
                    if (cudaFuncSetAttribute(kernel_for(bn, a, b), cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES) != cudaSuccess) rc = -4;
        const char* e;
        if ((e = getenv("ACCO_GEMM_CLUSTER")) && e[0] && e[1] == ',') { g_pm = e[0] - '0'; g_pn = e[2] - '0'; }
        if ((e = getenv("ACCO_GEMM_PDL")) && e[0] == '0') g_pdl = 0;
    });
    return rc;
}

// How many clusters of `cl` CTAs can be co-resident (persistent grid size); GPC boundaries can strand SMs for cl > 1.
static int max_clusters(int cl, int sms) {
    static int cache[17] = {0};
    static std::mutex mu;
    std::lock_guard<std::mutex> g(mu);
    if (cl < 2 || cl > 16) return sms;
    if (!cache[cl]) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(cl * 64);
        cfg.blockDim = dim3(THREADS);
        cfg.dynamicSmemBytes = SMEM_BYTES;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = cl;
        attr[0].val.clusterDim.y = 1;
        attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        int n = 0;
        if (cudaOccupancyMaxActiveClusters(&n, gemm_kernel<256, 0, 0>, &cfg) != cudaSuccess || n <= 0) { cudaGetLastError(); n = -1; }
        cache[cl] = n;
    }
    const int n = cache[cl];
    if (n <= 0) return 0;
    return n < sms / cl ? n : sms / cl;       // honour a caller-imposed SM cap
}

struct Config {
    int bn, splits, pm, pn;
};

// Tile / split-K / cluster choice: minimise (waves x per-unit cost).  Per k-block a CTA's tensor cores need 4 * bn cycles
// (128 x bn x 64 multiply-adds at 2048 per clock on an H100 SM) and the operand bytes must come in through L2 (~64 B/clk/SM
// assumed); the epilogue is not overlapped with the CTA's own mainloop.  Split-K needs an adding epilogue: accumulating GEMMs
// (wgrad), or a zero-filled output.
static Config choose_config(int M, int N, int K, int a_mn, int b_mn, int reduce, int sms, int bn_req, int splits_req, int pm_req, int pn_req) {
    (void)a_mn; (void)b_mn;
    const int num_k = (K + BK - 1) / BK;
    double best = 1e30;
    Config bc{256, 1, 1, 1};
    const int cands[3] = {256, 128, 64};
    const int num_mb = (M + BM - 1) / BM;
    for (int ci = 0; ci < 3; ++ci) {
        const int bn = cands[ci];
        if (bn_req > 0 && bn != bn_req) continue;
        if (bn_req <= 0 && bn > 64 && bn / 2 >= N) continue;                  // a narrower tile already covers N
        const int num_n = (N + bn - 1) / bn;
        for (int pm = 1; pm <= 2; ++pm) {
            for (int pn = 1; pn <= 2; ++pn) {
                if ((pm_req > 0 && pm != pm_req) || (pm_req <= 0 && pm != 1)) continue;    // multicast only on request
                if ((pn_req > 0 && pn != pn_req) || (pn_req <= 0 && pn != 1)) continue;
                if (b_mn ? ((bn / 64) % pm != 0) : ((bn / pm) % 8 != 0)) continue;
                if (a_mn && (BM / 64) % pn != 0) continue;
                const int cl = pm * pn;
                const int slots = cl > 1 ? max_clusters(cl, sms) * cl : sms;
                if (slots <= 0) continue;
                const long long tiles = (long long)((num_mb + pm - 1) / pm) * ((num_n + pn - 1) / pn) * cl;
                // non-accumulating GEMMs may split K too when K dwarfs the output (LM-head dgrad): the output is zero-filled first
                const int max_s = reduce ? 16 : (num_k >= 128 ? 4 : 1);
                for (int s = 1; s <= max_s; ++s) {
                    if (splits_req > 0 && s != 1) break;
                    int sp = splits_req > 0 ? splits_req : s;
                    if (sp > num_k) sp = num_k;
                    const int kbs = (num_k + sp - 1) / sp;
                    if (splits_req <= 0 && s > 1 && kbs < 8) break;
                    const int s_eff = (num_k + kbs - 1) / kbs;
                    if (splits_req <= 0 && s_eff != s) continue;                       // same unit count as a smaller s
                    const long long units = tiles * s_eff;
                    const long long waves = (units + slots - 1) / slots;
                    const double feed = (A_BYTES / (double)pn + bn * BK * 2 / (double)pm) / 64.0;   // cycles to pull one stage
                    const double mma = 4.0 * bn;
                    const double per_kb = feed > mma ? feed : mma;
                    const double epi = 128.0 * bn * 2.0 / 16.0 + 800.0;                // bf16 stores of the tile + drain
                    const double unit = kbs * per_kb + 600.0 + epi;
                    double cost = waves * unit + 1000.0 * (cl > 1);
                    if (reduce && s_eff > 1) cost += 0.05 * unit * s_eff + (double)M * N * s_eff * 4.0 / 3000.0;   // atomic adds
                    if (!reduce && s_eff > 1) cost += 3000.0 + (double)M * N * 2.0 / 2000.0 + (double)M * N * s_eff * 4.0 / 3000.0;  // zero-fill pass
                    if (cost < best) { best = cost; bc = Config{bn, s_eff, pm, pn}; }
                }
            }
        }
    }
    return bc;
}

struct GatherArgs {
    const void* const* peers;
    int n_peers;
    const int* tile_owner;
    uint32_t* flags;
    uint32_t* epoch;
    uint32_t* done;
};

static int launch(const void* a, long long lda, int a_mn, const void* b, long long ldb, int b_mn, void* d, long long ldd, const void* bias, int M,
                  int N, int K, int accumulate, int bn_req, int splits_req, int pm_req, int pn_req, int msub_req, const GatherArgs* ga, int sms,
                  cudaStream_t st) {
    if (M <= 0 || N <= 0 || K <= 0) return -1;
    if ((lda % 8) || (ldb % 8) || (ldd % 8) || (N % 8)) return -1;
    if (((uintptr_t)a % 16) || ((uintptr_t)b % 16) || ((uintptr_t)d % 16) || (bias && ((uintptr_t)bias % 16))) return -1;
    if (msub_req > 1) return -1;                                           // one 128-row tile per CTA
    int rc = init_once();
    if (rc) return rc;
    const int gather = (ga && ga->n_peers > 0) ? 1 : 0;
    if (gather && (ga->n_peers > MAX_PEERS || a_mn || b_mn || accumulate)) return -1;
    if (bn_req > 0 && bn_req != 64 && bn_req != 128 && bn_req != 256) return -1;
    if ((pm_req > 2) || (pn_req > 2)) return -1;
    Config cfgc{BN_MAX, 1, 1, 1};                                          // gather mode: 256-row weight tiles (GatheredWeight)
    if (!gather) {
        if (g_pm > 0 && pm_req <= 0) pm_req = g_pm;
        if (g_pn > 0 && pn_req <= 0) pn_req = g_pn;
        cfgc = choose_config(M, N, K, a_mn, b_mn, accumulate, sms, bn_req, splits_req, pm_req, pn_req);
    }
    const int bn = cfgc.bn, pm = cfgc.pm, pn = cfgc.pn;
    int splits = cfgc.splits;
    if ((bn_req > 0 && bn != bn_req) || (pm_req > 0 && pm != pm_req) || (pn_req > 0 && pn != pn_req)) return -1;   // request not realisable
    if (b_mn ? ((bn / 64) % pm != 0) : ((bn / pm) % 8 != 0)) return -1;
    if (a_mn && (BM / 64) % pn != 0) return -1;
    Params P;
    if (a_mn) rc = make_map(&P.map_a, a, (uint64_t)M, (uint64_t)K, (uint64_t)lda, 64, BK);
    else rc = make_map(&P.map_a, a, (uint64_t)K, (uint64_t)M, (uint64_t)lda, BK, (uint32_t)(BM / pn));
    if (rc) return rc;
    if (b_mn) rc = make_map(&P.map_b, b, (uint64_t)N, (uint64_t)K, (uint64_t)ldb, 64, BK);
    else rc = make_map(&P.map_b, b, (uint64_t)K, (uint64_t)N, (uint64_t)ldb, BK, (uint32_t)(bn / pm));
    if (rc) return rc;
    for (int i = 0; i < MAX_PEERS; ++i) {
        if (gather && i < ga->n_peers) {
            rc = make_map(&P.map_b_peer[i], ga->peers[i], (uint64_t)K, (uint64_t)N, (uint64_t)ldb, BK, (uint32_t)bn);
            if (rc) return rc;
        } else {
            P.map_b_peer[i] = P.map_b;
        }
    }
    P.bias = (const __nv_bfloat16*)bias;
    P.out = (__nv_bfloat16*)d;
    P.ldd = ldd;
    P.dbg = g_dbg;
    P.tile_owner = gather ? ga->tile_owner : nullptr;
    P.flags = gather ? ga->flags : nullptr;
    P.epoch = gather ? ga->epoch : nullptr;
    P.done_ctas = gather ? ga->done : nullptr;
    P.M = M; P.N = N; P.K = K;
    const int num_k = (K + BK - 1) / BK;
    if (splits < 1) splits = 1;
    if (splits > num_k) splits = num_k;
    P.kb_per_split = (num_k + splits - 1) / splits;
    P.splits = (num_k + P.kb_per_split - 1) / P.kb_per_split;      // no empty split
    P.reduce = accumulate ? 1 : 0;
    bool pdl = g_pdl != 0;
    if (P.splits > 1 && !P.reduce) {
        // split-K of a non-accumulating GEMM: zero-fill D, then every split adds its partial
        if (cudaMemset2DAsync(d, (size_t)ldd * 2, 0, (size_t)N * 2, (size_t)M, st) != cudaSuccess) return -6;
        P.reduce = 1;
        pdl = false;                    // a programmatic edge needs a kernel as its upstream node
    }
    P.atomic = P.splits > 1 ? 1 : 0;
    P.gather = gather;
    P.pm = pm; P.pn = pn;
    P.stage_bytes = A_BYTES + bn * BK * 2;
    P.stages = RING_BYTES / P.stage_bytes;
    if (P.stages > MAX_STAGES) P.stages = MAX_STAGES;
    const int num_n = (N + bn - 1) / bn;
    const int num_mb = (M + BM - 1) / BM;
    const int cl = pm * pn;
    const long long units = (long long)((num_mb + pm - 1) / pm) * ((num_n + pn - 1) / pn) * P.splits;
    const int slots = cl > 1 ? max_clusters(cl, sms) : sms;
    if (slots <= 0) return -5;
    const int grid = (int)(units < (long long)slots ? units : (long long)slots) * cl;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(THREADS);
    cfg.dynamicSmemBytes = SMEM_BYTES;
    cfg.stream = st;
    cudaLaunchAttribute attr[2];
    int na = 0;
    if (cl > 1) {
        attr[na].id = cudaLaunchAttributeClusterDimension;
        attr[na].val.clusterDim.x = cl;
        attr[na].val.clusterDim.y = 1;
        attr[na].val.clusterDim.z = 1;
        ++na;
    }
    if (pdl) {
        attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[na].val.programmaticStreamSerializationAllowed = 1;
        ++na;
    }
    cfg.attrs = attr;
    cfg.numAttrs = na;
    return (int)cudaLaunchKernelEx(&cfg, kernel_for(bn, a_mn, b_mn), P);
}

}  // namespace acco_gemm

// D[M,N] (+)= A * B^T (+ bias).  a_mn / b_mn = 0: operand stored [rows, K] (K contiguous, leading dimension ld);
// = 1: operand stored [K, rows] (rows contiguous).  accumulate: D += (enables split-K).
// bn_req / splits_req / pm_req / pn_req: 0 = heuristic; msub_req: 0 or 1 (one 128-row tile per CTA).
extern "C" int acco_gemm_run(const void* a, long long lda, int a_mn, const void* b, long long ldb, int b_mn, void* d, long long ldd, const void* bias,
                             int M, int N, int K, int accumulate, int bn_req, int splits_req, int pm_req, int pn_req, int msub_req, int sms,
                             cudaStream_t st) {
    return acco_gemm::launch(a, lda, a_mn, b, ldb, b_mn, d, ldd, bias, M, N, K, accumulate, bn_req, splits_req, pm_req, pn_req, msub_req, nullptr, sms,
                             st);
}

// Y = X * W^T with the remote row-blocks of W gathered over NVLink inside the kernel.  peers: n_peers base addresses of W on
// every rank (peer mapped); tile_owner/flags/epoch/done: device pointers.
extern "C" int acco_gemm_tn_gather(const void* x, const void* w_local, void* y, int M, int N, int K, const void* const* peers, int n_peers,
                                   const int* tile_owner, uint32_t* flags, uint32_t* epoch, uint32_t* done, int sms, cudaStream_t st) {
    acco_gemm::GatherArgs ga{peers, n_peers, tile_owner, flags, epoch, done};
    return acco_gemm::launch(x, K, 0, w_local, K, 0, y, N, nullptr, M, N, K, 0, 0, 0, 0, 0, 0, n_peers > 0 ? &ga : nullptr, sms, st);
}

extern "C" int acco_gemm_tile_n() { return acco_gemm::BN_MAX; }
extern "C" int acco_gemm_tile_k() { return acco_gemm::BK; }
extern "C" long long acco_gemm_map_encodes() { return acco_gemm::g_map_encodes; }
extern "C" void acco_gemm_set_debug(unsigned long long* buf) { acco_gemm::g_dbg = buf; }
extern "C" int acco_gemm_max_clusters(int cl, int sms) {
    acco_gemm::init_once();
    return acco_gemm::max_clusters(cl, sms);
}
// the heuristic's pick for a shape (introspection for tools / tests): {bn, splits, pm, pn, rows-per-CTA / 128}
extern "C" void acco_gemm_choose(int M, int N, int K, int a_mn, int b_mn, int accumulate, int sms, int* out5) {
    const acco_gemm::Config c = acco_gemm::choose_config(M, N, K, a_mn, b_mn, accumulate, sms, 0, 0, acco_gemm::g_pm, acco_gemm::g_pn);
    out5[0] = c.bn; out5[1] = c.splits; out5[2] = c.pm; out5[3] = c.pn; out5[4] = 1;
}
