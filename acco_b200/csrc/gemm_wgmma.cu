// KERNEL B - persistent, warp-specialised wgmma GEMM (Hopper, sm_90a).  One kernel serves every contraction of the training step
//
//        D[M, N] (+)= A[M, K] * B[N, K]^T  (+ bias[N])        bf16 in, fp32 accumulate in registers, bf16 out
//
//   forward   Y  = X  * W^T      A = X  (K-major)    B = W  (K-major)                      ("TN")
//   dgrad     dX = dY * W        A = dY (K-major)    B = W  stored [K, N] -> MN-major      ("NN")
//   wgrad     dW += dY^T * X     A = dY stored [K, M] -> MN-major,  B = X stored [K, N] -> MN-major, split-K,
//                                epilogue = add into the bf16 gradient arena (beta = 1), or into an fp32 one (gemm_f32acc_kernel)
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
//                                  release a stage to every CTA that wrote into it, then the epilogue: +bias, bf16, staged through
//                                  shared memory in 64 x 64 sub-tiles and written by TMA (store / bulk bf16 add for split-K partial
//                                  sums); for beta = 1 with one K split the C sub-tile is TMA-loaded into the staging buffer while
//                                  the mainloop runs and added in fp32 (one rounding).  The warpgroup does not wait for the stores:
//                                  it goes on to its next tile and only reuses a staging buffer once its store has read it.
//
// Ping-pong schedule (gemm_pingpong_kernel, chosen by use_pingpong): the forward and dgrad GEMMs with a plain-store epilogue run on a
// second kernel with the same producer / ring / epilogue building blocks, in which each consumer warpgroup owns whole 128 x 128 tiles
// and the two warpgroups take turns on the tensor cores, so one warpgroup's epilogue runs under the other's wgmmas.  The cooperative
// kernel above keeps every other call: wgrad, split-K, beta = 1, FP8, fp32 D, gather mode, multicast and explicit tile requests.
//
// Operand layouts in shared memory (wgmma canonical layouts, 128-byte swizzle):
//   K-major  : rows of 64 k (128 B), 8-row swizzle atoms 1024 B apart (SBO); one TMA box {64 k, rows}
//   MN-major : one TMA box {64 mn, 64 k} gives 64 rows (k) of 128 B = 8 KiB per 64-mn chunk;
//              SBO = 1024 B between 8-k groups, LBO = 8192 B between 64-mn chunks; advancing K by 16 = +2048 B
// In both layouts the 64-row half of the A tile that consumer warpgroup w multiplies starts 8 KiB * w into the stage.
// Output staging: each consumer warpgroup owns two 8 KiB buffers of 64 rows x 64 columns (128 B per row, 128-byte swizzle: the
// 16-byte chunk c of row r sits at chunk c ^ (r % 8)), the box of the output tensor map.
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
constexpr int EPI_BUF_BYTES = 64 * 64 * 2;         // one 64 x 64 bf16 output sub-tile
constexpr int EPI_BYTES = 2 * 2 * EPI_BUF_BYTES;   // 2 consumer warpgroups x 2 buffers
constexpr int SMEM_BYTES = RING_BYTES + EPI_BYTES + 1024 /*align*/ + 256 /*barriers*/;   // 230,656 B of the 232,448 B opt-in
constexpr int THREADS = 384;
constexpr int MAX_PEERS = 8;
constexpr int MN_CHUNK_BYTES = 64 * BK * 2;        // one {64 mn, 64 k} box of an MN-major operand

struct Params {
    CUtensorMap map_a;                 // K-major: box {64 k, 128 / pn rows} of A [M, K]; MN-major: box {64 m, 64 k} of A^T [K, M]
    CUtensorMap map_b;                 // K-major: box {64 k, BN / pm rows} of B [N, K]; MN-major: box {64 n, 64 k} of B^T [K, N]
    CUtensorMap map_b_peer[MAX_PEERS]; // gather mode: B on each rank (peer-mapped), box {64 k, BN rows}
    CUtensorMap map_d;                 // D [M, N] with row stride ldd, box {64 n, 64 m}: its extents clip ragged tiles
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
    int band;                          // tile order: bands of `band` super-tile columns (decode_unit)
    unsigned long long* dbg;          // optional: CTA 0 writes %globaltimer stamps of its phases (tools/gemm_timeline.py)
    const float* inv_scale_a;          // FP8: 1 / s of each operand (device memory, written by the quantiser); unused in bf16
    const float* inv_scale_b;
    int fold_a, fold_b;                // wgrad (A MN-major): map_a / map_b is a folded 3-D map (fold_mn_map), one box per stage
};

// Operand format of an instantiation.  FP8 (both operands K-major, B e4m3): a k-block is 128 one-byte k, so rows stay 128 B and
// the swizzle, stage bytes and ring geometry are those of bf16.  Each k-block accumulates into a fresh fp32 fragment that is then
// added to the tile's sum in registers ("promotion": the FP8 tensor-core accumulator keeps fewer bits than fp32).
constexpr int OP_BF16 = 0, OP_E4M3 = 1, OP_E5M2 = 2;    // A operand e4m3 (forward) / e5m2 (gradients)

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
// Tile order inside a split: bands of `band` super-tile columns; inside a band the columns go fastest, then the rows, then the next
// band.  band = num_sn is plain row-major order.  A narrower band keeps the B blocks of one band L2-resident while every row of A
// passes by (the host picks it only when all of A stays in L2), so B is read from HBM about once instead of once per wave.
// Gather mode uses band = num_sn: every waiter unit (m-block > 0) of a column comes after that column's gatherer unit (m-block 0)
// in every CTA's sequence of units, which its flag protocol needs.
struct Unit {
    int mb, n_blk, kb0, kb1;
};
__device__ __forceinline__ Unit decode_unit(int t, int tiles, int num_smb, int num_sn, int band, int num_k, int kb_per_split, int pm, int pn,
                                            int pi, int pj) {
    Unit u;
    const int s = t / tiles, tile = t - s * tiles;
    const int bi = tile / (band * num_smb), sn0 = bi * band;
    const int width = min(band, num_sn - sn0);
    const int r = tile - sn0 * num_smb;
    const int smb = r / width;
    u.mb = smb * pm + pi;
    u.n_blk = (sn0 + r - smb * width) * pn + pj;
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

template <int BN, int OP>
__device__ __forceinline__ void mma_k32(float (&acc)[BN / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
    static_assert(BN <= 128, "FP8 tiles: the promoted fragment doubles the accumulator registers");
    if constexpr (BN == 128) wgmma_m64n128k32_f8<OP == OP_E5M2>(acc, da, db, scale_d);
    else wgmma_m64n64k32_f8<OP == OP_E5M2>(acc, da, db, scale_d);
}

// |v| = m 2^e with m in [1, 2), for a finite non-zero fp32 (subnormals included: read from the bits, not flushed)
__device__ __forceinline__ void split_exponent(uint32_t u, int& e, float& m) {
    u &= 0x7FFFFFFFu;
    uint32_t frac = u & 0x7FFFFFu;
    if ((u >> 23) == 0) {
        const int lead = 31 - __clz(frac);
        e = -149 + lead;
        frac = (frac << (23 - lead)) & 0x7FFFFFu;
    } else {
        e = (int)(u >> 23) - 127;
    }
    m = __uint_as_float(0x3F800000u | frac);
}

// FP8 output scale 1 / (s_a s_b) = inv_a * inv_b, applied as (acc * pre) * post.  The quantiser emits inverses from 2^-127 (a subnormal,
// which this fast-math build would read as 0) to 2^120, so their product spans 2^-254 .. 2^240.  post is that product at its exponent
// clamped to the normal range, pre = 2^(the rest): pre = 1 whenever the product is a normal fp32 (the epilogue is then one fma per
// element), otherwise pre rescales the fp32 sum first, exactly (a power of two; whenever the result is a normal number, so is acc * pre).
// Launch-uniform: every thread derives the same pair from the same two words.
__device__ __forceinline__ void fp8_out_scale(float inv_a, float inv_b, float& pre, float& post) {
    const uint32_t ua = __float_as_uint(inv_a), ub = __float_as_uint(inv_b);
    pre = 1.f;
    if ((ua & 0x7FFFFFFFu) == 0 || (ub & 0x7FFFFFFFu) == 0 || (ua & 0x7F800000u) == 0x7F800000u || (ub & 0x7F800000u) == 0x7F800000u) {
        post = inv_a * inv_b;                              // 0, Inf or NaN (a NaN / Inf tensor's scale): propagate
        return;
    }
    int ea, eb;
    float ma, mb;
    split_exponent(ua, ea, ma);
    split_exponent(ub, eb, mb);
    float m = ma * mb;                                     // [1, 4); exact for powers of two
    int e = ea + eb;
    if (m >= 2.f) { m *= 0.5f; ++e; }
    const int ec = min(max(e, -126), 127), d = e - ec;    // d in [-172, 127]
    post = __uint_as_float(((ua ^ ub) & 0x80000000u) | (__float_as_uint(m) + ((uint32_t)ec << 23)));
    pre = d < -126 ? 0.f : __uint_as_float((uint32_t)(d + 127) << 23);   // below 2^-126 the output is far below bf16's normal range
}

__device__ __forceinline__ float2 ld_shared_f32x2(uint32_t addr) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void st_shared_f32x2(uint32_t addr, float a, float b) {
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}

// F32D: D is fp32 (an fp32 gradient accumulator under bf16 weights).  The epilogue then stages 64 x 32 fp32 sub-tiles - a 128-byte
// swizzled row holds 32 floats - through the same 8 KiB buffers, and the TMA unit reads C / writes and reduce-adds D in fp32: with one
// K split D += tile is exact up to the one fp32 add per element, with split-K each split's partial is added in fp32.
template <int BN, int A_MN, int B_MN, int OP, bool F32D = false>
__device__ __forceinline__ void gemm_body(const Params& P) {
    static_assert(OP == OP_BF16 || (A_MN == 0 && B_MN == 0), "FP8 wgmma has no transpose: both operands K-major");
    constexpr int BKE = OP ? 2 * BK : BK;                  // elements per k-block (128 bytes per row in both formats)
    extern __shared__ uint8_t smem_raw[];
    if (threadIdx.x == 0) stamp(P, 0);
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);   // SWIZZLE_128B needs 1024 B alignment
    uint8_t* epi_smem = smem + RING_BYTES;                    // [2 x 2] output staging buffers (1024 B aligned)
    uint64_t* full_bar = (uint64_t*)(epi_smem + EPI_BYTES);   // [MAX_STAGES]  TMA bytes landed
    uint64_t* empty_bar = full_bar + MAX_STAGES;              // [MAX_STAGES]  stage reusable (every consumer that reads it released it)
    uint64_t* c_bar = empty_bar + MAX_STAGES;                 // [2 x 2]       C sub-tile landed in a staging buffer (beta = 1)

    constexpr int B_BYTES = BN * BK * 2;
    const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
    const int n_stages = P.stages, stage_bytes = P.stage_bytes;
    const int pm = P.pm, pn = P.pn, cl_size = pm * pn;
    const uint32_t cl_rank = cl_size > 1 ? cluster_ctarank() : 0u;
    const int pi = (int)cl_rank / pn, pj = (int)cl_rank - pi * pn;
    const int unit0 = blockIdx.x / cl_size, unit_stride = gridDim.x / cl_size;
    const int num_n = (P.N + BN - 1) / BN, num_k = (P.K + BKE - 1) / BKE, num_mb = (P.M + BM - 1) / BM;
    const int num_sn = (num_n + pn - 1) / pn, num_smb = (num_mb + pm - 1) / pm;
    const int band = P.band;
    const int tiles = num_smb * num_sn;
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
        asm volatile("prefetch.tensormap [%0];" ::"l"(&P.map_d) : "memory");
        for (int s = 0; s < n_stages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 2u * (uint32_t)(pm + pn - 1));   // both consumer warpgroups of every CTA that reads what I (multi)cast
        }
        for (int b = 0; b < 4; ++b) mbar_init(&c_bar[b], 1);
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
                const Unit u = decode_unit(t, tiles, num_smb, num_sn, band, num_k, kbs, pm, pn, pi, pj);
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
                    if (A_MN && P.fold_a) {
                        // one box of nach 64-m chunks ({64 m, 64 k, nach} of the folded map): the chunks land 8 KiB apart, as below
                        if (mc_a) tma_load_3d_mc(&P.map_a, &full_bar[stage], sa + a_ch0 * MN_CHUNK_BYTES, 0, kb * BKE, m0 / 64 + a_ch0, mask_a);
                        else tma_load_3d(&P.map_a, &full_bar[stage], sa, 0, kb * BKE, m0 / 64);
                    } else if (A_MN) {
                        for (int c = a_ch0; c < a_ch0 + nach; ++c) {
                            if (mc_a) tma_load_2d_mc(&P.map_a, &full_bar[stage], sa + c * MN_CHUNK_BYTES, m0 + c * 64, kb * BKE, mask_a);
                            else tma_load_2d(&P.map_a, &full_bar[stage], sa + c * MN_CHUNK_BYTES, m0 + c * 64, kb * BKE);
                        }
                    } else {
                        if (mc_a) tma_load_2d_mc(&P.map_a, &full_bar[stage], sa + a_off * 128, kb * BKE, m0 + a_off, mask_a);
                        else tma_load_2d(&P.map_a, &full_bar[stage], sa, kb * BKE, m0);
                    }
                    if (A_MN && B_MN && P.fold_b) {
                        if (mc_b) tma_load_3d_mc(bmap, &full_bar[stage], sb + b_ch0 * MN_CHUNK_BYTES, 0, kb * BKE, n0 / 64 + b_ch0, mask_b);
                        else tma_load_3d(bmap, &full_bar[stage], sb, 0, kb * BKE, n0 / 64);
                    } else if (B_MN) {
                        for (int c = b_ch0; c < b_ch0 + nbch; ++c) {
                            if (mc_b) tma_load_2d_mc(bmap, &full_bar[stage], sb + c * MN_CHUNK_BYTES, n0 + c * 64, kb * BKE, mask_b);
                            else tma_load_2d(bmap, &full_bar[stage], sb + c * MN_CHUNK_BYTES, n0 + c * 64, kb * BKE);
                        }
                    } else {
                        if (mc_b) tma_load_2d_mc(bmap, &full_bar[stage], sb + b_off * 128, kb * BKE, n0 + b_off, mask_b);
                        else tma_load_2d(bmap, &full_bar[stage], sb, kb * BKE, n0);
                    }
                    if (gatherer) {
                        // write the pulled tile through to the local copy of W, then publish it (both halves of the 256-row tile)
                        mbar_wait(&full_bar[stage], phase);
                        fence_async_smem();
                        tma_store_2d(&P.map_b, sb, kb * BKE, n0);
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
        // epilogue: BN / 64 sub-tiles of 64 x 64 through this warpgroup's two staging buffers (sub-tile s uses buffer s % 2); thread 0
        // of the warpgroup issues the TMA traffic.  Before a buffer is rewritten, the store that last read it must be done reading:
        // the bulk group two commits back (one back with a single sub-tile per tile).
        constexpr int SUBW = F32D ? 32 : 64;               // output columns per staged sub-tile (128 B rows)
        constexpr int NSUB = BN / SUBW;
        constexpr int NPRE = NSUB < 2 ? NSUB : 2;          // C sub-tiles prefetched during the mainloop (beta = 1, one split)
        uint8_t* epi = epi_smem + cw * 2 * EPI_BUF_BYTES;
        uint64_t* cbar = c_bar + cw * 2;
        const bool load_c = P.reduce && !P.atomic;
        const int bar_id = 1 + cw;                         // named barrier of this warpgroup (0 is __syncthreads)
        uint32_t c_phase = 0;                              // bit b: parity of cbar[b]
        auto wait_buffer_free = [&]() {
            if (NSUB == 1) bulk_wait_read<0>();
            else bulk_wait_read<1>();
        };
        auto load_c_sub = [&](const Unit& u, int s) {
            mbar_expect_tx(&cbar[s & 1], (uint32_t)EPI_BUF_BYTES);
            tma_load_2d(&P.map_d, &cbar[s & 1], epi + (s & 1) * EPI_BUF_BYTES, u.n_blk * BN + s * SUBW, u.mb * BM + cw * 64);
        };
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        float part[OP ? BN / 2 : 1];                       // FP8: the current k-block's fragment
        float out_scale = 1.f, pre_scale = 1.f;
        if constexpr (OP != OP_BF16) fp8_out_scale(P.inv_scale_a[0], P.inv_scale_b[0], pre_scale, out_scale);
        int stage = 0;
        uint32_t phase = 0;
        for (int t = unit0; t < num_units; t += unit_stride) {
            const Unit u = decode_unit(t, tiles, num_smb, num_sn, band, num_k, kbs, pm, pn, pi, pj);
            int prev = -1;
            if constexpr (OP != OP_BF16) {
#pragma unroll
                for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
            }
            for (int kb = u.kb0; kb < u.kb1; ++kb) {
                mbar_wait(&full_bar[stage], phase);
                if (cw == 0 && tid == 0 && t == unit0 && kb == u.kb0) stamp(P, 4);
                const uint32_t a_addr = smem_u32(smem + stage * stage_bytes) + (uint32_t)(cw * 8192);
                const uint32_t b_addr = smem_u32(smem + stage * stage_bytes + A_BYTES);
                wgmma_fence();
                if constexpr (OP != OP_BF16) {
#pragma unroll
                    for (int k = 0; k < BKE / 32; ++k) {
                        const uint64_t da = make_smem_desc(a_addr + k * 32, 1, 1024 >> 4);
                        const uint64_t db = make_smem_desc(b_addr + k * 32, 1, 1024 >> 4);
                        mma_k32<BN, OP>(part, da, db, (uint32_t)(k != 0));
                    }
                } else {
#pragma unroll
                    for (int k = 0; k < BK / 16; ++k) {
                        const uint64_t da = make_smem_desc(a_addr + k * a_kstep, a_lbo, a_sbo);
                        const uint64_t db = make_smem_desc(b_addr + k * b_kstep, b_lbo, b_sbo);
                        mma_k16<BN, A_MN, B_MN>(acc, da, db, (uint32_t)((kb > u.kb0) | (k != 0)));
                    }
                }
                wgmma_commit();
                if (load_c && kb == u.kb0 && tid == 0) {
                    // beta = 1: fetch the first C sub-tiles now, their latency hides behind this tile's mainloop
                    bulk_wait_read<0>();
                    for (int s = 0; s < NPRE; ++s) load_c_sub(u, s);
                }
                if constexpr (OP != OP_BF16) {
                    // promotion: the k-block's fragment is complete, add it to the tile's fp32 sum (the other consumer
                    // warpgroup's wgmmas keep the tensor cores busy meanwhile)
                    wgmma_wait<0>();
                    reg_fence(part);
                    release(stage);
#pragma unroll
                    for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
                } else {
                    if (prev >= 0) {
                        wgmma_wait<1>();                   // the previous stage's wgmmas have retired: hand it back
                        release(prev);
                    }
                    prev = stage;
                }
                if (++stage == n_stages) { stage = 0; phase ^= 1; }
            }
            if constexpr (OP == OP_BF16) {
                wgmma_wait<0>();
                reg_fence(acc);
                release(prev);
            } else if (pre_scale != 1.f) {                 // an output scale outside fp32's normal range (fp8_out_scale)
#pragma unroll
                for (int i = 0; i < BN / 2; ++i) acc[i] *= pre_scale;
            }
            // ---------------- epilogue: fragment (row 16 warp + lane/4 (+8), columns 8 j + 2 (lane % 4) (+1)) -> staging -> TMA
            const int m0 = u.mb * BM + cw * 64;
            // my rows r = 16 warp + lane / 4 (+8) of the 64-row half; r % 8 = lane / 4 sets the swizzle of both.  My two columns of
            // a fragment group are 4 bf16 bytes at 4 (lane % 4) of its 16-byte chunk, or 8 fp32 bytes at 8 (lane % 2) of chunk lane % 4 / 2
            // of its two chunks.
            const uint32_t row_addr = smem_u32(epi) + (uint32_t)((warp * 16 + (lane >> 2)) * 128 + (F32D ? 8 * (lane & 1) : 4 * (lane & 3)));
            const int colb = u.n_blk * BN + 2 * (lane & 3);
            const bool bias_on = P.bias != nullptr && u.kb0 == 0;
#pragma unroll
            for (int s = 0; s < NSUB; ++s) {
                uint8_t* buf = epi + (s & 1) * EPI_BUF_BYTES;
                const uint32_t buf_addr = row_addr + (uint32_t)((s & 1) * EPI_BUF_BYTES);
                if (load_c) {
                    if (s >= NPRE && tid == 0) {
                        wait_buffer_free();
                        load_c_sub(u, s);
                    }
                    mbar_wait(&cbar[s & 1], (c_phase >> (s & 1)) & 1u);
                    c_phase ^= 1u << (s & 1);
                } else {
                    if (tid == 0) wait_buffer_free();
                    named_barrier(bar_id, 128);
                }
#pragma unroll
                for (int jj = 0; jj < SUBW / 8; ++jj) {
                    const int j = s * (SUBW / 8) + jj;
                    const int col = colb + 8 * j;
                    float b0 = 0.f, b1 = 0.f;
                    if (bias_on && col < P.N) {                    // N % 8 == 0: col < N implies col + 1 < N
                        const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(P.bias + col));
                        b0 = f.x; b1 = f.y;
                    }
                    const int chunk = F32D ? 2 * jj + ((lane & 3) >> 1) : jj;
                    const uint32_t chunk_addr = buf_addr + (uint32_t)((chunk ^ (lane >> 2)) << 4);
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const uint32_t dst = chunk_addr + h * 8 * 128;
                        float v0, v1;
                        if constexpr (OP != OP_BF16) {
                            v0 = acc[4 * j + 2 * h] * out_scale + b0;
                            v1 = acc[4 * j + 2 * h + 1] * out_scale + b1;
                        } else {
                            v0 = acc[4 * j + 2 * h] + b0;
                            v1 = acc[4 * j + 2 * h + 1] + b1;
                        }
                        if constexpr (F32D) {
                            if (load_c) {
                                const float2 c = ld_shared_f32x2(dst);
                                v0 += c.x; v1 += c.y;
                            }
                            st_shared_f32x2(dst, v0, v1);
                        } else {
                            if (load_c) {
                                // beta = 1 with a single K split: exact fp32 accumulate (one rounding), nobody else touches this tile
                                const uint32_t cv = ld_shared_u32(dst);
                                const float2 c = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&cv));
                                v0 += c.x; v1 += c.y;
                            }
                            st_shared_u32(dst, pack_bf16x2(v0, v1));
                        }
                    }
                }
                fence_async_smem();                        // my st.shared -> visible to the TMA engine
                named_barrier(bar_id, 128);
                if (tid == 0) {
                    // ragged rows / columns fall outside map_d's extents and are dropped by the TMA unit
                    if (P.atomic) tma_reduce_add_2d(&P.map_d, buf, u.n_blk * BN + s * SUBW, m0);
                    else tma_store_2d(&P.map_d, buf, u.n_blk * BN + s * SUBW, m0);
                    bulk_commit();
                }
            }
        }
        if (tid == 0) bulk_wait<0>();                      // the stores have landed before this CTA retires
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

template <int BN, int A_MN, int B_MN>
__global__ void __launch_bounds__(THREADS, 1) gemm_kernel(const __grid_constant__ Params P) {
    gemm_body<BN, A_MN, B_MN, OP_BF16>(P);
}

// FP8 (OP = OP_E4M3 / OP_E5M2): D = A * B^T / (s_a s_b) (+ bias), both operands K-major one-byte [rows, K]; BN 64 or 128
template <int BN, int OP>
__global__ void __launch_bounds__(THREADS, 1) gemm_fp8_kernel(const __grid_constant__ Params P) {
    gemm_body<BN, 0, 0, OP>(P);
}

// Accumulating GEMMs into an fp32 D (F32D): the wgrad layout (both operands MN-major) at every tile width, and the FP8 GEMM
template <int BN>
__global__ void __launch_bounds__(THREADS, 1) gemm_f32acc_kernel(const __grid_constant__ Params P) {
    gemm_body<BN, 1, 1, OP_BF16, true>(P);
}
template <int BN, int OP>
__global__ void __launch_bounds__(THREADS, 1) gemm_fp8_f32acc_kernel(const __grid_constant__ Params P) {
    gemm_body<BN, 0, 0, OP, true>(P);
}

// PING-PONG schedule for the bf16 GEMMs whose epilogue is a plain store: the forward (B K-major) and the dgrad (B MN-major), one K
// split, no gather, no cluster.  A unit is a whole 128 x 128 tile and belongs to ONE consumer warpgroup (two m64n128k16 wgmmas per
// k16 step, 2 x 64 fp32 accumulators per thread); the warpgroups take alternate units of the CTA's persistent sequence (the tile order
// of decode_unit).  The producer walks that same sequence into one ring, so the i-th unit of the CTA starts at ring position
// i * num_k.  An order barrier passes the tensor cores from unit i to unit i + 1: a warpgroup waits for its turn, issues its mainloop,
// hands the turn over as soon as its last wgmma group is issued, and then runs its epilogue (+bias, bf16, 64 x 64 staging, TMA stores)
// while the other warpgroup's wgmmas run.  The turn barrier of warpgroup w completes once per unit of the other warpgroup; unit i
// (i >= 1) waits for completion (i - 1) / 2 of turn[i % 2], i.e. parity ((i - 1) >> 1) & 1.  Every stage has one reader, so the
// empty barriers count one arrival.  tests/test_gemm_pingpong_protocol.py model-checks this protocol.
template <int B_MN>
__global__ void __launch_bounds__(THREADS, 1) gemm_pingpong_kernel(const __grid_constant__ Params P) {
    constexpr int BN = 128;
    constexpr int B_BYTES = BN * BK * 2;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint8_t* epi_smem = smem + RING_BYTES;
    uint64_t* full_bar = (uint64_t*)(epi_smem + EPI_BYTES);
    uint64_t* empty_bar = full_bar + MAX_STAGES;
    uint64_t* turn_bar = empty_bar + MAX_STAGES;              // [2]  turn[w]: warpgroup w may issue its next mainloop
    const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
    const int n_stages = P.stages, stage_bytes = P.stage_bytes;
    const int num_n = (P.N + BN - 1) / BN, num_k = (P.K + BK - 1) / BK, num_mb = (P.M + BM - 1) / BM;
    const int tiles = num_mb * num_n;

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&P.map_a) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&P.map_b) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&P.map_d) : "memory");
        for (int s = 0; s < n_stages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 1);
        }
        mbar_init(&turn_bar[0], 1);
        mbar_init(&turn_bar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

    if (wg == 0) {
        // ============================ TMA PRODUCER: every k-block of every unit of the CTA, in sequence order ============================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (tid == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
                const Unit u = decode_unit(t, tiles, num_mb, num_n, P.band, num_k, num_k, 1, 1, 0, 0);
                const int m0 = u.mb * BM, n0 = u.n_blk * BN;
                for (int kb = 0; kb < num_k; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    uint8_t* sa = smem + stage * stage_bytes;
                    uint8_t* sb = sa + A_BYTES;
                    mbar_expect_tx(&full_bar[stage], (uint32_t)(A_BYTES + B_BYTES));
                    tma_load_2d(&P.map_a, &full_bar[stage], sa, kb * BK, m0);
                    if (B_MN) {
                        tma_load_2d(&P.map_b, &full_bar[stage], sb, n0, kb * BK);
                        tma_load_2d(&P.map_b, &full_bar[stage], sb + MN_CHUNK_BYTES, n0 + 64, kb * BK);
                    } else {
                        tma_load_2d(&P.map_b, &full_bar[stage], sb, kb * BK, n0);
                    }
                    if (++stage == n_stages) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ============================ CONSUMERS: warpgroup cw computes units cw, cw + 2, ... of the CTA's sequence ============================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        const int cw = wg - 1;
        const int warp = tid >> 5, lane = tid & 31;
        constexpr uint32_t b_lbo = B_MN ? (MN_CHUNK_BYTES >> 4) : 1, b_sbo = 1024 >> 4, b_kstep = B_MN ? 2048 : 32;
        uint8_t* epi = epi_smem + cw * 2 * EPI_BUF_BYTES;
        const int bar_id = 1 + cw;
        float acc0[BN / 2], acc1[BN / 2];                  // rows [0, 64) and [64, 128) of the unit
        for (int i = cw;; i += 2) {                        // i: the unit's index in the CTA's sequence
            const int t = blockIdx.x + i * gridDim.x;
            if (t >= tiles) break;
            const Unit u = decode_unit(t, tiles, num_mb, num_n, P.band, num_k, num_k, 1, 1, 0, 0);
            const int pos = i * num_k;                     // the unit's first ring position
            int stage = pos % n_stages;
            uint32_t phase = (uint32_t)(pos / n_stages) & 1u;
            if (i > 0) mbar_wait(&turn_bar[cw], (uint32_t)((i - 1) >> 1) & 1u);
            int prev = -1;
            for (int kb = 0; kb < num_k; ++kb) {
                mbar_wait(&full_bar[stage], phase);
                const uint32_t a_addr = smem_u32(smem + stage * stage_bytes);
                const uint32_t b_addr = a_addr + A_BYTES;
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / 16; ++k) {
                    const uint64_t db = make_smem_desc(b_addr + k * b_kstep, b_lbo, b_sbo);
                    const uint32_t sd = (uint32_t)((kb > 0) | (k != 0));
                    wgmma_m64n128k16<0, B_MN>(acc0, make_smem_desc(a_addr + k * 32, 1, 1024 >> 4), db, sd);
                    wgmma_m64n128k16<0, B_MN>(acc1, make_smem_desc(a_addr + 8192 + k * 32, 1, 1024 >> 4), db, sd);
                }
                wgmma_commit();
                if (prev >= 0) {
                    wgmma_wait<1>();
                    if (tid == 0) mbar_arrive(&empty_bar[prev]);
                }
                prev = stage;
                if (++stage == n_stages) { stage = 0; phase ^= 1; }
            }
            if (tid == 0) mbar_arrive(&turn_bar[cw ^ 1]);  // every wgmma of this unit is issued: the other warpgroup's turn
            wgmma_wait<0>();
            reg_fence(acc0);
            reg_fence(acc1);
            if (tid == 0) mbar_arrive(&empty_bar[prev]);
            // ---------------- epilogue: 4 sub-tiles of 64 x 64 (row half h, column half s) through the two staging buffers, as in gemm_body
            const uint32_t row_addr = smem_u32(epi) + (uint32_t)((warp * 16 + (lane >> 2)) * 128 + 4 * (lane & 3));
            const int colb = u.n_blk * BN + 2 * (lane & 3);
            const bool bias_on = P.bias != nullptr;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int h = q >> 1, s = q & 1;
                float(&acc)[BN / 2] = h ? acc1 : acc0;
                uint8_t* buf = epi + (q & 1) * EPI_BUF_BYTES;
                const uint32_t buf_addr = row_addr + (uint32_t)((q & 1) * EPI_BUF_BYTES);
                if (tid == 0) bulk_wait_read<1>();         // the store that last read this buffer (two commits back) is done reading
                named_barrier(bar_id, 128);
#pragma unroll
                for (int jj = 0; jj < 8; ++jj) {
                    const int j = s * 8 + jj;
                    const int col = colb + 8 * j;
                    uint32_t braw = 0;                     // bf16 pair (the register budget is tight with 128 accumulators)
                    if (bias_on && col < P.N) braw = *reinterpret_cast<const uint32_t*>(P.bias + col);
                    const float2 bf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&braw));
                    const float b0 = bf.x, b1 = bf.y;
                    const uint32_t chunk_addr = buf_addr + (uint32_t)((jj ^ (lane >> 2)) << 4);
#pragma unroll
                    for (int r = 0; r < 2; ++r)
                        st_shared_u32(chunk_addr + r * 8 * 128, pack_bf16x2(acc[4 * j + 2 * r] + b0, acc[4 * j + 2 * r + 1] + b1));
                }
                fence_async_smem();
                named_barrier(bar_id, 128);
                if (tid == 0) {
                    tma_store_2d(&P.map_d, buf, u.n_blk * BN + s * 64, u.mb * BM + h * 64);
                    bulk_commit();
                }
            }
        }
        if (tid == 0) bulk_wait<0>();
    }
    __syncthreads();
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
    uint32_t fold;                     // 0: 2-D map; else a folded 3-D map (fold_mn_map) with boxes of `fold` chunks
    bool operator==(const MapKey& o) const {
        return base == o.base && inner == o.inner && outer == o.outer && ld == o.ld && box_inner == o.box_inner && box_outer == o.box_outer &&
               elem_bytes == o.elem_bytes && fold == o.fold;
    }
};
struct MapKeyHash {
    size_t operator()(const MapKey& k) const {
        size_t h = (size_t)k.base;
        auto mix = [&h](uint64_t v) { h ^= v + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2); };
        mix(k.inner); mix(k.outer); mix(k.ld); mix(((uint64_t)k.box_inner << 32) | k.box_outer); mix((uint64_t)k.elem_bytes | ((uint64_t)k.fold << 32));
        return h;
    }
};
static std::mutex g_map_mu;
static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_maps;
static long long g_map_encodes = 0;

static int encode_cached(CUtensorMap* m, const MapKey& key) {
    {
        std::lock_guard<std::mutex> g(g_map_mu);
        auto it = g_maps.find(key);
        if (it != g_maps.end()) { *m = it->second; return 0; }
    }
    EncodeFn enc = get_encode();
    if (!enc) return -2;
    const uint64_t eb = (uint64_t)key.elem_bytes;
    // 2-D: {inner, outer}, row stride ld.  Folded: {64, outer, inner / 64} with strides {ld, 64} elements - the 64-element chunks of a
    // row become the third dimension, so one box {64, box_outer, fold} gathers `fold` adjacent chunks of box_outer rows.
    const cuuint32_t rank = key.fold ? 3 : 2;
    cuuint64_t dims[3] = {key.inner, key.outer, 1};
    cuuint64_t strides[2] = {key.ld * eb, 0};
    cuuint32_t box[3] = {key.box_inner, key.box_outer, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    if (key.fold) {
        dims[0] = 64; dims[2] = key.inner / 64;
        strides[1] = 64 * eb;
        box[2] = key.fold;
    }
    const CUtensorMapDataType dt = key.elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                   : key.elem_bytes == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    CUresult r = enc(m, dt, rank, const_cast<void*>(key.base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r == CUDA_ERROR_INVALID_CONTEXT && bind_primary_context()) {
        r = enc(m, dt, rank, const_cast<void*>(key.base), dims, strides, box, estr,
                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    }
    if (r != CUDA_SUCCESS) return -3;
    std::lock_guard<std::mutex> g(g_map_mu);
    if (g_maps.size() > 8192) g_maps.clear();      // unbounded address churn (eager mode without the caching allocator): start over
    g_maps.emplace(key, *m);
    ++g_map_encodes;
    return 0;
}

// row-major matrix (fp8: elem_bytes 1, bf16: 2, fp32: 4) with `outer` rows of `inner` contiguous elements (row stride `ld` elements),
// box {box_inner, box_outer}, 128-byte swizzle (box_inner * elem_bytes = 128 B)
int make_map_typed(CUtensorMap* m, const void* base, uint64_t inner, uint64_t outer, uint64_t ld, uint32_t box_inner, uint32_t box_outer,
                   int elem_bytes) {
    return encode_cached(m, MapKey{base, inner, outer, ld, box_inner, box_outer, elem_bytes, 0});
}
// An MN-major bf16 operand stored [K, rows] (rows % 64 == 0), folded so that one TMA box {64 mn, 64 k, chunks} brings `chunks`
// adjacent 64-mn chunks of a k-block: they land 8 KiB apart, the layout of one 2-D box {64 mn, 64 k} per chunk.  The wgrad GEMMs load
// each operand of a stage with one box instead of one per chunk: with a box per chunk their k-block rate fell with the number of boxes
// per stage (on an H100, 128-wide tiles with two, three and four boxes: about 440, 570 and 770 ns per k-block), and with the folded
// boxes the Llama-125M qkv wgrad takes 69 us instead of 98.
static int fold_mn_map(CUtensorMap* m, const void* base, uint64_t rows, uint64_t K, uint64_t ld, uint32_t chunks) {
    return encode_cached(m, MapKey{base, rows, K, ld, 64, BK, 2, chunks});
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
// FP8 instantiations: BN in {64, 128} x A format (e4m3 forward, e5m2 gradients)
static KernelFn fp8_kernel_for(int bn, int op) {
    if (bn == 128) return op == OP_E5M2 ? gemm_fp8_kernel<128, OP_E5M2> : gemm_fp8_kernel<128, OP_E4M3>;
    return op == OP_E5M2 ? gemm_fp8_kernel<64, OP_E5M2> : gemm_fp8_kernel<64, OP_E4M3>;
}

static KernelFn f32acc_kernel_for(int bn) {
    return bn == 256 ? gemm_f32acc_kernel<256> : bn == 128 ? gemm_f32acc_kernel<128> : gemm_f32acc_kernel<64>;
}
static KernelFn fp8_f32acc_kernel_for(int bn, int op) {
    if (bn == 128) return op == OP_E5M2 ? gemm_fp8_f32acc_kernel<128, OP_E5M2> : gemm_fp8_f32acc_kernel<128, OP_E4M3>;
    return op == OP_E5M2 ? gemm_fp8_f32acc_kernel<64, OP_E5M2> : gemm_fp8_f32acc_kernel<64, OP_E4M3>;
}

static KernelFn pingpong_kernel_for(int b_mn) { return b_mn ? gemm_pingpong_kernel<1> : gemm_pingpong_kernel<0>; }

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
        for (int bn : {64, 128})
            for (int op : {OP_E4M3, OP_E5M2})
                if (cudaFuncSetAttribute(fp8_kernel_for(bn, op), cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES) != cudaSuccess ||
                    cudaFuncSetAttribute(fp8_f32acc_kernel_for(bn, op), cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES) != cudaSuccess)
                    rc = -4;
        for (int bn : {64, 128, 256})
            if (cudaFuncSetAttribute(f32acc_kernel_for(bn), cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES) != cudaSuccess) rc = -4;
        for (int b_mn = 0; b_mn < 2; ++b_mn)
            if (cudaFuncSetAttribute(pingpong_kernel_for(b_mn), cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES) != cudaSuccess) rc = -4;
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
// assumed); `epi` charges the epilogue as if it were not overlapped.  On the cooperative kernel only the TMA stores drain under the
// next tile's mainloop; the ping-pong kernel (use_pingpong) hides most of the epilogue under the other warpgroup's wgmmas, so for
// the calls it runs this over-estimates the epilogue.  The picks are kept as they are: use_pingpong starts from them.
// Split-K needs an adding epilogue: accumulating GEMMs (wgrad), or a zero-filled output.  FP8 passes K / 2: its 128-deep k-block moves the bytes of a bf16 one and takes the same tensor-core
// time (twice the rate), and caps the tile at bn_max = 128.
static Config choose_config(int M, int N, int K, int a_mn, int b_mn, int reduce, int sms, int bn_req, int splits_req, int pm_req, int pn_req,
                            int bn_max = BN_MAX) {
    (void)a_mn; (void)b_mn;
    const int num_k = (K + BK - 1) / BK;
    double best = 1e30;
    Config bc{bn_max, 1, 1, 1};
    const int cands[3] = {256, 128, 64};
    const int num_mb = (M + BM - 1) / BM;
    for (int ci = 0; ci < 3; ++ci) {
        const int bn = cands[ci];
        if (bn_req > 0 && bn != bn_req) continue;
        if (bn > bn_max) continue;
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

// Schedule of a call: the ping-pong kernel (gemm_pingpong_kernel) for the non-accumulating bf16 GEMMs with a K-major A - the forward
// and the dgrad - when the call requests nothing (tile width, K splits, multicast) and the cost model picks one K split and either
// 128-wide tiles, or 256-wide tiles with K <= 1024; everything else keeps the cooperative kernel and choose_config's pick.
//   * 64-wide picks (N <= 64, or too few tiles to fill the GPU): a 128 x 128 unit would compute wasted columns or leave SMs idle.
//   * 256-wide picks: a 128 x 128 unit pulls 1.5x the operand bytes per FLOP of a 128 x 256 tile, which only pays while the epilogue is
//     a large share of the tile (27-30 % at K = 768 by the cost model, 10-15 % at K = 2048-4096).  Measured on an H100 SXM (700 W):
//     the Llama-125M K = 768 forward / dgrad calls with 256-wide picks run 8-20 % faster on ping-pong, the Llama-3.2-1B ones at K >= 2048
//     from 6 % faster to 1.65x the time (the LM-head dgrad at K = 128256).
static bool use_pingpong(const Config& c, int K, int a_mn, int accumulate, int op, int f32d, int gather, int bn_req, int splits_req,
                         int pm_req, int pn_req) {
    return op == OP_BF16 && !f32d && !gather && !accumulate && !a_mn && bn_req <= 0 && splits_req <= 0 && pm_req <= 0 && pn_req <= 0 &&
           c.splits == 1 && c.pm == 1 && c.pn == 1 && (c.bn == 128 || (c.bn == 256 && K <= 16 * BK));
}

// Tile order (decode_unit): bands of G super-tile columns.  When all of A [M, K] fits in a third of L2 it stays resident while
// the tiles of a band go by, and G is as wide as keeps the band's B blocks (bn_cols x K each) within an eighth of L2: each B block
// is then read from HBM once.  Otherwise (or when all of B fits anyway) row-major order, G = num_sn.  For the Llama-125M LM-head
// forward (A = 8192 x 768, B = 50304 x 768, 256-row blocks) on an H100 (50 MB L2) that is G = 16 instead of one 77 MB pass over
// the weight per 132-tile wave.
static int tile_band(int M, int K, int bn_cols, int num_sn) {
    static int l2_cache[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) { cudaGetLastError(); return num_sn; }
    if (l2_cache[dev] == 0) {
        int l2 = 0;
        if (cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, dev) != cudaSuccess || l2 <= 0) { cudaGetLastError(); l2 = -1; }
        l2_cache[dev] = l2;
    }
    const double l2 = (double)l2_cache[dev];
    if (l2 <= 0 || (double)M * K * 2.0 > l2 / 3.0) return num_sn;
    const long long g = (long long)(l2 / 8.0 / ((double)bn_cols * K * 2.0));
    return (int)(g < 1 ? 1 : (g > num_sn ? num_sn : g));
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
                  cudaStream_t st, int op = OP_BF16, const float* inv_a = nullptr, const float* inv_b = nullptr, int f32d = 0) {
    if (M <= 0 || N <= 0 || K <= 0) return -1;
    // fp32 D: accumulate only, no bias, and (bf16) the wgrad operand layout - the instantiations that exist
    if (f32d && (!accumulate || bias || (ga && ga->n_peers > 0) || (!op && !(a_mn && b_mn)))) return -1;
    if ((lda % 8) || (ldb % 8) || (ldd % 8) || (N % 8)) return -1;
    const int eb = op ? 1 : 2, bke = op ? 2 * BK : BK;                     // operand bytes per element, elements per k-block
    if (op && (a_mn || b_mn || (lda % 16) || (ldb % 16) || (K % 16) || bn_req > 128 || !inv_a || !inv_b || (ga && ga->n_peers > 0))) return -1;
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
        cfgc = choose_config(M, N, op ? (K + 1) / 2 : K, a_mn, b_mn, accumulate, sms, bn_req, splits_req, pm_req, pn_req, op ? 128 : BN_MAX);
    }
    const bool pingpong = use_pingpong(cfgc, K, a_mn, accumulate, op, f32d, gather, bn_req, splits_req, pm_req, pn_req);
    const int bn = pingpong ? 128 : cfgc.bn, pm = cfgc.pm, pn = cfgc.pn;   // ping-pong units are 128 x 128
    int splits = cfgc.splits;
    if ((bn_req > 0 && bn != bn_req) || (pm_req > 0 && pm != pm_req) || (pn_req > 0 && pn != pn_req)) return -1;   // request not realisable
    if (b_mn ? ((bn / 64) % pm != 0) : ((bn / pm) % 8 != 0)) return -1;
    if (a_mn && (BM / 64) % pn != 0) return -1;
    Params P;
    // wgrad layout (A MN-major): one folded box per MN-major operand and stage where its extent is whole 64-element chunks
    P.fold_a = a_mn && M % 64 == 0;
    P.fold_b = a_mn && b_mn && N % 64 == 0;
    if (P.fold_a) rc = fold_mn_map(&P.map_a, a, (uint64_t)M, (uint64_t)K, (uint64_t)lda, (uint32_t)((BM / 64) / pn));
    else if (a_mn) rc = make_map(&P.map_a, a, (uint64_t)M, (uint64_t)K, (uint64_t)lda, 64, BK);
    else rc = make_map_typed(&P.map_a, a, (uint64_t)K, (uint64_t)M, (uint64_t)lda, bke, (uint32_t)(BM / pn), eb);
    if (rc) return rc;
    if (P.fold_b) rc = fold_mn_map(&P.map_b, b, (uint64_t)N, (uint64_t)K, (uint64_t)ldb, (uint32_t)((bn / 64) / pm));
    else if (b_mn) rc = make_map(&P.map_b, b, (uint64_t)N, (uint64_t)K, (uint64_t)ldb, 64, BK);
    else rc = make_map_typed(&P.map_b, b, (uint64_t)K, (uint64_t)N, (uint64_t)ldb, bke, (uint32_t)(bn / pm), eb);
    if (rc) return rc;
    for (int i = 0; i < MAX_PEERS; ++i) {
        if (gather && i < ga->n_peers) {
            rc = make_map(&P.map_b_peer[i], ga->peers[i], (uint64_t)K, (uint64_t)N, (uint64_t)ldb, BK, (uint32_t)bn);
            if (rc) return rc;
        } else {
            P.map_b_peer[i] = P.map_b;
        }
    }
    // the output map spans exactly the (M, N) view of D: the TMA stores of ragged tiles cannot reach the elements around it
    rc = f32d ? make_map_typed(&P.map_d, d, (uint64_t)N, (uint64_t)M, (uint64_t)ldd, 32, 64, 4)
              : make_map(&P.map_d, d, (uint64_t)N, (uint64_t)M, (uint64_t)ldd, 64, 64);
    if (rc) return rc;
    P.bias = (const __nv_bfloat16*)bias;
    P.out = (__nv_bfloat16*)d;
    P.ldd = ldd;
    P.dbg = g_dbg;
    P.inv_scale_a = inv_a;
    P.inv_scale_b = inv_b;
    P.tile_owner = gather ? ga->tile_owner : nullptr;
    P.flags = gather ? ga->flags : nullptr;
    P.epoch = gather ? ga->epoch : nullptr;
    P.done_ctas = gather ? ga->done : nullptr;
    P.M = M; P.N = N; P.K = K;
    const int num_k = (K + bke - 1) / bke;
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
    const int num_sn = (num_n + pn - 1) / pn;
    const long long units = (long long)((num_mb + pm - 1) / pm) * num_sn * P.splits;
    const int slots = cl > 1 ? max_clusters(cl, sms) : sms;
    if (slots <= 0) return -5;
    P.band = gather ? num_sn : tile_band(M, op ? (K + 1) / 2 : K, bn * pn, num_sn);
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
    const KernelFn fn = pingpong ? pingpong_kernel_for(b_mn)
                        : f32d ? (op ? fp8_f32acc_kernel_for(bn, op) : f32acc_kernel_for(bn))
                               : (op ? fp8_kernel_for(bn, op) : kernel_for(bn, a_mn, b_mn));
    return (int)cudaLaunchKernelEx(&cfg, fn, P);
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

// FP8: D[M,N] (+)= A[M,K] * B[N,K]^T * (inv_a[0] * inv_b[0]) (+ bias).  a, b: one-byte K-major operands (row strides lda, ldb
// bytes, multiples of 16; K % 16 == 0); a_e5m2: A is e5m2 (gradients), else e4m3; B is e4m3.  inv_a / inv_b: device pointers to 1/s.
extern "C" int acco_gemm_fp8_run(const void* a, long long lda, const void* b, long long ldb, void* d, long long ldd, const void* bias, int M, int N,
                                 int K, int accumulate, int a_e5m2, const float* inv_a, const float* inv_b, int bn_req, int splits_req, int sms,
                                 cudaStream_t st) {
    return acco_gemm::launch(a, lda, 0, b, ldb, 0, d, ldd, bias, M, N, K, accumulate, bn_req, splits_req, 0, 0, 0, nullptr, sms, st,
                             a_e5m2 ? acco_gemm::OP_E5M2 : acco_gemm::OP_E4M3, inv_a, inv_b);
}

// wgrad into an fp32 gradient: D[M,N] (fp32, row stride ldd) += A * B^T with A stored [K, M] and B stored [K, N] (both MN-major,
// bf16).  One K split adds the tile to D exactly (one fp32 add per element); split-K adds each split's fp32 partial through the TMA unit.
extern "C" int acco_gemm_wgrad_f32(const void* a, long long lda, const void* b, long long ldb, float* d, long long ldd, int M, int N, int K,
                                   int bn_req, int splits_req, int sms, cudaStream_t st) {
    return acco_gemm::launch(a, lda, 1, b, ldb, 1, d, ldd, nullptr, M, N, K, 1, bn_req, splits_req, 0, 0, 0, nullptr, sms, st, acco_gemm::OP_BF16,
                             nullptr, nullptr, 1);
}

// FP8 into an fp32 D: D[M,N] += A[M,K] * B[N,K]^T * (inv_a[0] * inv_b[0]), operands as in acco_gemm_fp8_run
extern "C" int acco_gemm_fp8_acc_f32(const void* a, long long lda, const void* b, long long ldb, float* d, long long ldd, int M, int N, int K,
                                     int a_e5m2, const float* inv_a, const float* inv_b, int bn_req, int splits_req, int sms, cudaStream_t st) {
    return acco_gemm::launch(a, lda, 0, b, ldb, 0, d, ldd, nullptr, M, N, K, 1, bn_req, splits_req, 0, 0, 0, nullptr, sms, st,
                             a_e5m2 ? acco_gemm::OP_E5M2 : acco_gemm::OP_E4M3, inv_a, inv_b, 1);
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
// the schedule launch() runs an unrequested bf16 call of that shape on (introspection for tools / tests): 1 = ping-pong, 0 = cooperative.
// A call that requests a tile width, K splits or multicast always runs on the cooperative kernel.
extern "C" int acco_gemm_schedule(int M, int N, int K, int a_mn, int b_mn, int accumulate, int sms) {
    const acco_gemm::Config c = acco_gemm::choose_config(M, N, K, a_mn, b_mn, accumulate, sms, 0, 0, acco_gemm::g_pm, acco_gemm::g_pn);
    return acco_gemm::use_pingpong(c, K, a_mn, accumulate, acco_gemm::OP_BF16, 0, 0, 0, 0, acco_gemm::g_pm, acco_gemm::g_pn) ? 1 : 0;
}
