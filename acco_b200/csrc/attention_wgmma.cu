// Causal (optionally sliding-window) flash attention on the Hopper tensor cores (sm_90a) - forward and backward, head_dim 64.
//
// OPT-IN (ACCO_ATTN=own); the default attention path is the library SDPA (ops/attention.py).  tools/attn_check.py compares both
// directions with the fp32 reference.
//
// Layout contract (what the fused QKV GEMM of the models produces): q / k / v are column blocks of one row-major activation
// [B*S, (Hq + 2 Hk) * 64] (row stride `ld`), RoPE already applied in place; O and dO are [B*S, Hq*64].
//
// Forward (wgmma + TMA + mbarrier; one CTA = 128 queries of one head, two warpgroups of 64 rows): Q once and K_j / V_j blocks of
//   64 keys through a 2-stage TMA ring (128-byte swizzle, the same shared-memory layouts as the wgmma GEMM: K-major Q and K, MN-major
//   V); S = Q K_j^T by wgmma into registers, running-max softmax in the exp2 domain, P (rounded to bf16) fed from the registers as
//   the A operand of O += P V_j.  LSE = ln(sum exp) per row is kept for the backward.
// Backward (mma.sync m16n8k16; one CTA = 64 keys of one KV head, 4 warps x 16 keys; FlashAttention-2 schedule: K_n / V_n
//   stationary, loop over the
//   query heads of the GQA group and the visible 64-query blocks):  S^T = K Q^T, P^T = exp2(S^T c - LSE), dP^T = V dO^T,
//   dS^T = P^T (dP^T - Delta) * scale;  dV += P^T dO, dK += dS^T Q in registers;  dS goes through shared memory for dQ = dS K,
//   which is added (fp32 atomics) into a zero-filled dQ accumulator.  P and dS are rounded to bf16 before their products.
// Delta = rowsum(dO * O) comes from `attn_delta_kernel`.  `attention_blockwise_ref` / `attention_blockwise_bwd_ref`
// (ops/attention.py) give the fp32 reference semantics of the same masking and rounding points.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "wgmma.cuh"

namespace acco_attn {

using namespace acco_tc;

constexpr int HD = 64;                         // head dim
constexpr int LDS = HD + 8;                    // shared-memory row stride (elements): 144 B rows spread the 32-bit fragment loads over banks
constexpr float LOG2E = 1.4426950408889634f;
constexpr float LN2 = 0.6931471805599453f;

typedef __nv_bfloat16 bf16;

__device__ __forceinline__ uint32_t pack2(float a, float b) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ uint32_t ld32(const bf16* p) { return *reinterpret_cast<const uint32_t*>(p); }

__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// acc[16 x 8*NB] += A[16 x 16*KB] * B[8*NB x 16*KB]^T; A: shared, row-major (rows = the warp's 16 rows); B: shared, [n][k]
template <int NB, int KB>
__device__ __forceinline__ void warp_mma_ss(float (&acc)[NB][4], const bf16* A, const bf16* B, int lane) {
    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int kb = 0; kb < KB; ++kb) {
        uint32_t a[4];
        const bf16* a0 = A + g * LDS + kb * 16 + 2 * t;
        a[0] = ld32(a0); a[1] = ld32(a0 + 8 * LDS); a[2] = ld32(a0 + 8); a[3] = ld32(a0 + 8 * LDS + 8);
#pragma unroll
        for (int nb = 0; nb < NB; ++nb) {
            const bf16* b = B + (nb * 8 + g) * LDS + kb * 16 + 2 * t;
            mma16816(acc[nb], a, ld32(b), ld32(b + 8));
        }
    }
}
// acc[16 x 8*NB] += P[16 x 64] * B[8*NB x 64]^T with P given as accumulator fragments p[8][4] (16 x 64, fp32), rounded to bf16
template <int NB>
__device__ __forceinline__ void warp_mma_rs(float (&acc)[NB][4], const float (&p)[8][4], const bf16* B, int lane) {
    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int kb = 0; kb < 4; ++kb) {
        uint32_t a[4];
        a[0] = pack2(p[2 * kb][0], p[2 * kb][1]);
        a[1] = pack2(p[2 * kb][2], p[2 * kb][3]);
        a[2] = pack2(p[2 * kb + 1][0], p[2 * kb + 1][1]);
        a[3] = pack2(p[2 * kb + 1][2], p[2 * kb + 1][3]);
#pragma unroll
        for (int nb = 0; nb < NB; ++nb) {
            const bf16* b = B + (nb * 8 + g) * LDS + kb * 16 + 2 * t;
            mma16816(acc[nb], a, ld32(b), ld32(b + 8));
        }
    }
}

// rows x 64 tile of a row-major [*, ld] bf16 matrix -> shared [rows][LDS]; rows beyond `valid` are zero
__device__ __forceinline__ void load_tile(bf16* dst, const bf16* src, long long ld, int rows, int valid, int tid, int nthr) {
    for (int i = tid; i < rows * 8; i += nthr) {
        const int r = i >> 3, c = (i & 7) * 8;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (r < valid) v = *reinterpret_cast<const uint4*>(src + (long long)r * ld + c);
        *reinterpret_cast<uint4*>(dst + r * LDS + c) = v;
    }
}
// same, transposed: dst[d][row]
__device__ __forceinline__ void load_tile_t(bf16* dst, const bf16* src, long long ld, int rows, int tid, int nthr) {
    for (int i = tid; i < rows * 8; i += nthr) {
        const int r = i >> 3, c = (i & 7) * 8;
        const uint4 v = *reinterpret_cast<const uint4*>(src + (long long)r * ld + c);
        const bf16* e = reinterpret_cast<const bf16*>(&v);
#pragma unroll
        for (int j = 0; j < 8; ++j) dst[(c + j) * LDS + r] = e[j];
    }
}

__device__ __forceinline__ bool visible(int q, int kv, int window) { return kv <= q && kv > q - window; }

// ================================================================================================ forward
struct FwdParams {
    CUtensorMap map_q;                 // Q columns of the qkv activation: box {64 d, 128 queries}
    CUtensorMap map_k;                 // K columns: box {64 d, 64 keys}
    CUtensorMap map_v;                 // V columns: box {64 d, 64 keys}
    bf16* o;
    long long ld_o;
    float* lse;
    int B, S, Hq, Hk, window;
    float scale;
};

constexpr int FWD_Q = 128, FWD_KV = 64, FWD_THREADS = 256;
constexpr int FWD_TILE_KV = FWD_KV * HD * 2;                       // 8 KiB
constexpr int FWD_SMEM = FWD_Q * HD * 2 + 2 * 2 * FWD_TILE_KV + 1024 /*align*/ + 64 /*barriers*/;

// D[64 x 64] += A[64 x 16] (registers, bf16 pairs) * B[16 x 64] (shared, MN-major: rows = k)
__device__ __forceinline__ void wgmma_m64n64k16_rs_tb(float (&d)[32], const uint32_t (&a)[4], uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
        "{%32,%33,%34,%35}, %36, p, 1, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
          "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]),
          "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]),
          "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(1));
}

// One CTA = 128 queries of one head = two warpgroups of 64 rows.  Thread 0 TMA-loads Q once and the K / V blocks of 64 keys through a
// 2-stage ring (128-byte swizzle, mbarrier transaction counts); S = Q K^T and O += P V run as wgmma (P straight from the registers
// holding S); the CTA barrier at the end of a block is what frees its stage for the block two ahead.
__global__ void __launch_bounds__(FWD_THREADS) attn_fwd_kernel(const __grid_constant__ FwdParams P) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);   // SWIZZLE_128B needs 1024 B alignment
    uint8_t* sQ = smem;                                            // [128 q][64 d]
    uint8_t* sKV = smem + FWD_Q * HD * 2;                          // 2 stages x (K [64][64], V [64][64])
    uint64_t* full = (uint64_t*)(sKV + 2 * 2 * FWD_TILE_KV);       // [2] K / V of a stage landed;  [2]: Q landed
    const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int hk = h / (P.Hq / P.Hk);
    const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int q0 = qb * FWD_Q;
    const int row0 = b * P.S;
    const int lo_key = max(0, q0 - P.window + 1);
    const int j_lo = lo_key / FWD_KV, j_hi = (q0 + FWD_Q - 1) / FWD_KV;
    auto issue = [&](int j) {                                      // thread 0: K_j, V_j into stage (j - j_lo) & 1
        const int s = (j - j_lo) & 1;
        mbar_expect_tx(&full[s], 2 * FWD_TILE_KV);
        tma_load_2d(&P.map_k, &full[s], sKV + s * 2 * FWD_TILE_KV, hk * HD, row0 + j * FWD_KV);
        tma_load_2d(&P.map_v, &full[s], sKV + s * 2 * FWD_TILE_KV + FWD_TILE_KV, hk * HD, row0 + j * FWD_KV);
    };
    if (tid == 0) {
        mbar_init(&full[0], 1);
        mbar_init(&full[1], 1);
        mbar_init(&full[2], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        mbar_expect_tx(&full[2], FWD_Q * HD * 2);
        tma_load_2d(&P.map_q, &full[2], sQ, h * HD, row0 + q0);
        issue(j_lo);
        if (j_lo + 1 <= j_hi) issue(j_lo + 1);
    }
    __syncthreads();
    mbar_wait(&full[2], 0);
    const float c = P.scale * LOG2E;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    const int wq_lo = q0 + wg * 64, wq_hi = wq_lo + 63;
    const int qr[2] = {wq_lo + warp * 16 + g, wq_lo + warp * 16 + g + 8};
    const uint32_t q_addr = smem_u32(sQ) + (uint32_t)(wg * 8192);
    for (int j = j_lo; j <= j_hi; ++j) {
        const int kv0 = j * FWD_KV, s = (j - j_lo) & 1;
        mbar_wait(&full[s], (uint32_t)(((j - j_lo) >> 1) & 1));
        // this warpgroup's rows see nothing of this block: skip the math (uniform per warpgroup)
        if (!(kv0 > wq_hi || kv0 + FWD_KV - 1 <= wq_lo - P.window)) {
            const uint32_t k_addr = smem_u32(sKV + s * 2 * FWD_TILE_KV), v_addr = k_addr + FWD_TILE_KV;
            float sc[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) sc[i] = 0.f;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < HD / 16; ++k)
                wgmma_m64n64k16<0, 0>(sc, make_smem_desc(q_addr + k * 32, 1, 1024 >> 4), make_smem_desc(k_addr + k * 32, 1, 1024 >> 4), 1u);
            wgmma_commit();
            wgmma_wait<0>();
            reg_fence(sc);
            float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
            for (int nb = 0; nb < 8; ++nb)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int kv = kv0 + nb * 8 + 2 * t + (e & 1), r = e >> 1;
                    const float v = visible(qr[r], kv, P.window) ? sc[4 * nb + e] * c : -INFINITY;
                    sc[4 * nb + e] = v;
                    mx[r] = fmaxf(mx[r], v);
                }
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
                mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            }
            float alpha[2], base[2], rs[2] = {0.f, 0.f};
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const float m_new = fmaxf(m_run[r], mx[r]);
                base[r] = m_new == -INFINITY ? 0.f : m_new;
                alpha[r] = exp2f(m_run[r] - base[r]);              // m_run = -inf -> 0
                m_run[r] = m_new;
            }
#pragma unroll
            for (int i = 0; i < 32; ++i) {
                const int r = (i >> 1) & 1;
                const float p = exp2f(sc[i] - base[r]);
                sc[i] = p;
                rs[r] += p;
            }
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 1);
                rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 2);
                l_run[r] = l_run[r] * alpha[r] + rs[r];
            }
#pragma unroll
            for (int i = 0; i < 32; ++i) o[i] *= alpha[(i >> 1) & 1];
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < FWD_KV / 16; ++kk) {
                uint32_t a[4];
                a[0] = pack2(sc[8 * kk + 0], sc[8 * kk + 1]);
                a[1] = pack2(sc[8 * kk + 2], sc[8 * kk + 3]);
                a[2] = pack2(sc[8 * kk + 4], sc[8 * kk + 5]);
                a[3] = pack2(sc[8 * kk + 6], sc[8 * kk + 7]);
                wgmma_m64n64k16_rs_tb(o, a, make_smem_desc(v_addr + kk * 2048, 8192 >> 4, 1024 >> 4));
            }
            wgmma_commit();
            wgmma_wait<0>();
            reg_fence(o);
        }
        __syncthreads();                                           // every warpgroup is done with stage s
        if (tid == 0 && j + 2 <= j_hi) issue(j + 2);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int q = qr[r];
        const float inv = l_run[r] > 0.f ? 1.f / l_run[r] : 0.f;
        bf16* dst = P.o + ((long long)row0 + q) * P.ld_o + h * HD + 2 * t;
#pragma unroll
        for (int nb = 0; nb < 8; ++nb)
            *reinterpret_cast<uint32_t*>(dst + nb * 8) = pack2(o[4 * nb + 2 * r] * inv, o[4 * nb + 2 * r + 1] * inv);
        if (t == 0) P.lse[((long long)b * P.Hq + h) * P.S + q] = (m_run[r] + log2f(l_run[r])) * LN2;
    }
}

// ================================================================================================ backward
struct BwdParams {
    const bf16 *q, *k, *v;
    long long ld;
    const bf16* d_o;
    long long ld_do;
    const float *lse, *delta;
    float* dq;                                 // [B*S, Hq*64] fp32, zero-filled
    bf16 *dk, *dv;                             // [B*S, Hk*64]
    int B, S, Hq, Hk, window;
    float scale;
};

constexpr int BWD_KV = 64, BWD_Q = 64, BWD_THREADS = 128;
constexpr int BWD_SMEM = 8 * 64 * LDS * 2 + 2 * BWD_Q * 4;

__global__ void __launch_bounds__(BWD_THREADS) attn_bwd_kernel(const BwdParams P) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    bf16* sK = reinterpret_cast<bf16*>(smem_raw);   // [key][d]
    bf16* sKt = sK + 64 * LDS;                      // [d][key]
    bf16* sV = sKt + 64 * LDS;                      // [key][d]
    bf16* sQ = sV + 64 * LDS;                       // [q][d]
    bf16* sQt = sQ + 64 * LDS;                      // [d][q]
    bf16* sdO = sQt + 64 * LDS;                     // [q][d]
    bf16* sdOt = sdO + 64 * LDS;                    // [d][q]
    bf16* sdS = sdOt + 64 * LDS;                    // [q][key]
    float* sL = reinterpret_cast<float*>(sdS + 64 * LDS);   // LSE (log2 domain) of the 64 queries
    float* sD = sL + BWD_Q;                                  // Delta
    const int nb_k = blockIdx.x, hk = blockIdx.y, b = blockIdx.z;
    const int G = P.Hq / P.Hk;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int kv0 = nb_k * BWD_KV;
    const long long row0 = (long long)b * P.S;
    load_tile(sK, P.k + (row0 + kv0) * P.ld + hk * HD, P.ld, BWD_KV, BWD_KV, tid, BWD_THREADS);
    load_tile_t(sKt, P.k + (row0 + kv0) * P.ld + hk * HD, P.ld, BWD_KV, tid, BWD_THREADS);
    load_tile(sV, P.v + (row0 + kv0) * P.ld + hk * HD, P.ld, BWD_KV, BWD_KV, tid, BWD_THREADS);
    const float c = P.scale * LOG2E;
    float dk[8][4], dv[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e) dk[i][e] = dv[i][e] = 0.f;
    const int kr[2] = {kv0 + warp * 16 + g, kv0 + warp * 16 + g + 8};   // this thread's key rows
    const int m_lo = kv0 / BWD_Q;
    const int m_hi = min(P.S / BWD_Q - 1, (kv0 + BWD_KV - 1 + P.window - 1) / BWD_Q);
    for (int gi = 0; gi < G; ++gi) {
        const int hq = hk * G + gi;
        for (int m = m_lo; m <= m_hi; ++m) {
            const int q0 = m * BWD_Q;
            __syncthreads();                               // previous iteration's Q / dO / dS consumed
            load_tile(sQ, P.q + (row0 + q0) * P.ld + hq * HD, P.ld, BWD_Q, BWD_Q, tid, BWD_THREADS);
            load_tile_t(sQt, P.q + (row0 + q0) * P.ld + hq * HD, P.ld, BWD_Q, tid, BWD_THREADS);
            load_tile(sdO, P.d_o + (row0 + q0) * P.ld_do + hq * HD, P.ld_do, BWD_Q, BWD_Q, tid, BWD_THREADS);
            load_tile_t(sdOt, P.d_o + (row0 + q0) * P.ld_do + hq * HD, P.ld_do, BWD_Q, tid, BWD_THREADS);
            if (tid < BWD_Q) {
                const long long li = ((long long)b * P.Hq + hq) * P.S + q0 + tid;
                sL[tid] = P.lse[li] * LOG2E;
                sD[tid] = P.delta[li];
            }
            __syncthreads();
            // S^T = K Q^T and dP^T = V dO^T for this warp's 16 keys x 64 queries
            float s[8][4], dp[8][4];
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int e = 0; e < 4; ++e) s[i][e] = dp[i][e] = 0.f;
            warp_mma_ss<8, 4>(s, sK + warp * 16 * LDS, sQ, lane);
            warp_mma_ss<8, 4>(dp, sV + warp * 16 * LDS, sdO, lane);
#pragma unroll
            for (int nb = 0; nb < 8; ++nb)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int ql = nb * 8 + 2 * t + (e & 1), q = q0 + ql, r = e >> 1;
                    const float p = visible(q, kr[r], P.window) ? exp2f(s[nb][e] * c - sL[ql]) : 0.f;
                    const float pb = __bfloat162float(__float2bfloat16(p));
                    s[nb][e] = pb;                                                          // P^T (bf16 values)
                    dp[nb][e] = __bfloat162float(__float2bfloat16(p * (dp[nb][e] - sD[ql]) * P.scale));   // dS^T
                }
            // dS -> shared [q][key] for dQ = dS K
#pragma unroll
            for (int nb = 0; nb < 8; ++nb)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int ql = nb * 8 + 2 * t + (e & 1), kl = warp * 16 + g + 8 * (e >> 1);
                    sdS[ql * LDS + kl] = __float2bfloat16(dp[nb][e]);
                }
            warp_mma_rs<8>(dv, s, sdOt, lane);             // dV += P^T dO
            warp_mma_rs<8>(dk, dp, sQt, lane);             // dK += dS^T Q
            __syncthreads();
            // dQ[q, :] += dS[q, keys] K[keys, :] for this warp's 16 queries
            float dq[8][4];
#pragma unroll
            for (int i = 0; i < 8; ++i) dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f;
            warp_mma_ss<8, 4>(dq, sdS + warp * 16 * LDS, sKt, lane);
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                float* dst = P.dq + (row0 + q0 + warp * 16 + g + 8 * r) * (long long)(P.Hq * HD) + hq * HD + 2 * t;
#pragma unroll
                for (int nb = 0; nb < 8; ++nb) {
                    atomicAdd(dst + nb * 8, dq[nb][2 * r]);
                    atomicAdd(dst + nb * 8 + 1, dq[nb][2 * r + 1]);
                }
            }
        }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const long long off = (row0 + kr[r]) * (long long)(P.Hk * HD) + hk * HD + 2 * t;
#pragma unroll
        for (int nb = 0; nb < 8; ++nb) {
            *reinterpret_cast<uint32_t*>(P.dk + off + nb * 8) = pack2(dk[nb][2 * r], dk[nb][2 * r + 1]);
            *reinterpret_cast<uint32_t*>(P.dv + off + nb * 8) = pack2(dv[nb][2 * r], dv[nb][2 * r + 1]);
        }
    }
}

// Delta[b, h, s] = sum_d dO[b, s, h, d] * O[b, s, h, d]     (8 lanes per (row, head): 16 bytes of each operand per lane)
__global__ void __launch_bounds__(256) attn_delta_kernel(const bf16* __restrict__ o, const bf16* __restrict__ d_o, long long ld_o,
                                                         long long ld_do, float* __restrict__ delta, int B, int S, int Hq) {
    const long long item = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 3;   // (row, head)
    const int part = threadIdx.x & 7;
    const long long n_items = (long long)B * S * Hq;
    float acc = 0.f;
    long long row = 0;
    int h = 0;
    if (item < n_items) {
        row = item / Hq;
        h = (int)(item - row * Hq);
        const uint4 a = *reinterpret_cast<const uint4*>(o + row * ld_o + h * HD + part * 8);
        const uint4 d = *reinterpret_cast<const uint4*>(d_o + row * ld_do + h * HD + part * 8);
        const __nv_bfloat162* a2 = reinterpret_cast<const __nv_bfloat162*>(&a);
        const __nv_bfloat162* d2 = reinterpret_cast<const __nv_bfloat162*>(&d);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 x = __bfloat1622float2(a2[i]), y = __bfloat1622float2(d2[i]);
            acc += x.x * y.x + x.y * y.y;
        }
    }
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    acc += __shfl_xor_sync(0xffffffffu, acc, 4);
    if (item < n_items && part == 0) {
        const long long b = row / S, s = row - b * S;
        delta[(b * Hq + h) * S + s] = acc;
    }
}

// ------------------------------------------------------------------------------------------------ host side
static bool shape_ok(int B, int S, int Hq, int Hk, int D, float scale) {
    return B > 0 && S > 0 && S % 128 == 0 && Hk > 0 && Hq > 0 && Hq % Hk == 0 && D == HD && scale > 0.f;
}
static bool aligned(const void* p, long long ld) { return ((uintptr_t)p % 16) == 0 && (ld % 8) == 0; }
static int eff_window(int S, int window) { return (window <= 0 || window > S) ? S : window; }

}  // namespace acco_attn

// 1 when the kernels cover the shape (head_dim 64, S a multiple of 128, grouped heads dividing evenly, scale > 0)
extern "C" int acco_attn_supported(int B, int S, int Hq, int Hk, int D, float scale) {
    return acco_attn::shape_ok(B, S, Hq, Hk, D, scale) ? 1 : 0;
}

// O = softmax(scale * Q K^T + causal/window mask) V.   q, k, v: column blocks (row stride ld elements) of [B*S, .] activations;
// o [B*S, Hq*64] (row stride ld_o); lse [B, Hq, S] fp32.  window <= 0 or >= S: plain causal.
extern "C" int acco_attn_fwd(const void* q, const void* k, const void* v, long long ld, void* o, long long ld_o, float* lse, int B, int S, int Hq,
                             int Hk, int D, float scale, int window, cudaStream_t st) {
    using namespace acco_attn;
    if (!shape_ok(B, S, Hq, Hk, D, scale) || !aligned(q, ld) || !aligned(k, ld) || !aligned(v, ld) || !aligned(o, ld_o)) return -1;
    static int fwd_attr = (int)cudaFuncSetAttribute(attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FWD_SMEM);
    if (fwd_attr) return fwd_attr;
    FwdParams P;
    const uint64_t rows = (uint64_t)B * S;
    // each map spans the whole activation (B*S rows, row stride ld); the head's 64 columns are selected by the box coordinate
    int rc = acco_gemm::make_map_typed(&P.map_q, q, (uint64_t)Hq * HD, rows, (uint64_t)ld, HD, FWD_Q, 2);
    if (!rc) rc = acco_gemm::make_map_typed(&P.map_k, k, (uint64_t)Hk * HD, rows, (uint64_t)ld, HD, FWD_KV, 2);
    if (!rc) rc = acco_gemm::make_map_typed(&P.map_v, v, (uint64_t)Hk * HD, rows, (uint64_t)ld, HD, FWD_KV, 2);
    if (rc) return rc;
    P.o = (bf16*)o; P.ld_o = ld_o; P.lse = lse;
    P.B = B; P.S = S; P.Hq = Hq; P.Hk = Hk; P.window = eff_window(S, window); P.scale = scale;
    attn_fwd_kernel<<<dim3(S / FWD_Q, Hq, B), FWD_THREADS, FWD_SMEM, st>>>(P);
    return (int)cudaGetLastError();
}

// Gradients of acco_attn_fwd.  d_o [B*S, Hq*64] (row stride ld_do); delta [B, Hq, S] fp32 scratch; dq_acc fp32 [B*S, Hq*64]
// contiguous (zero-filled here, then added into by the kernel); dk, dv bf16 [B*S, Hk*64] contiguous.
extern "C" int acco_attn_bwd(const void* q, const void* k, const void* v, long long ld, const void* o, long long ld_o, const void* d_o,
                             long long ld_do, const float* lse, float* delta, float* dq_acc, void* dk, void* dv, int B, int S, int Hq, int Hk, int D,
                             float scale, int window, cudaStream_t st) {
    using namespace acco_attn;
    if (!shape_ok(B, S, Hq, Hk, D, scale) || !aligned(q, ld) || !aligned(k, ld) || !aligned(v, ld) || !aligned(o, ld_o) || !aligned(d_o, ld_do))
        return -1;
    static int attr_rc = (int)cudaFuncSetAttribute(attn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, BWD_SMEM);
    if (attr_rc) return attr_rc;
    const long long items = (long long)B * S * Hq;
    attn_delta_kernel<<<(unsigned)((items * 8 + 255) / 256), 256, 0, st>>>((const bf16*)o, (const bf16*)d_o, ld_o, ld_do, delta, B, S, Hq);
    if (cudaMemsetAsync(dq_acc, 0, (size_t)items * HD * sizeof(float), st) != cudaSuccess) return -6;
    BwdParams P{(const bf16*)q, (const bf16*)k, (const bf16*)v, ld, (const bf16*)d_o, ld_do, lse, delta, dq_acc, (bf16*)dk, (bf16*)dv,
                B, S, Hq, Hk, eff_window(S, window), scale};
    attn_bwd_kernel<<<dim3(S / BWD_KV, Hk, B), BWD_THREADS, BWD_SMEM, st>>>(P);
    return (int)cudaGetLastError();
}
