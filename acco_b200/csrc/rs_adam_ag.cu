// KERNEL A - one launch per communication round:
//
//     reduce-scatter (pull my slice of every rank's gradient accumulator over NVLink)
//   + global micro-batch count exchange
//   + [stash add / stash write]  (ACCO: the tentative round's half-batch sum is kept on the owner)
//   + scale by 1/count, AdamW on the fp32 master shard with *commit flags* (tentative steps write
//     nothing back, so no clone/restore of weights and Adam state is ever needed)
//   + all-gather (push the fresh bf16 slice into every rank's shadow parameter buffer)
//
// It replaces, per round, the reference's: all_reduce(count) + reduce_scatter_tensor + cast +
// mul_(1/count) + ~17 foreach AdamW kernels + cast + all_gather_into_tensor + up to 7 clone/restore
// copies (trainer_decoupled.py:67-126K11) - with NO NCCL call on the path.
//
// Transport (chosen at launch):
//   * NVLS multicast : `multimem.ld_reduce.add.acc::f32.v4.bf16x2` pulls the switch-reduced sum of all
//     W accumulators in one instruction; `multimem.st.v4` broadcasts the new weights to all W ranks.
//   * P2P            : W plain 16-byte loads from the peers' mapped buffers, fp32 accumulate in
//     registers; W 16-byte stores.
//   * W == 1         : the same kernel on local pointers (also used after an NCCL reduce-scatter by
//     the library-baseline backend).
// Cross-GPU ordering: a start barrier (every rank's accumulator is final; also carries the counts)
// and an end barrier (every rank's pushes have landed) on flag words in a symmetric signal pad,
// written with st.release.sys and polled with ld.acquire.sys; the epoch lives in device memory so
// the launch is CUDA-graph friendly.  Only CTA 0 signals, every CTA polls its *local* pad, the
// last CTA to finish runs the end barrier - no grid-wide co-residency is required.
#include <cstdio>

#include <stdlib.h>

#include "common.cuh"

namespace acco {

constexpr int kMaxWorld = 16;
constexpr int kAdamThreads = 512;

struct RoundParams {
    // transport
    const void* acc_peer[kMaxWorld];   // each rank's accumulator for this round (peer-mapped); [0] only if world==1
    void* theta_peer[kMaxWorld];       // each rank's shadow parameter buffer
    uint32_t* pad_peer[kMaxWorld];     // each rank's signal pad
    const void* acc_mc;                // multicast address of the accumulator (0 -> P2P)
    void* theta_mc;                    // multicast address of the shadow buffer (0 -> P2P)
    // shard state (local)
    float* master;
    float* exp_avg;
    float* exp_avg_sq;
    float* stash;
    int* stash_count;                  // device: global count represented by the stash
    int* total_out;                    // device: global count of the update applied this round
    uint32_t* epoch;                   // device: last completed barrier epoch
    uint32_t* done_ctas;               // device: CTA completion counter (self-resetting)
    const float* inv_count_in;         // optional device scalar 1/count (world==1 library path); else nullptr
    const long long* skip;             // sorted, disjoint [lo, hi) element ranges that are NOT pushed to peers (they are pulled
    int n_skip;                        //   later by the gather-GEMM, KERNEL B); the owner still updates its own copy
    int watchdog_s;                    // trap if a peer has not reached a barrier after this many seconds (0 = wait forever)
    int gated;                         // 1: the start barrier already ran in round_gate_kernel (tiny, so waiting for a slow peer
                                       //    does not pin registers / SM slots that the overlapping compute needs)
    long long slice;                   // elements per rank (multiple of 8)
    int rank, world, local_count;
    float lr, beta1, beta2, eps, weight_decay, bc1, bc2_rsqrt;   // bc1 = 1-b1^t ; bc2_rsqrt = 1/sqrt(1-b2^t)
    int commit, add_stash, write_stash;
};

// signal pad layout (uint32 words): [0,W) start flags, [W,2W) end flags, [2W,3W) counts
ACCO_DEVINL void st_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
ACCO_DEVINL uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// Spin until *p >= epoch (wrap-safe).  Failure detection: a peer that never arrives (crashed / hung rank) would hang
// this kernel - and with it the whole job - forever (the reference has the same property through NCCL);
// after `watchdog_s` seconds the kernel traps instead, which surfaces as a CUDA error on the host.
ACCO_DEVINL void wait_flag(const uint32_t* p, uint32_t epoch, int watchdog_s) {
    unsigned long long t0 = 0;
    unsigned spins = 0;
    while ((int32_t)(ld_acquire_sys(p) - epoch) < 0) {
        __nanosleep(40);
        if ((++spins & 0xFFFF) == 0) {
            unsigned long long now;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
            if (t0 == 0) t0 = now;
            else if (watchdog_s > 0 && now - t0 > (unsigned long long)watchdog_s * 1000000000ull) {
                printf("acco_b200: rs_adam_ag_kernel watchdog - a peer did not reach the round barrier within %d s\n", watchdog_s);
                __trap();
            }
        }
    }
}
ACCO_DEVINL void st_relaxed_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

ACCO_DEVINL uint4 ld_peer16(const void* p) {   // peer memory is not L2-cached locally; keep it out of L1 too
    uint4 r;
    asm volatile("ld.relaxed.sys.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p)
                 : "memory");
    return r;
}
ACCO_DEVINL void st_peer16(void* p, const uint4& r) {
    asm volatile("st.relaxed.sys.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(r.x), "r"(r.y),
                 "r"(r.z), "r"(r.w)
                 : "memory");
}
// NVLS: switch-side reduction of 8 bf16 across all ranks mapped behind the multicast address
ACCO_DEVINL uint4 multimem_ld_reduce_bf16x8(const void* mc) {
    uint4 r;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(mc)
                 : "memory");
    return r;
}
ACCO_DEVINL float4 multimem_ld_reduce_f32x4(const void* mc) {
    float4 r;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
                 : "l"(mc)
                 : "memory");
    return r;
}
ACCO_DEVINL void multimem_st16(void* mc, const uint4& r) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "f"(__uint_as_float(r.x)),
                 "f"(__uint_as_float(r.y)), "f"(__uint_as_float(r.z)), "f"(__uint_as_float(r.w))
                 : "memory");
}

template <typename T> struct Elem;
template <> struct Elem<__nv_bfloat16> { static constexpr int kVec = 8; };   // elements per 16 bytes
template <> struct Elem<float> { static constexpr int kVec = 4; };

// true iff element e lies in one of the sorted, disjoint skip ranges (binary search; ranges are 8-aligned)
ACCO_DEVINL bool in_skip(const RoundParams& P, long long e) {
    int lo = 0, hi = P.n_skip;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(P.skip + 2 * mid + 1) <= e) lo = mid + 1;
        else hi = mid;
    }
    return lo < P.n_skip && __ldg(P.skip + 2 * lo) <= e;
}

// Load 8 consecutive gradient elements (sum over ranks) starting at element `e` of the full buffer.
template <typename G, int MODE /*0 local, 1 p2p, 2 multimem*/>
ACCO_DEVINL void load_grad8(const RoundParams& P, long long e, float (&g)[8]) {
    if constexpr (sizeof(G) == 2) {
        if constexpr (MODE == 2) {
            uint4 r = multimem_ld_reduce_bf16x8((const char*)P.acc_mc + e * 2);
            unpack8(*reinterpret_cast<bf16x8*>(&r), g);
        } else if constexpr (MODE == 1) {
            uint4 r[kMaxWorld];
#pragma unroll
            for (int q = 0; q < kMaxWorld; ++q)
                if (q < P.world) r[q] = ld_peer16((const char*)P.acc_peer[(P.rank + q) % P.world] + e * 2);
#pragma unroll
            for (int j = 0; j < 8; ++j) g[j] = 0.f;
#pragma unroll
            for (int q = 0; q < kMaxWorld; ++q)
                if (q < P.world) {
                    float f[8];
                    unpack8(*reinterpret_cast<bf16x8*>(&r[q]), f);
#pragma unroll
                    for (int j = 0; j < 8; ++j) g[j] += f[j];
                }
        } else {
            unpack8(ld_stream_rw((const char*)P.acc_peer[0] + e * 2), g);
        }
    } else {
        if constexpr (MODE == 2) {
            float4 a = multimem_ld_reduce_f32x4((const char*)P.acc_mc + e * 4);
            float4 b = multimem_ld_reduce_f32x4((const char*)P.acc_mc + e * 4 + 16);
            g[0] = a.x; g[1] = a.y; g[2] = a.z; g[3] = a.w; g[4] = b.x; g[5] = b.y; g[6] = b.z; g[7] = b.w;
        } else if constexpr (MODE == 1) {
#pragma unroll
            for (int j = 0; j < 8; ++j) g[j] = 0.f;
            for (int q = 0; q < P.world; ++q) {
                const char* src = (const char*)P.acc_peer[(P.rank + q) % P.world] + e * 4;
                uint4 a = ld_peer16(src), b = ld_peer16(src + 16);
                g[0] += __uint_as_float(a.x); g[1] += __uint_as_float(a.y); g[2] += __uint_as_float(a.z); g[3] += __uint_as_float(a.w);
                g[4] += __uint_as_float(b.x); g[5] += __uint_as_float(b.y); g[6] += __uint_as_float(b.z); g[7] += __uint_as_float(b.w);
            }
        } else {
            const float4* src = reinterpret_cast<const float4*>((const char*)P.acc_peer[0] + e * 4);
            float4 a = src[0], b = src[1];
            g[0] = a.x; g[1] = a.y; g[2] = a.z; g[3] = a.w; g[4] = b.x; g[5] = b.y; g[6] = b.z; g[7] = b.w;
        }
    }
}

// Store 8 consecutive new parameter values at element `e` of every rank's shadow buffer.
template <typename O, int MODE>
ACCO_DEVINL void store_param8(const RoundParams& P, long long e, const float (&p)[8], bool local_only) {
    if constexpr (sizeof(O) == 2) {
        bf16x8 v = pack8(p);
        const uint4& r = *reinterpret_cast<const uint4*>(&v);
        if (MODE != 0 && local_only) {
            st_peer16((char*)P.theta_peer[P.rank] + e * 2, r);       // own copy only; peers pull it inside their GEMM
        } else if constexpr (MODE == 2) {
            multimem_st16((char*)P.theta_mc + e * 2, r);
        } else if constexpr (MODE == 1) {
#pragma unroll
            for (int q = 0; q < kMaxWorld; ++q)
                if (q < P.world) st_peer16((char*)P.theta_peer[(P.rank + q) % P.world] + e * 2, r);
        } else {
            st_stream((char*)P.theta_peer[0] + e * 2, v);
        }
    } else {
        uint4 a = make_uint4(__float_as_uint(p[0]), __float_as_uint(p[1]), __float_as_uint(p[2]), __float_as_uint(p[3]));
        uint4 b = make_uint4(__float_as_uint(p[4]), __float_as_uint(p[5]), __float_as_uint(p[6]), __float_as_uint(p[7]));
        if constexpr (MODE == 2) {
            multimem_st16((char*)P.theta_mc + e * 4, a);
            multimem_st16((char*)P.theta_mc + e * 4 + 16, b);
        } else if constexpr (MODE == 1) {
            for (int q = 0; q < P.world; ++q) {
                char* dst = (char*)P.theta_peer[(P.rank + q) % P.world] + e * 4;
                st_peer16(dst, a);
                st_peer16(dst + 16, b);
            }
        } else {
            float4* dst = reinterpret_cast<float4*>((char*)P.theta_peer[0] + e * 4);
            dst[0] = *reinterpret_cast<float4*>(&a);
            dst[1] = *reinterpret_cast<float4*>(&b);
        }
    }
}

// Start barrier of a round as its own one-warp kernel: publish my micro-batch count + "my accumulator is final" to every
// peer, then wait until every peer has done the same.  A rank that is ahead of its peers (heterogeneous speeds are the whole
// point of ACCO) waits HERE, holding 32 threads instead of a grid of 512-thread CTAs, so its next micro-batches keep the SMs.
__global__ void __launch_bounds__(32) round_gate_kernel(const __grid_constant__ RoundParams P) {
    const int W = P.world;
    const uint32_t epoch = *((volatile uint32_t*)P.epoch) + 1;
    if (threadIdx.x < W) {
        uint32_t* pad = P.pad_peer[threadIdx.x];
        st_relaxed_sys(pad + 2 * W + P.rank, (uint32_t)P.local_count);
        st_release_sys(pad + P.rank, epoch);
        wait_flag(P.pad_peer[P.rank] + threadIdx.x, epoch, P.watchdog_s);
    }
}

// NVLS rounds run as 256-thread x 64-register CTAs (16 K registers), one per SM.  The wgmma GEMM CTA (384 threads x 168 registers)
// takes the whole register file of its SM, so a round CTA and a GEMM CTA never share an SM: the round overlaps the compute only on
// SMs that no GEMM CTA holds (between GEMMs, or when a GEMM's grid is smaller than the GPU).  How much overlap that leaves on 8 GPUs
// is not measured.
// kSmall (experimental, ACCO_ROUND_LOCAL_SMALL=1, local mode only): give the single-GPU round the NVLS variant's footprint (256
// threads x <= 64 registers, one CTA per SM, max shared-memory carve-out).  Not measured; the default instantiations do not use it.
template <int MODE, bool kSmall = false> constexpr int round_threads() { return (MODE == 2 || kSmall) ? 256 : kAdamThreads; }

template <typename G, typename O, int MODE, bool kSmall = false>
__global__ void __launch_bounds__(round_threads<MODE, kSmall>(), (MODE == 2 || kSmall) ? 4 : 1) rs_adam_ag_kernel(const __grid_constant__ RoundParams P) {
    __shared__ int s_total;
    const int W = P.world;
    uint32_t epoch = 0;
    // ---------------- start barrier + count exchange ----------------
    if (MODE != 0) {
        epoch = *((volatile uint32_t*)P.epoch) + 1;
        if (!P.gated && blockIdx.x == 0 && threadIdx.x < W) {
            uint32_t* pad = P.pad_peer[threadIdx.x];                       // peer's pad
            st_relaxed_sys(pad + 2 * W + P.rank, (uint32_t)P.local_count);  // my count, then my flag (release orders both)
            st_release_sys(pad + P.rank, epoch);
        }
        if (!P.gated && threadIdx.x < W) {
            const uint32_t* mine = P.pad_peer[P.rank];
            wait_flag(mine + threadIdx.x, epoch, P.watchdog_s);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        int total = 0;
        if (MODE != 0) {
            const uint32_t* mine = P.pad_peer[P.rank];
            for (int q = 0; q < W; ++q) total += (int)ld_acquire_sys(mine + 2 * W + q);
        } else {
            total = P.local_count;
        }
        int upd = total + (P.add_stash ? *P.stash_count : 0);
        s_total = upd;
        if (blockIdx.x == 0) {
            *P.total_out = upd;
        }
    }
    __syncthreads();
    const float inv_count = P.inv_count_in ? *P.inv_count_in : 1.f / (float)max(s_total, 1);

    // ---------------- streaming pass over my slice ----------------
    const long long base = (long long)P.rank * P.slice;
    const long long nvec = P.slice >> 3;
    const float lr = P.lr, b1 = P.beta1, b2 = P.beta2, eps = P.eps;
    const float decay = 1.f - lr * P.weight_decay;
    const float step_size = lr / P.bc1;
    const bool cp = P.commit & 1, cs = P.commit & 2;
    // Memory-level parallelism: the NVSwitch round trip of a multimem.ld_reduce is several microseconds, so ONE load in flight per
    // thread leaves the reduce-scatter latency-bound (round 1: 0.43 of the link roofline).  Every thread therefore owns kU
    // independent vectors per iteration: all kU switch-reduced gradient loads (and the 3 x kU optimizer-state loads) are issued
    // back to back before the first result is consumed, and the kU multicast stores of the new weights leave while the next
    // iteration's loads are already in flight - reduce-scatter ingress and all-gather egress overlap inside one pass.
    // (measured at 8 GPUs: 4 loads in flight per thread bought nothing over 2 - 0.659 vs 0.648 ms, the round already runs at NCCL's
    // own NVLS all-reduce rate for the same bytes - while 128 registers/thread = the whole register file per 512-thread CTA kept
    // the round kernel from co-residing with the compute kernels it is supposed to overlap; hence 2, and <= 64 registers)
    constexpr int kU = kSmall ? 2 : ((MODE == 0) ? 4 : (MODE == 2 ? 2 : 1));      // p2p already has W peer loads in flight per vector
    const long long vstride = (long long)gridDim.x * blockDim.x;
    for (long long v0 = (long long)blockIdx.x * blockDim.x + threadIdx.x; v0 < nvec; v0 += vstride * kU) {
        float g[kU][8];
        if constexpr (MODE == 2 && sizeof(G) == 2) {
            uint4 raw[kU];
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                const long long v = v0 + u * vstride;
                if (v < nvec) raw[u] = multimem_ld_reduce_bf16x8((const char*)P.acc_mc + (base + (v << 3)) * 2);
            }
#pragma unroll
            for (int u = 0; u < kU; ++u) unpack8(*reinterpret_cast<bf16x8*>(&raw[u]), g[u]);
        } else {
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                const long long v = v0 + u * vstride;
                if (v < nvec) load_grad8<G, MODE>(P, base + (v << 3), g[u]);
            }
        }
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            const long long v = v0 + u * vstride;
            if (v >= nvec) continue;
            const long long i = v << 3;       // index inside my shard
            const float4* m4 = reinterpret_cast<const float4*>(P.exp_avg + i);
            const float4* v4 = reinterpret_cast<const float4*>(P.exp_avg_sq + i);
            const float4* p4 = reinterpret_cast<const float4*>(P.master + i);
            const float4 ma = m4[0], mb = m4[1], va = v4[0], vb = v4[1], pa = p4[0], pb = p4[1];
            float m[8] = {ma.x, ma.y, ma.z, ma.w, mb.x, mb.y, mb.z, mb.w};
            float vv[8] = {va.x, va.y, va.z, va.w, vb.x, vb.y, vb.z, vb.w};
            float p[8] = {pa.x, pa.y, pa.z, pa.w, pb.x, pb.y, pb.z, pb.w};
            float (&gg)[8] = g[u];
            if (P.add_stash) {
                const float4* s4 = reinterpret_cast<const float4*>(P.stash + i);
                const float4 sa = s4[0], sb = s4[1];
                gg[0] += sa.x; gg[1] += sa.y; gg[2] += sa.z; gg[3] += sa.w;
                gg[4] += sb.x; gg[5] += sb.y; gg[6] += sb.z; gg[7] += sb.w;
            }
            if (P.write_stash) {
                float4* s4 = reinterpret_cast<float4*>(P.stash + i);
                s4[0] = make_float4(gg[0], gg[1], gg[2], gg[3]);
                s4[1] = make_float4(gg[4], gg[5], gg[6], gg[7]);
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float gj = gg[j] * inv_count;
                m[j] = m[j] + (1.f - b1) * (gj - m[j]);                 // lerp, as torch
                vv[j] = b2 * vv[j] + (1.f - b2) * gj * gj;
                const float denom = sqrtf(vv[j]) * P.bc2_rsqrt + eps;
                p[j] = p[j] * decay - step_size * (m[j] / denom);
            }
            if (cp) {
                float4* o = reinterpret_cast<float4*>(P.master + i);
                o[0] = make_float4(p[0], p[1], p[2], p[3]);
                o[1] = make_float4(p[4], p[5], p[6], p[7]);
            }
            if (cs) {
                float4* om = reinterpret_cast<float4*>(P.exp_avg + i);
                float4* ov = reinterpret_cast<float4*>(P.exp_avg_sq + i);
                om[0] = make_float4(m[0], m[1], m[2], m[3]);
                om[1] = make_float4(m[4], m[5], m[6], m[7]);
                ov[0] = make_float4(vv[0], vv[1], vv[2], vv[3]);
                ov[1] = make_float4(vv[4], vv[5], vv[6], vv[7]);
            }
            store_param8<O, MODE>(P, base + i, p, MODE != 0 && P.n_skip > 0 && in_skip(P, base + i));
        }
    }

    // ---------------- end barrier (last CTA) ----------------
    if (MODE != 0) __threadfence_system();
    __syncthreads();
    __shared__ bool s_last;
    if (threadIdx.x == 0) {
        __threadfence();
        const uint32_t prev = atomicAdd(P.done_ctas, 1u);
        s_last = (prev == gridDim.x - 1);
    }
    __syncthreads();
    if (!s_last) return;
    if (threadIdx.x == 0) {
        *P.done_ctas = 0;
        if (P.write_stash) *P.stash_count = s_total;          // count represented by the stash
        else if (P.add_stash) *P.stash_count = 0;
    }
    if (MODE != 0) {
        __threadfence_system();
        if (threadIdx.x < W) {
            st_release_sys(P.pad_peer[threadIdx.x] + W + P.rank, epoch);
            const uint32_t* mine = P.pad_peer[P.rank];
            wait_flag(mine + W + threadIdx.x, epoch, P.watchdog_s);
        }
        __syncthreads();
        if (threadIdx.x == 0) *P.epoch = epoch;
    }
}

// The round shares SMs with the wgmma GEMMs, which run with the maximum shared-memory carve-out.  An SM is only
// re-partitioned between L1 and shared memory when it is idle, so a kernel that prefers another carve-out can never be co-resident with
// them - it waits for the SM to drain (tools/coresidency_check.py checks this).
// Ask for the same configuration.
template <typename G, typename O, int MODE>
static void prefer_max_smem_carveout() {
    static bool done = false;
    if (!done) {
        cudaFuncSetAttribute(rs_adam_ag_kernel<G, O, MODE>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        done = true;
    }
}

static bool local_small() {
    static const bool on = [] { const char* e = getenv("ACCO_ROUND_LOCAL_SMALL"); return e && e[0] == '1'; }();
    return on;
}

template <typename G, typename O>
static void launch_mode(const RoundParams& P, int mode, int grid, cudaStream_t st) {
    if (mode == 1) prefer_max_smem_carveout<G, O, 1>();
    else if (mode == 2) prefer_max_smem_carveout<G, O, 2>();
    if (mode == 0 && local_small()) {
        static bool attr = false;
        static int sms = 0;
        if (!attr) {
            cudaFuncSetAttribute(rs_adam_ag_kernel<G, O, 0, true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
            int dev = 0;
            cudaGetDevice(&dev);
            cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
            attr = true;
        }
        if (sms > 0 && grid > sms) grid = sms;           // one 256-thread CTA per SM, like the NVLS rounds
        rs_adam_ag_kernel<G, O, 0, true><<<grid, round_threads<0, true>(), 0, st>>>(P);
        return;
    }
    if (mode == 0) rs_adam_ag_kernel<G, O, 0><<<grid, round_threads<0>(), 0, st>>>(P);
    else if (mode == 1) rs_adam_ag_kernel<G, O, 1><<<grid, round_threads<1>(), 0, st>>>(P);
    else rs_adam_ag_kernel<G, O, 2><<<grid, round_threads<2>(), 0, st>>>(P);
}

}  // namespace acco

// grad_bf16 / out_bf16: element types of accumulator and shadow parameter buffer.
// mode: 0 local (world==1), 1 P2P, 2 NVLS multicast.
extern "C" int acco_rs_adam_ag(const acco::RoundParams* P, int grad_bf16, int out_bf16, int mode, int grid, cudaStream_t st) {
    using namespace acco;
    if (P->slice % 8 != 0 || P->world > kMaxWorld) return -1;
    if (mode != 0 && P->gated) {
        static bool gate_attr = false;
        if (!gate_attr) { cudaFuncSetAttribute(round_gate_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared); gate_attr = true; }
        round_gate_kernel<<<1, 32, 0, st>>>(*P);
    }
    if (grad_bf16 && out_bf16) launch_mode<__nv_bfloat16, __nv_bfloat16>(*P, mode, grid, st);
    else if (!grad_bf16 && !out_bf16) launch_mode<float, float>(*P, mode, grid, st);
    else if (grad_bf16 && !out_bf16) launch_mode<__nv_bfloat16, float>(*P, mode, grid, st);
    else launch_mode<float, __nv_bfloat16>(*P, mode, grid, st);
    return (int)cudaGetLastError();
}

extern "C" int acco_round_params_size() { return (int)sizeof(acco::RoundParams); }
