// ovc_b200.cu — sm_90a (H100) kernels + C ABI (include/ovc_b200.h) of the batched Overcooked engine.
//
// K1  step_kernel<S, IO>     one joint transition of a tile of TILE environments per CTA.
//     IO = 1  the tile [TILE][S] int32 is brought into shared memory by ONE 2-D tensor-map TMA load
//             (cp.async.bulk.tensor.2d, SASS UTMALDG) with the hardware 64B/128B swizzle, so that the
//             per-thread 16-byte record-chunk accesses (stride = one record) are bank-conflict free;
//             threads update their record in place; one TMA tensor store (UTMASTG) writes it back.
//     IO = 2  same, with a 1-D bulk copy (cp.async.bulk, SASS UBLKCP) and a linear tile.
//     IO = 3  no staging: each thread reads / writes its record's chunks in global memory.
// K5  rollout_kernel<S, IO>  T transitions with the tile resident in shared memory.
// K4  reset_kernel           masked copy of the per-layout start record.
// The observation kernels (K2 lossless encode, K3 featurize) live in ovc_obs.cuh, K7 (first policy layer on the
// encoding, evaluated from the record) and the draw / return kernels in ovc_encfc.cuh, K8 (dense tail of the policy +
// the draw, one kernel) in ovc_tail.cuh, K9 (the policy's two wide layers as one wgmma kernel) in ovc_wide.cuh, K10 (the
// behaviour-cloned partner: featurize_state + its MLP + the draw, one kernel) and the partner seat draw in ovc_partner.cuh.
//
// The environment path is integer, branchy and HBM-bound (no contraction anywhere): no tensor cores there.  The policy-in-
// the-loop kernels K8 / K9 (config 5) are the contractions and use them.
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/ovc_b200.h"
#include "ovc_step.cuh"

namespace ovc {

// ------------------------------------------------------------------------------------------------
// error plumbing
// ------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";

static int fail(int code, const char *msg) {
    snprintf(g_err, sizeof g_err, "%s", msg);
    return code;
}
static int fail(int code, const char *msg, long long value) {
    snprintf(g_err, sizeof g_err, "%s (got %lld)", msg, value);
    return code;
}
static int cuda_fail(cudaError_t e, const char *what) {
    snprintf(g_err, sizeof g_err, "%s: %s", what, cudaGetErrorString(e));
    return OVC_E_CUDA;
}

// ------------------------------------------------------------------------------------------------
// PTX helpers: mbarrier + TMA (bulk async copies)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    } while (!ok);
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, int c0, int c1, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
        ::"r"(smem_u32(dst)), "l"((uint64_t)map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap *map, int c0, int c1, const void *src) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%1, %2}], [%3];" ::"l"((uint64_t)map),
                 "r"(c0), "r"(c1), "r"(smem_u32(src))
                 : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap *map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)map) : "memory");
}
// brings the line holding p into L2 (no register written, nothing to wait on)
__device__ __forceinline__ void prefetch_l2(const void *p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
__device__ __forceinline__ void bulk_load_1d(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"((uint64_t)src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void bulk_store_1d(void *dst, const void *src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"((uint64_t)dst), "r"(smem_u32(src)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}

// ------------------------------------------------------------------------------------------------
// record accessors
// ------------------------------------------------------------------------------------------------
// Shared-memory tile.  SWZ = number of 16-byte-chunk index bits the TMA swizzle XORs with address
// bits 7.. (2: CU_TENSOR_MAP_SWIZZLE_64B for 64-byte records, 3: SWIZZLE_128B, 0: linear tile).
template <int S, int SWZ>
struct SmemRec {
    char *tile;     // 1024-byte aligned tile base
    uint32_t base;  // byte offset of this thread's record inside the tile
    __device__ __forceinline__ uint32_t phys(uint32_t off) const {
        if (SWZ == 0) return off;
        return off ^ (((off >> 7) & ((1u << SWZ) - 1u)) << 4);
    }
    __device__ __forceinline__ int4 ld4(int c) const { return *reinterpret_cast<const int4 *>(tile + phys(base + c * 16)); }
    __device__ __forceinline__ void st4(int c, int4 v) { *reinterpret_cast<int4 *>(tile + phys(base + c * 16)) = v; }
    __device__ __forceinline__ int ldw(int w) const { return *reinterpret_cast<const int *>(tile + phys(base + w * 4)); }
    __device__ __forceinline__ void stw(int w, int v) { *reinterpret_cast<int *>(tile + phys(base + w * 4)) = v; }
};

struct GlobalRec {
    int32_t *rec;
    __device__ __forceinline__ int4 ld4(int c) const { return *reinterpret_cast<const int4 *>(rec + c * 4); }
    __device__ __forceinline__ void st4(int c, int4 v) { *reinterpret_cast<int4 *>(rec + c * 4) = v; }
    __device__ __forceinline__ int ldw(int w) const { return rec[w]; }
    __device__ __forceinline__ void stw(int w, int v) { rec[w] = v; }
};

#ifndef OVC_TILE16
#define OVC_TILE16 128
#endif

template <int S>
struct Cfg {
    static constexpr int TILE = S <= 16 ? OVC_TILE16 : S <= 32 ? 128 : 64;  // environments (= threads) per CTA
    static constexpr int ROW_WORDS = S == 16 ? 16 : 32;     // tensor-map row: 64 B or 128 B
    static constexpr int ROWS_PER_ENV = S / ROW_WORDS;      // 1, 1, 2, 4
    static constexpr int BOX_ROWS = TILE * ROWS_PER_ENV;    // <= 256
    static constexpr int SWZ = S == 16 ? 2 : 3;
    static constexpr int TILE_BYTES = TILE * S * 4;
};

struct StepArgs {
    const ovc_layout_t *layouts;
    const int32_t *start_records;
    int32_t *state;
    const int32_t *actions;
    int32_t *sparse, *shaped, *done, *events;
    long long n_envs;
    int n_layouts;
    int n_steps;  // rollout only
    int horizon, flags;
    int has_rs;
    ovc_random_start_t rs;
};

// 25-bit event mask (+ delivered recipe in bits 25-28) of ONE agent -> 5-bit code (see OVC_F_OUT_PACKED)
__device__ __forceinline__ unsigned event_code(unsigned ev) {
    if ((ev & 0x1FFFFFFu) == 0) return 0;
    if (ev & (1u << OVC_EV_SOUP_DELIVERY)) {
        const unsigned row = (ev >> OVC_EV_RECIPE_SHIFT) & 15u;  // rows 1,2,3,4,5,6,8,9,12 -> ranks 0..8
        return 23u + (unsigned)((0x0008007605432100ull >> (row * 4)) & 15u);
    }
    if (ev & ((1u << OVC_EV_POTTING_ONION) | (1u << OVC_EV_POTTING_TOMATO))) {
        const unsigned tom = (ev >> OVC_EV_POTTING_TOMATO) & 1u;
        const unsigned viable = (ev >> (OVC_EV_VIABLE_ONION_POTTING + tom)) & 1u, optimal = (ev >> (OVC_EV_OPTIMAL_ONION_POTTING + tom)) & 1u;
        const unsigned cata = (ev >> (OVC_EV_CATASTROPHIC_ONION_POTTING + tom)) & 1u;
        return 15u + tom * 4u + (viable ? (optimal ? 0u : 1u) : (cata ? 2u : 3u));
    }
    if (ev & (1u << OVC_EV_SOUP_PICKUP)) return 7;
    if (ev & (1u << OVC_EV_SOUP_DROP)) return 14;
    if (ev & (1u << OVC_EV_ONION_PICKUP)) return 1u + ((ev >> OVC_EV_USEFUL_ONION_PICKUP) & 1u);
    if (ev & (1u << OVC_EV_TOMATO_PICKUP)) return 3u + ((ev >> OVC_EV_USEFUL_TOMATO_PICKUP) & 1u);
    if (ev & (1u << OVC_EV_DISH_PICKUP)) return 5u + ((ev >> OVC_EV_USEFUL_DISH_PICKUP) & 1u);
    if (ev & (1u << OVC_EV_ONION_DROP)) return 8u + ((ev >> OVC_EV_USEFUL_ONION_DROP) & 1u);
    if (ev & (1u << OVC_EV_TOMATO_DROP)) return 10u + ((ev >> OVC_EV_USEFUL_TOMATO_DROP) & 1u);
    return 12u + ((ev >> OVC_EV_USEFUL_DISH_DROP) & 1u);  // dish_drop
}

// WIDE: the kernel instantiation for int32 actions and int32 outputs (the device-resident formats) — it carries
// none of the format tests below, which cost 3 % of a fused-rollout transition when they sat in every instantiation.
template <bool WIDE>
__device__ __forceinline__ void write_outputs(const StepArgs &a, long long idx, const StepOut &o) {
    if (!WIDE && (a.flags & OVC_F_OUT_CODES)) {  // 2 bytes per env-step: rewards are functions of the codes + two grant bits
        reinterpret_cast<unsigned short *>(a.events)[idx] =
            (unsigned short)(event_code(o.ev0) | (event_code(o.ev1) << 5) | ((unsigned)o.done << 10) |
                             ((o.ev0 & OVC_EVF_STEPPED_DONE) ? 1u << 11 : 0u) | (o.shaped0 != 0 ? 1u << 12 : 0u) |
                             (o.shaped1 != 0 ? 1u << 13 : 0u));
        return;
    }
    if (!WIDE && (a.flags & OVC_F_OUT_PACKED)) {  // 6 bytes per env-step for host transfer
        reinterpret_cast<short *>(a.sparse)[idx] = (short)o.sparse;
        reinterpret_cast<char2 *>(a.shaped)[idx] = make_char2((signed char)o.shaped0, (signed char)o.shaped1);
        reinterpret_cast<unsigned short *>(a.events)[idx] =
            (unsigned short)(event_code(o.ev0) | (event_code(o.ev1) << 5) | ((unsigned)o.done << 10) |
                             ((o.ev0 & OVC_EVF_STEPPED_DONE) ? 1u << 11 : 0u));
        return;
    }
    if (!WIDE && (a.flags & OVC_F_OUT_NARROW)) {  // uniform branch: int16 / int8x2 / uint8 for host transfer
        reinterpret_cast<short *>(a.sparse)[idx] = (short)o.sparse;
        reinterpret_cast<unsigned char *>(a.done)[idx] = (unsigned char)o.done;
        reinterpret_cast<char2 *>(a.shaped)[idx] = make_char2((signed char)o.shaped0, (signed char)o.shaped1);
    } else {
        a.sparse[idx] = o.sparse;
        a.done[idx] = o.done;
        reinterpret_cast<int2 *>(a.shaped)[idx] = make_int2(o.shaped0, o.shaped1);
    }
    reinterpret_cast<int2 *>(a.events)[idx] = make_int2((int)o.ev0, (int)o.ev1);
}

// address of joint-action element idx: int32 pairs (8 B), OVC_F_ACT_U8 (2 B) or OVC_F_ACT_PACKED (1 B)
template <bool WIDE, typename I>
__device__ __forceinline__ const void *action_addr(const StepArgs &a, I idx) {
    if (!WIDE && (a.flags & OVC_F_ACT_PACKED)) return reinterpret_cast<const unsigned char *>(a.actions) + idx;
    if (!WIDE && (a.flags & OVC_F_ACT_U8)) return reinterpret_cast<const uchar2 *>(a.actions) + idx;
    return reinterpret_cast<const int2 *>(a.actions) + idx;
}

template <bool WIDE, typename I>
__device__ __forceinline__ int2 load_action(const StepArgs &a, I idx) {
    if (!WIDE && (a.flags & OVC_F_ACT_PACKED)) {
        const unsigned u = *static_cast<const unsigned char *>(action_addr<WIDE>(a, idx));
        return make_int2((int)(u & 15u), (int)(u >> 4));
    }
    if (!WIDE && (a.flags & OVC_F_ACT_U8)) {
        const uchar2 u = *static_cast<const uchar2 *>(action_addr<WIDE>(a, idx));
        return make_int2(u.x, u.y);
    }
    return *static_cast<const int2 *>(action_addr<WIDE>(a, idx));
}

// Shared-memory plan of one CTA (dynamic, 1024-byte aligned so the TMA swizzle pattern lines up with
// the tile offsets): [ tile: TILE*S*4 bytes ][ layout tables: n_tbl*1024 bytes ][ mbarrier: 8 bytes ].
constexpr int MAX_SMEM_LAYOUTS = 8;

// One CTA = one tile of TILE records.  n_steps == 1: the step kernel K1; n_steps > 1: the fused rollout K5.
template <int S, int IO, bool RS, bool WIDE>
__global__ void __launch_bounds__(Cfg<S>::TILE)
step_kernel(const __grid_constant__ CUtensorMap tmap, const StepArgs a) {
    using C = Cfg<S>;
    const long long env0 = (long long)blockIdx.x * C::TILE;
    const long long env = env0 + threadIdx.x;
    const bool live = env < a.n_envs;
    const int T = a.n_steps;

    if (IO == 3) {
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
        asm volatile("griddepcontrol.wait;" ::: "memory");
        if (!live) return;
        GlobalRec r{a.state + env * S};
        const TblG tb{reinterpret_cast<const char *>(a.layouts)};
        for (int t = 0; t < T; t++) {
            const long long idx = (long long)t * a.n_envs + env;
            const int2 act = load_action<WIDE>(a, idx);
            StepOut o;
            step_core<RS>(r, tb, a.start_records, S, act.x, act.y, a.horizon, a.flags, RS ? &a.rs : nullptr, env, a.n_layouts, o);
            write_outputs<WIDE>(a, idx, o);
        }
        return;
    }

    extern __shared__ __align__(1024) char smem[];
    char *tile = smem;
    const int n_tbl = a.n_layouts <= MAX_SMEM_LAYOUTS ? a.n_layouts : 0;  // 0: tables stay in global memory
    const uint32_t tbl_bytes = (uint32_t)n_tbl * (uint32_t)sizeof(ovc_layout_t);
    char *tbl = smem + C::TILE_BYTES;
    uint64_t *bar = reinterpret_cast<uint64_t *>(smem + C::TILE_BYTES + tbl_bytes);  // host sizes the buffer the same way
    const long long rem = a.n_envs - env0;
    const uint32_t live_bytes = (uint32_t)((rem < C::TILE ? rem : C::TILE) * S * 4);

    if (threadIdx.x == 0) {
        mbar_init(bar, 1);
        mbar_expect_tx(bar, (IO == 1 ? (uint32_t)C::TILE_BYTES : live_bytes) + tbl_bytes);
        if (IO == 1) prefetch_tmap(&tmap);
        if (n_tbl) bulk_load_1d(tbl, a.layouts, tbl_bytes, bar);  // the constant table rides on the same barrier
    }
    // Programmatic dependent launch: everything above touches only constants, so it may overlap the
    // previous kernel of the stream; state and actions are read after the dependency resolves.
    // (Both instructions are no-ops when the kernel was launched without the PDL attribute.)
    asm volatile("griddepcontrol.wait;" ::: "memory");
    if (threadIdx.x == 0) {
        if (IO == 1) tma_load_2d(tile, &tmap, 0, (int)(env0 * C::ROWS_PER_ENV), bar);  // out-of-range rows: zero fill, still counted
        else bulk_load_1d(tile, a.state + env0 * S, live_bytes, bar);
    }
    // the first action fetch overlaps the tile load
    int2 act = make_int2(OVC_A_STAY, OVC_A_STAY);
    if (live) act = load_action<WIDE>(a, env);
    __syncthreads();  // barrier initialised and visible before anyone polls it
    mbar_wait(bar, 0);
    // Programmatic dependent launch: once the tile has landed, the next kernel of the stream may be
    // scheduled; its prologue (barrier init, tensor-map prefetch, table fetch) then overlaps this
    // kernel's compute, and its griddepcontrol.wait holds it until this grid has completed.
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

    if (live) {
        SmemRec<S, IO == 1 ? C::SWZ : 0> r{tile, (uint32_t)threadIdx.x * S * 4};
        auto run = [&](auto tb) {
            for (int t = 0; t < T; t++) {
                const long long idx = (long long)t * a.n_envs + env;
                int2 nxt = act;
                if (t + 1 < T) nxt = load_action<WIDE>(a, idx + a.n_envs);  // prefetch
                StepOut o;
                step_core<RS>(r, tb, a.start_records, S, act.x, act.y, a.horizon, a.flags, RS ? &a.rs : nullptr, env, a.n_layouts, o);
                write_outputs<WIDE>(a, idx, o);
                act = nxt;
            }
        };
        if (n_tbl) run(TblS{tbl});
        else run(TblG{reinterpret_cast<const char *>(a.layouts)});
    }
    fence_async_smem();  // generic-proxy writes -> visible to the async proxy (TMA store)
    __syncthreads();
    if (threadIdx.x == 0) {
        if (IO == 1) tma_store_2d(&tmap, 0, (int)(env0 * C::ROWS_PER_ENV), tile);  // rows past the end are clipped
        else bulk_store_1d(a.state + env0 * S, tile, live_bytes);
        bulk_commit();
        bulk_wait_read<0>();  // shared memory must stay alive until the TMA engine has read it
    }
}

}  // namespace ovc

#include "ovc_rollout.cuh"

namespace ovc {

__global__ void reset_kernel(const int32_t *__restrict__ start_records, int n_layouts, int32_t *__restrict__ state,
                             const int32_t *__restrict__ env_layout, const int32_t *__restrict__ mask,
                             long long n_envs, int S) {
    // one thread per 16-byte chunk: coalesced int4 stores
    const int cpr = S / 4;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_envs * cpr) return;
    const long long env = i / cpr;
    const int c = (int)(i % cpr);
    if (mask && mask[env] == 0) return;
    int lid = env_layout ? env_layout[env] : (state[env * S + 3] & 0xFF);
    if (lid < 0 || lid >= n_layouts) lid = 0;
    reinterpret_cast<int4 *>(state)[i] = __ldg(reinterpret_cast<const int4 *>(start_records) + (long long)lid * cpr + c);
}

// Random start states: one thread per environment draws its record (get_random_start_state_fn :1307-1369).
__global__ void reset_random_kernel(const ovc_layout_t *__restrict__ layouts, int n_layouts,
                                    const int32_t *__restrict__ start_records, int32_t *__restrict__ state,
                                    const int32_t *__restrict__ env_layout, const int32_t *__restrict__ mask,
                                    long long n_envs, int S, const ovc_random_start_t rs) {
    const long long env = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= n_envs) return;
    if (mask && mask[env] == 0) return;
    int32_t *rec = state + env * S;
    const unsigned old = (unsigned)rec[3];
    int lid = env_layout ? env_layout[env] : (int)(old & 0xFF);
    const unsigned episode = ((old >> 16) + 1u) & 0xFFFFu;
    if (rs.random_layout) lid = random_layout_id(rs, (uint64_t)env, episode, n_layouts);  // variable MDP
    if (lid < 0 || lid >= n_layouts) lid = 0;
    const ovc_layout_t *L = layouts + lid;
    random_start_record([&](int w, int32_t v) { rec[w] = v; }, S, start_records + (size_t)lid * S, L->cook_time, L->free_pos,
                        L->n_free, L->n_pots, lid, rs, (uint64_t)env, episode);
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*encode_tiled_fn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                    const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static encode_tiled_fn get_encode_fn() {
    static encode_tiled_fn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (encode_tiled_fn)p;
    }
    return fn;
}

template <int S>
static int make_tmap(CUtensorMap *m, int32_t *state, long long n_envs, int box_rows = Cfg<S>::BOX_ROWS) {
    using C = Cfg<S>;
    encode_tiled_fn enc = get_encode_fn();
    if (!enc) return fail(OVC_E_CUDA, "cuTensorMapEncodeTiled entry point not available");
    cuuint64_t dims[2] = {(cuuint64_t)C::ROW_WORDS, (cuuint64_t)(n_envs * C::ROWS_PER_ENV)};
    cuuint64_t strides[1] = {(cuuint64_t)C::ROW_WORDS * 4};
    cuuint32_t box[2] = {(cuuint32_t)C::ROW_WORDS, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_INT32, 2, state, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     S == 16 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(OVC_E_CUDA, "cuTensorMapEncodeTiled failed", (long long)r);
    return OVC_OK;
}

template <int S, int IO>
static cudaError_t launch_one(const CUtensorMap &tmap, const StepArgs &a, unsigned grid, size_t smem, cudaStream_t st) {
    using C = Cfg<S>;
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.gridDim = dim3(grid), cfg.blockDim = dim3(C::TILE), cfg.dynamicSmemBytes = smem, cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = (a.flags & OVC_F_PDL) ? 1 : 0;
    const bool wide = !(a.flags & (OVC_F_ACT_U8 | OVC_F_ACT_PACKED | OVC_F_OUT_NARROW | OVC_F_OUT_PACKED | OVC_F_OUT_CODES));
    if (a.has_rs)
        return wide ? cudaLaunchKernelEx(&cfg, step_kernel<S, IO, true, true>, tmap, a)
                    : cudaLaunchKernelEx(&cfg, step_kernel<S, IO, true, false>, tmap, a);
    return wide ? cudaLaunchKernelEx(&cfg, step_kernel<S, IO, false, true>, tmap, a)
                : cudaLaunchKernelEx(&cfg, step_kernel<S, IO, false, false>, tmap, a);
}

// ---- K5: the fused rollout kernel (ovc_rollout.cuh) ----
template <int S, int TILE>
static int launch_rollout(const StepArgs &a, cudaStream_t st) {
    using C = RollCfg<S, TILE>;
    CUtensorMap tmap;
    memset(&tmap, 0, sizeof tmap);
    int rc = make_tmap<S>(&tmap, a.state, a.n_envs, C::BOX_ROWS);
    if (rc) return rc;
    const size_t smem = C::smem_bytes(a.n_layouts);
    const bool wide = !(a.flags & (OVC_F_ACT_U8 | OVC_F_ACT_PACKED | OVC_F_OUT_NARROW | OVC_F_OUT_PACKED | OVC_F_OUT_CODES | OVC_F_OUT_STREAM));
    const bool stream = a.flags & OVC_F_OUT_STREAM;
    void (*kern)(const CUtensorMap, const StepArgs) =
        a.has_rs ? (wide ? rollout_kernel<S, TILE, true, FMT_WIDE> : stream ? rollout_kernel<S, TILE, true, FMT_STREAM> : rollout_kernel<S, TILE, true, FMT_HOST>)
                 : (wide ? rollout_kernel<S, TILE, false, FMT_WIDE> : stream ? rollout_kernel<S, TILE, false, FMT_STREAM> : rollout_kernel<S, TILE, false, FMT_HOST>);
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return cuda_fail(e, "rollout kernel shared-memory attribute");
    }
    const long long grid = (a.n_envs + TILE - 1) / TILE;
    StepArgs ka = a;
    ka.flags &= ~F_K5_NO_PREFETCH;
#if OVC_K5_PREFETCH > 1
    // The action prefetch pays in a middle range of warps per SM.  With many warps the others hide the action load; with
    // very few, a transition's own chain outlasts the (then short) DRAM latency, so the load is not on the path either, and
    // in both cases the prefetch only adds instructions.  The last wave of a grid larger than one wave runs with few
    // warps while the rest of the SM is idle, so there the prefetch stays on.  cramped_room, TILE = 64, on an H100 (132 SMs):
    // 16 384 envs (3.9 warps per SM) 4 % slower with it, 32 768 (7.8) about even, 65 536 (15.5) 13 % faster, 131 072
    // (31, one wave) 3 % slower; asymmetric_advantages at 131 072 envs (two waves) 17 % faster.
    {
        int dev = 0, n_sm = 0, per_sm = 0;
        cudaError_t e = cudaGetDevice(&dev);
        if (e == cudaSuccess) e = cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
        if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, TILE, smem);
        if (e != cudaSuccess) return cuda_fail(e, "rollout kernel occupancy");
        const long long warps = grid * (TILE / 32);
        if (grid <= (long long)per_sm * n_sm && (warps >= 24LL * n_sm || warps < 12LL * n_sm)) ka.flags |= F_K5_NO_PREFETCH;
    }
#endif
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.gridDim = dim3((unsigned)grid), cfg.blockDim = dim3(TILE), cfg.dynamicSmemBytes = smem, cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    // Programmatic dependent launch is for the microsecond-long per-transition kernel.  Here it only lets the next launch's
    // CTAs sit on the SMs beside a kernel that runs for hundreds of microseconds: slower with back-to-back launches of
    // 1-warp CTAs, nothing gained with larger CTAs.  Not used.
    cfg.numAttrs = 0;
    cudaError_t e = cudaLaunchKernelEx(&cfg, kern, tmap, ka);
    if (e != cudaSuccess) return cuda_fail(e, "rollout kernel launch");
    return OVC_OK;
}

// environments per CTA of the rollout kernel: 2 warps per CTA; a many-layout
// table set (4.5 KB of shared memory per layout and CTA) wants the largest tile so that enough CTAs fit an SM.  One warp
// per CTA is as fast at 65 536 environments and slower above.  OVC_K5_TILE overrides (tuning hook).
static int rollout_tile(int S, long long n_envs, int n_layouts) {
    static int forced = -1;
    if (forced < 0) {
        const char *e = getenv("OVC_K5_TILE");
        forced = e ? atoi(e) : 0;
    }
    (void)n_envs;
    if (S > 32) return 64;
    if (forced == 32 || forced == 64 || forced == 128) return forced;
    return n_layouts >= 3 ? 128 : 64;
}

// true: handled by the rollout kernel; false: the caller falls back to step_kernel with n_steps > 1
static bool use_rollout_kernel(const StepArgs &a, int io) {
    static int off = -1;
    if (off < 0) {
        const char *e = getenv("OVC_K5_LEGACY");  // measure / test the pre-round-2 fused path
        off = e && atoi(e) ? 1 : 0;
    }
    const bool stream = a.flags & OVC_F_OUT_STREAM;  // only the rollout kernel produces the sparse stream (step_impl checked it can)
    return (!off || stream) && (a.n_steps > 1 || stream) && a.n_steps <= ROLLOUT_MAX_STEPS && io == 1 && a.n_layouts <= MAX_SMEM_LAYOUTS;
}

template <int S>
static int launch_rollout_tiled(const StepArgs &a, cudaStream_t st) {
    if constexpr (S > 32) {
        return launch_rollout<S, 64>(a, st);
    } else {
        switch (rollout_tile(S, a.n_envs, a.n_layouts)) {
        case 32: return launch_rollout<S, 32>(a, st);
        case 64: return launch_rollout<S, 64>(a, st);
        default: return launch_rollout<S, 128>(a, st);
        }
    }
}

// The rollout kernel addresses its action / output rows with 32-bit element indices: a rollout of more than 2^32
// env-steps is cut into consecutive launches (same stream, same semantics).
template <int S>
static int launch_rollout_any(const StepArgs &a0, cudaStream_t st) {
    long long max_steps = 0xFFFFFFFFLL / a0.n_envs - 1;
    {
        static long long cap = -1;  // OVC_K5_MAX_LAUNCH_STEPS: test hook, cuts rollouts into launches of at most that many transitions
        if (cap < 0) {
            const char *e = getenv("OVC_K5_MAX_LAUNCH_STEPS");
            cap = e ? atoll(e) : 0;
        }
        if (cap > 0 && cap < max_steps && !(a0.flags & OVC_F_OUT_STREAM)) max_steps = cap;
    }
    if (a0.n_steps <= max_steps) return launch_rollout_tiled<S>(a0, st);
    if (max_steps < 1 || (a0.flags & OVC_F_OUT_STREAM)) return fail(OVC_E_UNSUPPORTED, "rollout too large for one launch (n_steps * n_envs must stay below 2^32)");
    // bytes per env-step of each array in this transfer format (the table of ovc_host.cuh: formats_of)
    const int f = a0.flags;
    const int b_act = (f & OVC_F_ACT_PACKED) ? 1 : (f & OVC_F_ACT_U8) ? 2 : 8;
    int b_sparse = 4, b_shaped = 8, b_done = 4, b_events = 8;
    if (f & OVC_F_OUT_CODES) b_sparse = 0, b_shaped = 0, b_done = 0, b_events = 2;
    else if (f & OVC_F_OUT_PACKED) b_sparse = 2, b_shaped = 2, b_done = 0, b_events = 2;
    else if (f & OVC_F_OUT_NARROW) b_sparse = 2, b_shaped = 2, b_done = 1, b_events = 8;
    for (long long t0 = 0; t0 < a0.n_steps; t0 += max_steps) {
        StepArgs a = a0;
        const long long off = t0 * a0.n_envs;
        a.n_steps = (int)(a0.n_steps - t0 < max_steps ? a0.n_steps - t0 : max_steps);
        a.actions = reinterpret_cast<const int32_t *>(reinterpret_cast<const char *>(a0.actions) + off * b_act);
        if (a0.sparse) a.sparse = reinterpret_cast<int32_t *>(reinterpret_cast<char *>(a0.sparse) + off * b_sparse);
        if (a0.shaped) a.shaped = reinterpret_cast<int32_t *>(reinterpret_cast<char *>(a0.shaped) + off * b_shaped);
        if (a0.done) a.done = reinterpret_cast<int32_t *>(reinterpret_cast<char *>(a0.done) + off * b_done);
        a.events = reinterpret_cast<int32_t *>(reinterpret_cast<char *>(a0.events) + off * b_events);
        const int rc = launch_rollout_tiled<S>(a, st);
        if (rc) return rc;
    }
    return OVC_OK;
}

template <int S>
static int launch_step(const StepArgs &a, int io, cudaStream_t st) {
    using C = Cfg<S>;
    if (use_rollout_kernel(a, io)) return launch_rollout_any<S>(a, st);
    const unsigned grid = (unsigned)((a.n_envs + C::TILE - 1) / C::TILE);
    CUtensorMap tmap;
    memset(&tmap, 0, sizeof tmap);
    const int n_tbl = a.n_layouts <= MAX_SMEM_LAYOUTS ? a.n_layouts : 0;
    const size_t smem = io == 3 ? 0 : C::TILE_BYTES + (size_t)n_tbl * sizeof(ovc_layout_t) + 16;
    cudaError_t e;
    if (io == 1) {
        int rc = make_tmap<S>(&tmap, a.state, a.n_envs);
        if (rc) return rc;
        e = launch_one<S, 1>(tmap, a, grid, smem, st);
    } else if (io == 2) {
        e = launch_one<S, 2>(tmap, a, grid, smem, st);
    } else {
        e = launch_one<S, 3>(tmap, a, grid, smem, st);
    }
    if (e != cudaSuccess) return cuda_fail(e, "step kernel launch");
    return OVC_OK;
}

static int check_common(const void *layouts, int n_layouts, const void *state, long long n_envs, int S) {
    if (!layouts || !state) return fail(OVC_E_BADARG, "null pointer argument");
    if (n_layouts <= 0 || n_layouts > 256) return fail(OVC_E_BADARG, "n_layouts must be 1..256", (long long)(n_layouts));
    if (n_envs < 0) return fail(OVC_E_BADARG, "negative n_envs");
    if (S != 16 && S != 32 && S != 64 && S != 128)
        return fail(OVC_E_BADARG, "state_words must be 16, 32, 64 or 128", (long long)(S));
    if (((uintptr_t)state & 15) != 0) return fail(OVC_E_BADARG, "state must be 16-byte aligned");
    return OVC_OK;
}

static int step_impl(const void *layouts, int n_layouts, const int32_t *start_records, int32_t *state,
                     const int32_t *actions, int32_t *sparse, int32_t *shaped, int32_t *done, int32_t *events,
                     long long n_envs, int n_steps, int S, int horizon, int flags, const ovc_random_start_t *rs,
                     void *stream) {
    int rc = check_common(layouts, n_layouts, state, n_envs, S);
    if (rc) return rc;
    const bool codes = flags & OVC_F_OUT_CODES;
    const bool is_stream = flags & OVC_F_OUT_STREAM;
    if (is_stream && (flags & (OVC_F_OUT_CODES | OVC_F_OUT_PACKED | OVC_F_OUT_NARROW)))
        return fail(OVC_E_BADARG, "OVC_F_OUT_STREAM excludes the other output formats");
    if (!actions || !events || !start_records || (!codes && !sparse) || (!codes && !is_stream && !shaped) ||
        (!done && !(flags & (OVC_F_OUT_PACKED | OVC_F_OUT_CODES | OVC_F_OUT_STREAM))))
        return fail(OVC_E_BADARG, "null pointer argument");
    if (codes) sparse = nullptr, shaped = nullptr, done = nullptr;
    if (is_stream) {
        shaped = nullptr;
        if ((((unsigned)flags >> OVC_F_STREAM_CAP_SHIFT) & 0xFFFFu) == 0) return fail(OVC_E_BADARG, "OVC_F_OUT_STREAM needs a capacity in flags bits 16-31");
        if (((uintptr_t)events & 3) || ((uintptr_t)sparse & 1) || ((uintptr_t)done & 1)) return fail(OVC_E_BADARG, "stream buffers are misaligned");
    }
    const bool small_out = flags & (OVC_F_OUT_NARROW | OVC_F_OUT_PACKED | OVC_F_OUT_CODES | OVC_F_OUT_STREAM);
    const bool small_ev = flags & (OVC_F_OUT_PACKED | OVC_F_OUT_CODES | OVC_F_OUT_STREAM);
    const bool small_act = flags & (OVC_F_ACT_U8 | OVC_F_ACT_PACKED);
    if (((small_act ? 0 : (uintptr_t)actions) | (small_out ? 0 : (uintptr_t)shaped) | (small_ev ? 0 : (uintptr_t)events)) & 7)
        return fail(OVC_E_BADARG, "actions / shaped / events must be 8-byte aligned");
    if ((((flags & OVC_F_ACT_U8) ? (uintptr_t)actions : 0) | (small_out ? ((uintptr_t)shaped | (uintptr_t)sparse) : 0) |
         (small_ev ? (uintptr_t)events : 0)) & 1)
        return fail(OVC_E_BADARG, "narrow actions / shaped / sparse must be 2-byte aligned");
    if (n_steps < 1) return fail(OVC_E_BADARG, "n_steps must be >= 1");
    if (n_envs == 0) return OVC_OK;
    int io = (flags & OVC_F_IO_MASK) >> OVC_F_IO_SHIFT;
    if (io == 0) io = 1;
    if (io < 1 || io > 3) return fail(OVC_E_BADARG, "unknown record I/O strategy", (long long)(io));
    if (io == 1 && (n_envs * (S / (S == 16 ? 16 : 32))) > 0x7FFFFFFFLL) io = 2;  // tensor coordinates are int32
    if (is_stream && (io != 1 || n_layouts > MAX_SMEM_LAYOUTS || n_steps > ROLLOUT_MAX_STEPS))
        return fail(OVC_E_UNSUPPORTED, "OVC_F_OUT_STREAM needs the rollout kernel: default record I/O, at most 8 layouts");
    StepArgs a{(const ovc_layout_t *)layouts, start_records, state, actions, sparse, shaped, done, events,
               n_envs, n_layouts, n_steps, horizon, flags, rs != nullptr, rs ? *rs : ovc_random_start_t{0, 0, 0}};
    cudaStream_t st = (cudaStream_t)stream;
    switch (S) {
    case 16: return launch_step<16>(a, io, st);
    case 32: return launch_step<32>(a, io, st);
    case 64: return launch_step<64>(a, io, st);
    default: return launch_step<128>(a, io, st);
    }
}

}  // namespace ovc

#include "ovc_obs.cuh"
#include "ovc_encfc.cuh"
#include "ovc_tail.cuh"
#include "ovc_wide.cuh"
#include "ovc_partner.cuh"
#include "ovc_potential.cuh"
#include "ovc_host.cuh"

// ------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------
extern "C" {

int ovc_abi_version(void) { return OVC_ABI_VERSION; }
size_t ovc_layout_table_size(void) { return sizeof(ovc_layout_t); }
size_t ovc_feat_lut_entry_size(void) { return sizeof(ovc_feat_lut_entry_t); }
const char *ovc_last_error(void) { return ovc::g_err; }

int ovc_step(const void *layouts, int n_layouts, const int32_t *start_records, int32_t *state, const int32_t *actions,
             int32_t *sparse, int32_t *shaped, int32_t *done, int32_t *events, int64_t n_envs, int state_words,
             int horizon, int flags, const ovc_random_start_t *random_start, void *stream) {
    return ovc::step_impl(layouts, n_layouts, start_records, state, actions, sparse, shaped, done, events, n_envs, 1,
                          state_words, horizon, flags, random_start, stream);
}

int ovc_rollout(const void *layouts, int n_layouts, const int32_t *start_records, int32_t *state,
                const int32_t *actions, int32_t *sparse, int32_t *shaped, int32_t *done, int32_t *events,
                int64_t n_envs, int n_steps, int state_words, int horizon, int flags,
                const ovc_random_start_t *random_start, void *stream) {
    return ovc::step_impl(layouts, n_layouts, start_records, state, actions, sparse, shaped, done, events, n_envs,
                          n_steps, state_words, horizon, flags, random_start, stream);
}

int ovc_reset(const void *layouts, int n_layouts, const int32_t *start_records, int32_t *state, const int32_t *env_layout,
              const int32_t *mask, int64_t n_envs, int state_words, const ovc_random_start_t *random_start, void *stream) {
    int rc = ovc::check_common(layouts, n_layouts, state, n_envs, state_words);
    if (rc) return rc;
    if (!start_records) return ovc::fail(OVC_E_BADARG, "null pointer argument");
    if (n_envs == 0) return OVC_OK;
    const int threads = 256;
    if (random_start) {
        ovc::reset_random_kernel<<<(unsigned)((n_envs + threads - 1) / threads), threads, 0, (cudaStream_t)stream>>>(
            (const ovc_layout_t *)layouts, n_layouts, start_records, state, env_layout, mask, n_envs, state_words,
            *random_start);
    } else {
        const long long chunks = (long long)n_envs * (state_words / 4);
        ovc::reset_kernel<<<(unsigned)((chunks + threads - 1) / threads), threads, 0, (cudaStream_t)stream>>>(
            start_records, n_layouts, state, env_layout, mask, n_envs, state_words);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return ovc::cuda_fail(e, "reset kernel launch");
    return OVC_OK;
}

int ovc_encode_lossless(const void *layouts, int n_layouts, const int32_t *state, const int32_t *view_swap,
                        void *out, int dtype, int64_t n_envs, int state_words, int width, int height, int horizon,
                        void *stream) {
    int rc = ovc::check_common(layouts, n_layouts, state, n_envs, state_words);
    if (rc) return rc;
    return ovc::encode_lossless_impl((const ovc_layout_t *)layouts, state, view_swap, out, dtype, n_envs, state_words,
                                     width, height, horizon, (cudaStream_t)stream);
}

int ovc_encode_linear(const void *layouts, int n_layouts, const int32_t *state, const int32_t *view_swap, const void *wt,
                      const float *bias, void *out, int64_t n_envs, int state_words, int width, int height, int horizon,
                      int n_out, float neg_slope, void *stream) {
    int rc = ovc::check_common(layouts, n_layouts, state, n_envs, state_words);
    if (rc) return rc;
    return ovc::encode_linear_impl((const ovc_layout_t *)layouts, n_layouts, state, view_swap, wt, bias, out, n_envs,
                                   state_words, width, height, horizon, n_out, neg_slope, (cudaStream_t)stream);
}

int ovc_sample_actions(const float *scores, int ld, int n_actions, int64_t n_rows, uint64_t seed, uint64_t *counter,
                       int32_t *actions, void *stream) {
    return ovc::sample_actions_impl(scores, ld, n_actions, n_rows, seed, (unsigned long long *)counter, actions, nullptr, (cudaStream_t)stream);
}

int ovc_sample_actions_logp(const float *scores, int ld, int n_actions, int64_t n_rows, uint64_t seed, uint64_t *counter,
                            int32_t *actions, float *logp, void *stream) {
    return ovc::sample_actions_impl(scores, ld, n_actions, n_rows, seed, (unsigned long long *)counter, actions, logp, (cudaStream_t)stream);
}

int ovc_accumulate_returns(const int32_t *sparse, const int32_t *shaped, float factor, int64_t n_envs, int64_t *ret_sparse,
                           float *ret_mixed, void *stream) {
    return ovc::accumulate_returns_impl(sparse, shaped, factor, n_envs, (long long *)ret_sparse, ret_mixed, nullptr, nullptr, nullptr,
                                        nullptr, nullptr, (cudaStream_t)stream);
}

int ovc_record_transition(const int32_t *sparse, const int32_t *shaped, const int32_t *done, const float *factor, int64_t n_envs,
                          float *rewards, uint8_t *dones, int64_t *ret_sparse, float *ret_mixed, void *stream) {
    if (!factor) return ovc::fail(OVC_E_BADARG, "null pointer argument");
    return ovc::accumulate_returns_impl(sparse, shaped, 0.f, n_envs, (long long *)ret_sparse, ret_mixed, factor, done, rewards, dones,
                                        nullptr, (cudaStream_t)stream);
}

int ovc_record_transition_stats(const int32_t *sparse, const int32_t *shaped, const int32_t *done, const float *factor, int64_t n_envs,
                                float *rewards, uint8_t *dones, int64_t *ret_sparse, float *ret_mixed, const ovc_episode_stats_t *stats,
                                void *stream) {
    if (!factor || !stats) return ovc::fail(OVC_E_BADARG, "null pointer argument");
    return ovc::accumulate_returns_impl(sparse, shaped, 0.f, n_envs, (long long *)ret_sparse, ret_mixed, factor, done, rewards, dones,
                                        stats, (cudaStream_t)stream);
}

int ovc_gae(const float *rewards, const float *values, const uint8_t *dones, const float *last_values, int64_t n_steps, int64_t n_rows,
            float gamma, float lambda, float *advantages, float *value_targets, void *stream) {
    return ovc::gae_impl(rewards, values, dones, last_values, n_steps, n_rows, gamma, lambda, advantages, value_targets,
                         (cudaStream_t)stream);
}

int ovc_policy_tail_logp(const void *x, int64_t n_rows, int k0, float in_slope, const void *w_first, const float *b_first,
                         const void *w_hidden, const float *b_hidden, int n_hidden, const void *w_heads, const float *b_heads,
                         float slope, int n_actions, uint64_t seed, uint64_t *counter, int32_t *actions, float *values, float *scores,
                         float *logp, void *stream) {
    ovc::PolicyTailArgs a;
    a.x = (const __nv_bfloat16 *)x, a.w_first = (const __nv_bfloat16 *)w_first, a.b_first = b_first;
    a.w_hidden = (const __nv_bfloat16 *)w_hidden, a.b_hidden = b_hidden, a.w_heads = (const __nv_bfloat16 *)w_heads, a.b_heads = b_heads;
    a.n_rows = n_rows, a.n_hidden = n_hidden, a.n_actions = n_actions, a.in_slope = in_slope, a.slope = slope, a.seed = seed;
    a.counter = (unsigned long long *)counter, a.actions = actions, a.values = values, a.scores = scores, a.logp = logp;
    return ovc::policy_tail_impl(a, k0, (cudaStream_t)stream);
}

int ovc_policy_tail(const void *x, int64_t n_rows, int k0, float in_slope, const void *w_first, const float *b_first,
                    const void *w_hidden, const float *b_hidden, int n_hidden, const void *w_heads, const float *b_heads,
                    float slope, int n_actions, uint64_t seed, uint64_t *counter, int32_t *actions, float *values, float *scores,
                    void *stream) {
    return ovc_policy_tail_logp(x, n_rows, k0, in_slope, w_first, b_first, w_hidden, b_hidden, n_hidden, w_heads, b_heads, slope,
                                n_actions, seed, counter, actions, values, scores, nullptr, stream);
}

int ovc_wide_layers(const void *a0, int64_t m, int k0, const void *w1, const float *b1, int n1, const void *w2, const float *b2, int n2,
                    float slope, void *z2, void *stream) {
    return ovc::wide_layers_impl(a0, m, k0, w1, b1, n1, w2, b2, n2, slope, z2, (cudaStream_t)stream);
}

int ovc_partner_policy(const void *layouts, int n_layouts, const void *lut, const int32_t *state, const int32_t *partner_seat,
                       int64_t n_envs, int state_words, int n_features, int width, const void *w_first, const float *b_first,
                       const void *w_hidden, const float *b_hidden, int n_hidden, const void *w_heads, const float *b_heads, int n_actions,
                       uint64_t seed, uint64_t *counter, int32_t *actions, float *scores, void *stream) {
    int rc = ovc::check_common(layouts, n_layouts, state, n_envs, state_words);
    if (rc) return rc;
    ovc::PartnerArgs a;
    a.f.layouts = (const ovc_layout_t *)layouts, a.f.lut = (const ovc_feat_lut_entry_t *)lut, a.f.state = state, a.f.view_swap = nullptr;
    a.f.out = nullptr, a.f.n_envs = n_envs, a.f.S = state_words, a.f.num_pots = 2, a.f.B = ovc::PP_B, a.f.F = ovc::PP_F, a.f.E = ovc::FEAT_E;
    a.partner_seat = partner_seat, a.w_first = (const __nv_bfloat16 *)w_first, a.b_first = b_first, a.w_hidden = (const __nv_bfloat16 *)w_hidden;
    a.b_hidden = b_hidden, a.w_heads = (const __nv_bfloat16 *)w_heads, a.b_heads = b_heads, a.n_hidden = n_hidden, a.n_actions = n_actions;
    a.seed = seed, a.counter = (unsigned long long *)counter, a.actions = actions, a.scores = scores;
    return ovc::partner_policy_impl(a, n_features, width, (cudaStream_t)stream);
}

int ovc_assign_partners(const int32_t *done, const float *bc_factor, int64_t n_envs, uint64_t seed, uint64_t *counter, int32_t *partner_seat,
                        void *stream) {
    return ovc::assign_partners_impl(done, bc_factor, n_envs, seed, (unsigned long long *)counter, partner_seat, (cudaStream_t)stream);
}

int ovc_featurize(const void *layouts, int n_layouts, const void *lut, const int32_t *state,
                  const int32_t *view_swap, float *out, int64_t n_envs, int state_words, int num_pots, void *stream) {
    int rc = ovc::check_common(layouts, n_layouts, state, n_envs, state_words);
    if (rc) return rc;
    return ovc::featurize_impl((const ovc_layout_t *)layouts, (const ovc_feat_lut_entry_t *)lut, state, view_swap, out,
                               n_envs, state_words, num_pots, (cudaStream_t)stream);
}

int ovc_potential(const void *layouts, int n_layouts, const void *pot_tables, const void *cost_lut, const double *gpow,
                  int n_pow, const int32_t *state, double *out, int64_t n_envs, int state_words, void *stream) {
    int rc = ovc::check_common(layouts, n_layouts, state, n_envs, state_words);
    if (rc) return rc;
    return ovc::potential_impl((const ovc_layout_t *)layouts, (const ovc_potential_t *)pot_tables,
                               (const ovc_cost_lut_entry_t *)cost_lut, gpow, n_pow, state, out, n_envs, state_words,
                               (cudaStream_t)stream);
}
size_t ovc_potential_table_size(void) { return sizeof(ovc_potential_t); }

int ovc_pipeline_create(const ovc_pipeline_desc_t *desc, ovc_pipeline_t **out) { return ovc::pipeline_create(desc, out); }
int ovc_pipeline_run(ovc_pipeline_t *p, const void *h_actions, void *h_sparse, void *h_shaped, void *h_done, void *h_events,
                     int n_steps, void *stream, int join, int64_t *ticket) {
    if (!p) return ovc::fail(OVC_E_BADARG, "null pipeline");
    return ovc::pipeline_run(p, h_actions, h_sparse, h_shaped, h_done, h_events, n_steps, (cudaStream_t)stream, join, ticket);
}
int ovc_pipeline_wait(ovc_pipeline_t *p, int64_t ticket) {
    if (!p) return ovc::fail(OVC_E_BADARG, "null pipeline");
    return ovc::pipeline_wait(p, ticket);
}
int ovc_pipeline_join(ovc_pipeline_t *p, void *stream) {
    if (!p) return ovc::fail(OVC_E_BADARG, "null pipeline");
    return ovc::pipeline_join(p, (cudaStream_t)stream);
}
void ovc_pipeline_destroy(ovc_pipeline_t *p) { ovc::pipeline_destroy(p); }

int ovc_expand_stream_host(const uint32_t *masks, const uint16_t *values, int64_t n_steps, int64_t chunk, int64_t cap,
                           int64_t n_envs, const int32_t *env_layout, const int32_t *reward_tbl, int n_layouts, int16_t *sparse,
                           int8_t *shaped, uint8_t *done, int32_t *events, int n_threads, int64_t *overflow) {
    return ovc::expand_stream_host(masks, values, n_steps, chunk, cap, n_envs, env_layout, reward_tbl, n_layouts, sparse, shaped,
                                   done, events, n_threads, overflow);
}

int ovc_expand_codes_host(const uint16_t *codes, int64_t n_steps, int64_t n_envs, const int32_t *env_layout,
                          const int32_t *reward_tbl, int n_layouts, int16_t *sparse, int8_t *shaped, uint8_t *done,
                          int32_t *events, int n_threads) {
    return ovc::expand_codes_host(codes, n_steps, n_envs, env_layout, reward_tbl, n_layouts, sparse, shaped, done, events,
                                  n_threads);
}

}  // extern "C"
