// ovc_obs.cuh — observation kernels (included by ovc_b200.cu, after the PTX helpers).
//
// K2  encode_kernel<T>   lossless_state_encoding (reference overcooked_mdp.py:2385-2561):
//     out[env][player][x][y][26].  A CTA builds the observations of a tile of E environments in
//     shared memory (zero fill with 16-byte stores, then a sparse scatter of the few non-zero
//     entries) and ships the tile — one contiguous byte range of the output — with ONE bulk
//     async store (cp.async.bulk.global.shared::cta, SASS UBLKCP), so every HBM write is a full,
//     coalesced line no matter how scattered the non-zeros are.  Write-bound: 2*W*H*26*sizeof(T)
//     bytes per environment (4160 B fp32 on cramped_room) against 64-128 B read.
// K3  featurize_kernel   featurize_state (:2579-2898) for the default planner parameters,
//     [env][player][F] float32: per-player feature blocks staged feature-major in shared memory
//     (conflict free), then assembled and written as coalesced float4 rows.
#pragma once
#include <cuda_bf16.h>

namespace ovc {

template <class T>
__device__ __forceinline__ T plane_value(int v) { return (T)v; }
template <>
__device__ __forceinline__ __nv_bfloat16 plane_value<__nv_bfloat16>(int v) { return __float2bfloat16((float)v); }


// plane indices, order of LAYERS at :2393-2442 (SURVEY.md appendix B)
enum {
    PL_LOC = 0, PL_ORI = 2, PL_POT = 10, PL_COUNTER = 11, PL_ONION_DISP = 12, PL_TOMATO_DISP = 13, PL_DISH_DISP = 14,
    PL_SERVE = 15, PL_ONIONS_IN_POT = 16, PL_TOMATOES_IN_POT = 17, PL_ONIONS_IN_SOUP = 18, PL_TOMATOES_IN_SOUP = 19,
    PL_COOK_TIME_REMAINING = 20, PL_SOUP_DONE = 21, PL_DISHES = 22, PL_ONIONS = 23, PL_TOMATOES = 24, PL_URGENCY = 25,
    N_PLANES = 26
};

struct EncodeArgs {
    const ovc_layout_t *layouts;
    const int32_t *state;
    const int32_t *view_swap;  // nullable
    void *out;
    long long n_envs;
    int S, W, H, horizon;
    int E;          // environments per tile
    int obs_elems;  // 2*W*H*26
    unsigned inv_items, inv_h;  // ceil(2^32 / d): n / d == __umulhi(n, inv) exactly while n * d < 2^32
};

// writes value v of plane c at cell (x,y) into BOTH players' views of one environment
template <class T>
__device__ __forceinline__ void put_both(T *obs, int WH26, int H, int x, int y, int c, int v) {
    const int i = (x * H + y) * N_PLANES + c;
    obs[i] = plane_value<T>(v);
    obs[WH26 + i] = plane_value<T>(v);
}

// object planes :2482-2534.  in_pot: the object sits in a pot cell (only soups do).
template <class T>
__device__ __forceinline__ void put_object(T *obs, int WH26, int H, const ovc_layout_t *__restrict__ L, unsigned code,
                                           int x, int y, bool in_pot) {
    const int type = code & 7;
    if (type == OVC_O_SOUP) {
        const int n = (code >> 3) & 3;
        const int nt = __popc((code >> 5) & ((1u << n) - 1u));
        const int tp1 = (code >> 8) & 0x3FFF;
        if (in_pot && tp1 == 0) {  // idle soup in a pot: ingredients can still be added (:2490-2497)
            put_both(obs, WH26, H, x, y, PL_ONIONS_IN_POT, n - nt);
            put_both(obs, WH26, H, x, y, PL_TOMATOES_IN_POT, nt);
        } else {
            put_both(obs, WH26, H, x, y, PL_ONIONS_IN_SOUP, n - nt);
            put_both(obs, WH26, H, x, y, PL_TOMATOES_IN_SOUP, nt);
            if (in_pot) {  // cooking or ready (:2498-2513)
                const int ct = __ldg(&L->cook_time[((n - nt) << 2) | nt]);
                put_both(obs, WH26, H, x, y, PL_COOK_TIME_REMAINING, ct - (tp1 - 1));
                if (tp1 - 1 >= ct) put_both(obs, WH26, H, x, y, PL_SOUP_DONE, 1);
            } else {  // held or on a counter: treated as done (:2515-2525)
                put_both(obs, WH26, H, x, y, PL_SOUP_DONE, 1);
            }
        }
    } else if (type == OVC_O_DISH) put_both(obs, WH26, H, x, y, PL_DISHES, 1);
    else if (type == OVC_O_ONION) put_both(obs, WH26, H, x, y, PL_ONIONS, 1);
    else if (type == OVC_O_TOMATO) put_both(obs, WH26, H, x, y, PL_TOMATOES, 1);
}

template <class T>
__global__ void __launch_bounds__(256) encode_kernel(const EncodeArgs a) {
    extern __shared__ char smem_raw[];
    T *buf = reinterpret_cast<T *>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~(uintptr_t)127);
    const long long env0 = (long long)blockIdx.x * a.E;
    const long long rem = a.n_envs - env0;
    const int ne = (int)(rem < a.E ? rem : a.E);
    const int WH = a.W * a.H, WH26 = WH * N_PLANES;
    const size_t tile_bytes = (size_t)ne * a.obs_elems * sizeof(T);

    // ---- phase A: zero fill (16-byte stores; the buffer is 128-byte aligned and padded) ----
    {
        int4 *b4 = reinterpret_cast<int4 *>(buf);
        const int n16 = (int)((tile_bytes + 15) / 16);
        for (int i = threadIdx.x; i < n16; i += blockDim.x) b4[i] = make_int4(0, 0, 0, 0);
    }
    __syncthreads();

    // ---- phase B: scatter.  Work items per environment: W*H terrain cells, 2 players, n_slots
    //      object cells (an upper bound S-4 is used so the item count is layout independent).
    //      The two integer divisions per item (item -> environment, cell -> column) are multiplications by
    //      host-computed reciprocals.  (A variant with a power-of-two lane group per environment measured
    //      slower: its idle lanes cost more than the divisions did.) ----
    const int items_per_env = WH + 2 + (a.S - 4);
    for (int it = threadIdx.x; it < ne * items_per_env; it += blockDim.x) {
        const int el = (int)__umulhi((unsigned)it, a.inv_items), k = it - el * items_per_env;
        const int32_t *__restrict__ rec = a.state + (env0 + el) * a.S;
        const ovc_layout_t *__restrict__ L = a.layouts + (__ldg(rec + 3) & 0xFF);
        T *obs = buf + (size_t)el * a.obs_elems;
        if (k < WH) {  // static terrain planes :2449-2465 and the urgency plane :2446-2447
            const int x = (int)__umulhi((unsigned)k, a.inv_h), y = k - x * a.H;
            const int terr = __ldg(&L->cell[(y << 4) | x]) & 7;
            // terrain code -> plane: X 11, O 12, T 13, D 14, P 10, S 15 (0 = none)
            const int plane = (int)((0x0F0A0E0D0C0B00ull >> (terr * 8)) & 0xFF);
            if (terr != OVC_T_FLOOR && terr != OVC_T_OUTSIDE) put_both(obs, WH26, a.H, x, y, plane, 1);
            if (a.horizon - __ldg(rec) < 40) put_both(obs, WH26, a.H, x, y, PL_URGENCY, 1);
        } else if (k < WH + 2) {  // player layers :2468-2479 (+ the held object, at the holder's cell)
            const int j = k - WH;
            const unsigned w = (unsigned)__ldg(rec + 1 + j);
            const int x = w & 15, y = (w >> 4) & 15, ori = (w >> 8) & 3;
            const int base = (x * a.H + y) * N_PLANES;
            // view p: own layers first — loc plane (j==p ? 0 : 1), orientation planes 2+4*(j!=p)+ori;
            // player j's own view lands in output slot j, or 1-j where view_swap says so
            const int own = (a.view_swap && __ldg(a.view_swap + env0 + el)) ? 1 - j : j;
            const T one = plane_value<T>(1);
            obs[(size_t)own * WH26 + base + PL_LOC] = one;
            obs[(size_t)own * WH26 + base + PL_ORI + ori] = one;
            obs[(size_t)(1 - own) * WH26 + base + PL_LOC + 1] = one;
            obs[(size_t)(1 - own) * WH26 + base + PL_ORI + 4 + ori] = one;
            put_object(obs, WH26, a.H, L, w >> 10, x, y, false);
        } else {  // loose objects: one per object-capable cell
            const int slot = k - WH - 2;
            if (slot < __ldg(&L->n_slots)) {
                const unsigned code = (unsigned)__ldg(rec + 4 + slot) & OVC_OBJ_MASK;
                if (code) {
                    const int pb = __ldg(&L->slot_pos[slot]);
                    put_object(obs, WH26, a.H, L, code, pb & 15, pb >> 4, slot < __ldg(&L->n_pots));
                }
            }
        }
    }

    // ---- phase C: ship the tile ----
    char *dst = reinterpret_cast<char *>(a.out) + (size_t)env0 * a.obs_elems * sizeof(T);
    if ((tile_bytes & 15) == 0) {
        fence_async_smem();
        __syncthreads();
        if (threadIdx.x == 0) {
            bulk_store_1d(dst, buf, (uint32_t)tile_bytes);
            bulk_commit();
            bulk_wait_read<0>();
        }
    } else {  // ragged last tile whose byte count is not a multiple of 16: plain coalesced stores
        __syncthreads();
        T *d = reinterpret_cast<T *>(dst);
        const int n = ne * a.obs_elems;
        for (int i = threadIdx.x; i < n; i += blockDim.x) d[i] = buf[i];
    }
}

static int gcd_int(int a, int b) { return b ? gcd_int(b, a % b) : a; }

static int encode_lossless_impl(const ovc_layout_t *layouts, const int32_t *state, const int32_t *view_swap, void *out,
                                int dtype, long long n_envs, int S, int W, int H, int horizon, cudaStream_t st) {
    if (!out) return fail(OVC_E_BADARG, "null output pointer");
    if (((uintptr_t)out & 15) != 0) return fail(OVC_E_BADARG, "output must be 16-byte aligned");
    if (W < 1 || W > 16 || H < 1 || H > 16) return fail(OVC_E_BADARG, "grid shape out of range");
    if (n_envs == 0) return OVC_OK;
    const int esize = dtype == OVC_DT_U8 ? 1 : dtype == OVC_DT_BF16 ? 2 : 4;
    if (dtype != OVC_DT_F32 && dtype != OVC_DT_U8 && dtype != OVC_DT_I32 && dtype != OVC_DT_BF16)
        return fail(OVC_E_BADARG, "unknown dtype", (long long)(dtype));
    EncodeArgs a;
    a.layouts = layouts, a.state = state, a.view_swap = view_swap, a.out = out, a.n_envs = n_envs;
    a.S = S, a.W = W, a.H = H, a.horizon = horizon;
    a.obs_elems = 2 * W * H * N_PLANES;
    a.inv_items = (unsigned)((0x100000000ull + (unsigned)(W * H + 2 + (S - 4)) - 1) / (unsigned)(W * H + 2 + (S - 4)));
    a.inv_h = (unsigned)((0x100000000ull + (unsigned)H - 1) / (unsigned)H);
    const int obs_bytes = a.obs_elems * esize;
    // Tile buffer size: small tiles keep ~8 CTAs per SM (228 KB of shared memory on an H100) in flight so that fill,
    // scatter and bulk store of different tiles overlap; larger tiles leave the SM waiting on fewer, longer stores.
    // OVC_ENC_BUF_KB overrides it for a sweep (tools/kbench.py).
    static int buf_kb = 0;
    if (buf_kb == 0) {
        const char *env = getenv("OVC_ENC_BUF_KB");  // tuning knob for experiments
        buf_kb = env ? atoi(env) : 24;
        if (buf_kb < 4 || buf_kb > 200) buf_kb = 24;
    }
    static int e_override = -1;
    if (e_override < 0) {
        const char *env = getenv("OVC_ENC_E");  // experiments: environments per tile, overrides the byte budget
        e_override = env ? atoi(env) : 0;
    }
    const int BUF = buf_kb * 1024;
    const int mult = 16 / gcd_int(16, obs_bytes);    // tiles must start 16-byte aligned in the output
    int E = e_override > 0 ? e_override : BUF / obs_bytes;
    if ((size_t)E * obs_bytes > 200 * 1024) E = 200 * 1024 / obs_bytes;
    E -= E % mult;
    if (E < mult) E = mult;
    a.E = E;
    const size_t smem = (size_t)E * obs_bytes + 128 + 16;
    const unsigned grid = (unsigned)((n_envs + E - 1) / E);
    cudaError_t e;
#define OVC_LAUNCH_ENCODE(TT)                                                                                    \
    do {                                                                                                         \
        e = cudaFuncSetAttribute(encode_kernel<TT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);     \
        if (e != cudaSuccess) return cuda_fail(e, "encode kernel attribute");                                    \
        encode_kernel<TT><<<grid, 256, smem, st>>>(a);                                                           \
    } while (0)
    if (dtype == OVC_DT_F32) OVC_LAUNCH_ENCODE(float);
    else if (dtype == OVC_DT_U8) OVC_LAUNCH_ENCODE(uint8_t);
    else if (dtype == OVC_DT_BF16) OVC_LAUNCH_ENCODE(__nv_bfloat16);
    else OVC_LAUNCH_ENCODE(int32_t);
#undef OVC_LAUNCH_ENCODE
    e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "encode kernel launch");
    return OVC_OK;
}

// ------------------------------------------------------------------------------------------------
// K3 featurize_state
// ------------------------------------------------------------------------------------------------
// Two phases per CTA (tile of E environments = 2E player views):
//   1. one thread per (environment, player) computes that player's feature block (26 + 10*num_pots
//      small integers) into shared memory in FEATURE-MAJOR order blk[feature][view] — consecutive
//      lanes hit consecutive words, so the writes are bank-conflict free (a view-major tile would
//      put every lane on the same bank: the view stride F is a multiple of 32 words);
//   2. all threads assemble the output rows [own block, other block, other-self offset, self position]
//      (:2877-2896) as float4 and write them straight to global memory, consecutive threads ->
//      consecutive 16-byte pieces of the contiguous output tile (fully coalesced, full lines).
struct FeatArgs {
    const ovc_layout_t *layouts;
    const ovc_feat_lut_entry_t *lut;
    const int32_t *state;
    const int32_t *view_swap;  // nullable
    float *out;
    long long n_envs;
    int S, num_pots, B, F, E;
};

constexpr int FEAT_E = 64;              // environments per tile
constexpr int FEAT_LD = 2 * FEAT_E + 1;  // odd leading dimension: phase-2 reads (stride LD) stay conflict free

// Block of player `me` (:2748-2840).  `own` points at column `view` of the feature-major tile
// asm_[F][FEAT_LD]; the same values are the "other player" block of the partner view (`oth` = rows B.. of
// column view^1), so phase 2 is a pure transpose.
__device__ __forceinline__ void feat_block(const FeatArgs &a, const ovc_layout_t *__restrict__ L,
                                           const ovc_feat_lut_entry_t *__restrict__ le, const int32_t *__restrict__ rec,
                                           unsigned me, short *own, short *oth) {
    int n = 0;
    auto put = [&](int v) {
        own[n * FEAT_LD] = (short)v;
        oth[n * FEAT_LD] = (short)v;
        n++;
    };
    const int x = me & 15, y = (me >> 4) & 15, ori = (me >> 8) & 3;
    const unsigned held = me >> 10;
    const int ht = held & 7;
    // the 12-byte LUT entry as three words: {d_onion, d_tomato}, {d_dish, d_serve}, pot_order
    const unsigned lw0 = __ldg(reinterpret_cast<const unsigned *>(le)), lw1 = __ldg(reinterpret_cast<const unsigned *>(le) + 1),
                   lw2 = __ldg(reinterpret_cast<const unsigned *>(le) + 2);
    auto sb = [](unsigned w, int k) { return (int)(signed char)((w >> (8 * k)) & 0xFF); };
    for (int k = 0; k < 4; k++) put(ori == k);  // pi_orientation :2750-2753
    // pi_objs one-hot over IDX_TO_OBJ = [onion, soup, dish, tomato] :2742-2764
    put(ht == OVC_O_ONION), put(ht == OVC_O_SOUP), put(ht == OVC_O_DISH), put(ht == OVC_O_TOMATO);
    // closest onion / tomato / dish source: (0,0) when that object is held :2632-2641
    put(ht == OVC_O_ONION ? 0 : sb(lw0, 0)), put(ht == OVC_O_ONION ? 0 : sb(lw0, 1));
    put(ht == OVC_O_TOMATO ? 0 : sb(lw0, 2)), put(ht == OVC_O_TOMATO ? 0 : sb(lw0, 3));
    put(ht == OVC_O_DISH ? 0 : sb(lw1, 0)), put(ht == OVC_O_DISH ? 0 : sb(lw1, 1));
    // closest soup: counters are never motion goals (NO_COUNTERS_PARAMS) -> (0,0); counts from a held soup
    put(0), put(0);
    int son = 0, sto = 0;
    if (ht == OVC_O_SOUP) {
        const int ns = (held >> 3) & 3;
        sto = __popc((held >> 5) & ((1u << ns) - 1u));
        son = ns - sto;
    }
    put(son), put(sto);
    put(sb(lw1, 2)), put(sb(lw1, 3));
    put(0), put(0);  // closest empty counter: unreachable goal -> (0,0)
    for (int k = 0; k < a.num_pots; k++) {  // make_pot_feature :2658-2740, pots by planner cost :2820-2831
        const int slot = k < OVC_MAX_POTS ? (int)((lw2 >> (8 * k)) & 0xFF) : OVC_NO_SLOT;
        if (slot == OVC_NO_SLOT) {
            for (int z = 0; z < 10; z++) put(0);
            continue;
        }
        const unsigned w = (unsigned)__ldg(rec + 4 + slot);
        const bool empty = (w & 7) == 0;
        const int ns = (w >> 3) & 3;
        const int nt = __popc((w >> 5) & ((1u << ns) - 1u));
        const int tp1 = (w >> 8) & 0x3FFF;
        const int ct = empty ? 0 : __ldg(&L->cook_time[((ns - nt) << 2) | nt]);
        const bool ready = !empty && tp1 != 0 && tp1 - 1 >= ct;
        const bool cooking = !empty && tp1 != 0 && !ready;
        const bool full = !empty && (tp1 != 0 || ns == 3);
        int remaining = (!empty && tp1 != 0) ? ct - (tp1 - 1) : 0;
        if (remaining < 0) remaining = 0;
        const int pb = __ldg(&L->slot_pos[slot]);
        put(1), put(empty), put(full), put(cooking), put(ready);
        put(empty ? 0 : ns - nt), put(empty ? 0 : nt), put(remaining);
        put((pb & 15) - x), put((pb >> 4) - y);
    }
    for (int d = 0; d < 4; d++)  // pi_wall_d :2833-2840
        put((__ldg(&L->cell[(((y << 4) | x) + dir_delta(d)) & 0xFF]) & 7) != OVC_T_FLOOR);
}

__global__ void __launch_bounds__(256) featurize_kernel(const FeatArgs a) {
    extern __shared__ __align__(16) char fsm[];
    short *asm_ = reinterpret_cast<short *>(fsm);  // [F][FEAT_LD] int16 (cook times go up to 16382), feature-major
    const long long env0 = (long long)blockIdx.x * FEAT_E;
    const long long rem = a.n_envs - env0;
    const int ne = (int)(rem < FEAT_E ? rem : FEAT_E);
    const int nv = ne * 2;
    // ---- phase 1: one thread per view builds its row pieces ----
    if ((int)threadIdx.x < nv) {
        const int v = threadIdx.x, el = v >> 1, j = v & 1;
        const int32_t *__restrict__ rec = a.state + (env0 + el) * a.S;
        const int lid = __ldg(rec + 3) & 0xFF;
        const ovc_layout_t *__restrict__ L = a.layouts + lid;
        const unsigned me = (unsigned)__ldg(rec + 1 + j), ot = (unsigned)__ldg(rec + 2 - j);
        const ovc_feat_lut_entry_t *le = a.lut + (size_t)lid * 1024 + ((me & 0xFF) << 2 | ((me >> 8) & 3));
        feat_block(a, L, le, rec, me, asm_ + v, asm_ + (size_t)a.B * FEAT_LD + (v ^ 1));
        // :2877-2896 tail of the row: other - self, then self position
        short *tail = asm_ + (size_t)2 * a.B * FEAT_LD + v;
        tail[0 * FEAT_LD] = (short)((int)(ot & 15) - (int)(me & 15));
        tail[1 * FEAT_LD] = (short)((int)((ot >> 4) & 15) - (int)((me >> 4) & 15));
        tail[2 * FEAT_LD] = (short)(me & 15);
        tail[3 * FEAT_LD] = (short)((me >> 4) & 15);
    }
    __syncthreads();
    // ---- phase 2: transpose to rows, float4 per thread, coalesced ----
    const int G = a.F / 4;  // F = 20*num_pots + 56 is a multiple of 4
    float4 *dst = reinterpret_cast<float4 *>(a.out + (size_t)env0 * 2 * a.F);
    for (int idx = threadIdx.x; idx < nv * G; idx += blockDim.x) {
        const int row = idx / G, g = idx - row * G;
        // output row `row` of the tile is player (row & 1)'s view, or the partner's where view_swap is set
        const int v = (a.view_swap && __ldg(a.view_swap + env0 + (row >> 1))) ? row ^ 1 : row;
        const short *src = asm_ + (size_t)(4 * g) * FEAT_LD + v;
        dst[idx] = make_float4((float)src[0], (float)src[FEAT_LD], (float)src[2 * FEAT_LD], (float)src[3 * FEAT_LD]);
    }
}

static int featurize_impl(const ovc_layout_t *layouts, const ovc_feat_lut_entry_t *lut, const int32_t *state,
                          const int32_t *view_swap, float *out, long long n_envs, int S, int num_pots, cudaStream_t st) {
    if (!out || !lut) return fail(OVC_E_BADARG, "null pointer argument");
    if (((uintptr_t)out & 15) != 0) return fail(OVC_E_BADARG, "output must be 16-byte aligned");
    if (num_pots < 0 || num_pots > 16) return fail(OVC_E_BADARG, "num_pots out of range");
    if (n_envs == 0) return OVC_OK;
    FeatArgs a;
    a.layouts = layouts, a.lut = lut, a.state = state, a.view_swap = view_swap, a.out = out, a.n_envs = n_envs, a.S = S;
    a.num_pots = num_pots, a.B = 10 * num_pots + 26, a.F = 2 * a.B + 4;
    a.E = FEAT_E;
    const size_t smem = 2 * (size_t)a.F * FEAT_LD + 16;
    cudaError_t e;
    if (smem > 48 * 1024) {
        e = cudaFuncSetAttribute(featurize_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return cuda_fail(e, "featurize kernel attribute");
    }
    featurize_kernel<<<(unsigned)((n_envs + FEAT_E - 1) / FEAT_E), 256, smem, st>>>(a);
    e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "featurize kernel launch");
    return OVC_OK;
}

}  // namespace ovc
