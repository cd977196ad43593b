// ovc_encfc.cuh — K7 encode_linear_kernel (included by ovc_b200.cu after ovc_obs.cuh).
//
// out[2N][n_out] = leaky_relu(W0 . lossless_state_encoding(s) + b): the FIRST LAYER of a policy that consumes the
// reference's lossless encoding (overcooked_mdp.py:2385-2561; consumer: ppo_rllib.py:43-79, the 5x5 'same' convolution,
// folded into one matrix by the host) evaluated straight from the packed record — the observation tensor
// (2*W*H*26 elements per environment, 2080 B of bf16 on cramped_room) is never written to or read back from HBM.
//
// Not a GEMM: the encoding is sparse.  Of the W*H*26 inputs of a view, the six terrain planes are constants of the
// layout (-> folded into a per-layout bias in the prologue), the urgency plane is all-or-nothing (-> one pre-summed
// vector), and what is left is a handful of entries: own / other player cell and orientation (4 per view), and one to
// four entries per object in the game (shared by both views).  So a view's row of the product is
//     bias_l + [urgent] u + sum over ~8 entries of value_k * Wt[feature_k][:]
// i.e. ~8 row gathers of a table instead of W*H*26 = 520 multiply-adds per output: 40-60x fewer operations than the
// dense contraction, which is why this runs on the CUDA cores out of shared memory and not on wgmma.
//
// One CTA per SM keeps a column slice Wt[:, slice] of the 19 dynamic planes in shared memory (380 rows x 256 columns
// of bf16 = 190 KB on a 5x4 grid); a warp owns one environment at a time: lane l decodes object slot l, the entries go
// round the warp by shuffle, every lane accumulates its CPL columns in fp32 (one 16-byte LDS per entry and lane,
// conflict free), the object part is computed once and shared by both views.  Output rows leave as 16-byte stores,
// 512 contiguous bytes per warp and row.
#pragma once
#include <cuda_bf16.h>
#include <type_traits>

namespace ovc {

constexpr int EL_DYN = 19;          // dynamic planes kept in the table: 0-9 (players) and 16-24 (objects)
constexpr int EL_THREADS = 1024;
constexpr int EL_MAX_LAYOUTS = 8;

struct EncLinArgs {
    const ovc_layout_t *layouts;
    const int32_t *state;
    const int32_t *view_swap;  // nullable
    const __nv_bfloat16 *wt;   // [W*H*26][n_out], row = feature in K2's element order (x*H + y)*26 + plane
    const float *bias;         // [n_out]
    __nv_bfloat16 *out;        // [2 n_envs][n_out]
    long long n_envs;
    int n_layouts, S, W, H, horizon, n_out, n_workers;
    float neg_slope;
};

__device__ __forceinline__ int el_dyn_plane(int plane) { return plane < 10 ? plane : plane - 6; }

// entry word: table row << 16 | value (int16); value 0 = no entry
__device__ __forceinline__ unsigned el_entry(int row, int value) { return ((unsigned)row << 16) | ((unsigned)value & 0xFFFFu); }

// the object planes of put_object (ovc_obs.cuh, :2482-2534) as up to four (row, value) entries
__device__ __forceinline__ void el_object(unsigned code, int rowbase, bool in_pot, const int *cook, unsigned e[4]) {
    e[0] = e[1] = e[2] = e[3] = 0;
    const int type = code & 7;
    if (type == OVC_O_SOUP) {
        const int n = (code >> 3) & 3;
        const int nt = __popc((code >> 5) & ((1u << n) - 1u));
        const int tp1 = (code >> 8) & 0x3FFF;
        if (in_pot && tp1 == 0) {
            e[0] = el_entry(rowbase + el_dyn_plane(PL_ONIONS_IN_POT), n - nt);
            e[1] = el_entry(rowbase + el_dyn_plane(PL_TOMATOES_IN_POT), nt);
        } else {
            e[0] = el_entry(rowbase + el_dyn_plane(PL_ONIONS_IN_SOUP), n - nt);
            e[1] = el_entry(rowbase + el_dyn_plane(PL_TOMATOES_IN_SOUP), nt);
            if (in_pot) {
                const int ct = cook[((n - nt) << 2) | nt];
                e[2] = el_entry(rowbase + el_dyn_plane(PL_COOK_TIME_REMAINING), ct - (tp1 - 1));
                if (tp1 - 1 >= ct) e[3] = el_entry(rowbase + el_dyn_plane(PL_SOUP_DONE), 1);
            } else {
                e[3] = el_entry(rowbase + el_dyn_plane(PL_SOUP_DONE), 1);
            }
        }
    } else if (type == OVC_O_DISH) e[0] = el_entry(rowbase + el_dyn_plane(PL_DISHES), 1);
    else if (type == OVC_O_ONION) e[0] = el_entry(rowbase + el_dyn_plane(PL_ONIONS), 1);
    else if (type == OVC_O_TOMATO) e[0] = el_entry(rowbase + el_dyn_plane(PL_TOMATOES), 1);
}

template <int CPL>
struct ElCols;  // CPL bf16 columns of one table row, as one vector load
template <>
struct ElCols<8> { using vec = uint4; };
template <>
struct ElCols<4> { using vec = uint2; };
template <>
struct ElCols<2> { using vec = unsigned; };

template <int CPL>
__device__ __forceinline__ void el_words(const typename ElCols<CPL>::vec &v, unsigned w[CPL / 2]);
template <>
__device__ __forceinline__ void el_words<8>(const uint4 &v, unsigned w[4]) { w[0] = v.x, w[1] = v.y, w[2] = v.z, w[3] = v.w; }
template <>
__device__ __forceinline__ void el_words<4>(const uint2 &v, unsigned w[2]) { w[0] = v.x, w[1] = v.y; }
template <>
__device__ __forceinline__ void el_words<2>(const unsigned &v, unsigned w[1]) { w[0] = v; }

// acc[:] += value * table[row][lane's columns]
template <int CPL>
__device__ __forceinline__ void el_gather(float acc[CPL], const __nv_bfloat16 *tab_lane, int row, float value) {
    constexpr int CS = 32 * CPL;
    const typename ElCols<CPL>::vec v = *reinterpret_cast<const typename ElCols<CPL>::vec *>(tab_lane + (size_t)row * CS);
    unsigned w[CPL / 2];
    el_words<CPL>(v, w);
#pragma unroll
    for (int i = 0; i < CPL / 2; i++) {
        acc[2 * i] = fmaf(__uint_as_float(w[i] << 16), value, acc[2 * i]);
        acc[2 * i + 1] = fmaf(__uint_as_float(w[i] & 0xFFFF0000u), value, acc[2 * i + 1]);
    }
}

template <int CPL>
__global__ void __launch_bounds__(EL_THREADS, 1) encode_linear_kernel(const EncLinArgs a) {
    constexpr int CS = 32 * CPL;  // columns per CTA
    extern __shared__ __align__(16) char el_smem[];
    const int WH = a.W * a.H;
    const int n_rows = WH * EL_DYN;
    __nv_bfloat16 *tab = reinterpret_cast<__nv_bfloat16 *>(el_smem);                      // [n_rows][CS]
    float *bias_eff = reinterpret_cast<float *>(el_smem + (size_t)n_rows * CS * 2);       // [n_layouts][CS]
    float *urg = bias_eff + a.n_layouts * CS;                                             // [CS]
    int *cook = reinterpret_cast<int *>(urg + CS);                                        // [n_layouts][16]
    int *nslots = cook + a.n_layouts * 16;                                                // [n_layouts][2]: n_slots, n_pots
    unsigned short *srow = reinterpret_cast<unsigned short *>(nslots + a.n_layouts * 2);  // [n_layouts][128] slot -> row base

    const int n_slices = a.n_out / CS;
    const int slice = blockIdx.x % n_slices, worker = blockIdx.x / n_slices;
    const int col0 = slice * CS;

    // ---- prologue: the table slice and the per-layout constants ----
    unsigned char *tplane = reinterpret_cast<unsigned char *>(srow + a.n_layouts * 128);  // [n_layouts][256] terrain plane of a cell, 0 = none
    for (int i = threadIdx.x; i < a.n_layouts * WH; i += EL_THREADS) {  // terrain code -> plane: X 11, O 12, T 13, D 14, P 10, S 15 (:2449-2465)
        const int l = i / WH, cell = i - l * WH, x = cell / a.H, y = cell - x * a.H;
        tplane[l * 256 + cell] = (unsigned char)((0x000F0A0E0D0C0B00ull >> ((a.layouts[l].cell[(y << 4) | x] & 7) * 8)) & 0xFF);
    }
    __syncthreads();
    {
        constexpr int CH = CS * 2 / 16;  // 16-byte chunks per row
        for (int i = threadIdx.x; i < n_rows * CH; i += EL_THREADS) {
            const int r = i / CH, c = i - r * CH;
            const int cell = r / EL_DYN, d = r - cell * EL_DYN;
            const int plane = d < 10 ? d : d + 6;
            const uint4 *src = reinterpret_cast<const uint4 *>(a.wt + (size_t)(cell * N_PLANES + plane) * a.n_out + col0) + c;
            reinterpret_cast<uint4 *>(tab)[i] = __ldg(src);
        }
        // terrain and urgency sums: one thread per (layout, column); the cells' loads are independent (plane ids staged in
        // shared memory first), issued four at a time, added in cell order
        for (int i = threadIdx.x; i < (a.n_layouts + 1) * CS; i += EL_THREADS) {
            const int l = i / CS, c = i - l * CS;
            const unsigned char *tp = tplane + l * 256;
            const __nv_bfloat16 *w = a.wt + col0 + c;
            float s = l == a.n_layouts ? 0.f : a.bias[col0 + c];
            for (int cell = 0; cell < WH; cell += 4) {
                float v[4];
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const int pl = cell + u < WH ? (l == a.n_layouts ? (int)PL_URGENCY : (int)tp[cell + u]) : 0;
                    v[u] = pl ? __bfloat162float(w[(size_t)((cell + u) * N_PLANES + pl) * a.n_out]) : 0.f;
                }
                s = (((s + v[0]) + v[1]) + v[2]) + v[3];
            }
            if (l == a.n_layouts) urg[c] = s;
            else bias_eff[i] = s;
        }
        for (int i = threadIdx.x; i < a.n_layouts * 128; i += EL_THREADS) {
            const ovc_layout_t *L = a.layouts + (i >> 7);
            const int pb = L->slot_pos[i & 127];
            srow[i] = (unsigned short)((((pb & 15) * a.H + (pb >> 4)) * EL_DYN) & 0xFFFF);
        }
        for (int i = threadIdx.x; i < a.n_layouts * 16; i += EL_THREADS) cook[i] = a.layouts[i >> 4].cook_time[i & 15];
        for (int i = threadIdx.x; i < a.n_layouts; i += EL_THREADS) {
            nslots[2 * i] = a.layouts[i].n_slots;
            nslots[2 * i + 1] = a.layouts[i].n_pots;
        }
    }
    __syncthreads();

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    constexpr int NW = EL_THREADS / 32;
    const __nv_bfloat16 *tab_lane = tab + lane * CPL;
    const long long stride = (long long)a.n_workers * NW;
    const int max_slot_chunks = (a.S - 4 + 31) / 32;

    for (long long env = (long long)worker * NW + warp; env < a.n_envs; env += stride) {
        const int32_t *__restrict__ rec = a.state + env * a.S;
        const int4 head = __ldg(reinterpret_cast<const int4 *>(rec));  // timestep, player 0, player 1, misc (same address in every lane)
        const int lid = head.w & 0xFF;
        const int n_slots = nslots[2 * lid], n_pots = nslots[2 * lid + 1];
        const int *ck = cook + lid * 16;
        const unsigned short *sr = srow + lid * 128;

        float common[CPL];
        {   // vector loads: consecutive lanes read consecutive CPL-float pieces (conflict free)
            const bool urgent = a.horizon - head.x < 40;
            constexpr int V = CPL >= 4 ? 4 : 2;
            using fv = typename std::conditional<CPL >= 4, float4, float2>::type;
#pragma unroll
            for (int i = 0; i < CPL / V; i++) {
                const fv b = reinterpret_cast<const fv *>(bias_eff + lid * CS + lane * CPL)[i];
                const fv u = reinterpret_cast<const fv *>(urg + lane * CPL)[i];
                const float *bp = reinterpret_cast<const float *>(&b), *up = reinterpret_cast<const float *>(&u);
#pragma unroll
                for (int k = 0; k < V; k++) common[i * V + k] = bp[k] + (urgent ? up[k] : 0.f);
            }
        }
        // objects on pots / counters: lane l of chunk c decodes slot 32 c + l; entries travel by shuffle
        for (int c = 0; c < max_slot_chunks; c++) {
            if (c * 32 >= n_slots) break;
            const int slot = c * 32 + lane;
            unsigned e[4] = {0, 0, 0, 0};
            if (slot < n_slots) {
                const unsigned code = (unsigned)__ldg(rec + 4 + slot) & OVC_OBJ_MASK;
                if (code) el_object(code, sr[slot], slot < n_pots, ck, e);
            }
            unsigned m = __ballot_sync(0xFFFFFFFFu, (e[0] | e[1] | e[2] | e[3]) != 0);
            while (m) {
                const int j = __ffs(m) - 1;
                m &= m - 1;
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    const unsigned w = __shfl_sync(0xFFFFFFFFu, e[q], j);
                    if (w & 0xFFFFu) el_gather<CPL>(common, tab_lane, (int)(w >> 16), (float)(short)(w & 0xFFFFu));
                }
            }
        }
        // held objects: at the holder's cell, in both views (computed by every lane, no exchange needed)
        const unsigned p0 = (unsigned)head.y, p1 = (unsigned)head.z;
        const int cell0 = ((p0 & 15) * a.H + ((p0 >> 4) & 15)) * EL_DYN, cell1 = ((p1 & 15) * a.H + ((p1 >> 4) & 15)) * EL_DYN;
#pragma unroll
        for (int j = 0; j < 2; j++) {
            const unsigned held = (j ? p1 : p0) >> 10;
            if (held) {
                unsigned e[4];
                el_object(held, j ? cell1 : cell0, false, ck, e);
#pragma unroll
                for (int q = 0; q < 4; q++)
                    if (e[q] & 0xFFFFu) el_gather<CPL>(common, tab_lane, (int)(e[q] >> 16), (float)(short)(e[q] & 0xFFFFu));
            }
        }
        // the two views: own cell / orientation in planes 0, 2..5, the partner's in planes 1, 6..9 (:2468-2479)
        const int ori0 = (p0 >> 8) & 3, ori1 = (p1 >> 8) & 3;
        const int swap = a.view_swap ? (__ldg(a.view_swap + env) != 0) : 0;
#pragma unroll
        for (int p = 0; p < 2; p++) {  // p = the player whose view this is
            float acc[CPL];
#pragma unroll
            for (int i = 0; i < CPL; i++) acc[i] = common[i];
            const int own_cell = p ? cell1 : cell0, oth_cell = p ? cell0 : cell1;
            const int own_ori = p ? ori1 : ori0, oth_ori = p ? ori0 : ori1;
            el_gather<CPL>(acc, tab_lane, own_cell + PL_LOC, 1.f);
            el_gather<CPL>(acc, tab_lane, own_cell + PL_ORI + own_ori, 1.f);
            el_gather<CPL>(acc, tab_lane, oth_cell + PL_LOC + 1, 1.f);
            el_gather<CPL>(acc, tab_lane, oth_cell + PL_ORI + 4 + oth_ori, 1.f);
            unsigned packed[CPL / 2];
#pragma unroll
            for (int i = 0; i < CPL / 2; i++) {
                const float x0 = acc[2 * i], x1 = acc[2 * i + 1];
                const __nv_bfloat162 h = __floats2bfloat162_rn(fmaxf(x0, x0 * a.neg_slope), fmaxf(x1, x1 * a.neg_slope));
                packed[i] = *reinterpret_cast<const unsigned *>(&h);
            }
            const long long row = 2 * env + (swap ? 1 - p : p);
            __nv_bfloat16 *dst = a.out + row * a.n_out + col0 + lane * CPL;
            if constexpr (CPL == 8) *reinterpret_cast<uint4 *>(dst) = make_uint4(packed[0], packed[1], packed[2], packed[3]);
            else if constexpr (CPL == 4) *reinterpret_cast<uint2 *>(dst) = make_uint2(packed[0], packed[1]);
            else *reinterpret_cast<unsigned *>(dst) = packed[0];
        }
    }
}

static size_t encode_linear_smem(int cpl, int n_rows, int n_layouts) {
    const size_t CS = 32 * (size_t)cpl;
    return (size_t)n_rows * CS * 2 + ((size_t)n_layouts + 1) * CS * 4 + (size_t)n_layouts * (16 * 4 + 2 * 4 + 128 * 2 + 256) + 16;
}

static int encode_linear_impl(const ovc_layout_t *layouts, int n_layouts, const int32_t *state, const int32_t *view_swap,
                              const void *wt, const float *bias, void *out, long long n_envs, int S, int W, int H, int horizon,
                              int n_out, float neg_slope, cudaStream_t st) {
    if (!out || !wt || !bias) return fail(OVC_E_BADARG, "null pointer argument");
    if ((((uintptr_t)out | (uintptr_t)wt) & 15) != 0) return fail(OVC_E_BADARG, "weights and output must be 16-byte aligned");
    if (W < 1 || W > 16 || H < 1 || H > 16) return fail(OVC_E_BADARG, "grid shape out of range");
    if (n_out < 64 || n_out % 64) return fail(OVC_E_BADARG, "n_out must be a positive multiple of 64", n_out);
    if (!(neg_slope >= 0.f && neg_slope <= 1.f)) return fail(OVC_E_BADARG, "negative slope must lie in [0, 1]");
    if (n_layouts > EL_MAX_LAYOUTS) return fail(OVC_E_UNSUPPORTED, "encode_linear: more than 8 layouts per call", n_layouts);
    if (n_envs == 0) return OVC_OK;
    int dev = 0, n_sm = 0, max_smem = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    const int n_rows = W * H * EL_DYN;
    int cpl = 0;
    for (int c = 8; c >= 2; c >>= 1)
        if (n_out % (32 * c) == 0 && encode_linear_smem(c, n_rows, n_layouts) <= (size_t)max_smem) {
            cpl = c;
            break;
        }
    if (!cpl) return fail(OVC_E_UNSUPPORTED, "encode_linear: the weight table of this grid does not fit shared memory", W * H);
    EncLinArgs a;
    a.layouts = layouts, a.state = state, a.view_swap = view_swap, a.wt = (const __nv_bfloat16 *)wt, a.bias = bias;
    a.out = (__nv_bfloat16 *)out, a.n_envs = n_envs, a.n_layouts = n_layouts, a.S = S, a.W = W, a.H = H, a.horizon = horizon;
    a.n_out = n_out, a.neg_slope = neg_slope;
    const int n_slices = n_out / (32 * cpl);
    const long long want = (n_envs + EL_THREADS / 32 - 1) / (EL_THREADS / 32);
    int workers = n_sm / n_slices;
    if (workers < 1) workers = 1;
    if (workers > want) workers = (int)want;
    a.n_workers = workers;
    const size_t smem = encode_linear_smem(cpl, n_rows, n_layouts);
    cudaError_t e;
#define OVC_LAUNCH_EL(C)                                                                                           \
    do {                                                                                                           \
        e = cudaFuncSetAttribute(encode_linear_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); \
        if (e != cudaSuccess) return cuda_fail(e, "encode_linear kernel attribute");                               \
        encode_linear_kernel<C><<<(unsigned)(workers * n_slices), EL_THREADS, smem, st>>>(a);                      \
    } while (0)
    if (cpl == 8) OVC_LAUNCH_EL(8);
    else if (cpl == 4) OVC_LAUNCH_EL(4);
    else OVC_LAUNCH_EL(2);
#undef OVC_LAUNCH_EL
    e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "encode_linear kernel launch");
    return OVC_OK;
}

}  // namespace ovc

// ------------------------------------------------------------------------------------------------
// The two ends of a policy-in-the-loop transition around ovc_step (config 5): drawing the joint action from the
// policy's logits, and folding the transition's rewards into the running returns.  One small kernel each, where the
// tensor-library formulation launches five and four.
// ------------------------------------------------------------------------------------------------
namespace ovc {

// Gumbel-max draw: argmax_i (logit_i - log(-log u_i)) picks i with probability softmax(logits)_i.
// u_i from Philox4x32-10, key = seed, counter = (row lo, row hi, step lo, 2 * step hi + block): reproducible from
// (seed, step, row) alone.  counter[0] = the step; counter[1] = arrival count of the CTAs of the current launch: the
// last CTA to finish advances the step (every CTA has read it by then), so a captured CUDA graph draws fresh numbers at
// every replay without any host involvement.
__global__ void __launch_bounds__(256) sample_actions_kernel(const float *__restrict__ scores, int ld, int n_actions, long long n_rows,
                                                             unsigned long long seed, unsigned long long *counter,
                                                             int32_t *__restrict__ actions) {
    const unsigned long long step = *reinterpret_cast<volatile unsigned long long *>(counter);
    const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (row < n_rows) {
        const float *s = scores + row * ld;
        const uint32_t c3 = (uint32_t)(step >> 32) << 1;
        const Philox4 A = philox4x32_10(seed, (uint32_t)row, (uint32_t)((unsigned long long)row >> 32), (uint32_t)step, c3);
        Philox4 B = A;
        if (n_actions > 4) B = philox4x32_10(seed, (uint32_t)row, (uint32_t)((unsigned long long)row >> 32), (uint32_t)step, c3 | 1u);
        int best = 0;
        float best_v = -INFINITY;
        for (int i = 0; i < n_actions; i++) {
            const uint32_t r = i < 4 ? A.v[i] : B.v[i - 4];
            const float u = ((float)(r >> 9) + 0.5f) * 1.1920928955078125e-7f;  // (k + 0.5) / 2^23, exact in float32: never 0 or 1
            const float v = s[i] - logf(-logf(u));
            if (v > best_v) best_v = v, best = i;
        }
        actions[row] = best;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned long long arrived = atomicAdd(counter + 1, 1ull);
        if (arrived == (unsigned long long)gridDim.x - 1) {
            counter[1] = 0;
            counter[0] = step + 1;
            __threadfence();
        }
    }
}

// ret_sparse[e] += sparse[e];  ret_mixed[e] += sparse[e] + factor * (shaped[e][0] + shaped[e][1])   (rllib.py:328-329)
__global__ void __launch_bounds__(256) accumulate_returns_kernel(const int32_t *__restrict__ sparse, const int32_t *__restrict__ shaped,
                                                                 float factor, long long n_envs, long long *__restrict__ ret_sparse,
                                                                 float *__restrict__ ret_mixed) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_envs) return;
    const int sp = sparse[e];
    const int2 sh = reinterpret_cast<const int2 *>(shaped)[e];
    if (ret_sparse) ret_sparse[e] += sp;
    if (ret_mixed) ret_mixed[e] = ((ret_mixed[e] + (float)sp) + factor * (float)sh.x) + factor * (float)sh.y;
}

static int sample_actions_impl(const float *scores, int ld, int n_actions, long long n_rows, unsigned long long seed,
                               unsigned long long *counter, int32_t *actions, cudaStream_t st) {
    if (!scores || !counter || !actions) return fail(OVC_E_BADARG, "null pointer argument");
    if (n_actions < 1 || n_actions > 8 || ld < n_actions) return fail(OVC_E_BADARG, "n_actions must be 1..8 and <= ld", n_actions);
    if (n_rows < 0) return fail(OVC_E_BADARG, "negative row count");
    if (n_rows == 0) return OVC_OK;
    sample_actions_kernel<<<(unsigned)((n_rows + 255) / 256), 256, 0, st>>>(scores, ld, n_actions, n_rows, seed, counter, actions);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "sample_actions kernel launch");
    return OVC_OK;
}

static int accumulate_returns_impl(const int32_t *sparse, const int32_t *shaped, float factor, long long n_envs, long long *ret_sparse,
                                   float *ret_mixed, cudaStream_t st) {
    if (!sparse || !shaped) return fail(OVC_E_BADARG, "null pointer argument");
    if (n_envs < 0) return fail(OVC_E_BADARG, "negative env count");
    if (n_envs == 0) return OVC_OK;
    accumulate_returns_kernel<<<(unsigned)((n_envs + 255) / 256), 256, 0, st>>>(sparse, shaped, factor, n_envs, ret_sparse, ret_mixed);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "accumulate_returns kernel launch");
    return OVC_OK;
}

}  // namespace ovc
