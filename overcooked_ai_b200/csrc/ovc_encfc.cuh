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
constexpr int EL_MAX_MEMBERS = 64;

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
    int seat;                  // one view (encode_linear_kernel<CPL, true>): the agent's seat, view_swap its per-env swap
    const int32_t *rows;       // the rows map (encode_linear_kernel<CPL, true, true>): compact row r is environment rows[r]
    const int32_t *range;      //   for r in [range[0], range[1]) (device memory)
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

// VIEW: one view per environment, player p(e) = seat ^ (view_swap[e] != 0), written to out[e] ([n_envs][n_out]); the
// object part and that view's gathers run in the same order as in the two-view kernel, so the row is bit-identical to
// row 2 e + p(e) of it.  ROWS (with VIEW): compact rows r in [range[0], range[1]) only, environment rows[r] written to
// out[r]; a CTA whose share of the range is empty leaves before its prologue.
// MASKED (encode_linear_masked_kernel, without view_swap): entry r < n_envs of the list is environment list[r] >> 2 with the
// views of mask list[r] & 3 (bit v: view v); the object part is computed once, and the views in the mask go to consecutive
// rows from first[r] in ascending view order, each bit for bit row 2 e + v of the two-view kernel.
// GROUPED (encode_linear_grouped_kernel, two views, without view_swap): n_members members, member k's tables entry k of
// stacked wt / bias and its environments [offsets[k], offsets[k + 1]); the CTAs are split over (member, column slice,
// worker), a.n_workers workers per member, so a CTA loads its member's column slice once and walks only that member's
// environments.
template <int CPL, bool VIEW, bool ROWS, bool MASKED, bool GROUPED = false>
__device__ __forceinline__ void encode_linear_body(const EncLinArgs &a, const int32_t *list = nullptr, const int32_t *first = nullptr,
                                                   const int32_t *offsets = nullptr) {
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
    const __nv_bfloat16 *wt = a.wt;
    const float *bias = a.bias;
    long long r_beg = 0, r_end = a.n_envs;
    int slice = blockIdx.x % n_slices, worker = blockIdx.x / n_slices;
    if constexpr (GROUPED) {
        int bx = blockIdx.x;
        const int per = n_slices * a.n_workers, k = bx / per;
        bx -= k * per;
        wt += (size_t)k * a.W * a.H * N_PLANES * a.n_out, bias += (size_t)k * a.n_out;
        r_beg = min(max((long long)__ldg(offsets + k), 0ll), a.n_envs);
        r_end = max(min((long long)__ldg(offsets + k + 1), a.n_envs), r_beg);
        slice = bx % n_slices, worker = bx / n_slices;
    }
    const int col0 = slice * CS;
    if constexpr (ROWS) {
        r_beg = max(__ldg(a.range), 0);
        r_end = min((long long)__ldg(a.range + 1), a.n_envs);
        if (r_beg + (long long)worker * (EL_THREADS / 32) >= r_end) return;
    }
    if constexpr (MASKED) {
        if ((long long)worker * (EL_THREADS / 32) >= r_end) return;
    }
    if constexpr (GROUPED) {
        if (r_beg + (long long)worker * (EL_THREADS / 32) >= r_end) return;
    }

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
            const uint4 *src = reinterpret_cast<const uint4 *>(wt + (size_t)(cell * N_PLANES + plane) * a.n_out + col0) + c;
            reinterpret_cast<uint4 *>(tab)[i] = __ldg(src);
        }
        // terrain and urgency sums: one thread per (layout, column); the cells' loads are independent (plane ids staged in
        // shared memory first), issued four at a time, added in cell order
        for (int i = threadIdx.x; i < (a.n_layouts + 1) * CS; i += EL_THREADS) {
            const int l = i / CS, c = i - l * CS;
            const unsigned char *tp = tplane + l * 256;
            const __nv_bfloat16 *w = wt + col0 + c;
            float s = l == a.n_layouts ? 0.f : bias[col0 + c];
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

    for (long long r = r_beg + (long long)worker * NW + warp; r < r_end; r += stride) {
        long long env, row0 = 0;
        int vmask = 3;
        if constexpr (MASKED) {
            const int entry = __ldg(list + r);
            env = entry >> 2, vmask = entry & 3;
            if (!vmask) continue;  // the whole warp holds entry r
            row0 = __ldg(first + r);
        } else {
            env = ROWS ? (long long)__ldg(a.rows + r) : r;
        }
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
        auto view = [&](int p, long long row) {  // p = the player whose view this is
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
            __nv_bfloat16 *dst = a.out + row * a.n_out + col0 + lane * CPL;
            if constexpr (CPL == 8) *reinterpret_cast<uint4 *>(dst) = make_uint4(packed[0], packed[1], packed[2], packed[3]);
            else if constexpr (CPL == 4) *reinterpret_cast<uint2 *>(dst) = make_uint2(packed[0], packed[1]);
            else *reinterpret_cast<unsigned *>(dst) = packed[0];
        };
        if constexpr (MASKED) {
            if (vmask & 1) view(0, row0);
            if (vmask & 2) view(1, row0 + (vmask & 1));
        } else if constexpr (VIEW) {
            view(a.seat ^ swap, r);
        } else {
#pragma unroll
            for (int p = 0; p < 2; p++) view(p, 2 * env + (swap ? 1 - p : p));
        }
    }
}

template <int CPL, bool VIEW, bool ROWS = false>
__global__ void __launch_bounds__(EL_THREADS, 1) encode_linear_kernel(const EncLinArgs a) {
    encode_linear_body<CPL, VIEW, ROWS, false>(a);
}

// A kernel of its own, so that the list and first-row pointers stay out of EncLinArgs and encode_linear_kernel's code
template <int CPL>
__global__ void __launch_bounds__(EL_THREADS, 1) encode_linear_masked_kernel(const EncLinArgs a, const int32_t *list, const int32_t *first) {
    encode_linear_body<CPL, false, false, true>(a, list, first);
}

template <int CPL>
__global__ void __launch_bounds__(EL_THREADS, 1) encode_linear_grouped_kernel(const EncLinArgs a, const int32_t *offsets) {
    encode_linear_body<CPL, false, false, false, true>(a, nullptr, nullptr, offsets);
}

// MASKED and GROUPED together (population play): member k walks list entries [offsets[k], offsets[k + 1]) with its table
template <int CPL>
__global__ void __launch_bounds__(EL_THREADS, 1) encode_linear_grouped_masked_kernel(const EncLinArgs a, const int32_t *list,
                                                                                     const int32_t *first, const int32_t *offsets) {
    encode_linear_body<CPL, false, false, true, true>(a, list, first, offsets);
}

static size_t encode_linear_smem(int cpl, int n_rows, int n_layouts) {
    const size_t CS = 32 * (size_t)cpl;
    return (size_t)n_rows * CS * 2 + ((size_t)n_layouts + 1) * CS * 4 + (size_t)n_layouts * (16 * 4 + 2 * 4 + 128 * 2 + 256) + 16;
}

// seat < 0: both views (ovc_encode_linear); 0 / 1: one view per environment (ovc_encode_linear_view, view_swap = swap);
// with rows / range: the rows map (ovc_encode_linear_rows); with list / first: n_envs list entries (ovc_encode_linear_masked);
// n_members > 0: a population's stacked tables over its environment offsets (ovc_encode_linear_grouped), or with list / first
// over its list entry offsets (ovc_encode_linear_grouped_masked)
static int encode_linear_impl(const ovc_layout_t *layouts, int n_layouts, const int32_t *state, const int32_t *view_swap,
                              const void *wt, const float *bias, void *out, long long n_envs, int S, int W, int H, int horizon,
                              int n_out, float neg_slope, cudaStream_t st, int seat = -1, const int32_t *rows = nullptr,
                              const int32_t *range = nullptr, const int32_t *list = nullptr, const int32_t *first = nullptr,
                              const int32_t *offsets = nullptr, int n_members = 0) {
    const bool rows_map = rows || range, masked = list || first, grouped = n_members != 0;
    if (!out || !wt || !bias || (rows_map && (!rows || !range)) || (masked && (!list || !first)) || (grouped && !offsets))
        return fail(OVC_E_BADARG, "null pointer argument");
    if (grouped && (n_members < 1 || n_members > EL_MAX_MEMBERS)) return fail(OVC_E_BADARG, "n_members must be 1..64", n_members);
    if (grouped && ((uintptr_t)offsets & 3) != 0) return fail(OVC_E_BADARG, "offsets must be 4-byte aligned");
    if ((((uintptr_t)out | (uintptr_t)wt) & 15) != 0) return fail(OVC_E_BADARG, "weights and output must be 16-byte aligned");
    if (seat >= 0 && ((uintptr_t)view_swap & 3) != 0) return fail(OVC_E_BADARG, "swap must be 4-byte aligned");
    if ((((uintptr_t)rows | (uintptr_t)range) & 3) != 0) return fail(OVC_E_BADARG, "rows and range must be 4-byte aligned");
    if ((((uintptr_t)list | (uintptr_t)first) & 3) != 0) return fail(OVC_E_BADARG, "list and first must be 4-byte aligned");
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
    a.n_out = n_out, a.neg_slope = neg_slope, a.seat = seat, a.rows = rows, a.range = range;
    const int n_slices = n_out / (32 * cpl);
    const long long want = (n_envs + EL_THREADS / 32 - 1) / (EL_THREADS / 32);
    int workers = n_sm / n_slices;
    if (grouped) workers /= n_members;  // workers per member: one wave of CTAs in all
    if (workers < 1) workers = 1;
    if (workers > want) workers = (int)want;
    a.n_workers = workers;
    const size_t smem = encode_linear_smem(cpl, n_rows, n_layouts);
    cudaError_t e;
#define OVC_LAUNCH_EL(C, ...)                                                                                                 \
    do {                                                                                                                      \
        e = cudaFuncSetAttribute(encode_linear_kernel<C, __VA_ARGS__>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); \
        if (e != cudaSuccess) return cuda_fail(e, "encode_linear kernel attribute");                                          \
        encode_linear_kernel<C, __VA_ARGS__><<<(unsigned)(workers * n_slices), EL_THREADS, smem, st>>>(a);                    \
    } while (0)
#define OVC_LAUNCH_ELM(C)                                                                                                     \
    do {                                                                                                                      \
        e = cudaFuncSetAttribute(encode_linear_masked_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);     \
        if (e != cudaSuccess) return cuda_fail(e, "encode_linear kernel attribute");                                          \
        encode_linear_masked_kernel<C><<<(unsigned)(workers * n_slices), EL_THREADS, smem, st>>>(a, list, first);             \
    } while (0)
#define OVC_LAUNCH_ELG(C)                                                                                                     \
    do {                                                                                                                      \
        e = cudaFuncSetAttribute(encode_linear_grouped_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);    \
        if (e != cudaSuccess) return cuda_fail(e, "encode_linear kernel attribute");                                          \
        encode_linear_grouped_kernel<C><<<grid, EL_THREADS, smem, st>>>(a, offsets);                                          \
    } while (0)
#define OVC_LAUNCH_ELGM(C)                                                                                                    \
    do {                                                                                                                      \
        e = cudaFuncSetAttribute(encode_linear_grouped_masked_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); \
        if (e != cudaSuccess) return cuda_fail(e, "encode_linear kernel attribute");                                          \
        encode_linear_grouped_masked_kernel<C><<<grid, EL_THREADS, smem, st>>>(a, list, first, offsets);                      \
    } while (0)
    if (grouped && masked) {
        const unsigned grid = (unsigned)(workers * n_slices * n_members);
        if (cpl == 8) OVC_LAUNCH_ELGM(8);
        else if (cpl == 4) OVC_LAUNCH_ELGM(4);
        else OVC_LAUNCH_ELGM(2);
    } else if (grouped) {
        const unsigned grid = (unsigned)(workers * n_slices * n_members);
        if (cpl == 8) OVC_LAUNCH_ELG(8);
        else if (cpl == 4) OVC_LAUNCH_ELG(4);
        else OVC_LAUNCH_ELG(2);
    } else if (masked) {
        if (cpl == 8) OVC_LAUNCH_ELM(8);
        else if (cpl == 4) OVC_LAUNCH_ELM(4);
        else OVC_LAUNCH_ELM(2);
    } else if (rows_map) {
        if (cpl == 8) OVC_LAUNCH_EL(8, true, true);
        else if (cpl == 4) OVC_LAUNCH_EL(4, true, true);
        else OVC_LAUNCH_EL(2, true, true);
    } else if (seat >= 0) {
        if (cpl == 8) OVC_LAUNCH_EL(8, true);
        else if (cpl == 4) OVC_LAUNCH_EL(4, true);
        else OVC_LAUNCH_EL(2, true);
    } else {
        if (cpl == 8) OVC_LAUNCH_EL(8, false);
        else if (cpl == 4) OVC_LAUNCH_EL(4, false);
        else OVC_LAUNCH_EL(2, false);
    }
#undef OVC_LAUNCH_EL
#undef OVC_LAUNCH_ELM
#undef OVC_LAUNCH_ELG
#undef OVC_LAUNCH_ELGM
    e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "encode_linear kernel launch");
    return OVC_OK;
}

// ------------------------------------------------------------------------------------------------
// K12 encode_linear_wgrad_kernel: the weight gradient of K7's layer, from the same packed records,
//     dwt[f][c] += sum over rows r of enc(r)[f] * dz[r][c]
// with enc(r) the lossless encoding of row r's record and view (never materialised) and dz the gradient at the layer's
// pre-activation.  K7's decomposition read backwards: each dynamic entry (value, feature row) of a row scatters
// value * dz[r][:] into its row of the gradient; the object entries, held objects included, are shared by both views of a
// record, so they scatter value * (dz[2m] + dz[2m + 1]) once; the terrain rows of layout l get the column sum of dz over
// the rows on l, the urgency rows the column sum over the urgent rows.
//
// One CTA per SM holds the float32 gradient of its column slice of the 19 dynamic planes in shared memory ([W*H*19][CS],
// 190 KB on a 5x4 grid at 128 columns; 32 columns reach K7's largest grid).  A warp takes one record at a time; lane l
// owns columns l, l + 32, ... of the slice (conflict-free shared accesses, coalesced dz loads); lanes decode object slots
// and pass the entries round by shuffle, as K7 does.  Warps of a CTA meet in shared memory through atomicAdd; each CTA
// adds its non-zero sums to dwt once, with global reductions.  Summation order is unspecified (it depends on the grid and
// on scheduling); on operands whose float32 sums are exact in any order the result is exact.
// ------------------------------------------------------------------------------------------------
constexpr int WG_SMEM_LIMIT = 227 * 1024;  // sm_90's opt-in shared memory per block: the grids K12 takes are checked against it

struct EncWgradArgs {
    const ovc_layout_t *layouts;
    const int32_t *state;     // [n_rec][S]
    const int32_t *swap;      // one view: nullable
    const float *dz;          // [n_rec or 2 n_rec][n_out]
    float *dwt;               // [W*H*26][n_out]
    long long n_rec;
    int n_layouts, S, W, H, horizon, n_out, n_workers;
    int seat;                 // -1: two views (row 2 m + v); 0 / 1: one view (row m, player seat ^ (swap[m] != 0))
};

static size_t encode_linear_wgrad_smem(int cpl, int n_dyn_rows, int n_layouts) {
    const size_t CS = 32 * (size_t)cpl;
    return (size_t)n_dyn_rows * CS * 4 + ((size_t)n_layouts + 1) * CS * 4 + (size_t)n_layouts * (16 * 4 + 2 * 4 + 128 * 2 + 256) + 16;
}

template <int CPL>
__device__ __forceinline__ void wg_scatter(float *g_lane, int row, float value, const float d[CPL]) {
#pragma unroll
    for (int i = 0; i < CPL; i++) atomicAdd(g_lane + row * (32 * CPL) + 32 * i, value * d[i]);
}

template <int CPL>
__global__ void __launch_bounds__(EL_THREADS, 1) encode_linear_wgrad_kernel(const EncWgradArgs a) {
    constexpr int CS = 32 * CPL;
    constexpr int NW = EL_THREADS / 32;
    extern __shared__ __align__(16) char wg_smem[];
    const int WH = a.W * a.H;
    const int n_rows = WH * EL_DYN;
    float *g = reinterpret_cast<float *>(wg_smem);                                       // [n_rows][CS]
    float *tsum = g + (size_t)n_rows * CS;                                               // [n_layouts][CS]
    float *urg = tsum + a.n_layouts * CS;                                                // [CS]
    int *cook = reinterpret_cast<int *>(urg + CS);                                       // [n_layouts][16]
    int *nslots = cook + a.n_layouts * 16;                                               // [n_layouts][2]
    unsigned short *srow = reinterpret_cast<unsigned short *>(nslots + a.n_layouts * 2);  // [n_layouts][128]
    unsigned char *tplane = reinterpret_cast<unsigned char *>(srow + a.n_layouts * 128);  // [n_layouts][256]

    const int n_slices = a.n_out / CS;
    const int slice = blockIdx.x % n_slices, worker = blockIdx.x / n_slices;
    const int col0 = slice * CS;

    for (int i = threadIdx.x; i < (n_rows + a.n_layouts + 1) * CS; i += EL_THREADS) g[i] = 0.f;  // g, tsum, urg
    for (int i = threadIdx.x; i < a.n_layouts * WH; i += EL_THREADS) {
        const int l = i / WH, cell = i - l * WH, x = cell / a.H, y = cell - x * a.H;
        tplane[l * 256 + cell] = (unsigned char)((0x000F0A0E0D0C0B00ull >> ((a.layouts[l].cell[(y << 4) | x] & 7) * 8)) & 0xFF);
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
    __syncthreads();

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float *g_lane = g + lane;
    const long long stride = (long long)a.n_workers * NW;
    const int max_slot_chunks = (a.S - 4 + 31) / 32;
    const bool two = a.seat < 0;
    // the warp's terrain sum for layout t_lid and its urgency sum, in registers: one shared-memory add per layout change
    float t_acc[CPL], u_acc[CPL];
    int t_lid = -1;
#pragma unroll
    for (int i = 0; i < CPL; i++) t_acc[i] = 0.f, u_acc[i] = 0.f;

    for (long long m = (long long)worker * NW + warp; m < a.n_rec; m += stride) {
        const int32_t *__restrict__ rec = a.state + m * a.S;
        const int4 head = __ldg(reinterpret_cast<const int4 *>(rec));
        const int lid = head.w & 0xFF;
        const int n_slots = nslots[2 * lid], n_pots = nslots[2 * lid + 1];
        const int *ck = cook + lid * 16;
        const unsigned short *sr = srow + lid * 128;
        // the rows' gradients in this lane's columns: d0 (view 0, or the one view), d1 (view 1), ds = their sum
        float d0[CPL], d1[CPL], ds[CPL];
        const float *dz0 = a.dz + (two ? 2 * m : m) * a.n_out + col0 + lane;
#pragma unroll
        for (int i = 0; i < CPL; i++) d0[i] = __ldcs(dz0 + 32 * i);
        if (two) {
#pragma unroll
            for (int i = 0; i < CPL; i++) d1[i] = __ldcs(dz0 + a.n_out + 32 * i), ds[i] = d0[i] + d1[i];
        } else {
#pragma unroll
            for (int i = 0; i < CPL; i++) d1[i] = 0.f, ds[i] = d0[i];
        }
        // terrain (per layout) and urgency column sums
        if (lid != t_lid) {
            if (t_lid >= 0) {
#pragma unroll
                for (int i = 0; i < CPL; i++) atomicAdd(tsum + t_lid * CS + 32 * i + lane, t_acc[i]), t_acc[i] = 0.f;
            }
            t_lid = lid;
        }
        const bool urgent = a.horizon - head.x < 40;
#pragma unroll
        for (int i = 0; i < CPL; i++) {
            t_acc[i] += ds[i];
            if (urgent) u_acc[i] += ds[i];
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
            unsigned msk = __ballot_sync(0xFFFFFFFFu, (e[0] | e[1] | e[2] | e[3]) != 0);
            while (msk) {
                const int j = __ffs(msk) - 1;
                msk &= msk - 1;
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    const unsigned w = __shfl_sync(0xFFFFFFFFu, e[q], j);
                    if (w & 0xFFFFu) wg_scatter<CPL>(g_lane, (int)(w >> 16), (float)(short)(w & 0xFFFFu), ds);
                }
            }
        }
        // held objects, at the holder's cell in both views
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
                    if (e[q] & 0xFFFFu) wg_scatter<CPL>(g_lane, (int)(e[q] >> 16), (float)(short)(e[q] & 0xFFFFu), ds);
            }
        }
        // each view's own cell / orientation (planes 0, 2..5) and the partner's (planes 1, 6..9)
        const int ori0 = (p0 >> 8) & 3, ori1 = (p1 >> 8) & 3;
        auto view = [&](int p, const float d[CPL]) {
            const int own_cell = p ? cell1 : cell0, oth_cell = p ? cell0 : cell1;
            const int own_ori = p ? ori1 : ori0, oth_ori = p ? ori0 : ori1;
            wg_scatter<CPL>(g_lane, own_cell + PL_LOC, 1.f, d);
            wg_scatter<CPL>(g_lane, own_cell + PL_ORI + own_ori, 1.f, d);
            wg_scatter<CPL>(g_lane, oth_cell + PL_LOC + 1, 1.f, d);
            wg_scatter<CPL>(g_lane, oth_cell + PL_ORI + 4 + oth_ori, 1.f, d);
        };
        if (two) {
            view(0, d0);
            view(1, d1);
        } else {
            view(a.seat ^ (a.swap ? (__ldg(a.swap + m) != 0) : 0), d0);
        }
    }
#pragma unroll
    for (int i = 0; i < CPL; i++) {
        if (t_lid >= 0) atomicAdd(tsum + t_lid * CS + 32 * i + lane, t_acc[i]);
        atomicAdd(urg + 32 * i + lane, u_acc[i]);
    }
    __syncthreads();

    // flush: the dynamic rows, then each layout's terrain sum at its terrain cells and the urgency sum at every cell
    for (int i = threadIdx.x; i < n_rows * CS; i += EL_THREADS) {
        const float v = g[i];
        if (v != 0.f) {
            const int r = i / CS, c = i - r * CS;
            const int cell = r / EL_DYN, d = r - cell * EL_DYN;
            const int plane = d < 10 ? d : d + 6;
            atomicAdd(a.dwt + (size_t)(cell * N_PLANES + plane) * a.n_out + col0 + c, v);
        }
    }
    for (int i = threadIdx.x; i < (a.n_layouts + 1) * WH * CS; i += EL_THREADS) {
        const int l = i / (WH * CS), rem = i - l * WH * CS, cell = rem / CS, c = rem - cell * CS;
        const int pl = l == a.n_layouts ? (int)PL_URGENCY : (int)tplane[l * 256 + cell];
        const float v = l == a.n_layouts ? urg[c] : tsum[l * CS + c];
        if (pl && v != 0.f) atomicAdd(a.dwt + (size_t)(cell * N_PLANES + pl) * a.n_out + col0 + c, v);
    }
}

// seat < 0: two views (row 2 m + v); 0 / 1: one view per record (row m, player seat ^ (swap[m] != 0))
static int encode_linear_wgrad_impl(const ovc_layout_t *layouts, int n_layouts, const int32_t *state, const int32_t *swap, int seat,
                                    const float *dz, float *dwt, long long n_rec, int S, int W, int H, int horizon, int n_out,
                                    cudaStream_t st) {
    if (!dz || !dwt) return fail(OVC_E_BADARG, "null pointer argument");
    if ((((uintptr_t)dz | (uintptr_t)dwt) & 15) != 0) return fail(OVC_E_BADARG, "dz and dwt must be 16-byte aligned");
    if (((uintptr_t)swap & 3) != 0) return fail(OVC_E_BADARG, "swap must be 4-byte aligned");
    if (W < 1 || W > 16 || H < 1 || H > 16) return fail(OVC_E_BADARG, "grid shape out of range");
    if (n_out < 64 || n_out % 64) return fail(OVC_E_BADARG, "n_out must be a positive multiple of 64", n_out);
    if (n_layouts > EL_MAX_LAYOUTS) return fail(OVC_E_UNSUPPORTED, "encode_linear_wgrad: more than 8 layouts per call", n_layouts);
    const int n_rows = W * H * EL_DYN;
    if (encode_linear_wgrad_smem(1, n_rows, n_layouts) > (size_t)WG_SMEM_LIMIT)
        return fail(OVC_E_UNSUPPORTED, "encode_linear_wgrad: the gradient table of this grid does not fit shared memory", W * H);
    if (n_rec == 0) return OVC_OK;
    int dev = 0, n_sm = 0, max_smem = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    int cpl = 0;
    for (int c = 4; c >= 1; c >>= 1)
        if (n_out % (32 * c) == 0 && encode_linear_wgrad_smem(c, n_rows, n_layouts) <= (size_t)max_smem) {
            cpl = c;
            break;
        }
    if (!cpl) return fail(OVC_E_UNSUPPORTED, "encode_linear_wgrad: the gradient table of this grid does not fit shared memory", W * H);
    EncWgradArgs a;
    a.layouts = layouts, a.state = state, a.swap = seat >= 0 ? swap : nullptr, a.dz = dz, a.dwt = dwt, a.n_rec = n_rec;
    a.n_layouts = n_layouts, a.S = S, a.W = W, a.H = H, a.horizon = horizon, a.n_out = n_out, a.seat = seat;
    const int n_slices = n_out / (32 * cpl);
    const long long want = (n_rec + EL_THREADS / 32 - 1) / (EL_THREADS / 32);
    int workers = n_sm / n_slices;
    if (workers < 1) workers = 1;
    if (workers > want) workers = (int)want;
    a.n_workers = workers;
    const size_t smem = encode_linear_wgrad_smem(cpl, n_rows, n_layouts);
    cudaError_t e;
#define OVC_LAUNCH_WG(C)                                                                                                      \
    do {                                                                                                                      \
        e = cudaFuncSetAttribute(encode_linear_wgrad_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);      \
        if (e != cudaSuccess) return cuda_fail(e, "encode_linear_wgrad kernel attribute");                                    \
        encode_linear_wgrad_kernel<C><<<(unsigned)(workers * n_slices), EL_THREADS, smem, st>>>(a);                           \
    } while (0)
    if (cpl == 4) OVC_LAUNCH_WG(4);
    else if (cpl == 2) OVC_LAUNCH_WG(2);
    else OVC_LAUNCH_WG(1);
#undef OVC_LAUNCH_WG
    e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "encode_linear_wgrad kernel launch");
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

// u = (k + 0.5) / 2^23 from the top 23 bits k of a Philox word: exact in float32, never 0 or 1
__device__ __forceinline__ float draw_uniform(uint32_t r) { return ((float)(r >> 9) + 0.5f) * 1.1920928955078125e-7f; }

// The last CTA of a launch to get here advances the draw step (every CTA has read it by then): counter[1] counts arrivals.
__device__ __forceinline__ void advance_step(unsigned long long *counter, unsigned long long step) {
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

// Where a row of a draw's input goes (the draw kernel below, K8):
//   Identity: row r is joint row r;
//   View: row r is one agent's row of environment r, at player p(r) = seat ^ (swap[r] != 0) (swap nullable): drawn on the
//     joint row 2 r + p(r), which indexes actions; every other output stays indexed by r;
//   Rows: compact rows r in [range[0], range[1]) only, environment e = rows[r] at player p(e): drawn on the joint row
//     2 e + p(e), which indexes actions; every other output stays indexed by r;
//   Joint (K8 only): compact rows r in [range[0], range[1]) only, drawn on the joint row rows[r], which indexes every output.
enum class RowMap { Identity, View, Rows, Joint };

// LOGP: also logp[row] = scores[row][a] - (m + log(sum_i exp(scores[row][i] - m))), m = max_i scores[row][i], at the drawn a.
// Every CTA, with rows in the range or not, takes part in the counter's advance.
template <bool LOGP, RowMap MAP>
__global__ void __launch_bounds__(256) sample_actions_kernel(const float *__restrict__ scores, int ld, int n_actions, long long n_rows,
                                                             unsigned long long seed, unsigned long long *counter,
                                                             int32_t *__restrict__ actions, float *__restrict__ logp,
                                                             const int32_t *__restrict__ swap, int seat, const int32_t *__restrict__ rows,
                                                             const int32_t *__restrict__ range) {
    static_assert(MAP != RowMap::Joint, "the draw has no joint-rows form");
    const unsigned long long step = *reinterpret_cast<volatile unsigned long long *>(counter);
    const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool in = MAP == RowMap::Rows ? row >= max(__ldg(range), 0) && row < min((long long)__ldg(range + 1), n_rows) : row < n_rows;
    if (in) {
        const float *s = scores + row * ld;
        long long g = row;
        if constexpr (MAP != RowMap::Identity) {
            const long long e = MAP == RowMap::Rows ? (long long)__ldg(rows + row) : row;
            g = 2 * e + (seat ^ (swap && swap[e] != 0));
        }
        const uint32_t c3 = (uint32_t)(step >> 32) << 1;
        const Philox4 A = philox4x32_10(seed, (uint32_t)g, (uint32_t)((unsigned long long)g >> 32), (uint32_t)step, c3);
        Philox4 B = A;
        if (n_actions > 4) B = philox4x32_10(seed, (uint32_t)g, (uint32_t)((unsigned long long)g >> 32), (uint32_t)step, c3 | 1u);
        int best = 0;
        float best_v = -INFINITY;
        for (int i = 0; i < n_actions; i++) {
            const uint32_t r = i < 4 ? A.v[i] : B.v[i - 4];
            const float v = s[i] - logf(-logf(draw_uniform(r)));
            if (v > best_v) best_v = v, best = i;
        }
        actions[g] = best;
        if constexpr (LOGP) {
            float m = s[0];
            for (int i = 1; i < n_actions; i++) m = fmaxf(m, s[i]);
            float se = 0.f;
            for (int i = 0; i < n_actions; i++) se += expf(s[i] - m);
            logp[row] = s[best] - (m + logf(se));
        }
    }
    advance_step(counter, step);
}

// ret_sparse[e] += sparse[e];  ret_mixed[e] += sparse[e] + factor * (shaped[e][0] + shaped[e][1])   (rllib.py:328-329)
// ovc_record_transition adds what a sample batch keeps of the transition: rewards[2 e + i] = sparse[e] + f * shaped[e][i]
// (rounded after the product, as a float32 restatement computes it) and dones[e]; f is read from factor_dev when given, so
// a captured graph follows a factor the host changes between replays.
// STATS (ovc_record_transition_stats): also the episode statistics of ovc_episode_stats_t.  The running sums are loaded
// together with the events and the layout ids, in one round trip to memory; a sum is only written back when its increment
// is not zero, and an event count is incremented with a reduction that does not wait for memory (each count belongs to
// one thread, so the result is the same as a load and a store).  Most transitions fire no event, deliver nothing and earn
// no reward: they write the episode length only.
__device__ __forceinline__ void episode_stats_update(const ovc_episode_stats_t &s, long long e, long long n_envs, int2 sh, float r0,
                                                     float r1, bool done) {
    longlong2 *spa = reinterpret_cast<longlong2 *>(s.sparse_by_agent) + e;
    longlong2 *sha = reinterpret_cast<longlong2 *>(s.shaped_by_agent) + e;
    float2 *rwa = s.reward_by_agent ? reinterpret_cast<float2 *>(s.reward_by_agent) + e : nullptr;
    const int2 ev = __ldg(reinterpret_cast<const int2 *>(s.events) + e);
    const int lid = s.layout_id[e];
    const int new_lid = __ldg(s.state + e * s.state_words + 3) & 0xFF;
    const int len = s.ep_length[e] + 1;
    const longlong2 spv = *spa, shv = *sha;
    const float2 rwv = rwa ? *rwa : make_float2(0.f, 0.f);
    long long d0 = 0, d1 = 0;
    if ((ev.x | ev.y) & (1 << OVC_EV_SOUP_DELIVERY)) {
        const int32_t *dv = static_cast<const ovc_layout_t *>(s.layouts)[lid].deliver_value;
        if ((ev.x >> OVC_EV_SOUP_DELIVERY) & 1) d0 = dv[(ev.x >> OVC_EV_RECIPE_SHIFT) & 15];
        if ((ev.y >> OVC_EV_SOUP_DELIVERY) & 1) d1 = dv[(ev.y >> OVC_EV_RECIPE_SHIFT) & 15];
    }
    int32_t *cnt = s.event_counts + e * (2 * OVC_NUM_EVENTS);
#pragma unroll
    for (int i = 0; i < 2; i++)
        for (unsigned m = (unsigned)(i ? ev.y : ev.x) & ((1u << OVC_NUM_EVENTS) - 1u); m; m &= m - 1)
            atomicAdd(cnt + i * OVC_NUM_EVENTS + __ffs(m) - 1, 1);
    // x + 0 == x: the reward sum never holds -0 (it starts at +0 and no reward is -0), so a zero reward may skip the add
    const float2 rw = make_float2(__fadd_rn(rwv.x, r0), __fadd_rn(rwv.y, r1));
    if (!done) {
        if (d0 | d1) *spa = make_longlong2(spv.x + d0, spv.y + d1);
        if (sh.x | sh.y) *sha = make_longlong2(shv.x + sh.x, shv.y + sh.y);
        if (rwa && (r0 != 0.f || r1 != 0.f)) *rwa = rw;
        s.ep_length[e] = len;
        if (new_lid != lid) s.layout_id[e] = new_lid;
        return;
    }
    // the episode ended: into slot count[e] of the records (or counted as dropped), then a fresh running state.  The event
    // counts are read and cleared with atomics, the same kind of access as their increments above.
    const int k = s.count[e];
    const bool keep = k < s.capacity;
    const long long slot = (long long)k * n_envs + e;
    int32_t *dst = keep ? s.rec_event_counts + slot * (2 * OVC_NUM_EVENTS) : nullptr;
#pragma unroll 10
    for (int j = 0; j < 2 * OVC_NUM_EVENTS; j++) {
        const int v = atomicExch(cnt + j, 0);
        if (keep) dst[j] = v;
    }
    if (keep) {
        s.rec_length[slot] = len;
        s.rec_layout[slot] = lid;
        s.rec_partner_seat[slot] = s.partner_seat ? __ldg(s.partner_seat + e) : -1;
        reinterpret_cast<longlong2 *>(s.rec_sparse_by_agent)[slot] = make_longlong2(spv.x + d0, spv.y + d1);
        reinterpret_cast<longlong2 *>(s.rec_shaped_by_agent)[slot] = make_longlong2(shv.x + sh.x, shv.y + sh.y);
        if (rwa) reinterpret_cast<float2 *>(s.rec_reward_by_agent)[slot] = rw;
        s.count[e] = k + 1;
    } else {
        s.dropped[e] += 1;
    }
    *spa = make_longlong2(0, 0);
    *sha = make_longlong2(0, 0);
    if (rwa) *rwa = make_float2(0.f, 0.f);
    s.ep_length[e] = 0;
    s.layout_id[e] = new_lid;
}

// The transition both record kernels write.  VIEW (record_transition_view_kernel): ONE reward per environment, the
// agent's at player p(e) = seat ^ (swap[e] != 0), bit for bit rewards[2 e + p(e)] of the two-row store.
template <bool STATS, bool VIEW>
__device__ __forceinline__ void record_body(long long e, const int32_t *__restrict__ sparse, const int32_t *__restrict__ shaped, float f,
                                            long long n_envs, long long *__restrict__ ret_sparse, float *__restrict__ ret_mixed,
                                            const int32_t *__restrict__ done, const int32_t *__restrict__ swap, int seat,
                                            float *__restrict__ rewards, uint8_t *__restrict__ dones, const ovc_episode_stats_t &stats) {
    const int sp = sparse[e];
    const int2 sh = reinterpret_cast<const int2 *>(shaped)[e];
    if (ret_sparse) ret_sparse[e] += sp;
    if (ret_mixed) ret_mixed[e] = ((ret_mixed[e] + (float)sp) + f * (float)sh.x) + f * (float)sh.y;
    if constexpr (VIEW) {
        const int p = seat ^ (swap && swap[e] != 0);
        rewards[e] = __fadd_rn((float)sp, __fmul_rn(f, (float)(p ? sh.y : sh.x)));
    } else if (rewards) {
        reinterpret_cast<float2 *>(rewards)[e] = make_float2(__fadd_rn((float)sp, __fmul_rn(f, (float)sh.x)), __fadd_rn((float)sp, __fmul_rn(f, (float)sh.y)));
    }
    if (dones) dones[e] = done[e] != 0;
    if constexpr (STATS)
        episode_stats_update(stats, e, n_envs, sh, __fadd_rn((float)sp, __fmul_rn(f, (float)sh.x)), __fadd_rn((float)sp, __fmul_rn(f, (float)sh.y)),
                             done[e] != 0);
}

template <bool STATS>
__global__ void __launch_bounds__(256) accumulate_returns_kernel(const int32_t *__restrict__ sparse, const int32_t *__restrict__ shaped,
                                                                 float factor, long long n_envs, long long *__restrict__ ret_sparse,
                                                                 float *__restrict__ ret_mixed, const float *__restrict__ factor_dev,
                                                                 const int32_t *__restrict__ done, float *__restrict__ rewards,
                                                                 uint8_t *__restrict__ dones, const ovc_episode_stats_t stats) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_envs) return;
    record_body<STATS, false>(e, sparse, shaped, factor_dev ? *factor_dev : factor, n_envs, ret_sparse, ret_mixed, done, nullptr, 0, rewards,
                              dones, stats);
}

// map Identity: rows are joint rows (ovc_sample_actions[_logp]); View: one agent's rows (ovc_sample_actions_view, which
// checks the seat); Rows: the rows map (ovc_sample_actions_rows)
static int sample_actions_impl(const float *scores, int ld, int n_actions, long long n_rows, unsigned long long seed,
                               unsigned long long *counter, int32_t *actions, float *logp, cudaStream_t st, RowMap map = RowMap::Identity,
                               const int32_t *swap = nullptr, int seat = 0, const int32_t *rows = nullptr, const int32_t *range = nullptr) {
    const bool listed = map == RowMap::Rows;
    if (!scores || !counter || !actions || (listed && (!rows || !range))) return fail(OVC_E_BADARG, "null pointer argument");
    if (listed && seat != 0 && seat != 1) return fail(OVC_E_BADARG, "seat must be 0 or 1", seat);
    if (n_actions < 1 || n_actions > 8 || ld < n_actions) return fail(OVC_E_BADARG, "n_actions must be 1..8 and <= ld", n_actions);
    if (n_rows < 0) return fail(OVC_E_BADARG, "negative row count");
    if (listed) {
        if ((((uintptr_t)scores | (uintptr_t)actions | (uintptr_t)logp | (uintptr_t)swap | (uintptr_t)rows | (uintptr_t)range) & 3) != 0)
            return fail(OVC_E_BADARG, "scores, actions, logp, swap, rows and range must be 4-byte aligned");
        if (((uintptr_t)counter & 7) != 0) return fail(OVC_E_BADARG, "counter must be 8-byte aligned");
    } else if (map == RowMap::View && (((uintptr_t)scores | (uintptr_t)actions | (uintptr_t)logp | (uintptr_t)swap) & 3) != 0) {
        return fail(OVC_E_BADARG, "scores, actions, logp and swap must be 4-byte aligned");
    }
    if (n_rows == 0) return OVC_OK;
    const unsigned grid = (unsigned)((n_rows + 255) / 256);
    auto kern = listed                ? (logp ? sample_actions_kernel<true, RowMap::Rows> : sample_actions_kernel<false, RowMap::Rows>)
                : map == RowMap::View ? (logp ? sample_actions_kernel<true, RowMap::View> : sample_actions_kernel<false, RowMap::View>)
                : logp                ? sample_actions_kernel<true, RowMap::Identity>
                                      : sample_actions_kernel<false, RowMap::Identity>;
    kern<<<grid, 256, 0, st>>>(scores, ld, n_actions, n_rows, seed, counter, actions, logp, swap, seat, rows, range);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, listed ? "sample_actions_rows kernel launch" : "sample_actions kernel launch");
    return OVC_OK;
}

// The argument checks of ovc_accumulate_returns / ovc_record_transition[_stats] / ovc_record_transition_view.
static int check_record_args(const int32_t *sparse, const int32_t *shaped, long long n_envs, const int32_t *done, const uint8_t *dones,
                             const ovc_episode_stats_t *stats) {
    if (!sparse || !shaped || (dones && !done)) return fail(OVC_E_BADARG, "null pointer argument");
    if (n_envs < 0) return fail(OVC_E_BADARG, "negative env count");
    if (stats) {
        const ovc_episode_stats_t &s = *stats;
        if (!done || !s.layouts || !s.state || !s.events || !s.event_counts || !s.sparse_by_agent || !s.shaped_by_agent || !s.ep_length ||
            !s.layout_id || !s.count || !s.dropped)
            return fail(OVC_E_BADARG, "null pointer argument (episode statistics)");
        if (s.capacity < 0) return fail(OVC_E_BADARG, "negative record capacity", s.capacity);
        if (s.capacity > 0 && (!s.rec_length || !s.rec_layout || !s.rec_partner_seat || !s.rec_sparse_by_agent || !s.rec_shaped_by_agent ||
                               !s.rec_event_counts || (s.reward_by_agent && !s.rec_reward_by_agent)))
            return fail(OVC_E_BADARG, "null pointer argument (episode records)");
        if (s.state_words < 4) return fail(OVC_E_BADARG, "state_words too small", s.state_words);
        if (((uintptr_t)s.event_counts | (uintptr_t)s.rec_event_counts | (uintptr_t)s.events | (uintptr_t)s.reward_by_agent |
             (uintptr_t)s.rec_reward_by_agent) & 7)
            return fail(OVC_E_BADARG, "event and reward buffers must be 8-byte aligned");
        if (((uintptr_t)s.sparse_by_agent | (uintptr_t)s.shaped_by_agent | (uintptr_t)s.rec_sparse_by_agent | (uintptr_t)s.rec_shaped_by_agent) & 15)
            return fail(OVC_E_BADARG, "int64 sums must be 16-byte aligned");
    }
    return OVC_OK;
}

static int accumulate_returns_impl(const int32_t *sparse, const int32_t *shaped, float factor, long long n_envs, long long *ret_sparse,
                                   float *ret_mixed, const float *factor_dev, const int32_t *done, float *rewards, uint8_t *dones,
                                   const ovc_episode_stats_t *stats, cudaStream_t st) {
    if (int rc = check_record_args(sparse, shaped, n_envs, done, dones, stats)) return rc;
    if (n_envs == 0) return OVC_OK;
    const unsigned grid = (unsigned)((n_envs + 255) / 256);
    if (stats)
        accumulate_returns_kernel<true><<<grid, 256, 0, st>>>(sparse, shaped, factor, n_envs, ret_sparse, ret_mixed, factor_dev, done,
                                                              rewards, dones, *stats);
    else
        accumulate_returns_kernel<false><<<grid, 256, 0, st>>>(sparse, shaped, factor, n_envs, ret_sparse, ret_mixed, factor_dev, done,
                                                               rewards, dones, ovc_episode_stats_t{});
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "accumulate_returns kernel launch");
    return OVC_OK;
}

// ovc_record_transition_view: accumulate_returns_kernel's transition with ONE reward per environment (record_body's VIEW)
template <bool STATS>
__global__ void __launch_bounds__(256) record_transition_view_kernel(const int32_t *__restrict__ sparse, const int32_t *__restrict__ shaped,
                                                                     long long n_envs, long long *__restrict__ ret_sparse,
                                                                     float *__restrict__ ret_mixed, const float *__restrict__ factor_dev,
                                                                     const int32_t *__restrict__ done, const int32_t *__restrict__ swap,
                                                                     int seat, float *__restrict__ rewards, uint8_t *__restrict__ dones,
                                                                     const ovc_episode_stats_t stats) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_envs) return;
    record_body<STATS, true>(e, sparse, shaped, *factor_dev, n_envs, ret_sparse, ret_mixed, done, swap, seat, rewards, dones, stats);
}

static int record_transition_view_impl(const int32_t *sparse, const int32_t *shaped, const int32_t *done, const float *factor_dev,
                                       long long n_envs, const int32_t *swap, int seat, float *rewards, uint8_t *dones,
                                       long long *ret_sparse, float *ret_mixed, const ovc_episode_stats_t *stats, cudaStream_t st) {
    if (!factor_dev || !rewards) return fail(OVC_E_BADARG, "null pointer argument");
    if (int rc = check_record_args(sparse, shaped, n_envs, done, dones, stats)) return rc;
    if (seat != 0 && seat != 1) return fail(OVC_E_BADARG, "seat must be 0 or 1", seat);
    if (((uintptr_t)rewards | (uintptr_t)swap) & 3) return fail(OVC_E_BADARG, "rewards and swap must be 4-byte aligned");
    if (n_envs == 0) return OVC_OK;
    const unsigned grid = (unsigned)((n_envs + 255) / 256);
    if (stats)
        record_transition_view_kernel<true><<<grid, 256, 0, st>>>(sparse, shaped, n_envs, ret_sparse, ret_mixed, factor_dev, done, swap,
                                                                  seat, rewards, dones, *stats);
    else
        record_transition_view_kernel<false><<<grid, 256, 0, st>>>(sparse, shaped, n_envs, ret_sparse, ret_mixed, factor_dev, done, swap,
                                                                   seat, rewards, dones, ovc_episode_stats_t{});
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "record_transition_view kernel launch");
    return OVC_OK;
}

// ovc_record_transition_dense: accumulate_returns_kernel's transition with the potential-based dense reward (use_phi,
// rllib.py:314-319): both agents get sparse + f * dense[e], every operation rounded on its own.  shaped still feeds the
// game statistics.  ONE_VIEW: rewards [n_envs] (the agents' rewards are equal, so no seat is needed), else [n_envs][2].
template <bool STATS, bool ONE_VIEW>
__global__ void __launch_bounds__(256) record_transition_dense_kernel(const int32_t *__restrict__ sparse, const int32_t *__restrict__ shaped,
                                                                      const float *__restrict__ dense, long long n_envs,
                                                                      long long *__restrict__ ret_sparse, float *__restrict__ ret_mixed,
                                                                      const float *__restrict__ factor_dev, const int32_t *__restrict__ done,
                                                                      float *__restrict__ rewards, uint8_t *__restrict__ dones,
                                                                      const ovc_episode_stats_t stats) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_envs) return;
    const float f = *factor_dev;
    const int sp = sparse[e];
    const float fd = __fmul_rn(f, dense[e]);
    const float r = __fadd_rn((float)sp, fd);
    if (ret_sparse) ret_sparse[e] += sp;
    if (ret_mixed) ret_mixed[e] = __fadd_rn(__fadd_rn(__fadd_rn(ret_mixed[e], (float)sp), fd), fd);
    if (rewards) {
        if (ONE_VIEW) rewards[e] = r;
        else reinterpret_cast<float2 *>(rewards)[e] = make_float2(r, r);
    }
    if (dones) dones[e] = done[e] != 0;
    if constexpr (STATS) episode_stats_update(stats, e, n_envs, reinterpret_cast<const int2 *>(shaped)[e], r, r, done[e] != 0);
}

static int record_transition_dense_impl(const int32_t *sparse, const int32_t *shaped, const float *dense, const int32_t *done,
                                        const float *factor_dev, long long n_envs, int one_view, float *rewards, uint8_t *dones,
                                        long long *ret_sparse, float *ret_mixed, const ovc_episode_stats_t *stats, cudaStream_t st) {
    if (!factor_dev || !dense) return fail(OVC_E_BADARG, "null pointer argument");
    if (int rc = check_record_args(sparse, shaped, n_envs, done, dones, stats)) return rc;
    if (one_view != 0 && one_view != 1) return fail(OVC_E_BADARG, "one_view must be 0 or 1", one_view);
    if (((uintptr_t)dense & 3) || ((uintptr_t)rewards & (one_view ? 3 : 7)))
        return fail(OVC_E_BADARG, "dense must be 4-byte aligned, rewards 4-byte (one view) or 8-byte (two rows)");
    if (n_envs == 0) return OVC_OK;
    const unsigned grid = (unsigned)((n_envs + 255) / 256);
    const ovc_episode_stats_t s = stats ? *stats : ovc_episode_stats_t{};
    auto kern = stats ? (one_view ? record_transition_dense_kernel<true, true> : record_transition_dense_kernel<true, false>)
                      : (one_view ? record_transition_dense_kernel<false, true> : record_transition_dense_kernel<false, false>);
    kern<<<grid, 256, 0, st>>>(sparse, shaped, dense, n_envs, ret_sparse, ret_mixed, factor_dev, done, rewards, dones, s);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "record_transition_dense kernel launch");
    return OVC_OK;
}

// Generalized advantage estimation over a window of T transitions (the postprocessing of RLlib's PPO sample batches),
// one thread per environment holding its rows (V = float2: both agents' rows, ovc_gae; V = float: one row, ovc_gae_view),
// walking t backwards.  Every operation is rounded on its own (no FMA contraction) in the order ovc_gae documents, so a
// float32 loop on the host reproduces it bit for bit.  A thread's chain is serial in t, so GAE_UNROLL timesteps of loads
// are issued before they are consumed: with one thread per environment there are too few threads per SM to cover the
// memory latency otherwise.  Without a minimum of 5 CTAs per SM ptxas gives both forms 255 registers (2 CTAs per SM);
// with it, 96 (two rows) and 64 (one row), no spills.
constexpr int GAE_THREADS = 128;
constexpr int GAE_UNROLL = 16;

// a row's advantage at step t from the one at t + 1 (a), its reward r, value v, the next value nv and not-done nt
__device__ __forceinline__ float gae_step(float a, float r, float v, float nv, float nt, float gamma, float gl) {
    const float d = __fsub_rn(__fadd_rn(r, __fmul_rn(__fmul_rn(gamma, nv), nt)), v);
    return __fadd_rn(d, __fmul_rn(__fmul_rn(gl, nt), a));
}
__device__ __forceinline__ float2 gae_step(float2 a, float2 r, float2 v, float2 nv, float nt, float gamma, float gl) {
    return make_float2(gae_step(a.x, r.x, v.x, nv.x, nt, gamma, gl), gae_step(a.y, r.y, v.y, nv.y, nt, gamma, gl));
}
__device__ __forceinline__ float gae_target(float a, float v) { return __fadd_rn(a, v); }
__device__ __forceinline__ float2 gae_target(float2 a, float2 v) { return make_float2(__fadd_rn(a.x, v.x), __fadd_rn(a.y, v.y)); }

template <class V>
__global__ void __launch_bounds__(GAE_THREADS, 5)
    gae_kernel(const V *__restrict__ rewards, const V *__restrict__ values, const uint8_t *__restrict__ dones, const V *__restrict__ last_values,
               long long T, long long n_envs, float gamma, float lambda, V *__restrict__ adv, V *__restrict__ targets) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_envs) return;
    const float gl = __fmul_rn(gamma, lambda);
    V a = {}, nv = last_values[e];
    for (long long t0 = T - 1; t0 >= 0; t0 -= GAE_UNROLL) {
        V r[GAE_UNROLL], v[GAE_UNROLL];
        float nt[GAE_UNROLL];
#pragma unroll
        for (int k = 0; k < GAE_UNROLL; k++)
            if (t0 - k >= 0) {
                const long long i = (t0 - k) * n_envs + e;
                r[k] = __ldcs(rewards + i), v[k] = __ldcs(values + i), nt[k] = dones[i] ? 0.f : 1.f;
            }
#pragma unroll
        for (int k = 0; k < GAE_UNROLL; k++)
            if (t0 - k >= 0) {
                const long long i = (t0 - k) * n_envs + e;
                a = gae_step(a, r[k], v[k], nv, nt[k], gamma, gl);
                __stcs(adv + i, a);
                __stcs(targets + i, gae_target(a, v[k]));
                nv = v[k];
            }
    }
}

// one_row: ovc_gae_view, n environments of one row each; otherwise ovc_gae, n rows, two per environment
static int gae_impl(const float *rewards, const float *values, const uint8_t *dones, const float *last_values, long long T, long long n,
                    float gamma, float lambda, float *adv, float *targets, cudaStream_t st, bool one_row = false) {
    if (!rewards || !values || !dones || !last_values || !adv || !targets) return fail(OVC_E_BADARG, "null pointer argument");
    if (T < 0 || n < 0 || (!one_row && n % 2))
        return fail(OVC_E_BADARG, one_row ? "T and n_envs must be >= 0" : "T must be >= 0 and n_rows even and >= 0");
    if (((uintptr_t)rewards | (uintptr_t)values | (uintptr_t)last_values | (uintptr_t)adv | (uintptr_t)targets) & (one_row ? 3 : 7))
        return fail(OVC_E_BADARG, one_row ? "float buffers must be 4-byte aligned" : "float buffers must be 8-byte aligned");
    const long long n_envs = one_row ? n : n / 2;
    if (T == 0 || n_envs == 0) return OVC_OK;
    const unsigned grid = (unsigned)((n_envs + GAE_THREADS - 1) / GAE_THREADS);
    if (one_row)
        gae_kernel<float><<<grid, GAE_THREADS, 0, st>>>(rewards, values, dones, last_values, T, n_envs, gamma, lambda, adv, targets);
    else
        gae_kernel<float2><<<grid, GAE_THREADS, 0, st>>>((const float2 *)rewards, (const float2 *)values, dones, (const float2 *)last_values, T,
                                                         n_envs, gamma, lambda, (float2 *)adv, (float2 *)targets);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, one_row ? "gae_view kernel launch" : "gae kernel launch");
    return OVC_OK;
}

}  // namespace ovc
