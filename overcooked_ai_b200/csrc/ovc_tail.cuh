// ovc_tail.cuh — K8 policy_tail_kernel (included by ovc_b200.cu after ovc_encfc.cuh).
//
// The narrow end of the rollout policy (reference model: human_aware_rl/ppo/ppo_rllib.py:43-79 — after the
// convolutions three dense layers of 64 and the action / value heads) and the action draw, in ONE kernel:
//
//   x [rows][K0] bf16 (pre-activation of the layer before, leaky ReLU applied on load)
//     -> dense K0 -> 64 -> leaky ReLU -> (64 -> 64 -> leaky ReLU) x n_hidden -> heads 64 -> 8 (logits + value)
//     -> Gumbel-max draw of the action (the ovc_sample_actions definition) -> actions int32, values float32
//
// As library calls this is 4 GEMMs with N <= 64, 4 activation passes, 2 copies and the draw: ~12 launches that are
// each latency bound around 2.5 GFLOP of arithmetic.  Here a warp owns 16 rows at a time and never leaves its registers: the first
// layer's A fragments are 16-byte global loads, every later layer's A fragments ARE the previous layer's accumulator
// fragments (the m16n8 C layout of two adjacent n-tiles is the m16k16 A layout), weights sit in shared memory in the
// order the B fragments are read (one 8- or 16-byte LDS per fragment pair, conflict free).  Tensor-core work is
// mma.sync m16n8k16 bf16 -> fp32: at K, N <= 160 x 64 per layer there is no tile a wgmma pipeline (64-row warpgroup
// tiles with operands staged through shared memory) could amortise its hand-offs over — the chain of four tiny layers is
// dependency bound, and registers are the shortest path between them.
#pragma once
#include <cuda_bf16.h>

namespace ovc {

constexpr int PT_THREADS = 512;
constexpr int PT_H = 64;        // hidden width
constexpr int PT_HS = 80;       // shared-memory row stride of the 64-wide weight matrices (elements): LDS.64 conflict free
constexpr int PT_NOUT = 8;      // heads: up to 7 logits + value, one n-tile

struct PolicyTailArgs {
    const __nv_bfloat16 *x;        // [n_rows][K0]
    const __nv_bfloat16 *w_first;  // [64][K0]
    const float *b_first;          // [64]
    const __nv_bfloat16 *w_hidden; // [n_hidden][64][64]
    const float *b_hidden;         // [n_hidden][64]
    const __nv_bfloat16 *w_heads;  // [8][64]
    const float *b_heads;          // [8]
    long long n_rows;
    int n_hidden, n_actions;
    float in_slope, slope;
    unsigned long long seed;
    unsigned long long *counter;   // [2]: step, arrival scratch (as ovc_sample_actions)
    int32_t *actions;              // [n_rows]
    float *values;                 // [n_rows] or null
    float *scores;                 // [n_rows][8] or null
    float *logp;                   // [n_rows] or null: log-probability of the drawn action (LOGP)
    __nv_bfloat16 *hidden;         // [n_rows][64]: the last 64-wide activation (HIDDEN)
    const int32_t *swap;           // View, Rows: per-environment seat swap, nullable
    int seat;                      // View, Rows: the agent's player
    const int32_t *rows, *range;   // Rows, Joint: the row map and its compact range [range[0], range[1])
    const int32_t *offsets;        // grouped: member k's rows [offsets[k], offsets[k + 1])
    int n_members;                 // grouped
};

__device__ __forceinline__ void mma_bf16_16816(float c[4], const unsigned a[4], unsigned b0, unsigned b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ unsigned pack_lrelu(float x0, float x1, float slope) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(fmaxf(x0, x0 * slope), fmaxf(x1, x1 * slope));
    return *reinterpret_cast<const unsigned *>(&h);
}

// leaky ReLU on a bf16 pair the way the tensor library's activation pass computes it: in float32, rounded once
__device__ __forceinline__ unsigned lrelu_bf16x2(unsigned v, float slope) {
    return pack_lrelu(__uint_as_float(v << 16), __uint_as_float(v & 0xFFFF0000u), slope);
}

// One 64-wide layer whose A operand is the previous layer's activations held as fragments a[4][4] (k-steps of 16).
// ws: weights [n][PT_HS] in the permuted order (position 16 s + 4 t + e  <->  k = 16 s + (e < 2 ? 2 t + e : 8 + 2 t + e - 2)),
// so the (b0, b1) pair of lane (g, t) for k-step s is ONE 8-byte load at ws[n][16 s + 4 t].
template <int NT>
__device__ __forceinline__ void dense64(float acc[NT][4], const unsigned a[4][4], const __nv_bfloat16 *ws, const float *bs, int g, int t) {
#pragma unroll
    for (int j = 0; j < NT; j++) {
        const float2 b = *reinterpret_cast<const float2 *>(bs + 8 * j + 2 * t);
        acc[j][0] = b.x, acc[j][1] = b.y, acc[j][2] = b.x, acc[j][3] = b.y;
    }
#pragma unroll
    for (int s = 0; s < 4; s++)
#pragma unroll
        for (int j = 0; j < NT; j++) {
            const uint2 b = *reinterpret_cast<const uint2 *>(ws + (8 * j + g) * PT_HS + 16 * s + 4 * t);
            mma_bf16_16816(acc[j], a[s], b.x, b.y);
        }
}

// accumulators of a 64-wide layer -> A fragments of the next one
__device__ __forceinline__ void to_fragments(unsigned a[4][4], const float acc[8][4], float slope) {
#pragma unroll
    for (int s = 0; s < 4; s++) {
        a[s][0] = pack_lrelu(acc[2 * s][0], acc[2 * s][1], slope);
        a[s][1] = pack_lrelu(acc[2 * s][2], acc[2 * s][3], slope);
        a[s][2] = pack_lrelu(acc[2 * s + 1][0], acc[2 * s + 1][1], slope);
        a[s][3] = pack_lrelu(acc[2 * s + 1][2], acc[2 * s + 1][3], slope);
    }
}

// Shared-memory copy of a tail's weights (K8, K10), in the orders the fragment loads read.  NT threads per CTA.
struct TailSmem {
    __nv_bfloat16 *w1, *wh, *wo;  // [64][FS] natural k order; [n_hidden][64][PT_HS] and [8][PT_HS] permuted k order
    float *b1, *bh, *bo;          // [64], [n_hidden][64], [8]
};

// row stride of the first layer's weights: 32 mod 64 elements, LDS.128 conflict free
__host__ __device__ constexpr int tail_fs(int k0) { return k0 % 64 == 32 ? k0 : k0 + 32; }

__host__ __device__ constexpr size_t tail_smem_bytes(int k0, int n_hidden) {
    return (size_t)PT_H * tail_fs(k0) * 2 + (size_t)(n_hidden * PT_H + PT_NOUT) * PT_HS * 2 + (size_t)(PT_H + n_hidden * PT_H + PT_NOUT) * 4;
}

template <int K0, int NT, class Args>
__device__ __forceinline__ TailSmem tail_weights_to_smem(char *smem, const Args &p) {
    constexpr int FS = tail_fs(K0);
    TailSmem w;
    w.w1 = reinterpret_cast<__nv_bfloat16 *>(smem);
    w.wh = w.w1 + PT_H * FS;
    w.wo = w.wh + p.n_hidden * PT_H * PT_HS;
    w.b1 = reinterpret_cast<float *>(w.wo + PT_NOUT * PT_HS);
    w.bh = w.b1 + PT_H;
    w.bo = w.bh + p.n_hidden * PT_H;
    for (int i = threadIdx.x; i < PT_H * (K0 / 8); i += NT) {
        const int n = i / (K0 / 8), c = i - n * (K0 / 8);
        *reinterpret_cast<uint4 *>(w.w1 + n * FS + 8 * c) = __ldg(reinterpret_cast<const uint4 *>(p.w_first + (size_t)n * K0) + c);
    }
    for (int i = threadIdx.x; i < (p.n_hidden * PT_H + PT_NOUT) * (PT_H / 8); i += NT) {
        // 8 consecutive inputs of one row (hidden layers' rows, then the heads' with the same stride): natural k = 16 s + r,
        // r = 8 h + 2 tt + e  ->  permuted position 16 s + 4 tt + 2 h + e: the four input pairs go to four 4-byte slots
        const int n = i >> 3, q = i & 7, s2 = q >> 1, h = q & 1;
        const __nv_bfloat16 *src = n < p.n_hidden * PT_H ? p.w_hidden + (size_t)n * PT_H : p.w_heads + (size_t)(n - p.n_hidden * PT_H) * PT_H;
        const uint4 v = __ldg(reinterpret_cast<const uint4 *>(src) + q);
        unsigned *dst = reinterpret_cast<unsigned *>(w.wh + n * PT_HS + 16 * s2 + 2 * h);
        dst[0] = v.x, dst[2] = v.y, dst[4] = v.z, dst[6] = v.w;
    }
    for (int i = threadIdx.x; i < PT_H; i += NT) w.b1[i] = p.b_first[i];
    for (int i = threadIdx.x; i < p.n_hidden * PT_H; i += NT) w.bh[i] = p.b_hidden[i];
    for (int i = threadIdx.x; i < PT_NOUT; i += NT) w.bo[i] = p.b_heads[i];
    return w;
}

// First layer K0 = 32 KS2 -> 64 of the 16 rows of a warp.  Lane (g, t) holds inputs 32 s2 + 8 t + 0..7 of rows g and g + 8:
// frag(s2, a_lo, a_hi) gives them as the A fragments of k-steps 2 s2 (a_lo) and 2 s2 + 1 (a_hi) — elements 0-3 of the
// eight feed a_lo (a0 / a2 for row g, a1 / a3 for row g + 8), 4-7 feed a_hi.  The B fragments use the same assignment,
// so the weights stay in their natural order.
template <int KS2, class Frag>
__device__ __forceinline__ void first_layer64(float acc[8][4], const TailSmem &w, int g, int t, Frag &&frag) {
    constexpr int FS = tail_fs(32 * KS2);
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const float2 b = *reinterpret_cast<const float2 *>(w.b1 + 8 * j + 2 * t);
        acc[j][0] = b.x, acc[j][1] = b.y, acc[j][2] = b.x, acc[j][3] = b.y;
    }
#pragma unroll
    for (int s2 = 0; s2 < KS2; s2++) {
        unsigned a_lo[4], a_hi[4];
        frag(s2, a_lo, a_hi);
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const uint4 b = *reinterpret_cast<const uint4 *>(w.w1 + (8 * j + g) * FS + 32 * s2 + 8 * t);
            mma_bf16_16816(acc[j], a_lo, b.x, b.y);
            mma_bf16_16816(acc[j], a_hi, b.z, b.w);
        }
    }
}

// The layers after the first: ReLU-family activation, n_hidden 64 -> 64 layers, then the heads.  out[0][0..1]: heads 2 t,
// 2 t + 1 of row g; out[0][2..3]: the same of row g + 8.  Without ``out`` (HEADS false) it stops before the heads and
// leaves the last layer's activations bf16(act(z)) in ``a`` as A fragments.
template <bool HEADS = true>
__device__ __forceinline__ void tail_layers(float out[1][4], float acc[8][4], const TailSmem &w, int n_hidden, float slope, int g, int t,
                                            unsigned (*a_out)[4] = nullptr) {
    unsigned a[4][4];
    to_fragments(a, acc, slope);
    for (int l = 0; l < n_hidden; l++) {
        dense64<8>(acc, a, w.wh + l * PT_H * PT_HS, w.bh + l * PT_H, g, t);
        to_fragments(a, acc, slope);
    }
    if constexpr (HEADS) {
        dense64<1>(out, a, w.wo, w.bo, g, t);
    } else {
#pragma unroll
        for (int s = 0; s < 4; s++)
#pragma unroll
            for (int i = 0; i < 4; i++) a_out[s][i] = a[s][i];
    }
}

// The draw of ovc_sample_actions on one row whose heads 2 t, 2 t + 1 (s0, s1) lane t of the row's four lanes holds: they
// use words 2 t, 2 t + 1 of Philox block t / 2 at counter (row, step).  Every lane returns the drawn action; with LOGP
// also its log-probability (lp).  All 32 lanes must take part (shuffles).
template <bool LOGP>
__device__ __forceinline__ int draw_row(float s0, float s1, unsigned long long seed, unsigned long long step, long long row, int n_actions,
                                        int lane, int t, float &lp) {
    const Philox4 P = philox4x32_10(seed, (uint32_t)row, (uint32_t)((unsigned long long)row >> 32), (uint32_t)step,
                                    ((uint32_t)(step >> 32) << 1) | (uint32_t)(t >> 1));
    const float u0 = draw_uniform(P.v[(2 * t) & 3]), u1 = draw_uniform(P.v[(2 * t + 1) & 3]);
    float v0 = 2 * t < n_actions ? s0 - logf(-logf(u0)) : -INFINITY;
    const float v1 = 2 * t + 1 < n_actions ? s1 - logf(-logf(u1)) : -INFINITY;
    int best = 2 * t;
    if (v1 > v0) v0 = v1, best = 2 * t + 1;
#pragma unroll
    for (int d = 1; d <= 2; d <<= 1) {  // argmax over the four lanes of the row (lowest index wins ties, as a serial scan does)
        const float ov = __shfl_xor_sync(0xFFFFFFFFu, v0, d);
        const int ob = __shfl_xor_sync(0xFFFFFFFFu, best, d);
        if (ov > v0 || (ov == v0 && ob < best)) v0 = ov, best = ob;
    }
    if constexpr (LOGP) {  // log-softmax at the drawn action over the same four lanes: max, then the sum of exp
        const bool in0 = 2 * t < n_actions, in1 = 2 * t + 1 < n_actions;
        float m = fmaxf(in0 ? s0 : -INFINITY, in1 ? s1 : -INFINITY);
#pragma unroll
        for (int d = 1; d <= 2; d <<= 1) m = fmaxf(m, __shfl_xor_sync(0xFFFFFFFFu, m, d));
        float se = (in0 ? expf(s0 - m) : 0.f) + (in1 ? expf(s1 - m) : 0.f);
#pragma unroll
        for (int d = 1; d <= 2; d <<= 1) se += __shfl_xor_sync(0xFFFFFFFFu, se, d);
        const int src = (lane & ~3) | (best >> 1);  // the lane holding head `best`
        const float b0 = __shfl_sync(0xFFFFFFFFu, s0, src), b1 = __shfl_sync(0xFFFFFFFFu, s1, src);
        lp = ((best & 1) ? b1 : b0) - (m + logf(se));
    }
    return best;
}

// The joint row 2 r + p(r) of compact row r, whose agent sits at player p(r) = seat ^ (swap[r] != 0) (swap nullable);
// rows past the end map to 2 r + seat (their draws are discarded)
__device__ __forceinline__ long long view_row(const int32_t *swap, int seat, long long r, long long n_rows) {
    return 2 * r + (seat ^ (swap && r < n_rows && __ldg(swap + r) != 0));
}

// K8's tile: rows r0 and r0 + 8 of x (g = r0 mod 8 within the warp's 16 rows; rows from r_end on read as zeros) through the
// first layer, the hidden layers and the heads into out; without HEADS, the last 64-wide layer's A fragments into a_out.
template <int KS2, bool HEADS = true, class Row>
__device__ __forceinline__ void tail_tile(float out[1][4], const PolicyTailArgs &p, const TailSmem &w, Row r0, Row r_end, int g, int t,
                                          unsigned (*a_out)[4] = nullptr) {
    constexpr int K0 = 32 * KS2;
    const Row r1 = r0 + 8;
    const float in_slope = p.in_slope;
    // ---- first layer: A fragments straight from global memory, 16 bytes (8 inputs) per load ----
    // The loads of PRE k-steps are issued before the first layer, the rest as it reaches them.  PRE is KS2 except at
    // KS2 = 6: holding all 48 registers of x under the 128-register cap made every drawing form spill 20 - 44 bytes
    // there, and with 4 up front none spills.
    constexpr int PRE = KS2 == 6 ? 4 : KS2;
    uint4 xa[KS2], xb[KS2];
    auto load = [&](int s2) {
        xa[s2] = r0 < r_end ? __ldg(reinterpret_cast<const uint4 *>(p.x + (long long)r0 * K0 + 32 * s2 + 8 * t)) : make_uint4(0, 0, 0, 0);
        xb[s2] = r1 < r_end ? __ldg(reinterpret_cast<const uint4 *>(p.x + (long long)r1 * K0 + 32 * s2 + 8 * t)) : make_uint4(0, 0, 0, 0);
    };
#pragma unroll
    for (int s2 = 0; s2 < PRE; s2++) load(s2);
    float acc[8][4];
    first_layer64<KS2>(acc, w, g, t, [&](int s2, unsigned a_lo[4], unsigned a_hi[4]) {
        if (s2 >= PRE) load(s2);
        a_lo[0] = lrelu_bf16x2(xa[s2].x, in_slope), a_lo[1] = lrelu_bf16x2(xb[s2].x, in_slope);
        a_lo[2] = lrelu_bf16x2(xa[s2].y, in_slope), a_lo[3] = lrelu_bf16x2(xb[s2].y, in_slope);
        a_hi[0] = lrelu_bf16x2(xa[s2].z, in_slope), a_hi[1] = lrelu_bf16x2(xb[s2].z, in_slope);
        a_hi[2] = lrelu_bf16x2(xa[s2].w, in_slope), a_hi[3] = lrelu_bf16x2(xb[s2].w, in_slope);
    });
    // ---- hidden layers and heads: fragments in, fragments out ----
    tail_layers<HEADS>(out, acc, w, p.n_hidden, p.slope, g, t, a_out);
}

// K8's epilogue on rows r0 and r0 + 8 of a tile (heads in out): per row the scores, the draw (ovc_sample_actions) and the
// action, logp and value, placed by MAP (RowMap): row r is drawn on joint row d, which indexes actions, and the other
// outputs are indexed by o.  Rows from r_end on are drawn with the others (the shuffles need all 32 lanes) and discarded.
template <bool LOGP, RowMap MAP, class Row>
__device__ __forceinline__ void tail_epilogue(const PolicyTailArgs &p, const float out[1][4], unsigned long long step, Row r0, Row r_end,
                                              int lane, int t) {
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const Row r = h ? r0 + 8 : r0;
        const bool in = r < r_end;
        const float s0 = out[0][2 * h], s1 = out[0][2 * h + 1];
        long long d = r, o = r;
        if constexpr (MAP == RowMap::View) d = view_row(p.swap, p.seat, r, p.n_rows);
        if constexpr (MAP == RowMap::Rows) {
            const long long e = in ? (long long)__ldg(p.rows + r) : 0;
            d = 2 * e + (p.seat ^ (p.swap && in && __ldg(p.swap + e) != 0));
        }
        if constexpr (MAP == RowMap::Joint) d = o = in ? (long long)__ldg(p.rows + r) : 0;
        if (p.scores && in) *reinterpret_cast<float2 *>(p.scores + o * PT_NOUT + 2 * t) = make_float2(s0, s1);
        float lp = 0.f;
        const int best = draw_row<LOGP>(s0, s1, p.seed, step, d, p.n_actions, lane, t, lp);
        if (in) {
            if (t == 0) p.actions[d] = best;
            if constexpr (LOGP) if (t == 0) p.logp[o] = lp;
            // the value head is head n_actions: lane n_actions / 2 holds it
            if (p.values && t == (p.n_actions >> 1)) p.values[o] = (p.n_actions & 1) ? s1 : s0;
        }
    }
}

// K8, K0 = 32 * KS2, over the rows MAP names (Rows, Joint: the compact range).  LOGP: also write p.logp; HIDDEN: stop after
// the last 64-wide layer and write its activations to p.hidden instead of the heads and the draw (the LSTM policy's input;
// the counter is neither read nor advanced).
template <int KS2, RowMap MAP, bool LOGP, bool HIDDEN = false>
__global__ void __launch_bounds__(PT_THREADS, 1) policy_tail_kernel(const PolicyTailArgs p) {
    static_assert(!HIDDEN || (MAP == RowMap::Identity && !LOGP), "the hidden form has no draw");
    constexpr int K0 = 32 * KS2;
    extern __shared__ __align__(16) char pt_smem[];

    const unsigned long long step = HIDDEN ? 0ull : *reinterpret_cast<volatile unsigned long long *>(p.counter);
    // ---- weights into shared memory ----
    const TailSmem w = tail_weights_to_smem<K0, PT_THREADS>(pt_smem, p);
    __syncthreads();

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    // the forms over a range count rows in 32 bits (a range of int32 entries), which keeps them within K8's registers
    constexpr bool RANGED = MAP == RowMap::Rows || MAP == RowMap::Joint;
    using Row = typename std::conditional<RANGED, int, long long>::type;
    Row r_beg = 0, r_end = p.n_rows;
    if constexpr (RANGED) {
        r_beg = max(__ldg(p.range), 0);
        r_end = max((int)min((long long)__ldg(p.range + 1), p.n_rows), r_beg);
    }
    const Row n_tiles = (r_end - r_beg + 15) / 16;
    for (Row tile = (Row)blockIdx.x * (PT_THREADS / 32) + warp; tile < n_tiles; tile += (Row)gridDim.x * (PT_THREADS / 32)) {
        const Row r0 = r_beg + tile * 16 + g, r1 = r0 + 8;
        if constexpr (HIDDEN) {  // the A fragments of the last layer's activations, written as [row][64]
            unsigned a[4][4];
            tail_tile<KS2, false>(nullptr, p, w, r0, r_end, g, t, a);
#pragma unroll
            for (int s = 0; s < 4; s++) {
                unsigned *h0 = reinterpret_cast<unsigned *>(p.hidden + r0 * PT_H + 16 * s + 2 * t);
                unsigned *h1 = reinterpret_cast<unsigned *>(p.hidden + r1 * PT_H + 16 * s + 2 * t);
                if (r0 < r_end) h0[0] = a[s][0], h0[4] = a[s][2];
                if (r1 < r_end) h1[0] = a[s][1], h1[4] = a[s][3];
            }
        } else {
            float out[1][4];
            tail_tile<KS2>(out, p, w, r0, r_end, g, t);
            tail_epilogue<LOGP, MAP>(p, out, step, r0, r_end, lane, t);
        }
    }
    if constexpr (!HIDDEN) advance_step(p.counter, step);
}

// Grouped K8 (ovc_policy_tail_grouped): a population of K tails, member k's tables entry k of stacked tables, its rows
// [offsets[k], offsets[k + 1]) (clipped to [0, n_rows)).  The launch's tile list is every member's 16-row tiles in member
// order (a member's last tile partial, never shared with the next member); CTA b takes the contiguous share
// [b T / G, (b + 1) T / G) of the T tiles, so a CTA holds at most a few members' tables, each staged once, and the work is
// balanced whatever the block sizes.  Each row is drawn on its own row index r with the call's step, exactly as
// ovc_policy_tail_logp draws row r, and every CTA advances the counter once.  MAP Joint (ovc_policy_tail_grouped_joint,
// population play): the rows are compact rows, row r drawn on and written at joint row rows[r], as in the joint form.
// 12 warps per CTA (a cap of 170 registers; ptxas uses 112 - 159 over the instantiations, no spills): under K8's 16 warps
// (a cap of 128) the member bookkeeping on top of K8's tile spilled.
constexpr int PT_MAX_MEMBERS = 64;
constexpr int PTG_THREADS = 384;

template <int KS2, bool LOGP, RowMap MAP = RowMap::Identity>
__global__ void __launch_bounds__(PTG_THREADS, 1) policy_tail_grouped_kernel(const PolicyTailArgs p) {
    static_assert(MAP == RowMap::Identity || (MAP == RowMap::Joint && LOGP), "the grouped forms: Identity, or Joint with logp");
    constexpr int K0 = 32 * KS2;
    extern __shared__ __align__(16) char pt_smem[];
    __shared__ int tile0[PT_MAX_MEMBERS + 1], rbeg[PT_MAX_MEMBERS], rend[PT_MAX_MEMBERS];

    const unsigned long long step = *reinterpret_cast<volatile unsigned long long *>(p.counter);
    if (threadIdx.x == 0) {
        int n = 0;
        for (int k = 0; k < p.n_members; k++) {
            const int lo = max(__ldg(p.offsets + k), 0), hi = max((int)min((long long)__ldg(p.offsets + k + 1), p.n_rows), lo);
            tile0[k] = n, rbeg[k] = lo, rend[k] = hi;
            n += (hi - lo + 15) / 16;
        }
        tile0[p.n_members] = n;
    }
    __syncthreads();
    const int total = tile0[p.n_members];
    const int t_lo = (int)((long long)blockIdx.x * total / gridDim.x), t_hi = (int)((long long)(blockIdx.x + 1) * total / gridDim.x);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    int tb = t_lo;
    for (int k = 0; k < p.n_members && tb < t_hi; k++) {
        const int te = min(t_hi, tile0[k + 1]);
        if (te <= tb) continue;
        PolicyTailArgs q = p;  // member k's tables
        q.w_first += (size_t)k * PT_H * K0, q.b_first += (size_t)k * PT_H;
        q.w_hidden += (size_t)k * p.n_hidden * PT_H * PT_H, q.b_hidden += (size_t)k * p.n_hidden * PT_H;
        q.w_heads += (size_t)k * PT_NOUT * PT_H, q.b_heads += (size_t)k * PT_NOUT;
        __syncthreads();  // the previous member's tiles no longer read the shared tables
        const TailSmem w = tail_weights_to_smem<K0, PTG_THREADS>(pt_smem, q);
        __syncthreads();
        const int r_end = rend[k];
        for (int tile = tb + warp; tile < te; tile += PTG_THREADS / 32) {
            const int r0 = rbeg[k] + (tile - tile0[k]) * 16 + g;
            float out[1][4];
            tail_tile<KS2>(out, p, w, r0, r_end, g, t);
            tail_epilogue<LOGP, MAP>(p, out, step, r0, r_end, lane, t);
        }
        tb = te;
    }
    advance_step(p.counter, step);
}

using PolicyTailKernel = void (*)(PolicyTailArgs);

template <int KS2>
static PolicyTailKernel policy_tail_pick(RowMap map, bool logp, bool hid, bool grouped) {
    if (grouped && map == RowMap::Joint) return policy_tail_grouped_kernel<KS2, true, RowMap::Joint>;
    if (grouped) return logp ? policy_tail_grouped_kernel<KS2, true> : policy_tail_grouped_kernel<KS2, false>;
    if (hid) return policy_tail_kernel<KS2, RowMap::Identity, false, true>;
    switch (map) {
    case RowMap::View: return logp ? policy_tail_kernel<KS2, RowMap::View, true> : policy_tail_kernel<KS2, RowMap::View, false>;
    case RowMap::Rows: return logp ? policy_tail_kernel<KS2, RowMap::Rows, true> : policy_tail_kernel<KS2, RowMap::Rows, false>;
    case RowMap::Joint: return policy_tail_kernel<KS2, RowMap::Joint, true>;
    default: return logp ? policy_tail_kernel<KS2, RowMap::Identity, true> : policy_tail_kernel<KS2, RowMap::Identity, false>;
    }
}

// The launch of every K8 form, its arguments checked: one wave of CTAs at most, never more than the SMs.  The grouped form
// runs 12 warps per CTA over at most n_rows / 16 + n_members tiles (a member's last tile partial).
static int policy_tail_launch(const PolicyTailArgs &a, int k0, cudaStream_t st, RowMap map, bool hid, bool grouped) {
    int dev = 0, n_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    const int threads = grouped ? PTG_THREADS : PT_THREADS;
    const size_t smem = tail_smem_bytes(k0, a.n_hidden) + 16;
    const long long n_tiles = (a.n_rows + 15) / 16 + (grouped ? a.n_members : 0), want = (n_tiles + threads / 32 - 1) / (threads / 32);
    const unsigned grid = (unsigned)(want < n_sm ? want : n_sm);
    PolicyTailKernel kern = nullptr;
#define OVC_PT_CASE(KS2) \
    case KS2: kern = policy_tail_pick<KS2>(map, a.logp, hid, grouped); break;
    switch (k0 / 32) {
        OVC_PT_CASE(1) OVC_PT_CASE(2) OVC_PT_CASE(3) OVC_PT_CASE(4) OVC_PT_CASE(5) OVC_PT_CASE(6) OVC_PT_CASE(7) OVC_PT_CASE(8)
    }
#undef OVC_PT_CASE
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return cuda_fail(e, grouped ? "policy_tail_grouped kernel attribute" : "policy_tail kernel attribute");
    kern<<<grid, threads, smem, st>>>(a);
    e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, grouped ? "policy_tail_grouped kernel launch" : "policy_tail kernel launch");
    return OVC_OK;
}

// map Identity: ovc_policy_tail_grouped; Joint: ovc_policy_tail_grouped_joint (a.rows = jrow, logp required)
static int policy_tail_grouped_impl(const PolicyTailArgs &a, int k0, cudaStream_t st, RowMap map = RowMap::Identity) {
    if (!a.x || !a.w_first || !a.b_first || !a.w_heads || !a.b_heads || !a.counter || !a.actions || !a.offsets ||
        (a.n_hidden > 0 && (!a.w_hidden || !a.b_hidden)) || (map == RowMap::Joint && (!a.rows || !a.logp)))
        return fail(OVC_E_BADARG, "null pointer argument");
    if ((((uintptr_t)a.x | (uintptr_t)a.w_first | (uintptr_t)a.w_hidden | (uintptr_t)a.w_heads) & 15) != 0)
        return fail(OVC_E_BADARG, "x and the weight tables must be 16-byte aligned");
    if ((((uintptr_t)a.b_first | (uintptr_t)a.b_hidden | (uintptr_t)a.b_heads | (uintptr_t)a.scores | (uintptr_t)a.counter) & 7) != 0)
        return fail(OVC_E_BADARG, "biases, scores and counter must be 8-byte aligned");
    if ((((uintptr_t)a.actions | (uintptr_t)a.values | (uintptr_t)a.logp | (uintptr_t)a.offsets) & 3) != 0)
        return fail(OVC_E_BADARG, "actions, values, logp and offsets must be 4-byte aligned");
    if (((uintptr_t)a.rows & 3) != 0) return fail(OVC_E_BADARG, "jrow must be 4-byte aligned");
    if (a.n_members < 1 || a.n_members > PT_MAX_MEMBERS) return fail(OVC_E_BADARG, "n_members must be 1..64", a.n_members);
    if (k0 < 32 || k0 > 256 || k0 % 32) return fail(OVC_E_BADARG, "k0 must be a multiple of 32 in 32..256", k0);
    if (a.n_hidden < 0 || a.n_hidden > 8) return fail(OVC_E_BADARG, "n_hidden must be 0..8", a.n_hidden);
    if (a.n_actions < 1 || a.n_actions > 7) return fail(OVC_E_BADARG, "n_actions must be 1..7 (head n_actions is the value)", a.n_actions);
    if (!(a.in_slope >= 0.f && a.in_slope <= 1.f && a.slope >= 0.f && a.slope <= 1.f)) return fail(OVC_E_BADARG, "slopes must lie in [0, 1]");
    if (a.n_rows < 0 || a.n_rows > 0x7FFFFFFFll) return fail(OVC_E_BADARG, "n_rows must lie in [0, 2^31)", a.n_rows);
    if (a.n_rows == 0) return OVC_OK;
    return policy_tail_launch(a, k0, st, map, false, true);
}

// map: ovc_policy_tail[_logp] Identity, ovc_policy_tail_view View, ovc_policy_tail_rows Rows, ovc_policy_tail_joint Joint.
// hid: the HIDDEN form into a.hidden (no heads, no draw; a.w_heads / a.b_heads are staged but never read, so the entry
// point passes the first layer's tables, which are at least as large, in their place).
static int policy_tail_impl(const PolicyTailArgs &a, int k0, cudaStream_t st, RowMap map = RowMap::Identity, bool hid = false) {
    const bool view = map != RowMap::Identity, ranged = map == RowMap::Rows || map == RowMap::Joint;
    if (!a.x || !a.w_first || !a.b_first || !a.w_heads || !a.b_heads || (hid ? !a.hidden : (!a.counter || !a.actions)) ||
        (a.n_hidden > 0 && (!a.w_hidden || !a.b_hidden)) || (ranged && (!a.rows || !a.range)) || (map == RowMap::Joint && !a.logp))
        return fail(OVC_E_BADARG, "null pointer argument");
    if ((((uintptr_t)a.x | (uintptr_t)a.w_first) & 15) != 0) return fail(OVC_E_BADARG, "x and w_first must be 16-byte aligned");
    if (hid && ((uintptr_t)a.hidden & 3) != 0) return fail(OVC_E_BADARG, "hidden must be 4-byte aligned");
    if (view && (((uintptr_t)a.actions | (uintptr_t)a.values | (uintptr_t)a.logp | (uintptr_t)a.swap) & 3) != 0)
        return fail(OVC_E_BADARG, "actions, values, logp and swap must be 4-byte aligned");
    if ((((uintptr_t)a.rows | (uintptr_t)a.range) & 3) != 0) return fail(OVC_E_BADARG, "rows and range must be 4-byte aligned");
    if (view && ((uintptr_t)a.scores & 7) != 0) return fail(OVC_E_BADARG, "scores must be 8-byte aligned");
    if (k0 < 32 || k0 > 256 || k0 % 32) return fail(OVC_E_BADARG, "k0 must be a multiple of 32 in 32..256", k0);
    if (a.n_hidden < 0 || a.n_hidden > 8) return fail(OVC_E_BADARG, "n_hidden must be 0..8", a.n_hidden);
    if (a.n_actions < 1 || a.n_actions > 7) return fail(OVC_E_BADARG, "n_actions must be 1..7 (head n_actions is the value)", a.n_actions);
    if (!(a.in_slope >= 0.f && a.in_slope <= 1.f && a.slope >= 0.f && a.slope <= 1.f)) return fail(OVC_E_BADARG, "slopes must lie in [0, 1]");
    if (a.n_rows < 0) return fail(OVC_E_BADARG, "negative row count");
    if (a.n_rows == 0) return OVC_OK;
    return policy_tail_launch(a, k0, st, map, hid, false);
}

}  // namespace ovc
