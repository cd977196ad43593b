// ovc_lstm.cuh — K11 lstm_head_kernel (included by ovc_b200.cu after ovc_tail.cuh).
//
// The recurrent end of the reference's LSTM PPO model (human_aware_rl/ppo/ppo_rllib.py:89-238, RllibLSTMPPOModel: the
// dense layers of 64, then tf.keras.layers.LSTM(256), then the logits and value heads on its output) and the action draw,
// in ONE kernel per transition:
//
//   gates  = [x | h_in] . W^T + b               x bf16 [rows][64], h_in bf16 [rows][256], W bf16 [1024][320], b float32
//   c_out  = sigmoid(f) * c_in + sigmoid(i) * tanh(g);   h_out = bf16(sigmoid(o) * tanh(c_out))
//   s      = h_out . W_heads^T + b_heads          W_heads bf16 [8][256]
//   draw / logp / value as K8 (draw_row, advance_step)
//
// Layout.  A warp owns 16 rows; a CTA of LH_WARPS warps walks row tiles of LH_ROWS (persistent grid).  The warp's A
// fragments of [x | h_in] (20 k-steps) are loaded once per tile into registers with K8's first-layer trick (lane (g, t)
// holds 8 consecutive inputs of rows g and g + 8 per 32-wide block, the B fragments read the same k assignment, so every
// operand stays in its natural order).  The gate rows arrive permuted by the host: slice j (64 rows) holds hidden units
// 16 j .. 16 j + 15, n-tile q = 4 half + gate of it units 16 j + 8 half + 0..7 of gate i / f / g / o.  Lane (g, t) then
// holds all four gates of units 16 j + 8 half + 2 t, + 1 for rows g and g + 8, and the cell update runs in the
// accumulators.  The two halves' h_out (m16n8 C layout) are directly the A fragment of k-step j of the heads (the m16k16
// identity K8 uses), so the heads accumulate slice by slice and h_out is never re-read.
//
// The 640 KB gate matrix does not fit shared memory: it streams slice by slice (40 KB) through a two-stage cp.async ring
// that all warps of the CTA consume, one pass per tile; LH_ROWS rows per pass amortise that L2 -> SM traffic.  Tensor
// work is mma.sync m16n8k16 (bf16 -> fp32), as in K8: the chain from gates to cell to heads lives in registers.
#pragma once
#include <cuda_bf16.h>

namespace ovc {

constexpr int LH_WARPS = 12;  // as many as the register file holds at one CTA per SM (<= 168 registers per thread)
constexpr int LH_THREADS = 32 * LH_WARPS;
constexpr int LH_ROWS = 16 * LH_WARPS;  // rows per tile
constexpr int LH_X = 64;                // LSTM input width
constexpr int LH_U = 256;               // cell size
constexpr int LH_K = LH_X + LH_U;       // 320
constexpr int LH_KS2 = LH_K / 32;       // 10 blocks of 32 inputs
constexpr int LH_SLICE = 64;            // gate rows per slice: 16 units x 4 gates
constexpr int LH_NSLICE = 4 * LH_U / LH_SLICE;
constexpr int LH_WS = LH_K + 32;        // shared row stride of a slice (elements): 32 mod 64, LDS.128 conflict free
constexpr int LH_HS = LH_U + 8;         // shared row stride of the heads (elements): LDS.32 conflict free
constexpr size_t LH_SMEM = (size_t)2 * LH_SLICE * LH_WS * 2 + (size_t)PT_NOUT * LH_HS * 2 + (size_t)4 * LH_U * 4 + PT_NOUT * 4;

struct LstmHeadArgs {
    const __nv_bfloat16 *x;        // [n_rows][64]
    const __nv_bfloat16 *h_in;     // [n_rows][256]
    const float *c_in;             // [n_rows][256]
    const int32_t *reset;          // [ceil(n_rows / 2)] or null: state zero for both rows of env e where reset[e] != 0
    long long n_rows;
    const __nv_bfloat16 *w;        // [1024][320], gate rows permuted (see above)
    const float *b;                // [1024], same permutation
    const __nv_bfloat16 *w_heads;  // [8][256]
    const float *b_heads;          // [8]
    int n_actions;
    unsigned long long seed;
    unsigned long long *counter;   // [2]: step, arrival scratch (as ovc_sample_actions)
    __nv_bfloat16 *h_out;          // [n_rows][256], may alias h_in
    float *c_out;                  // [n_rows][256], may alias c_in
    __nv_bfloat16 *snap_h;         // [n_rows][256] or null: the state the row used (after the reset rule)
    float *snap_c;                 // [n_rows][256] or null
    int32_t *actions;              // [n_rows]
    float *values, *logp, *scores; // [n_rows], [n_rows], [n_rows][8]; each nullable
    const int32_t *swap;           // one view (lstm_head_kernel<true>): [n_rows] or null, and the seat: row r is environment
    int seat;                      // r's agent at player seat ^ (swap[r] != 0), reset[r] its reset
};

__device__ __forceinline__ void lh_load_slice(__nv_bfloat16 *dst, const __nv_bfloat16 *w, int slice) {
    const __nv_bfloat16 *src = w + (size_t)slice * LH_SLICE * LH_K;
    for (int i = threadIdx.x; i < LH_SLICE * (LH_K / 8); i += LH_THREADS) {
        const int r = i / (LH_K / 8), c = i - r * (LH_K / 8);
        const unsigned d = (unsigned)__cvta_generic_to_shared(dst + r * LH_WS + 8 * c);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(src + (size_t)r * LH_K + 8 * c) : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
}

__device__ __forceinline__ float lh_sigmoid(float v) { return 1.f / (1.f + expf(-v)); }

__device__ __forceinline__ unsigned lh_pack(float a, float b) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const unsigned *>(&h);
}

// VIEW: one agent's row per environment: row r resets with reset[r], draws on the joint row g = view_row(r) and writes
// actions[g]; the state, values, logp and scores stay indexed by r.
template <bool VIEW>
__global__ void __launch_bounds__(LH_THREADS, 1) lstm_head_kernel(const LstmHeadArgs p) {
    extern __shared__ __align__(16) char lh_smem[];
    __nv_bfloat16 *ring = reinterpret_cast<__nv_bfloat16 *>(lh_smem);  // [2][64][LH_WS]
    __nv_bfloat16 *wh = ring + 2 * LH_SLICE * LH_WS;                    // [8][LH_HS]
    float *bs = reinterpret_cast<float *>(wh + PT_NOUT * LH_HS);        // [1024]
    float *bh = bs + 4 * LH_U;                                          // [8]

    const unsigned long long step = *reinterpret_cast<volatile unsigned long long *>(p.counter);
    const long long n_tiles = (p.n_rows + LH_ROWS - 1) / LH_ROWS;
    if ((long long)blockIdx.x < n_tiles) lh_load_slice(ring, p.w, 0);
    for (int i = threadIdx.x; i < PT_NOUT * (LH_U / 8); i += LH_THREADS) {
        const int r = i / (LH_U / 8), c = i - r * (LH_U / 8);
        *reinterpret_cast<uint4 *>(wh + r * LH_HS + 8 * c) = __ldg(reinterpret_cast<const uint4 *>(p.w_heads + r * LH_U) + c);
    }
    for (int i = threadIdx.x; i < 4 * LH_U; i += LH_THREADS) bs[i] = p.b[i];
    for (int i = threadIdx.x; i < PT_NOUT; i += LH_THREADS) bh[i] = p.b_heads[i];
    __syncthreads();  // the heads' bias is read at the start of every tile, before the ring's first barrier

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    int k = 0;  // slices consumed by this CTA: the ring stage is k & 1
    for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const long long r0 = tile * LH_ROWS + warp * 16 + g, r1 = r0 + 8;
        const bool in0 = r0 < p.n_rows, in1 = r1 < p.n_rows;
        const bool z0 = !in0 || (p.reset && p.reset[VIEW ? r0 : r0 >> 1]), z1 = !in1 || (p.reset && p.reset[VIEW ? r1 : r1 >> 1]);
        // ---- A fragments of [x | h_in]: 8 consecutive inputs of rows g, g + 8 per 32-wide block ----
        uint4 xa[LH_KS2], xb[LH_KS2];
#pragma unroll
        for (int s2 = 0; s2 < LH_KS2; s2++) {
            if (s2 < LH_X / 32) {
                xa[s2] = in0 ? __ldg(reinterpret_cast<const uint4 *>(p.x + r0 * LH_X + 32 * s2 + 8 * t)) : make_uint4(0, 0, 0, 0);
                xb[s2] = in1 ? __ldg(reinterpret_cast<const uint4 *>(p.x + r1 * LH_X + 32 * s2 + 8 * t)) : make_uint4(0, 0, 0, 0);
            } else {  // h_in may alias h_out: plain loads, all of this warp's rows read before any is written
                const int k0 = 32 * (s2 - LH_X / 32) + 8 * t;
                xa[s2] = z0 ? make_uint4(0, 0, 0, 0) : *reinterpret_cast<const uint4 *>(p.h_in + r0 * LH_U + k0);
                xb[s2] = z1 ? make_uint4(0, 0, 0, 0) : *reinterpret_cast<const uint4 *>(p.h_in + r1 * LH_U + k0);
                if (p.snap_h) {
                    if (in0) *reinterpret_cast<uint4 *>(p.snap_h + r0 * LH_U + k0) = xa[s2];
                    if (in1) *reinterpret_cast<uint4 *>(p.snap_h + r1 * LH_U + k0) = xb[s2];
                }
            }
        }
        float heads[4];
        {
            const float2 b = *reinterpret_cast<const float2 *>(bh + 2 * t);
            heads[0] = b.x, heads[1] = b.y, heads[2] = b.x, heads[3] = b.y;
        }
        for (int j = 0; j < LH_NSLICE; j++, k++) {
            // ---- the ring: slice k + 1 streams in while slice k is consumed ----
            const bool more = j + 1 < LH_NSLICE || tile + gridDim.x < n_tiles;
            if (more) {
                lh_load_slice(ring + ((k + 1) & 1) * LH_SLICE * LH_WS, p.w, (j + 1) % LH_NSLICE);
                asm volatile("cp.async.wait_group 1;" ::: "memory");
            } else {
                asm volatile("cp.async.wait_group 0;" ::: "memory");
            }
            __syncthreads();
            const __nv_bfloat16 *ws = ring + (k & 1) * LH_SLICE * LH_WS;
            unsigned ha[4];  // A fragment of k-step j of the heads: h_out of units 16 j .. 16 j + 15
#pragma unroll
            for (int half = 0; half < 2; half++) {
                float acc[4][4];
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    const float2 b = *reinterpret_cast<const float2 *>(bs + LH_SLICE * j + 8 * (4 * half + q) + 2 * t);
                    acc[q][0] = b.x, acc[q][1] = b.y, acc[q][2] = b.x, acc[q][3] = b.y;
                }
#pragma unroll
                for (int s2 = 0; s2 < LH_KS2; s2++) {
                    const unsigned a_lo[4] = {xa[s2].x, xb[s2].x, xa[s2].y, xb[s2].y};
                    const unsigned a_hi[4] = {xa[s2].z, xb[s2].z, xa[s2].w, xb[s2].w};
#pragma unroll
                    for (int q = 0; q < 4; q++) {
                        const uint4 b = *reinterpret_cast<const uint4 *>(ws + (8 * (4 * half + q) + g) * LH_WS + 32 * s2 + 8 * t);
                        mma_bf16_16816(acc[q], a_lo, b.x, b.y);
                        mma_bf16_16816(acc[q], a_hi, b.z, b.w);
                    }
                }
                // ---- the cell: lane (g, t) holds units u, u + 1 of rows g (e = 0, 1) and g + 8 (e = 2, 3) ----
                const int u = 16 * j + 8 * half + 2 * t;
                float h[4];
#pragma unroll
                for (int rr = 0; rr < 2; rr++) {
                    const long long row = rr ? r1 : r0;
                    const bool z = rr ? z1 : z0, in = rr ? in1 : in0;
                    const float2 c = z ? make_float2(0.f, 0.f) : *reinterpret_cast<const float2 *>(p.c_in + row * LH_U + u);
                    float cn[2];
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        const int ix = 2 * rr + e;
                        const float cv = e ? c.y : c.x;
                        cn[e] = lh_sigmoid(acc[1][ix]) * cv + lh_sigmoid(acc[0][ix]) * tanhf(acc[2][ix]);
                        h[ix] = lh_sigmoid(acc[3][ix]) * tanhf(cn[e]);
                    }
                    const unsigned hp = lh_pack(h[2 * rr], h[2 * rr + 1]);
                    ha[2 * half + rr] = hp;
                    if (in) {
                        if (p.snap_c) *reinterpret_cast<float2 *>(p.snap_c + row * LH_U + u) = c;
                        *reinterpret_cast<float2 *>(p.c_out + row * LH_U + u) = make_float2(cn[0], cn[1]);
                        *reinterpret_cast<unsigned *>(p.h_out + row * LH_U + u) = hp;
                    }
                }
            }
            // ---- heads: k-step j (units 16 j + 2 t, + 1 in ha[0..1], 16 j + 8 + 2 t, + 1 in ha[2..3]) ----
            const unsigned hf[4] = {ha[0], ha[1], ha[2], ha[3]};
            const unsigned b0 = *reinterpret_cast<const unsigned *>(wh + g * LH_HS + 16 * j + 2 * t);
            const unsigned b1 = *reinterpret_cast<const unsigned *>(wh + g * LH_HS + 16 * j + 8 + 2 * t);
            mma_bf16_16816(heads, hf, b0, b1);
            __syncthreads();  // every warp is done with this stage before the next iteration refills it
        }
        if (p.scores) {
            if (in0) *reinterpret_cast<float2 *>(p.scores + r0 * PT_NOUT + 2 * t) = make_float2(heads[0], heads[1]);
            if (in1) *reinterpret_cast<float2 *>(p.scores + r1 * PT_NOUT + 2 * t) = make_float2(heads[2], heads[3]);
        }
        // ---- the draw (ovc_sample_actions, as K8) ----
        auto draw = [&](long long row, float s0, float s1) {
            float lp = 0.f;
            const long long g = VIEW ? view_row(p.swap, p.seat, row, p.n_rows) : row;
            const int best = draw_row<true>(s0, s1, p.seed, step, g, p.n_actions, lane, t, lp);
            if (row < p.n_rows) {
                if (t == 0) p.actions[g] = best;
                if (p.logp && t == 0) p.logp[row] = lp;
                if (p.values && t == (p.n_actions >> 1)) p.values[row] = (p.n_actions & 1) ? s1 : s0;
            }
        };
        draw(r0, heads[0], heads[1]);
        draw(r1, heads[2], heads[3]);
    }
    advance_step(p.counter, step);
}

// view: the one-view instantiation (a.swap / a.seat, ovc_lstm_head_view)
static int lstm_head_impl(const LstmHeadArgs &a, cudaStream_t st, bool view = false) {
    if (!a.x || !a.h_in || !a.c_in || !a.w || !a.b || !a.w_heads || !a.b_heads || !a.counter || !a.h_out || !a.c_out || !a.actions)
        return fail(OVC_E_BADARG, "null pointer argument");
    if ((((uintptr_t)a.x | (uintptr_t)a.h_in | (uintptr_t)a.w | (uintptr_t)a.w_heads | (uintptr_t)a.snap_h) & 15) != 0)
        return fail(OVC_E_BADARG, "x, h_in, w, w_heads and snap_h must be 16-byte aligned");
    if ((((uintptr_t)a.c_in | (uintptr_t)a.c_out | (uintptr_t)a.snap_c | (uintptr_t)a.b | (uintptr_t)a.b_heads | (uintptr_t)a.scores) & 7) != 0 ||
        ((uintptr_t)a.h_out & 3) != 0)
        return fail(OVC_E_BADARG, "c_in, c_out, snap_c, b, b_heads and scores must be 8-byte aligned, h_out 4-byte aligned");
    if (view && (((uintptr_t)a.actions | (uintptr_t)a.values | (uintptr_t)a.logp | (uintptr_t)a.reset | (uintptr_t)a.swap) & 3) != 0)
        return fail(OVC_E_BADARG, "actions, values, logp, reset and swap must be 4-byte aligned");
    if (a.n_actions < 1 || a.n_actions > 7) return fail(OVC_E_BADARG, "n_actions must be 1..7 (head n_actions is the value)", a.n_actions);
    if (a.n_rows < 0) return fail(OVC_E_BADARG, "negative row count");
    if (a.n_rows == 0) return OVC_OK;
    int dev = 0, n_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    const long long n_tiles = (a.n_rows + LH_ROWS - 1) / LH_ROWS;
    const unsigned grid = (unsigned)(n_tiles < n_sm ? n_tiles : n_sm);
    cudaError_t e = cudaFuncSetAttribute(view ? lstm_head_kernel<true> : lstm_head_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)LH_SMEM);
    if (e != cudaSuccess) return cuda_fail(e, "lstm_head kernel attribute");
    if (view) lstm_head_kernel<true><<<grid, LH_THREADS, LH_SMEM, st>>>(a);
    else lstm_head_kernel<false><<<grid, LH_THREADS, LH_SMEM, st>>>(a);
    e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "lstm_head kernel launch");
    return OVC_OK;
}

}  // namespace ovc
