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

template <int KS2>  // K0 = 32 * KS2
__global__ void __launch_bounds__(PT_THREADS, 1) policy_tail_kernel(const PolicyTailArgs p) {
    constexpr int K0 = 32 * KS2;
    constexpr int FS = K0 % 64 == 32 ? K0 : K0 + 32;  // row stride of the first layer's weights: 32 mod 64 elements, LDS.128 conflict free
    extern __shared__ __align__(16) char pt_smem[];
    __nv_bfloat16 *w1 = reinterpret_cast<__nv_bfloat16 *>(pt_smem);            // [64][FS], natural k order
    __nv_bfloat16 *wh = w1 + PT_H * FS;                                       // [n_hidden][64][PT_HS], permuted k order
    __nv_bfloat16 *wo = wh + p.n_hidden * PT_H * PT_HS;                       // [8][PT_HS], permuted
    float *b1 = reinterpret_cast<float *>(wo + PT_NOUT * PT_HS);              // [64]
    float *bh = b1 + PT_H;                                                    // [n_hidden][64]
    float *bo = bh + p.n_hidden * PT_H;                                       // [8]

    const unsigned long long step = *reinterpret_cast<volatile unsigned long long *>(p.counter);
    // ---- weights into shared memory ----
    for (int i = threadIdx.x; i < PT_H * (K0 / 8); i += PT_THREADS) {
        const int n = i / (K0 / 8), c = i - n * (K0 / 8);
        *reinterpret_cast<uint4 *>(w1 + n * FS + 8 * c) = __ldg(reinterpret_cast<const uint4 *>(p.w_first + (size_t)n * K0) + c);
    }
    for (int i = threadIdx.x; i < (p.n_hidden * PT_H + PT_NOUT) * (PT_H / 8); i += PT_THREADS) {
        // 8 consecutive inputs of one row (hidden layers' rows, then the heads' with the same stride): natural k = 16 s + r,
        // r = 8 h + 2 tt + e  ->  permuted position 16 s + 4 tt + 2 h + e: the four input pairs go to four 4-byte slots
        const int n = i >> 3, q = i & 7, s2 = q >> 1, h = q & 1;
        const __nv_bfloat16 *src = n < p.n_hidden * PT_H ? p.w_hidden + (size_t)n * PT_H : p.w_heads + (size_t)(n - p.n_hidden * PT_H) * PT_H;
        const uint4 v = __ldg(reinterpret_cast<const uint4 *>(src) + q);
        unsigned *dst = reinterpret_cast<unsigned *>(wh + n * PT_HS + 16 * s2 + 2 * h);
        dst[0] = v.x, dst[2] = v.y, dst[4] = v.z, dst[6] = v.w;
    }
    for (int i = threadIdx.x; i < PT_H; i += PT_THREADS) b1[i] = p.b_first[i];
    for (int i = threadIdx.x; i < p.n_hidden * PT_H; i += PT_THREADS) bh[i] = p.b_hidden[i];
    for (int i = threadIdx.x; i < PT_NOUT; i += PT_THREADS) bo[i] = p.b_heads[i];
    __syncthreads();

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const float in_slope2 = p.in_slope;
    const long long n_tiles = (p.n_rows + 15) / 16;
    for (long long tile = (long long)blockIdx.x * (PT_THREADS / 32) + warp; tile < n_tiles; tile += (long long)gridDim.x * (PT_THREADS / 32)) {
        const long long r0 = tile * 16 + g, r1 = r0 + 8;
        // ---- first layer: A fragments straight from global memory, 16 bytes (8 inputs) per load.  Lane (g, t) holds inputs
        //      32 s2 + 8 t + 0..7 of rows g and g + 8: elements 0-3 feed k-step 2 s2 (a0/a2 resp. a1/a3), 4-7 feed k-step 2 s2 + 1;
        //      the B fragments use the same assignment, so the weights stay in their natural order. ----
        uint4 xa[KS2], xb[KS2];
#pragma unroll
        for (int s2 = 0; s2 < KS2; s2++) {
            xa[s2] = r0 < p.n_rows ? __ldg(reinterpret_cast<const uint4 *>(p.x + r0 * K0 + 32 * s2 + 8 * t)) : make_uint4(0, 0, 0, 0);
            xb[s2] = r1 < p.n_rows ? __ldg(reinterpret_cast<const uint4 *>(p.x + r1 * K0 + 32 * s2 + 8 * t)) : make_uint4(0, 0, 0, 0);
        }
        float acc[8][4];
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const float2 b = *reinterpret_cast<const float2 *>(b1 + 8 * j + 2 * t);
            acc[j][0] = b.x, acc[j][1] = b.y, acc[j][2] = b.x, acc[j][3] = b.y;
        }
#pragma unroll
        for (int s2 = 0; s2 < KS2; s2++) {
            unsigned a_lo[4], a_hi[4];
            a_lo[0] = lrelu_bf16x2(xa[s2].x, in_slope2), a_lo[1] = lrelu_bf16x2(xb[s2].x, in_slope2);
            a_lo[2] = lrelu_bf16x2(xa[s2].y, in_slope2), a_lo[3] = lrelu_bf16x2(xb[s2].y, in_slope2);
            a_hi[0] = lrelu_bf16x2(xa[s2].z, in_slope2), a_hi[1] = lrelu_bf16x2(xb[s2].z, in_slope2);
            a_hi[2] = lrelu_bf16x2(xa[s2].w, in_slope2), a_hi[3] = lrelu_bf16x2(xb[s2].w, in_slope2);
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const uint4 b = *reinterpret_cast<const uint4 *>(w1 + (8 * j + g) * FS + 32 * s2 + 8 * t);
                mma_bf16_16816(acc[j], a_lo, b.x, b.y);
                mma_bf16_16816(acc[j], a_hi, b.z, b.w);
            }
        }
        // ---- hidden layers and heads: fragments in, fragments out ----
        unsigned a[4][4];
        to_fragments(a, acc, p.slope);
        for (int l = 0; l < p.n_hidden; l++) {
            dense64<8>(acc, a, wh + l * PT_H * PT_HS, bh + l * PT_H, g, t);
            to_fragments(a, acc, p.slope);
        }
        float out[1][4];
        dense64<1>(out, a, wo, bo, g, t);  // lane (g, t): heads 2 t, 2 t + 1 of rows g (out[0][0..1]) and g + 8 (out[0][2..3])
        if (p.scores) {
            if (r0 < p.n_rows) *reinterpret_cast<float2 *>(p.scores + r0 * PT_NOUT + 2 * t) = make_float2(out[0][0], out[0][1]);
            if (r1 < p.n_rows) *reinterpret_cast<float2 *>(p.scores + r1 * PT_NOUT + 2 * t) = make_float2(out[0][2], out[0][3]);
        }
        // ---- the draw (ovc_sample_actions): heads 2 t, 2 t + 1 use words 2 t, 2 t + 1 of block t / 2 ----
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const long long row = h ? r1 : r0;
            const float s0 = out[0][2 * h], s1 = out[0][2 * h + 1];
            const Philox4 P = philox4x32_10(p.seed, (uint32_t)row, (uint32_t)((unsigned long long)row >> 32), (uint32_t)step,
                                            ((uint32_t)(step >> 32) << 1) | (uint32_t)(t >> 1));
            const uint32_t d0 = P.v[(2 * t) & 3], d1 = P.v[(2 * t + 1) & 3];
            const float u0 = ((float)(d0 >> 9) + 0.5f) * 1.1920928955078125e-7f, u1 = ((float)(d1 >> 9) + 0.5f) * 1.1920928955078125e-7f;
            float v0 = 2 * t < p.n_actions ? s0 - logf(-logf(u0)) : -INFINITY;
            const float v1 = 2 * t + 1 < p.n_actions ? s1 - logf(-logf(u1)) : -INFINITY;
            int best = 2 * t;
            if (v1 > v0) v0 = v1, best = 2 * t + 1;
#pragma unroll
            for (int d = 1; d <= 2; d <<= 1) {  // argmax over the four lanes of the row (lowest index wins ties, as a serial scan does)
                const float ov = __shfl_xor_sync(0xFFFFFFFFu, v0, d);
                const int ob = __shfl_xor_sync(0xFFFFFFFFu, best, d);
                if (ov > v0 || (ov == v0 && ob < best)) v0 = ov, best = ob;
            }
            if (row < p.n_rows) {
                if (t == 0) p.actions[row] = best;
                // the value head is head n_actions: lane n_actions / 2 holds it
                if (p.values && t == (p.n_actions >> 1)) p.values[row] = (p.n_actions & 1) ? s1 : s0;
            }
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned long long arrived = atomicAdd(p.counter + 1, 1ull);
        if (arrived == (unsigned long long)gridDim.x - 1) {
            p.counter[1] = 0;
            p.counter[0] = step + 1;
            __threadfence();
        }
    }
}

static int policy_tail_impl(const PolicyTailArgs &a, int k0, cudaStream_t st) {
    if (!a.x || !a.w_first || !a.b_first || !a.w_heads || !a.b_heads || !a.counter || !a.actions || (a.n_hidden > 0 && (!a.w_hidden || !a.b_hidden)))
        return fail(OVC_E_BADARG, "null pointer argument");
    if ((((uintptr_t)a.x | (uintptr_t)a.w_first) & 15) != 0) return fail(OVC_E_BADARG, "x and w_first must be 16-byte aligned");
    if (k0 < 32 || k0 > 256 || k0 % 32) return fail(OVC_E_BADARG, "k0 must be a multiple of 32 in 32..256", k0);
    if (a.n_hidden < 0 || a.n_hidden > 8) return fail(OVC_E_BADARG, "n_hidden must be 0..8", a.n_hidden);
    if (a.n_actions < 1 || a.n_actions > 7) return fail(OVC_E_BADARG, "n_actions must be 1..7 (head n_actions is the value)", a.n_actions);
    if (!(a.in_slope >= 0.f && a.in_slope <= 1.f && a.slope >= 0.f && a.slope <= 1.f)) return fail(OVC_E_BADARG, "slopes must lie in [0, 1]");
    if (a.n_rows < 0) return fail(OVC_E_BADARG, "negative row count");
    if (a.n_rows == 0) return OVC_OK;
    int dev = 0, n_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    const int fs = k0 % 64 == 32 ? k0 : k0 + 32;
    const size_t smem = (size_t)PT_H * fs * 2 + (size_t)(a.n_hidden * PT_H + PT_NOUT) * PT_HS * 2 + (size_t)(PT_H + a.n_hidden * PT_H + PT_NOUT) * 4 + 16;
    const long long n_tiles = (a.n_rows + 15) / 16, want = (n_tiles + PT_THREADS / 32 - 1) / (PT_THREADS / 32);
    const unsigned grid = (unsigned)(want < n_sm ? want : n_sm);
    cudaError_t e = cudaSuccess;
#define OVC_LAUNCH_PT(KS2)                                                                                              \
    case KS2:                                                                                                           \
        e = cudaFuncSetAttribute(policy_tail_kernel<KS2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);      \
        if (e == cudaSuccess) policy_tail_kernel<KS2><<<grid, PT_THREADS, smem, st>>>(a);                               \
        break;
    switch (k0 / 32) {
        OVC_LAUNCH_PT(1) OVC_LAUNCH_PT(2) OVC_LAUNCH_PT(3) OVC_LAUNCH_PT(4) OVC_LAUNCH_PT(5) OVC_LAUNCH_PT(6) OVC_LAUNCH_PT(7) OVC_LAUNCH_PT(8)
    }
#undef OVC_LAUNCH_PT
    if (e != cudaSuccess) return cuda_fail(e, "policy_tail kernel attribute");
    e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "policy_tail kernel launch");
    return OVC_OK;
}

}  // namespace ovc
