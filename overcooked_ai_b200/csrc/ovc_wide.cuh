// ovc_wide.cuh — K9 wide_layers_kernel (included by ovc_b200.cu after ovc_tail.cuh): the two wide layers of the rollout
// policy between K7 and K8 (reference model: human_aware_rl/ppo/ppo_rllib.py:54-62, the two 3x3 convolutions, each folded
// into one matrix by the host) as ONE Hopper wgmma kernel:
//
//     a1 = leaky_relu(a0 . W1^T + b1)        a0 [M][512] bf16 (K7's output), W1 [512][512] bf16
//     z2 = a1 . W2^T + b2                    W2 [160][512] bf16, z2 [M][160] bf16 (K8's input: its leaky ReLU is applied there)
//
// The 128 x 512 activation tile a1 never reaches HBM or even shared memory.  Layer 1 is computed 128 columns at a time
// (a 64 x 128 fp32 accumulator per warpgroup, in registers); the epilogue adds the bias, applies the leaky ReLU and rounds
// to bf16 straight into the register fragment layout wgmma takes for its A operand, and layer 2 then accumulates those
// 128 columns' contribution into its own 64 x 160 register accumulator (A from registers, W2 from shared memory).  As
// library calls the same work is two GEMMs and an activation pass with a1 written once and read twice (3 x 67 MB per
// 65 536 rows).
//
// Persistent: one CTA per SM walks 128-row tiles; three warpgroups: warps 0-7 = two consumer warpgroups (rows 0-63 and
// 64-127 of the tile), warpgroup 2 = TMA producer (one lane).  setmaxnreg moves registers from the producer (40 per thread)
// to the consumers (232): each SM sub-partition then holds one producer and two consumer warps within its 16 K registers.
// Operand tiles arrive by TMA (cp.async.bulk.tensor.2d, 128-byte swizzle) through two mbarrier rings: {a0 128 x 64, W1 128 x 64} = 32 KB per stage, four stages, for layer 1, and W2's 160 x 128
// columns of one chunk = 40 KB per stage, two stages, for layer 2 (208 KB of shared memory in all).  Every mbarrier wait
// is bounded (~10 s; a protocol error traps instead of hanging the GPU).
#pragma once
#include <cuda_bf16.h>

namespace ovc {

constexpr int WL_BM = 128, WL_BK = 64, WL_K0 = 512, WL_N1 = 512, WL_N2 = 160;
constexpr int WL_NC = 128;                  // layer-1 columns per chunk (one wgmma N)
constexpr int WL_KC = WL_K0 / WL_BK;        // k-chunks of layer 1 per column chunk
constexpr int WL_CHUNKS = WL_N1 / WL_NC;    // column chunks of layer 1 = k-chunks of layer 2
constexpr int WL_THREADS = 384;             // 2 consumer warpgroups + the producer warpgroup
constexpr int WL_STAGES = 4;
constexpr uint32_t WL_A_BYTES = WL_BM * WL_BK * 2;            // 16 KB
constexpr uint32_t WL_B1_BYTES = WL_NC * WL_BK * 2;           // 16 KB
constexpr uint32_t WL_STAGE = WL_A_BYTES + WL_B1_BYTES;       // 32 KB
constexpr uint32_t WL_B2_BOX = WL_N2 * WL_BK * 2;             // 20 KB: 64 columns of W2
constexpr uint32_t WL_B2_STAGE = (WL_NC / WL_BK) * WL_B2_BOX; // 40 KB: W2's columns of one chunk
constexpr uint32_t WL_TILE_BYTES = WL_STAGES * WL_STAGE + 2 * WL_B2_STAGE;  // 208 KB
constexpr uint32_t WL_SMEM = 1024 + WL_TILE_BYTES + (WL_N1 + WL_N2) * 4 + 128;  // tiles + biases + 12 mbarriers
static_assert(WL_SMEM <= 227 * 1024, "one CTA per SM within the opt-in shared memory of sm_90");

struct WideArgs {
    const float *b1, *b2;
    __nv_bfloat16 *z2;
    long long m;
    float slope;
    int n_tiles;
};

__device__ __forceinline__ void mbar_wait_bounded(uint64_t *bar, uint32_t parity) {
    const long long t0 = clock64();
    uint32_t ok;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
        if (!ok && clock64() - t0 > 20000000000ll) __trap();  // ~10 s: a protocol error must not hang the device
    } while (!ok);
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void regs_dealloc() {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void regs_alloc() {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}

// wgmma shared-memory descriptor of a K-major bf16 tile stored as rows of 128 bytes (64 elements) with the 128-byte swizzle
// (what TMA's CU_TENSOR_MAP_SWIZZLE_128B writes): start address >> 4, leading byte offset (unused for swizzled K-major) 1,
// stride byte offset 1024 (8 rows), layout type 1 = SWIZZLE_128B at bit 62.  Tile bases are 1024-byte aligned (base
// offset 0); a k-step of 16 elements advances the start address by 32 bytes inside the swizzle atom.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}

// d[64] (+)= A[smem desc] . B[smem desc]^T: m64n128k16, bf16 x bf16 -> fp32, both operands K-major
__device__ __forceinline__ void wgmma_m64n128_ss(float d[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}
// d[80] (+)= A[registers] . B[smem desc]^T: m64n160k16, A in the register fragment layout of m64nNk16 (that of mma.sync
// m16n8k16 per warp, warp w of the warpgroup holding rows 16w..16w+15), B K-major
__device__ __forceinline__ void wgmma_m64n160_rs(float d[80], const uint32_t a[4], uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %85, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n160k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79}, "
        "{%80, %81, %82, %83}, %84, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate)
        : "memory");
}

__device__ __forceinline__ uint32_t leaky_bf16x2(float x0, float x1, float slope) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(fmaxf(x0, x0 * slope), fmaxf(x1, x1 * slope));
    return *reinterpret_cast<const uint32_t *>(&h);
}

__global__ void __launch_bounds__(WL_THREADS, 1)
wide_layers_kernel(const __grid_constant__ CUtensorMap map_a0, const __grid_constant__ CUtensorMap map_w1,
                   const __grid_constant__ CUtensorMap map_w2, const WideArgs p) {
    extern __shared__ char wl_raw[];
    char *tile = reinterpret_cast<char *>((reinterpret_cast<uintptr_t>(wl_raw) + 1023) & ~(uintptr_t)1023);
    char *w2_tile = tile + WL_STAGES * WL_STAGE;
    float *bias1 = reinterpret_cast<float *>(tile + WL_TILE_BYTES);
    float *bias2 = bias1 + WL_N1;
    uint64_t *bars = reinterpret_cast<uint64_t *>(bias2 + WL_N2);
    uint64_t *full = bars, *empty = bars + WL_STAGES, *w2_full = bars + 2 * WL_STAGES, *w2_empty = w2_full + 2;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        // a stage is free again when all 8 consumer warps have seen their wgmma reading it complete
        for (int i = 0; i < WL_STAGES; i++) mbar_init(full + i, 1), mbar_init(empty + i, 8);
        for (int i = 0; i < 2; i++) mbar_init(w2_full + i, 1), mbar_init(w2_empty + i, 8);
        prefetch_tmap(&map_a0), prefetch_tmap(&map_w1), prefetch_tmap(&map_w2);
    }
    for (int i = threadIdx.x; i < WL_N1; i += WL_THREADS) bias1[i] = p.b1[i];
    for (int i = threadIdx.x; i < WL_N2; i += WL_THREADS) bias2[i] = p.b2[i];
    __syncthreads();

    if (warp >= 8) {
        regs_dealloc<40>();
        if (warp == 8 && lane == 0) {
            // ---- TMA producer: tiles blockIdx.x, + gridDim.x, ...; the rings' use counters run on across tiles ----
            int it1 = 0, it2 = 0;
            for (int tile_i = blockIdx.x; tile_i < p.n_tiles; tile_i += gridDim.x) {
                const int m0 = tile_i * WL_BM;
                for (int n = 0; n < WL_CHUNKS; n++) {
                    for (int c = 0; c < WL_KC; c++, it1++) {
                        const int s = it1 % WL_STAGES, u = it1 / WL_STAGES;
                        mbar_wait_bounded(empty + s, (u & 1) ^ 1);
                        char *st = tile + s * WL_STAGE;
                        mbar_expect_tx(full + s, WL_STAGE);
                        tma_load_2d(st, &map_a0, c * WL_BK, m0, full + s);  // rows past M: zero fill, still counted
                        tma_load_2d(st + WL_A_BYTES, &map_w1, c * WL_BK, n * WL_NC, full + s);
                    }
                    const int s = it2 & 1, u = it2 >> 1;
                    it2++;
                    mbar_wait_bounded(w2_empty + s, (u & 1) ^ 1);
                    mbar_expect_tx(w2_full + s, WL_B2_STAGE);
                    for (int h = 0; h < WL_NC / WL_BK; h++)
                        tma_load_2d(w2_tile + s * WL_B2_STAGE + h * WL_B2_BOX, &map_w2, n * WL_NC + h * WL_BK, 0, w2_full + s);
                }
            }
        }
        return;
    }

    // ---- consumer warpgroup g: rows 64 g .. 64 g + 63 of the tile; warp w of the group owns 16 of them ----
    regs_alloc<232>();
    const int g = warp >> 2, w = warp & 3;
    float acc1[64], acc2[80];
    uint32_t a1[WL_NC / 16][4];  // the activation chunk as layer 2's A fragments, one [4] per k-step of 16
#pragma unroll
    for (int i = 0; i < 80; i++) acc2[i] = 0.f;
    int it1 = 0, it2 = 0;
    for (int tile_i = blockIdx.x; tile_i < p.n_tiles; tile_i += gridDim.x) {
        for (int n = 0; n < WL_CHUNKS; n++) {
            // layer 1, columns n*128 .. n*128+127: 8 k-chunks, one stage each; a stage is released once the wgmma
            // group after it has been issued and it has itself completed (wait_group 1)
#pragma unroll
            for (int i = 0; i < 64; i++) acc1[i] = 0.f;
            int prev = 0;
            for (int c = 0; c < WL_KC; c++, it1++) {
                const int s = it1 % WL_STAGES, u = it1 / WL_STAGES;
                mbar_wait_bounded(full + s, u & 1);
                const uint32_t a_addr = smem_u32(tile + s * WL_STAGE) + g * (WL_A_BYTES / 2);
                const uint64_t da = wgmma_desc_sw128(a_addr), db = wgmma_desc_sw128(smem_u32(tile + s * WL_STAGE + WL_A_BYTES));
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < WL_BK / 16; k++) wgmma_m64n128_ss(acc1, da + 2 * k, db + 2 * k, (c | k) != 0);
                wgmma_commit();
                wgmma_wait<1>();
                if (c && lane == 0) mbar_arrive(empty + prev);
                prev = s;
            }
            wgmma_wait<0>();
            if (lane == 0) mbar_arrive(empty + prev);
            // epilogue 1: bias, leaky ReLU, bf16.  Accumulator n8-group j holds (row l/4, columns 8j + 2(l%4) + {0,1}) in
            // [4j], [4j+1] and row l/4 + 8 in [4j+2], [4j+3]; k-step q's A fragment is groups 2q (registers 0, 1) and 2q+1 (2, 3).
            const float *bn = bias1 + n * WL_NC + 2 * (lane & 3);
#pragma unroll
            for (int j = 0; j < WL_NC / 8; j++) {
                const float b0 = bn[8 * j], b1 = bn[8 * j + 1];
                a1[j >> 1][(j & 1) * 2] = leaky_bf16x2(acc1[4 * j] + b0, acc1[4 * j + 1] + b1, p.slope);
                a1[j >> 1][(j & 1) * 2 + 1] = leaky_bf16x2(acc1[4 * j + 2] + b0, acc1[4 * j + 3] + b1, p.slope);
            }
            // layer 2: z2 += a1[:, n*128 .. n*128+127] . W2[:, n*128 .. n*128+127]^T
            const int s = it2 & 1, u = it2 >> 1;
            it2++;
            mbar_wait_bounded(w2_full + s, u & 1);
            const uint32_t b_addr = smem_u32(w2_tile + s * WL_B2_STAGE);
            wgmma_fence();
#pragma unroll
            for (int q = 0; q < WL_NC / 16; q++)
                wgmma_m64n160_rs(acc2, a1[q], wgmma_desc_sw128(b_addr + (q >> 2) * WL_B2_BOX) + 2 * (q & 3), (n | q) != 0);
            wgmma_commit();
            wgmma_wait<0>();
            if (lane == 0) mbar_arrive(w2_empty + s);
        }
        // epilogue 2: bias, bf16, two rows of 160 columns per quad of lanes
        const long long row = (long long)tile_i * WL_BM + g * 64 + w * 16 + (lane >> 2);
#pragma unroll
        for (int j = 0; j < WL_N2 / 8; j++) {
            const int col = 8 * j + 2 * (lane & 3);
            const float b0 = bias2[col], b1 = bias2[col + 1];
            if (row < p.m)
                *reinterpret_cast<__nv_bfloat162 *>(p.z2 + row * WL_N2 + col) = __floats2bfloat162_rn(acc2[4 * j] + b0, acc2[4 * j + 1] + b1);
            if (row + 8 < p.m)
                *reinterpret_cast<__nv_bfloat162 *>(p.z2 + (row + 8) * WL_N2 + col) = __floats2bfloat162_rn(acc2[4 * j + 2] + b0, acc2[4 * j + 3] + b1);
        }
    }
}

static int make_tmap_bf16(CUtensorMap *m, const void *base, long long rows, int cols, int box_rows) {
    encode_tiled_fn enc = get_encode_fn();
    if (!enc) return fail(OVC_E_CUDA, "cuTensorMapEncodeTiled entry point not available");
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)cols * 2};
    cuuint32_t box[2] = {(cuuint32_t)WL_BK, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(OVC_E_CUDA, "cuTensorMapEncodeTiled failed", (long long)r);
    return OVC_OK;
}

static int wide_layers_impl(const void *a0, long long m, int k0, const void *w1, const float *b1, int n1, const void *w2, const float *b2,
                            int n2, float slope, void *z2, cudaStream_t st) {
    if (!a0 || !w1 || !b1 || !w2 || !b2 || !z2) return fail(OVC_E_BADARG, "null pointer argument");
    if (k0 != WL_K0 || n1 != WL_N1 || n2 != WL_N2) return fail(OVC_E_UNSUPPORTED, "wide_layers: built for 512 -> 512 -> 160", k0 * 1000000ll + n1 * 1000 + n2);
    if ((((uintptr_t)a0 | (uintptr_t)w1 | (uintptr_t)w2 | (uintptr_t)z2) & 15) != 0) return fail(OVC_E_BADARG, "operands must be 16-byte aligned");
    if (!(slope >= 0.f && slope <= 1.f)) return fail(OVC_E_BADARG, "negative slope must lie in [0, 1]");
    if (m < 0) return fail(OVC_E_BADARG, "negative row count");
    if (m == 0) return OVC_OK;
    CUtensorMap ma, mw1, mw2;
    int rc = make_tmap_bf16(&ma, a0, m, WL_K0, WL_BM);
    if (!rc) rc = make_tmap_bf16(&mw1, w1, WL_N1, WL_K0, WL_NC);  // one column chunk of a k-chunk per box
    if (!rc) rc = make_tmap_bf16(&mw2, w2, WL_N2, WL_N1, WL_N2);
    if (rc) return rc;
    cudaError_t e = cudaFuncSetAttribute(wide_layers_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WL_SMEM);
    if (e != cudaSuccess) return cuda_fail(e, "wide_layers kernel attribute");
    WideArgs p;
    int dev = 0, n_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    p.b1 = b1, p.b2 = b2, p.z2 = (__nv_bfloat16 *)z2, p.m = m, p.slope = slope;
    p.n_tiles = (int)((m + WL_BM - 1) / WL_BM);
    // persistent: one CTA per SM walks tiles blockIdx.x, + gridDim.x, ... (barriers and biases are set up once)
    wide_layers_kernel<<<(unsigned)(p.n_tiles < n_sm ? p.n_tiles : n_sm), WL_THREADS, WL_SMEM, st>>>(ma, mw1, mw2, p);
    e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "wide_layers kernel launch");
    return OVC_OK;
}

}  // namespace ovc
