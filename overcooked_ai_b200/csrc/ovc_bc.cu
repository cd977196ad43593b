// ovc_bc.cu — behaviour-cloning training (include/ovc_bc.h): one CTA trains one model for one epoch, its parameters, the
// minibatch's rows, activations and deltas resident in shared memory, the Adam moments read and written in global memory.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>

#include "../../include/ovc_b200.h"
#include "../../include/ovc_bc.h"

namespace ovc {

static thread_local char g_bc_err[512] = "";

static int bc_fail(int code, const char *msg, long long value = 0) {
    snprintf(g_bc_err, sizeof g_bc_err, "%s (%lld)", msg, value);
    return code;
}

constexpr int BC_THREADS = 256;
constexpr int BC_TM = 8;         // rows of the output each thread accumulates per weight it loads
constexpr int BC_FEATURES = 96;
constexpr int BC_HIDDEN = 64;
constexpr int BC_MAX_LAYERS = 2;
constexpr int BC_MAX_ACTIONS = 7;
constexpr int BC_ZW = 8;         // row stride of the logits / their gradient

// C(m, n) = sum_k A[m a_m + k a_k] * B[n b_n + k b_k] for m < M, n < N, one FFMA chain per output in k order, then
// epi(m, n, C).  A warp takes a block of BC_TM rows and 32 consecutive n: every A load is a broadcast, and the B loads of
// the 32 lanes fall in 32 banks when b_n is 1 or odd (the weights are stored with odd row strides for this).
template <class Epi>
__device__ __forceinline__ void smem_gemm(int M, int N, int K, const float *A, int a_m, int a_k, const float *B, int b_n, int b_k,
                                          Epi epi) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nc = (N + 31) >> 5, mt = (M + BC_TM - 1) / BC_TM;
    for (int item = warp; item < nc * mt; item += BC_THREADS / 32) {
        const int n = (item % nc) * 32 + lane, m0 = (item / nc) * BC_TM;
        int ao[BC_TM];
#pragma unroll
        for (int r = 0; r < BC_TM; r++) ao[r] = min(m0 + r, M - 1) * a_m;
        const float *b = B + min(n, N - 1) * b_n;
        float acc[BC_TM];
#pragma unroll
        for (int r = 0; r < BC_TM; r++) acc[r] = 0.f;
#pragma unroll 4
        for (int k = 0; k < K; k++) {
            const float bk = b[k * b_k];
#pragma unroll
            for (int r = 0; r < BC_TM; r++) acc[r] = fmaf(A[ao[r] + k * a_k], bk, acc[r]);
        }
        if (n < N) {
#pragma unroll
            for (int r = 0; r < BC_TM; r++)
                if (m0 + r < M) epi(m0 + r, n, acc[r]);
        }
    }
}

struct BcShape {
    int L, A, B;
    // shared-memory float offsets: layer l's padded weights [out][in + 1] and bias; then the rows
    __host__ __device__ int in(int l) const { return l == 0 ? BC_FEATURES : BC_HIDDEN; }
    __host__ __device__ int out(int l) const { return l == L ? A : BC_HIDDEN; }  // l == L: the logits layer
    __host__ __device__ int s_w(int l) const {
        int o = 0;
        for (int i = 0; i < l; i++) o += out(i) * (in(i) + 1) + out(i);
        return o;
    }
    __host__ __device__ int s_b(int l) const { return s_w(l) + out(l) * (in(l) + 1); }
    __host__ __device__ int g_w(int l) const {  // the same in the flat global vector (unpadded)
        int o = 0;
        for (int i = 0; i < l; i++) o += out(i) * in(i) + out(i);
        return o;
    }
    __host__ __device__ int g_b(int l) const { return g_w(l) + out(l) * in(l); }
    __host__ __device__ int n_params() const { return g_w(L + 1); }
    __host__ __device__ int s_x() const { return (s_w(L + 1) + 3) & ~3; }                    // x [B][96], 16-byte aligned
    __host__ __device__ int s_act(int l) const { return s_x() + B * BC_FEATURES + (l - 1) * B * BC_HIDDEN; }  // l = 1..L
    __host__ __device__ int s_extra() const { return s_act(L + 1); }                          // [B][64]
    __host__ __device__ int s_z() const { return s_extra() + B * BC_HIDDEN; }                 // [B][8]
    __host__ __device__ int s_loss() const { return s_z() + B * BC_ZW; }                      // [B]
    __host__ __device__ int s_label() const { return s_loss() + B; }                          // int [B]
    __host__ __device__ int s_correct() const { return s_label() + B; }                       // int [B]
    __host__ __device__ int s_end() const { return s_correct() + B; }
};

struct AdamStep {
    float alpha;
    __device__ __forceinline__ float operator()(float g, float *m, float *v, float p) const {
        float mm = *m, vv = *v;
        mm = mm + (g - mm) * 0.1f;
        vv = vv + (g * g - vv) * 0.001f;
        *m = mm, *v = vv;
        return p - (alpha * mm) / (sqrtf(vv) + 1e-7f);
    }
};

// Loads the rows of one minibatch: their labels and features.
__device__ __forceinline__ void load_rows(const BcShape &s, float *sm, const float *__restrict__ features, const int32_t *__restrict__ labels,
                                          const int32_t *rows, int n) {
    int *lab = reinterpret_cast<int *>(sm + s.s_label());
    for (int b = threadIdx.x; b < n; b += BC_THREADS) lab[b] = __ldg(labels + __ldg(rows + b));
    float4 *x = reinterpret_cast<float4 *>(sm + s.s_x());
    for (int i = threadIdx.x; i < n * (BC_FEATURES / 4); i += BC_THREADS) {
        const int b = i / (BC_FEATURES / 4), c = i % (BC_FEATURES / 4);
        x[i] = __ldg(reinterpret_cast<const float4 *>(features + (long long)__ldg(rows + b) * BC_FEATURES) + c);
    }
}

// Forward pass of n loaded rows to the logits (at s_z), then per row its loss, its correctness and (with grad) dz.
__device__ __forceinline__ void forward_loss(const BcShape &s, float *sm, int n, bool grad) {
    for (int l = 0; l <= s.L; l++) {
        const float *a = sm + (l == 0 ? s.s_x() : s.s_act(l));
        const int in = s.in(l), out = s.out(l);
        const float *w = sm + s.s_w(l), *bias = sm + s.s_b(l);
        if (l < s.L) {
            float *y = sm + s.s_act(l + 1);
            smem_gemm(n, out, in, a, in, 1, w, in + 1, 1, [&](int m, int j, float acc) { y[m * BC_HIDDEN + j] = fmaxf(acc + bias[j], 0.f); });
        } else {
            float *z = sm + s.s_z();
            smem_gemm(n, out, in, a, in, 1, w, in + 1, 1, [&](int m, int j, float acc) { z[m * BC_ZW + j] = acc + bias[j]; });
        }
        __syncthreads();
    }
    float *z = sm + s.s_z(), *loss = sm + s.s_loss();
    const int *lab = reinterpret_cast<const int *>(sm + s.s_label());
    int *corr = reinterpret_cast<int *>(sm + s.s_correct());
    for (int b = threadIdx.x; b < n; b += BC_THREADS) {
        float zz[BC_MAX_ACTIONS];
        const int y = lab[b];
        float mx = z[b * BC_ZW], zy = 0.f;
        int arg = 0;
#pragma unroll
        for (int a = 0; a < BC_MAX_ACTIONS; a++)
            if (a < s.A) {
                zz[a] = z[b * BC_ZW + a];
                if (zz[a] > mx) mx = zz[a], arg = a;
                if (a == y) zy = zz[a];
            }
        float sum = 0.f;
#pragma unroll
        for (int a = 0; a < BC_MAX_ACTIONS; a++)
            if (a < s.A) sum += expf(zz[a] - mx);
        const float lse = mx + logf(sum);
        loss[b] = lse - zy;
        corr[b] = arg == y;
        if (grad) {
#pragma unroll
            for (int a = 0; a < BC_MAX_ACTIONS; a++)
                if (a < s.A) z[b * BC_ZW + a] = (expf(zz[a] - lse) - (a == y ? 1.f : 0.f)) / (float)n;
        }
    }
    __syncthreads();
}

// Warp 0 adds the n row losses (float64, a fixed order) and correct flags to *loss_sum / *correct (lane 0's copies).
__device__ __forceinline__ void reduce_rows(const BcShape &s, const float *sm, int n, double *loss_sum, double *correct) {
    if (threadIdx.x >= 32) return;
    const float *loss = sm + s.s_loss();
    const int *corr = reinterpret_cast<const int *>(sm + s.s_correct());
    double l = 0.0, c = 0.0;
    for (int b = threadIdx.x; b < n; b += 32) l += (double)loss[b], c += corr[b];
#pragma unroll
    for (int d = 16; d; d >>= 1) l += __shfl_xor_sync(0xFFFFFFFFu, l, d), c += __shfl_xor_sync(0xFFFFFFFFu, c, d);
    *loss_sum += l, *correct += c;
}

// Gradient and Adam update of layer l's weights and biases from its input activations a (row stride in) and the delta of
// its outputs d (row stride dstride), over n rows.
__device__ __forceinline__ void update_layer(const BcShape &s, float *sm, int l, const float *a, const float *d, int dstride, int n,
                                             float *__restrict__ gm, float *__restrict__ gv, const AdamStep &adam) {
    const int in = s.in(l), out = s.out(l);
    float *w = sm + s.s_w(l), *bias = sm + s.s_b(l);
    float *mw = gm + s.g_w(l), *vw = gv + s.g_w(l);
    smem_gemm(out, in, n, d, 1, dstride, a, 1, in, [&](int j, int i, float g) {
        const int p = j * in + i;
        w[j * (in + 1) + i] = adam(g, mw + p, vw + p, w[j * (in + 1) + i]);
    });
    float *mb = gm + s.g_b(l), *vb = gv + s.g_b(l);
    for (int j = threadIdx.x; j < out; j += BC_THREADS) {
        float g = 0.f;
        for (int b = 0; b < n; b++) g += d[b * dstride + j];
        bias[j] = adam(g, mb + j, vb + j, bias[j]);
    }
}

__global__ void __launch_bounds__(BC_THREADS) bc_train_kernel(BcShape s, const float *__restrict__ features, const int32_t *__restrict__ labels,
                                                              const int32_t *__restrict__ train_rows, const int32_t *__restrict__ n_train,
                                                              const int32_t *__restrict__ val_rows, const int32_t *__restrict__ n_val,
                                                              long long row_stride, float *__restrict__ params, float *__restrict__ adam_m,
                                                              float *__restrict__ adam_v, int32_t *__restrict__ step,
                                                              const float *__restrict__ lr, const uint8_t *__restrict__ active,
                                                              double *__restrict__ stats) {
    extern __shared__ __align__(16) float sm[];
    const int k = blockIdx.x;
    if (!active[k]) return;
    const int P = s.n_params();
    float *gp = params + (long long)k * P, *gm = adam_m + (long long)k * P, *gv = adam_v + (long long)k * P;
    const int32_t *tr = train_rows + k * row_stride, *vr = val_rows + k * row_stride;
    const int nt = (int)min((long long)max(n_train[k], 0), row_stride), nv = (int)min((long long)max(n_val[k], 0), row_stride);
    for (int l = 0; l <= s.L; l++) {  // the flat parameters into the padded layout
        const int in = s.in(l), out = s.out(l);
        for (int i = threadIdx.x; i < out * in; i += BC_THREADS) sm[s.s_w(l) + (i / in) * (in + 1) + i % in] = gp[s.g_w(l) + i];
        for (int j = threadIdx.x; j < out; j += BC_THREADS) sm[s.s_b(l) + j] = gp[s.g_b(l) + j];
    }
    int t = step[k];
    const double lr_k = lr[k];
    double tr_loss = 0.0, tr_corr = 0.0, va_loss = 0.0, va_corr = 0.0;
    __syncthreads();
    for (int r0 = 0; r0 < nt; r0 += s.B) {
        const int n = min(s.B, nt - r0);
        load_rows(s, sm, features, labels, tr + r0, n);
        __syncthreads();
        forward_loss(s, sm, n, true);
        reduce_rows(s, sm, n, &tr_loss, &tr_corr);
        t += 1;
        const AdamStep adam{(float)(lr_k * sqrt(1.0 - pow(0.999, (double)t)) / (1.0 - pow(0.9, (double)t)))};
        // backward, top down: each layer's input delta is taken before the layer is updated; the delta of hidden layer l
        // goes to the extra buffer (l = L) or over a_{l+1}, which the update of layer l + 1 was the last to read
        const float *dz = sm + s.s_z();
        float *d = sm + s.s_extra();
        {
            const float *a = sm + s.s_act(s.L);
            const float *w = sm + s.s_w(s.L);
            smem_gemm(n, BC_HIDDEN, s.A, dz, BC_ZW, 1, w, 1, BC_HIDDEN + 1,
                      [&](int m, int i, float acc) { d[m * BC_HIDDEN + i] = a[m * BC_HIDDEN + i] > 0.f ? acc : 0.f; });
            __syncthreads();
            update_layer(s, sm, s.L, a, dz, BC_ZW, n, gm, gv, adam);
        }
        for (int l = s.L - 1; l >= 1; l--) {
            __syncthreads();
            const float *a = sm + s.s_act(l);
            const float *w = sm + s.s_w(l);
            float *dn = sm + s.s_act(l + 1);
            smem_gemm(n, BC_HIDDEN, BC_HIDDEN, d, BC_HIDDEN, 1, w, 1, BC_HIDDEN + 1,
                      [&](int m, int i, float acc) { dn[m * BC_HIDDEN + i] = a[m * BC_HIDDEN + i] > 0.f ? acc : 0.f; });
            __syncthreads();
            update_layer(s, sm, l, a, d, BC_HIDDEN, n, gm, gv, adam);
            d = dn;
        }
        update_layer(s, sm, 0, sm + s.s_x(), d, BC_HIDDEN, n, gm, gv, adam);
        __syncthreads();
    }
    for (int r0 = 0; r0 < nv; r0 += s.B) {
        const int n = min(s.B, nv - r0);
        load_rows(s, sm, features, labels, vr + r0, n);
        __syncthreads();
        forward_loss(s, sm, n, false);
        reduce_rows(s, sm, n, &va_loss, &va_corr);
        __syncthreads();
    }
    for (int l = 0; l <= s.L; l++) {
        const int in = s.in(l), out = s.out(l);
        for (int i = threadIdx.x; i < out * in; i += BC_THREADS) gp[s.g_w(l) + i] = sm[s.s_w(l) + (i / in) * (in + 1) + i % in];
        for (int j = threadIdx.x; j < out; j += BC_THREADS) gp[s.g_b(l) + j] = sm[s.s_b(l) + j];
    }
    if (threadIdx.x == 0) {
        step[k] = t;
        double *o = stats + 4ll * k;
        o[0] = tr_loss, o[1] = tr_corr, o[2] = va_loss, o[3] = va_corr;
    }
}

}  // namespace ovc

extern "C" {

int ovc_bc_abi_version(void) { return OVC_BC_ABI_VERSION; }

const char *ovc_bc_last_error(void) { return ovc::g_bc_err; }

int ovc_bc_train_epoch(const float *features, const int32_t *labels, int64_t n_rows, const int32_t *train_rows,
                       const int32_t *n_train, const int32_t *val_rows, const int32_t *n_val, int64_t row_stride, float *params,
                       float *adam_m, float *adam_v, int32_t *step, const float *lr, const uint8_t *active, double *stats,
                       int n_models, int n_features, int hidden, int num_hidden_layers, int num_actions, int batch, void *stream) {
    using ovc::bc_fail;
    if (!features || !labels || !train_rows || !n_train || !val_rows || !n_val || !params || !adam_m || !adam_v || !step || !lr ||
        !active || !stats)
        return bc_fail(OVC_E_BADARG, "null pointer argument");
    if (n_features != ovc::BC_FEATURES) return bc_fail(OVC_E_UNSUPPORTED, "n_features must be 96 (featurize_state at num_pots = 2)", n_features);
    if (hidden != ovc::BC_HIDDEN) return bc_fail(OVC_E_UNSUPPORTED, "hidden must be 64", hidden);
    if (num_hidden_layers < 1 || num_hidden_layers > ovc::BC_MAX_LAYERS)
        return bc_fail(OVC_E_UNSUPPORTED, "num_hidden_layers must be 1 or 2", num_hidden_layers);
    if (num_actions < 2 || num_actions > ovc::BC_MAX_ACTIONS) return bc_fail(OVC_E_UNSUPPORTED, "num_actions must be in [2, 7]", num_actions);
    if (batch < 1 || batch > OVC_BC_MAX_BATCH) return bc_fail(OVC_E_UNSUPPORTED, "batch must be in [1, 128]", batch);
    if (n_models < 0) return bc_fail(OVC_E_BADARG, "negative n_models", n_models);
    if (n_rows < 0 || n_rows >= (1ll << 31)) return bc_fail(OVC_E_BADARG, "n_rows must be in [0, 2^31)", (long long)n_rows);
    if (row_stride < 0 || row_stride >= (1ll << 31)) return bc_fail(OVC_E_BADARG, "row_stride must be in [0, 2^31)", (long long)row_stride);
    if ((uintptr_t)features & 15) return bc_fail(OVC_E_BADARG, "features must be 16-byte aligned");
    if ((uintptr_t)stats & 7) return bc_fail(OVC_E_BADARG, "stats must be 8-byte aligned");
    if (((uintptr_t)labels | (uintptr_t)train_rows | (uintptr_t)n_train | (uintptr_t)val_rows | (uintptr_t)n_val | (uintptr_t)params |
         (uintptr_t)adam_m | (uintptr_t)adam_v | (uintptr_t)step | (uintptr_t)lr) & 3)
        return bc_fail(OVC_E_BADARG, "the int32 and float32 buffers must be 4-byte aligned");
    if (n_models == 0) return OVC_OK;
    const ovc::BcShape s{num_hidden_layers, num_actions, batch};
    const size_t smem = sizeof(float) * (size_t)s.s_end();
    cudaError_t e = cudaFuncSetAttribute(ovc::bc_train_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) {
        ovc::bc_train_kernel<<<n_models, ovc::BC_THREADS, smem, (cudaStream_t)stream>>>(s, features, labels, train_rows, n_train, val_rows,
                                                                                       n_val, row_stride, params, adam_m, adam_v, step, lr,
                                                                                       active, stats);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) return bc_fail(OVC_E_CUDA, cudaGetErrorString(e));
    return OVC_OK;
}

}  // extern "C"
