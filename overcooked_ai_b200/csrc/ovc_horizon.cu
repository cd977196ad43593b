// ovc_horizon.cu — the horizon bootstrap's kernels (include/ovc_horizon.h): the compaction of the ended environments'
// learner rows, and GAE that bootstraps at the horizon cut from the learner's value of the terminal state.
#include <cuda_runtime.h>
#include <stdio.h>

#include "../../include/ovc_b200.h"
#include "../../include/ovc_horizon.h"

namespace ovc {

static thread_local char g_horizon_err[512] = "";

static int horizon_fail(int code, const char *msg, long long value = 0) {
    snprintf(g_horizon_err, sizeof g_horizon_err, "%s (%lld)", msg, value);
    return code;
}

constexpr int HORIZON_ROWS_THREADS = 256;

// One thread per environment.  Episodes usually end together, once per horizon, so most launches find no environment done:
// a warp with nothing to claim leaves after zeroing its value rows.  A warp that has rows claims them with one atomic.
__global__ void __launch_bounds__(HORIZON_ROWS_THREADS) horizon_rows_kernel(const int32_t *__restrict__ state, int S,
                                                                            const int32_t *__restrict__ done,
                                                                            const int32_t *__restrict__ partner_seat, int one_view,
                                                                            long long n_envs, int32_t *__restrict__ records,
                                                                            int32_t *__restrict__ view, int32_t *__restrict__ jrow,
                                                                            int32_t *__restrict__ range, float *__restrict__ values) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool in = e < n_envs;
    const int lane = threadIdx.x & 31;
    int n = 0, v0 = 0;  // the learner views of e: n of them, from v0
    if (in) {
        if (values) {
            if (one_view) values[e] = 0.f;
            else values[2 * e] = 0.f, values[2 * e + 1] = 0.f;
        }
        if (done[e]) {
            const int ps = partner_seat ? partner_seat[e] : -1;
            if (one_view || ps >= 0) n = 1, v0 = 1 - ps;
            else n = 2, v0 = 0;
        }
    }
    const unsigned any = __ballot_sync(0xFFFFFFFFu, n != 0);
    if (!any) return;
    int incl = n;  // inclusive prefix sum of n over the warp
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int y = __shfl_up_sync(0xFFFFFFFFu, incl, d);
        if (lane >= d) incl += y;
    }
    int base = 0;
    if (lane == 31) base = atomicAdd(range + 1, incl);
    base = __shfl_sync(0xFFFFFFFFu, base, 31);
    const int4 *src = reinterpret_cast<const int4 *>(state + e * S);
    for (int k = 0; k < n; k++) {
        const long long r = base + incl - n + k;
        const int v = v0 + k;
        view[r] = v;
        jrow[r] = (int32_t)(one_view ? e : 2 * e + v);
        int4 *dst = reinterpret_cast<int4 *>(records + r * S);
        for (int c = 0; c < S / 4; c++) dst[c] = __ldg(src + c);
    }
}

// Generalized advantage estimation with the horizon bootstrap: ovc_encfc.cuh's gae_kernel (one thread per environment
// holding its rows, GAE_UNROLL timesteps of loads issued before they are consumed) with the next value of an ended episode
// taken from terminal_values.  Every operation is rounded on its own, in the order include/ovc_horizon.h documents.  The
// terminal values are a third stream of loads: at gae_kernel's minimum of 5 CTAs per SM the two-row form spills 56 bytes;
// at 4 it takes 116 registers and the one-row form 68, no spills.
constexpr int GAE_THREADS = 128;
constexpr int GAE_UNROLL = 16;

__device__ __forceinline__ float gae_step(float a, float r, float v, float nv, float tv, bool d, float gamma, float gl) {
    const float next_v = d ? tv : nv;
    const float delta = __fsub_rn(__fadd_rn(r, __fmul_rn(gamma, next_v)), v);
    return __fadd_rn(delta, __fmul_rn(__fmul_rn(gl, d ? 0.f : 1.f), a));
}
__device__ __forceinline__ float2 gae_step(float2 a, float2 r, float2 v, float2 nv, float2 tv, bool d, float gamma, float gl) {
    return make_float2(gae_step(a.x, r.x, v.x, nv.x, tv.x, d, gamma, gl), gae_step(a.y, r.y, v.y, nv.y, tv.y, d, gamma, gl));
}
__device__ __forceinline__ float gae_target(float a, float v) { return __fadd_rn(a, v); }
__device__ __forceinline__ float2 gae_target(float2 a, float2 v) { return make_float2(__fadd_rn(a.x, v.x), __fadd_rn(a.y, v.y)); }

template <class V>
__global__ void __launch_bounds__(GAE_THREADS, 4)
    gae_horizon_kernel(const V *__restrict__ rewards, const V *__restrict__ values, const uint8_t *__restrict__ dones,
                       const V *__restrict__ terminal_values, const V *__restrict__ last_values, long long T, long long n_envs, float gamma,
                       float lambda, V *__restrict__ adv, V *__restrict__ targets) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_envs) return;
    const float gl = __fmul_rn(gamma, lambda);
    V a = {}, nv = last_values[e];
    for (long long t0 = T - 1; t0 >= 0; t0 -= GAE_UNROLL) {
        V r[GAE_UNROLL], v[GAE_UNROLL], tv[GAE_UNROLL];
        bool d[GAE_UNROLL];
#pragma unroll
        for (int k = 0; k < GAE_UNROLL; k++)
            if (t0 - k >= 0) {
                const long long i = (t0 - k) * n_envs + e;
                r[k] = __ldcs(rewards + i), v[k] = __ldcs(values + i), d[k] = dones[i] != 0;
                tv[k] = d[k] ? __ldcs(terminal_values + i) : V{};
            }
#pragma unroll
        for (int k = 0; k < GAE_UNROLL; k++)
            if (t0 - k >= 0) {
                const long long i = (t0 - k) * n_envs + e;
                a = gae_step(a, r[k], v[k], nv, tv[k], d[k], gamma, gl);
                __stcs(adv + i, a);
                __stcs(targets + i, gae_target(a, v[k]));
                nv = v[k];
            }
    }
}

static int gae_horizon_impl(const float *rewards, const float *values, const uint8_t *dones, const float *terminal_values,
                            const float *last_values, long long T, long long n, float gamma, float lambda, float *adv, float *targets,
                            cudaStream_t st, bool one_row) {
    if (!rewards || !values || !dones || !terminal_values || !last_values || !adv || !targets)
        return horizon_fail(OVC_E_BADARG, "null pointer argument");
    if (T < 0) return horizon_fail(OVC_E_BADARG, "negative n_steps", T);
    if (n < 0 || (!one_row && n % 2)) return horizon_fail(OVC_E_BADARG, one_row ? "negative n_envs" : "n_rows must be even and >= 0", n);
    if (((uintptr_t)rewards | (uintptr_t)values | (uintptr_t)terminal_values | (uintptr_t)last_values | (uintptr_t)adv |
         (uintptr_t)targets) & (one_row ? 3 : 7))
        return horizon_fail(OVC_E_BADARG, one_row ? "float buffers must be 4-byte aligned" : "float buffers must be 8-byte aligned");
    const long long n_envs = one_row ? n : n / 2;
    if (T == 0 || n_envs == 0) return OVC_OK;
    const unsigned grid = (unsigned)((n_envs + GAE_THREADS - 1) / GAE_THREADS);
    if (one_row)
        gae_horizon_kernel<float><<<grid, GAE_THREADS, 0, st>>>(rewards, values, dones, terminal_values, last_values, T, n_envs, gamma,
                                                                lambda, adv, targets);
    else
        gae_horizon_kernel<float2><<<grid, GAE_THREADS, 0, st>>>((const float2 *)rewards, (const float2 *)values, dones,
                                                                 (const float2 *)terminal_values, (const float2 *)last_values, T,
                                                                 n_envs, gamma, lambda, (float2 *)adv, (float2 *)targets);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return horizon_fail(OVC_E_CUDA, cudaGetErrorString(e));
    return OVC_OK;
}

}  // namespace ovc

extern "C" {

int ovc_horizon_abi_version(void) { return OVC_HORIZON_ABI_VERSION; }

const char *ovc_horizon_last_error(void) { return ovc::g_horizon_err; }

int ovc_horizon_rows(const int32_t *state, int state_words, const int32_t *done, const int32_t *partner_seat, int one_view,
                     int64_t n_envs, int32_t *records, int32_t *view, int32_t *jrow, int32_t *range, float *values, void *stream) {
    using ovc::horizon_fail;
    if (!state || !done || !records || !view || !jrow || !range) return horizon_fail(OVC_E_BADARG, "null pointer argument");
    if (one_view && !partner_seat) return horizon_fail(OVC_E_BADARG, "one_view needs partner_seat (agent 1's player)");
    if (n_envs < 0 || n_envs >= (1ll << 30)) return horizon_fail(OVC_E_BADARG, "n_envs must be in [0, 2^30)", (long long)n_envs);
    if (state_words != 16 && state_words != 32 && state_words != 64 && state_words != 128)
        return horizon_fail(OVC_E_BADARG, "state_words must be 16, 32, 64 or 128", state_words);
    if ((((uintptr_t)state | (uintptr_t)records) & 15) ||
        (((uintptr_t)done | (uintptr_t)partner_seat | (uintptr_t)view | (uintptr_t)jrow | (uintptr_t)range | (uintptr_t)values) & 3))
        return horizon_fail(OVC_E_BADARG, "state and records must be 16-byte aligned, the other buffers 4-byte aligned");
    if (n_envs == 0) return OVC_OK;
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t err = cudaMemsetAsync(range, 0, 2 * sizeof(int32_t), st);
    if (err == cudaSuccess) {
        const unsigned blocks = (unsigned)((n_envs + ovc::HORIZON_ROWS_THREADS - 1) / ovc::HORIZON_ROWS_THREADS);
        ovc::horizon_rows_kernel<<<blocks, ovc::HORIZON_ROWS_THREADS, 0, st>>>(state, state_words, done, partner_seat, one_view, n_envs,
                                                                               records, view, jrow, range, values);
        err = cudaGetLastError();
    }
    if (err != cudaSuccess) return horizon_fail(OVC_E_CUDA, cudaGetErrorString(err));
    return OVC_OK;
}

int ovc_gae_horizon(const float *rewards, const float *values, const uint8_t *dones, const float *terminal_values,
                    const float *last_values, int64_t n_steps, int64_t n_rows, float gamma, float lambda, float *advantages,
                    float *value_targets, void *stream) {
    return ovc::gae_horizon_impl(rewards, values, dones, terminal_values, last_values, n_steps, n_rows, gamma, lambda, advantages,
                                 value_targets, (cudaStream_t)stream, false);
}

int ovc_gae_horizon_view(const float *rewards, const float *values, const uint8_t *dones, const float *terminal_values,
                         const float *last_values, int64_t n_steps, int64_t n_envs, float gamma, float lambda, float *advantages,
                         float *value_targets, void *stream) {
    return ovc::gae_horizon_impl(rewards, values, dones, terminal_values, last_values, n_steps, n_envs, gamma, lambda, advantages,
                                 value_targets, (cudaStream_t)stream, true);
}

}  // extern "C"
