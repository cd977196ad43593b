// ovc_potential.cuh — K6 potential_kernel: the reference's shaped-reward potential phi(s)
// (overcooked_mdp.py:2920-3250), one thread per environment, double precision.
//
// The reference evaluates gamma ** (small integer) in Python floats and combines the factors with
// plain double multiplications and additions in a fixed order.  The kernel takes the powers from a
// host-built table (gpow[k] = gamma ** k as Python computes it) and performs every multiplication and
// addition with __dmul_rn / __dadd_rn in exactly that order (no FMA contraction), so phi is
// reproduced bit for bit, not merely within a tolerance.  Player "lists" are 2-bit masks walked in
// player order; soups are visited in the orders the reference's Python containers would yield
// (pot order, dict insertion order, CPython's set order for the partially full pots — from the table).
#pragma once

namespace ovc {

struct PotArgs {
    const ovc_layout_t *layouts;
    const ovc_potential_t *pt;
    const ovc_cost_lut_entry_t *cost;
    const double *gpow;
    const int32_t *state;
    double *out;
    long long n_envs;
    int S, n_pow;
};

#define OVC_BIG 1000000

__device__ __forceinline__ double gpw(const PotArgs &a, int k) { return __ldg(a.gpow + (k < a.n_pow ? k : a.n_pow - 1)); }

__global__ void __launch_bounds__(128) potential_kernel(const PotArgs a) {
    const long long env = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= a.n_envs) return;
    const int32_t *__restrict__ rec = a.state + env * a.S;
#include "ovc_potential_phi.inc"
    a.out[env] = potential;
}

static int potential_impl(const ovc_layout_t *layouts, const ovc_potential_t *pt, const ovc_cost_lut_entry_t *cost,
                          const double *gpow, int n_pow, const int32_t *state, double *out, long long n_envs, int S,
                          cudaStream_t st) {
    if (!pt || !cost || !gpow || !out) return fail(OVC_E_BADARG, "null pointer argument");
    if (n_pow < 2) return fail(OVC_E_BADARG, "gamma power table too short");
    if (n_envs == 0) return OVC_OK;
    PotArgs a{layouts, pt, cost, gpow, state, out, n_envs, S, n_pow};
    potential_kernel<<<(unsigned)((n_envs + 127) / 128), 128, 0, st>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "potential kernel launch");
    return OVC_OK;
}

// ovc_potential_shaping: the potential-based dense reward of the transition ovc_step has just made with auto-reset off,
// then that auto-reset.  K1 resets a finishing environment inside the step, where phi(s') of the terminal record would be
// lost; here phi is taken first and the record is reset after.
struct ShapingArgs {
    PotArgs p;  // p.state: the records, p.out unused
    const int32_t *start_records;
    int32_t *state;
    const int32_t *done;
    const double *phi_s;
    float *dense;
    int n_layouts;
    ovc_random_start_t rs;
};

// RS: compiled with the random-start draw, as K1's RS instantiation.
template <bool RS>
__global__ void __launch_bounds__(128) potential_shaping_kernel(const ShapingArgs s) {
    const long long env = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= s.p.n_envs) return;
    const int S = s.p.S;
    const PotArgs &a = s.p;
    const int32_t *rec = s.state + env * S;
#include "ovc_potential_phi.inc"
    s.dense[env] = __double2float_rn(__dsub_rn(potential, s.phi_s[env]));
    if (s.done[env] == 0) return;
    // The record was read through the read-only path: those reads are ordered before the reset's stores to it.
    __threadfence_block();
    // K1's OVC_F_AUTO_RESET (step_core): the start record of the record's layout, or a random start of the next episode
    GlobalRec r{s.state + env * S};
    int nl = lid;  // the layout id of word 3 (h: the record's header, read above)
    if (RS) {
        const unsigned episode = (((unsigned)h.w >> 16) + 1u) & 0xFFFFu;
        if (s.rs.random_layout) nl = random_layout_id(s.rs, (uint64_t)env, episode, s.n_layouts);
        const ovc_layout_t *Ln = s.p.layouts + nl;
        random_start_record([&](int w, int32_t v) { r.stw(w, v); }, S, s.start_records + (size_t)nl * S, Ln->cook_time, Ln->free_pos,
                            Ln->n_free, Ln->n_pots, nl, s.rs, (uint64_t)env, episode);
    } else {
        const int4 *__restrict__ src = reinterpret_cast<const int4 *>(s.start_records + (size_t)nl * S);
#pragma unroll 4
        for (int c = 0; c < S / 4; c++) r.st4(c, __ldg(src + c));
    }
}

static int potential_shaping_impl(const ovc_layout_t *layouts, int n_layouts, const int32_t *start_records, const ovc_potential_t *pt,
                                  const ovc_cost_lut_entry_t *cost, const double *gpow, int n_pow, int32_t *state, const int32_t *done,
                                  const double *phi_s, float *dense, long long n_envs, int S, const ovc_random_start_t *rs,
                                  cudaStream_t st) {
    if (!start_records || !pt || !cost || !gpow || !done || !phi_s || !dense) return fail(OVC_E_BADARG, "null pointer argument");
    if (n_pow < 2) return fail(OVC_E_BADARG, "gamma power table too short");
    if (((uintptr_t)phi_s & 7) != 0) return fail(OVC_E_BADARG, "phi_s must be 8-byte aligned");
    if ((((uintptr_t)dense | (uintptr_t)done) & 3) != 0) return fail(OVC_E_BADARG, "dense and done must be 4-byte aligned");
    if (n_envs == 0) return OVC_OK;
    ShapingArgs a{PotArgs{layouts, pt, cost, gpow, state, nullptr, n_envs, S, n_pow}, start_records, state, done, phi_s, dense, n_layouts,
                  rs ? *rs : ovc_random_start_t{0, 0, 0}};
    const unsigned grid = (unsigned)((n_envs + 127) / 128);
    if (rs) potential_shaping_kernel<true><<<grid, 128, 0, st>>>(a);
    else potential_shaping_kernel<false><<<grid, 128, 0, st>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "potential_shaping kernel launch");
    return OVC_OK;
}

}  // namespace ovc
