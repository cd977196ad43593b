// ovc_host.cuh — host-side helpers of the C ABI (no device code): expansion of the 2-byte
// OVC_F_OUT_CODES transfer words into the dense reward / done / event arrays a host consumer indexes.
// The result of a rollout crosses PCIe as codes; this runs on the host cores at memory speed.
#pragma once
#include <sched.h>
#include <stdint.h>
#include <string.h>
#include <unistd.h>
#if defined(__x86_64__)
#include <immintrin.h>
#endif

#include <condition_variable>
#include <functional>
#include <mutex>
#include <thread>
#include <vector>

#include "../../include/ovc_b200.h"

namespace ovc {

// One OVC_F_OUT_CODES word -> element i of each requested dense array; tb: the reward table of the word's layout
static inline void expand_word(unsigned w, size_t i, const int32_t *tb, const int32_t *mask, int16_t *sparse, int8_t *shaped,
                               uint8_t *done, int32_t *events) {
    const unsigned c0 = w & 31u, c1 = (w >> 5) & 31u;
    if (sparse) sparse[i] = (int16_t)(tb[c0] + tb[c1]);
    if (shaped) {
        shaped[2 * i] = (int8_t)((w >> 12) & 1u ? tb[32 + c0] : 0);
        shaped[2 * i + 1] = (int8_t)((w >> 13) & 1u ? tb[32 + c1] : 0);
    }
    if (done) done[i] = (uint8_t)((w >> 10) & 1u);
    if (events) {
        const bool stepped = (w >> 11) & 1u;  // a finished env was stepped: nothing happened, only the flag is set
        events[2 * i] = stepped ? (int32_t)OVC_EVF_STEPPED_DONE : mask[c0];
        events[2 * i + 1] = stepped ? (int32_t)OVC_EVF_STEPPED_DONE : mask[c1];
    }
}

static void expand_range(const uint16_t *codes, int64_t lo, int64_t hi, int64_t n_envs, const int32_t *env_layout,
                         const int32_t *reward_tbl, int16_t *sparse, int8_t *shaped, uint8_t *done, int32_t *events,
                         const int32_t *mask) {
    int64_t e = n_envs > 0 ? lo % n_envs : 0;  // env index of word i, carried instead of a 64-bit modulo per word
    for (int64_t i = lo; i < hi; i++, e = e + 1 == n_envs ? 0 : e + 1)
        expand_word(codes[i], (size_t)i, reward_tbl + (env_layout ? (size_t)env_layout[e] * 64 : 0), mask, sparse, shaped, done, events);
}

// A small persistent worker pool: spawning a hundred threads per call costs more than expanding 26 M words.
class HostPool {
public:
    static HostPool &get() {
        static HostPool *p = new HostPool();  // never destroyed: its detached workers may outlive static destruction
        return *p;
    }
    // runs job(k) for k in [0, n_jobs) on n_threads threads (the caller is one of them); slices are claimed
    // dynamically, so a core that is shared with somebody else's process only delays its current slice
    void run(int n_jobs, int n_threads, const std::function<void(int)> &job) {
        std::unique_lock<std::mutex> call(call_mu_);  // one parallel region at a time
        grow(n_threads - 1);
        {
            std::lock_guard<std::mutex> g(mu_);
            job_ = &job, n_jobs_ = n_jobs, next_ = 0, pending_ = n_jobs, limit_ = n_threads - 1, active_ = 0;
        }
        cv_.notify_all();
        for (;;) {
            int k;
            {
                std::lock_guard<std::mutex> g(mu_);
                if (next_ >= n_jobs_) break;
                k = next_++;
            }
            job(k);
            std::lock_guard<std::mutex> g(mu_);
            --pending_;
        }
        std::unique_lock<std::mutex> g(mu_);
        done_cv_.wait(g, [&] { return pending_ == 0; });
        job_ = nullptr, n_jobs_ = 0;
    }

private:
    void grow(int n) {
        while ((int)workers_.size() < n) {
            workers_.emplace_back([this] { loop(); });
            workers_.back().detach();
        }
    }
    void loop() {
        for (;;) {
            int k;
            const std::function<void(int)> *job;
            {
                std::unique_lock<std::mutex> g(mu_);
                // an unclaimed slice of the current region, and room among the threads this region asked for
                cv_.wait(g, [&] { return next_ < n_jobs_ && active_ < limit_; });
                k = next_++;
                job = job_;
                active_++;
            }
            for (;;) {
                (*job)(k);
                std::lock_guard<std::mutex> g(mu_);
                if (--pending_ == 0) done_cv_.notify_all();
                if (next_ >= n_jobs_) {
                    active_--;
                    break;
                }
                k = next_++;
            }
        }
    }
    std::mutex call_mu_, mu_;
    std::condition_variable cv_, done_cv_;
    std::vector<std::thread> workers_;
    const std::function<void(int)> *job_ = nullptr;
    int n_jobs_ = 0, next_ = 0, pending_ = 0, limit_ = 0, active_ = 0;
};

static int default_host_threads() {  // every CPU of the process's affinity mask (a fractional-node lease sees the whole machine online)
    cpu_set_t set;
    int n = sched_getaffinity(0, sizeof set, &set) == 0 ? CPU_COUNT(&set) : 0;
    if (n <= 0) {
        const long c = sysconf(_SC_NPROCESSORS_ONLN);
        n = c > 0 ? (int)c : 1;
    }
    return n;
}

static int expand_codes_host(const uint16_t *codes, int64_t n_steps, int64_t n_envs, const int32_t *env_layout,
                             const int32_t *reward_tbl, int n_layouts, int16_t *sparse, int8_t *shaped, uint8_t *done,
                             int32_t *events, int n_threads) {
    if (!codes || !reward_tbl) return fail(OVC_E_BADARG, "null pointer argument");
    if (n_steps < 0 || n_envs < 0 || n_layouts < 1) return fail(OVC_E_BADARG, "bad sizes");
    if (env_layout)
        for (int64_t e = 0; e < n_envs; e++)
            if (env_layout[e] < 0 || env_layout[e] >= n_layouts) return fail(OVC_E_BADARG, "layout id out of range", (long long)e);
    int32_t mask[32];  // code -> int32 event mask incl. the delivered-recipe bits
    for (int c = 0; c < 32; c++) mask[c] = (int32_t)code_mask_of(c);
    const int64_t n = n_steps * n_envs;
    if (n_threads <= 0) n_threads = default_host_threads();
    if (n_threads > 256) n_threads = 256;
    if (n < (int64_t)n_threads * 4096) n_threads = (int)(n / 4096) + 1;
    if (n_threads == 1) {
        expand_range(codes, 0, n, n_envs, env_layout, reward_tbl, sparse, shaped, done, events, mask);
        return OVC_OK;
    }
    const int n_slices = n_threads * 8;  // ~50 k words per slice at the bench's size
    HostPool::get().run(n_slices, n_threads, [&](int k) {
        expand_range(codes, n * k / n_slices, n * (k + 1) / n_slices, n_envs, env_layout, reward_tbl, sparse, shaped, done,
                     events, mask);
    });
    return OVC_OK;
}

// Row segments of the dense arrays are built in a small thread-local buffer (L1 resident) and then written out ONCE with
// non-temporal stores: the arrays are written, never read, by the expander, so ordinary stores would first fetch every
// line from DRAM (read-for-ownership) and double the memory traffic — measured: 16 threads expanded 26 M env-steps in
// 3.3 ms with memset + scatter into the arrays, which is the memory bandwidth of 2 x 131 MB, not the work.
static int nt_store_mode() {  // OVC_EXPAND_NT (measurement hook): 0 = ordinary stores, 1 = 16-byte streaming stores only, unset = widest
    static int v = -1;
    if (v < 0) {
        const char *e = getenv("OVC_EXPAND_NT");
        v = e ? atoi(e) : 2;
    }
    return v;
}
static bool use_nt_stores() { return nt_store_mode() != 0; }

#if defined(__x86_64__)
// whole cache lines per store where the CPU has 512-bit vectors (one write-combining buffer per instruction)
__attribute__((target("avx512f"))) static void stream_out_avx512(void *dst, const void *src, size_t bytes) {
    const __m512i *s = (const __m512i *)src;
    __m512i *d = (__m512i *)dst;
    for (size_t i = 0; i < bytes / 64; i++) _mm512_stream_si512(d + i, _mm512_load_si512(s + i));
}
static bool cpu_has_avx512() {
    static int v = -1;
    if (v < 0) v = __builtin_cpu_supports("avx512f") ? 1 : 0;
    return v != 0;
}
#endif

static inline void stream_out(void *dst, const void *src, size_t bytes) {
#if defined(__x86_64__)
    if (use_nt_stores()) {
        if (nt_store_mode() >= 2 && (((uintptr_t)dst | (uintptr_t)src | bytes) & 63) == 0 && cpu_has_avx512()) return stream_out_avx512(dst, src, bytes);
        if ((((uintptr_t)dst | bytes) & 15) == 0) {
            const __m128i *s = (const __m128i *)src;
            __m128i *d = (__m128i *)dst;
            for (size_t i = 0; i < bytes / 16; i++) _mm_stream_si128(d + i, _mm_load_si128(s + i));
            return;
        }
    }
#endif
    memcpy(dst, src, bytes);
}

// OVC_F_OUT_STREAM -> dense arrays.  A thread owns a range of groups [g0, g1) = environments [32 g0, 32 g1): per
// transition it builds its segment of every output row (zeros + the few non-zero words its masks name, each group's
// value slice read sequentially; the cursor restarts at every chunk) and streams it out.
static void expand_stream_range(const uint32_t *masks, const uint16_t *values, int64_t n_steps, int64_t chunk, int64_t cap,
                                int64_t n_envs, int64_t G, int64_t g0, int64_t g1, const int32_t *env_layout,
                                const int32_t *reward_tbl, int16_t *sparse, int8_t *shaped, uint8_t *done, int32_t *events,
                                const int32_t *mask, int64_t *overflow) {
    constexpr int SEG_GROUPS = 32;  // 1024 environments per segment: 2 + 2 + 1 + 8 KB of row buffers
    alignas(64) int16_t b_sparse[SEG_GROUPS * 32];
    alignas(64) int8_t b_shaped[SEG_GROUPS * 64];
    alignas(64) uint8_t b_done[SEG_GROUPS * 32];
    alignas(64) int32_t b_events[SEG_GROUPS * 64];
    int16_t *const r_sparse = sparse ? b_sparse : nullptr;  // the row buffers of the requested arrays
    int8_t *const r_shaped = shaped ? b_shaped : nullptr;
    uint8_t *const r_done = done ? b_done : nullptr;
    int32_t *const r_events = events ? b_events : nullptr;
    int64_t over = 0;
    for (int64_t s0 = g0; s0 < g1; s0 += SEG_GROUPS) {
        const int64_t s1 = s0 + SEG_GROUPS < g1 ? s0 + SEG_GROUPS : g1;
        const int64_t e0 = s0 * 32, e1 = s1 * 32 < n_envs ? s1 * 32 : n_envs;
        if (e1 <= e0) break;
        const size_t ne = (size_t)(e1 - e0);
        uint32_t cur[SEG_GROUPS] = {0};
        for (int64_t t = 0; t < n_steps; t++) {
            const int64_t c = t / chunk;
            if (t % chunk == 0)
                for (int k = 0; k < SEG_GROUPS; k++) over += cur[k] > (uint64_t)cap, cur[k] = 0;
            if (sparse) memset(b_sparse, 0, ne * sizeof(int16_t));
            if (shaped) memset(b_shaped, 0, ne * 2);
            if (done) memset(b_done, 0, ne);
            if (events) memset(b_events, 0, ne * 2 * sizeof(int32_t));
            const uint32_t *mrow = masks + t * G;
            for (int64_t g = s0; g < s1; g++) {
                uint32_t m = mrow[g];
                if (!m) continue;
                const uint16_t *vals = values + ((size_t)c * (size_t)G + (size_t)g) * (size_t)cap;
                uint32_t &k = cur[g - s0];
                while (m) {
                    const int l = __builtin_ctz(m);
                    m &= m - 1;
                    const uint32_t kk = k++;
                    if (kk >= (uint64_t)cap) continue;  // dropped by the kernel: counted at the chunk boundary
                    const int64_t e = g * 32 + l;
                    expand_word(vals[kk], (size_t)(e - e0), reward_tbl + (env_layout ? (size_t)env_layout[e] * 64 : 0), mask, r_sparse,
                                r_shaped, r_done, r_events);
                }
            }
            const size_t row = (size_t)t * (size_t)n_envs + (size_t)e0;
            if (sparse) stream_out(sparse + row, b_sparse, ne * sizeof(int16_t));
            if (shaped) stream_out(shaped + 2 * row, b_shaped, ne * 2);
            if (done) stream_out(done + row, b_done, ne);
            if (events) stream_out(events + 2 * row, b_events, ne * 2 * sizeof(int32_t));
        }
        for (int k = 0; k < SEG_GROUPS; k++) over += cur[k] > (uint64_t)cap;
    }
#if defined(__x86_64__)
    _mm_sfence();  // non-temporal stores are weakly ordered: make them visible before the caller is told we are done
#endif
    if (over) __atomic_fetch_add(overflow, over, __ATOMIC_RELAXED);
}

static int expand_stream_host(const uint32_t *masks, const uint16_t *values, int64_t n_steps, int64_t chunk, int64_t cap,
                              int64_t n_envs, const int32_t *env_layout, const int32_t *reward_tbl, int n_layouts, int16_t *sparse,
                              int8_t *shaped, uint8_t *done, int32_t *events, int n_threads, int64_t *overflow) {
    if (!masks || !values || !reward_tbl) return fail(OVC_E_BADARG, "null pointer argument");
    if (n_steps < 0 || n_envs < 0 || n_layouts < 1 || chunk < 1 || cap < 1) return fail(OVC_E_BADARG, "bad sizes");
    if (env_layout)
        for (int64_t e = 0; e < n_envs; e++)
            if (env_layout[e] < 0 || env_layout[e] >= n_layouts) return fail(OVC_E_BADARG, "layout id out of range", (long long)e);
    int32_t mask[32];
    for (int c = 0; c < 32; c++) mask[c] = (int32_t)code_mask_of(c);
    const int64_t G = (n_envs + 31) / 32;
    int64_t over = 0;
    if (n_threads <= 0) n_threads = default_host_threads();
    if (n_threads > 256) n_threads = 256;
    if (G < (int64_t)n_threads * 4) n_threads = (int)(G / 4) + 1;
    if (n_threads == 1) {
        expand_stream_range(masks, values, n_steps, chunk, cap, n_envs, G, 0, G, env_layout, reward_tbl, sparse, shaped, done, events, mask, &over);
    } else {
        const int n_slices = n_threads * 4;
        HostPool::get().run(n_slices, n_threads, [&](int k) {
            expand_stream_range(masks, values, n_steps, chunk, cap, n_envs, G, G * k / n_slices, G * (k + 1) / n_slices, env_layout, reward_tbl,
                                sparse, shaped, done, events, mask, &over);
        });
    }
    if (overflow) *overflow = over;
    return OVC_OK;
}

// ------------------------------------------------------------------------------------------------
// host-buffer rollout pipeline (ovc_pipeline_*): H2D / rollout kernel / D2H on three streams
// ------------------------------------------------------------------------------------------------
}  // namespace ovc

struct ovc_pipeline {
    ovc_pipeline_desc_t d;
    ovc::OutFmt fmt;
    cudaStream_t s_h2d, s_comp, s_d2h;
    cudaEvent_t ev_start, ev_in[2], ev_comp[2], ev_d2h[2], ev_join[3];
    bool comp_rec[2], d2h_rec[2];
    static constexpr int RING = 8;
    cudaEvent_t ev_pass[RING];
    int64_t n_pass;
    int64_t k;  // chunk counter: buffer parity carries across passes
};

namespace ovc {

#define OVC_CK(call, what)                                 \
    do {                                                   \
        cudaError_t e_ = (call);                           \
        if (e_ != cudaSuccess) return cuda_fail(e_, what); \
    } while (0)

static int pipeline_create(const ovc_pipeline_desc_t *desc, ovc_pipeline_t **out) {
    if (!desc || !out) return fail(OVC_E_BADARG, "null pointer argument");
    if (desc->chunk < 1) return fail(OVC_E_BADARG, "chunk must be >= 1", (long long)desc->chunk);
    int rc = check_common(desc->layouts, desc->n_layouts, desc->state, desc->n_envs, desc->state_words);
    if (rc) return rc;
    const OutFmt f = formats_of(desc->flags);
    for (int b = 0; b < 2; b++)
        if (f.missing(desc->d_actions[b], desc->d_sparse[b], desc->d_shaped[b], desc->d_done[b], desc->d_events[b]))
            return fail(OVC_E_BADARG, "missing device staging buffer");
    if (f.stream && (desc->stream_cap < 1 || desc->stream_cap > OVC_F_STREAM_CAP_MAX))
        return fail(OVC_E_BADARG, "stream_cap must be 1..65535", (long long)desc->stream_cap);
    ovc_pipeline_t *p = new ovc_pipeline_t();
    p->d = *desc;
    p->fmt = f;
    p->n_pass = 0, p->k = 0;
    p->comp_rec[0] = p->comp_rec[1] = p->d2h_rec[0] = p->d2h_rec[1] = false;
    cudaError_t e = cudaSuccess;
    auto mk_stream = [&](cudaStream_t *s) { if (e == cudaSuccess) e = cudaStreamCreateWithFlags(s, cudaStreamNonBlocking); };
    auto mk_event = [&](cudaEvent_t *v) { if (e == cudaSuccess) e = cudaEventCreateWithFlags(v, cudaEventDisableTiming); };
    mk_stream(&p->s_h2d), mk_stream(&p->s_comp), mk_stream(&p->s_d2h);
    mk_event(&p->ev_start);
    for (int b = 0; b < 2; b++) mk_event(&p->ev_in[b]), mk_event(&p->ev_comp[b]), mk_event(&p->ev_d2h[b]);
    for (int i = 0; i < 3; i++) mk_event(&p->ev_join[i]);
    for (int i = 0; i < ovc_pipeline::RING; i++) mk_event(&p->ev_pass[i]);
    if (e != cudaSuccess) {
        delete p;  // streams / events created so far are leaked only on an already failing device
        return cuda_fail(e, "pipeline stream / event creation");
    }
    *out = p;
    return OVC_OK;
}

static int pipeline_join(ovc_pipeline_t *p, cudaStream_t caller) {
    cudaStream_t ss[3] = {p->s_h2d, p->s_comp, p->s_d2h};
    for (int i = 0; i < 3; i++) {
        OVC_CK(cudaEventRecord(p->ev_join[i], ss[i]), "pipeline join record");
        OVC_CK(cudaStreamWaitEvent(caller, p->ev_join[i], 0), "pipeline join wait");
    }
    return OVC_OK;
}

static int pipeline_run(ovc_pipeline_t *p, const void *h_actions, void *h_sparse, void *h_shaped, void *h_done, void *h_events,
                        int n_steps, cudaStream_t caller, int join, int64_t *ticket) {
    const OutFmt &f = p->fmt;
    if (f.missing(h_actions, h_sparse, h_shaped, h_done, h_events)) return fail(OVC_E_BADARG, "null host buffer");
    if (n_steps < 1) return fail(OVC_E_BADARG, "n_steps must be >= 1");
    const ovc_pipeline_desc_t &d = p->d;
    const size_t N = (size_t)d.n_envs, G = (N + 31) / 32;
    void *const codes_full = f.stream ? d.d_codes_full[p->n_pass & 1] : nullptr;
    OVC_CK(cudaEventRecord(p->ev_start, caller), "pipeline start record");
    OVC_CK(cudaStreamWaitEvent(p->s_h2d, p->ev_start, 0), "pipeline start wait");
    OVC_CK(cudaStreamWaitEvent(p->s_comp, p->ev_start, 0), "pipeline start wait");
    OVC_CK(cudaStreamWaitEvent(p->s_d2h, p->ev_start, 0), "pipeline start wait");
    for (int t0 = 0; t0 < n_steps; t0 += d.chunk) {
        const int tc = n_steps - t0 < d.chunk ? n_steps - t0 : d.chunk;
        const int b = (int)(p->k++ & 1);
        const size_t off = (size_t)t0 * N, cnt = (size_t)tc * N;
        // stage 1: this chunk's actions, once the kernel two chunks ago has consumed the staging buffer
        if (p->comp_rec[b]) OVC_CK(cudaStreamWaitEvent(p->s_h2d, p->ev_comp[b], 0), "pipeline wait");
        OVC_CK(cudaMemcpyAsync(d.d_actions[b], (const char *)h_actions + off * f.act, cnt * f.act, cudaMemcpyHostToDevice, p->s_h2d),
               "pipeline H2D copy");
        OVC_CK(cudaEventRecord(p->ev_in[b], p->s_h2d), "pipeline record");
        // stage 2: the fused rollout kernel, once the outputs of two chunks ago have left the staging buffers
        OVC_CK(cudaStreamWaitEvent(p->s_comp, p->ev_in[b], 0), "pipeline wait");
        if (p->d2h_rec[b]) OVC_CK(cudaStreamWaitEvent(p->s_comp, p->ev_d2h[b], 0), "pipeline wait");
        int rc;
        if (f.stream)  // masks + compacted values of this chunk; the dense words (if kept) go to their rows of the pass buffer
            rc = step_impl(d.layouts, d.n_layouts, d.start_records, d.state, (const int32_t *)d.d_actions[b], (int32_t *)d.d_sparse[b], nullptr,
                           codes_full ? (int32_t *)((char *)codes_full + off * 2) : nullptr, (int32_t *)d.d_events[b], d.n_envs, tc,
                           d.state_words, d.horizon, (int)((unsigned)d.flags | ((unsigned)d.stream_cap << OVC_F_STREAM_CAP_SHIFT)),
                           d.has_random_start ? &d.random_start : nullptr, p->s_comp);
        else
            rc = step_impl(d.layouts, d.n_layouts, d.start_records, d.state, (const int32_t *)d.d_actions[b], (int32_t *)d.d_sparse[b],
                           (int32_t *)d.d_shaped[b], (int32_t *)d.d_done[b], (int32_t *)d.d_events[b], d.n_envs, tc, d.state_words,
                           d.horizon, d.flags, d.has_random_start ? &d.random_start : nullptr, p->s_comp);
        if (rc) return rc;
        OVC_CK(cudaEventRecord(p->ev_comp[b], p->s_comp), "pipeline record");
        p->comp_rec[b] = true;
        // stage 3: results to the host
        OVC_CK(cudaStreamWaitEvent(p->s_d2h, p->ev_comp[b], 0), "pipeline wait");
        if (f.stream) {  // the lane masks and the value slots; the dense backup stays on the device
            const size_t c = (size_t)(t0 / d.chunk), vbytes = G * (size_t)d.stream_cap * f.sparse;
            OVC_CK(cudaMemcpyAsync((char *)h_events + (size_t)t0 * G * f.events, d.d_events[b], (size_t)tc * G * f.events, cudaMemcpyDeviceToHost, p->s_d2h), "pipeline D2H copy");
            OVC_CK(cudaMemcpyAsync((char *)h_sparse + c * vbytes, d.d_sparse[b], vbytes, cudaMemcpyDeviceToHost, p->s_d2h), "pipeline D2H copy");
        } else {
            if (f.sparse) OVC_CK(cudaMemcpyAsync((char *)h_sparse + off * f.sparse, d.d_sparse[b], cnt * f.sparse, cudaMemcpyDeviceToHost, p->s_d2h), "pipeline D2H copy");
            if (f.shaped) OVC_CK(cudaMemcpyAsync((char *)h_shaped + off * f.shaped, d.d_shaped[b], cnt * f.shaped, cudaMemcpyDeviceToHost, p->s_d2h), "pipeline D2H copy");
            if (f.done) OVC_CK(cudaMemcpyAsync((char *)h_done + off * f.done, d.d_done[b], cnt * f.done, cudaMemcpyDeviceToHost, p->s_d2h), "pipeline D2H copy");
            OVC_CK(cudaMemcpyAsync((char *)h_events + off * f.events, d.d_events[b], cnt * f.events, cudaMemcpyDeviceToHost, p->s_d2h), "pipeline D2H copy");
        }
        OVC_CK(cudaEventRecord(p->ev_d2h[b], p->s_d2h), "pipeline record");
        p->d2h_rec[b] = true;
    }
    const int64_t id = p->n_pass++;
    OVC_CK(cudaEventRecord(p->ev_pass[id % ovc_pipeline::RING], p->s_d2h), "pipeline record");
    if (ticket) *ticket = id;
    if (join) return pipeline_join(p, caller);
    return OVC_OK;
}

static int pipeline_wait(ovc_pipeline_t *p, int64_t ticket) {
    if (ticket < 0 || ticket >= p->n_pass) return fail(OVC_E_BADARG, "unknown pass ticket", (long long)ticket);
    // the ring slot may by now hold the event of a LATER pass: it was recorded later on the same copy stream, so
    // waiting for it implies the asked-for pass has landed too
    OVC_CK(cudaEventSynchronize(p->ev_pass[ticket % ovc_pipeline::RING]), "pipeline wait");
    return OVC_OK;
}

static void pipeline_destroy(ovc_pipeline_t *p) {
    if (!p) return;
    cudaStreamSynchronize(p->s_h2d), cudaStreamSynchronize(p->s_comp), cudaStreamSynchronize(p->s_d2h);
    cudaEventDestroy(p->ev_start);
    for (int b = 0; b < 2; b++) cudaEventDestroy(p->ev_in[b]), cudaEventDestroy(p->ev_comp[b]), cudaEventDestroy(p->ev_d2h[b]);
    for (int i = 0; i < 3; i++) cudaEventDestroy(p->ev_join[i]);
    for (int i = 0; i < ovc_pipeline::RING; i++) cudaEventDestroy(p->ev_pass[i]);
    cudaStreamDestroy(p->s_h2d), cudaStreamDestroy(p->s_comp), cudaStreamDestroy(p->s_d2h);
    delete p;
}
#undef OVC_CK

}  // namespace ovc
