// ovc_partner.cuh — the behaviour-cloned partner of PPO_BC (included by ovc_b200.cu after ovc_obs.cuh and ovc_tail.cuh).
//
// K10 partner_policy_kernel: the BC agent's action from the packed record, features never materialised
// (reference: human_aware_rl/imitation/behavior_cloning_tf2.py — featurize_state, Dense 64 ReLU, Dense 64 ReLU, 6 logits,
// the action sampled from the softmax):
//   phase 1  K3's feat_block for both players of each environment of a 64-environment tile, into a feature-major int16
//            tile laid out exactly as K3's (column 2 e + j = player j's view: own block, other block, other - self,
//            self position); only environments with a partner are built
//   phase 2  warps own 16 environments each and run K8's layer chain on the partner's view column: A fragments read from
//            the tile and converted to bf16, ReLU between layers, heads padded to 8, then K8's Gumbel-max draw on row
//            2 e + seat
// assign_partners_kernel: the per-episode seat draw of OvercookedMultiAgent._populate_agents.
#pragma once

namespace ovc {

constexpr int PP_THREADS = 128;          // 4 warps x 16 environments = one K3 tile (FEAT_E = 64 environments, 2 views each)
constexpr int PP_F = 96;                 // featurize_state width at num_pots = 2
constexpr int PP_B = 46;                 // one player's block at num_pots = 2
constexpr int PP_TILE_BYTES = PP_F * FEAT_LD * 2;

struct PartnerArgs {
    FeatArgs f;                          // layouts, lut, state, n_envs, S, num_pots = 2 (the fields feat_block reads)
    const int32_t *partner_seat;         // [n_envs]: -1 self-play, 0 / 1 the partner's player index
    const __nv_bfloat16 *w_first;        // [64][96]
    const float *b_first;
    const __nv_bfloat16 *w_hidden;       // [n_hidden][64][64]
    const float *b_hidden;
    const __nv_bfloat16 *w_heads;        // [8][64]
    const float *b_heads;
    int n_hidden, n_actions;
    unsigned long long seed;
    unsigned long long *counter;         // [2]: step, arrival scratch (as ovc_sample_actions)
    int32_t *actions;                    // [n_envs][2]: only [e][seat] of partnered environments is written
    float *scores;                       // [n_envs][8] or null
};

__global__ void __launch_bounds__(PP_THREADS) partner_policy_kernel(const PartnerArgs p) {
    constexpr int KS2 = PP_F / 32;
    extern __shared__ __align__(16) char pp_smem[];
    const unsigned long long step = *reinterpret_cast<volatile unsigned long long *>(p.counter);
    const TailSmem w = tail_weights_to_smem<PP_F, PP_THREADS>(pp_smem, p);
    short *tile = reinterpret_cast<short *>(pp_smem + tail_smem_bytes(PP_F, p.n_hidden));  // [96][FEAT_LD], feature-major

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const long long n_tiles = (p.f.n_envs + FEAT_E - 1) / FEAT_E;
    for (long long tl = blockIdx.x; tl < n_tiles; tl += gridDim.x) {
        const long long env0 = tl * FEAT_E;
        __syncthreads();  // the previous tile's reads are done (first pass: the weights are in place)
        // ---- phase 1: thread (el, j) builds player j's block, as K3 does ----
        {
            const int v = threadIdx.x, el = v >> 1, j = v & 1;
            const long long e = env0 + el;
            const int seat = e < p.f.n_envs ? __ldg(p.partner_seat + e) : -1;
            if (seat >= 0) {
                const int32_t *__restrict__ rec = p.f.state + e * p.f.S;
                const int lid = __ldg(rec + 3) & 0xFF;
                const ovc_layout_t *__restrict__ L = p.f.layouts + lid;
                const unsigned me = (unsigned)__ldg(rec + 1 + j), ot = (unsigned)__ldg(rec + 2 - j);
                const ovc_feat_lut_entry_t *le = p.f.lut + (size_t)lid * 1024 + ((me & 0xFF) << 2 | ((me >> 8) & 3));
                feat_block(p.f, L, le, rec, me, tile + v, tile + (size_t)PP_B * FEAT_LD + (v ^ 1));
                if (j == seat) {  // :2877-2896 tail of the partner's row: other - self, then self position
                    short *tl4 = tile + (size_t)2 * PP_B * FEAT_LD + v;
                    tl4[0 * FEAT_LD] = (short)((int)(ot & 15) - (int)(me & 15));
                    tl4[1 * FEAT_LD] = (short)((int)((ot >> 4) & 15) - (int)((me >> 4) & 15));
                    tl4[2 * FEAT_LD] = (short)(me & 15);
                    tl4[3 * FEAT_LD] = (short)((me >> 4) & 15);
                }
            }
        }
        __syncthreads();
        // ---- phase 2: warp w evaluates environments 16 w + g and 16 w + g + 8 of the tile ----
        const int el0 = 16 * warp + g, el1 = el0 + 8;
        const long long e0 = env0 + el0, e1 = env0 + el1;
        const int seat0 = e0 < p.f.n_envs ? __ldg(p.partner_seat + e0) : -1, seat1 = e1 < p.f.n_envs ? __ldg(p.partner_seat + e1) : -1;
        if (__all_sync(0xFFFFFFFFu, seat0 < 0 && seat1 < 0)) continue;  // no partner among the warp's 16 environments
        // the partner's view column; an environment without a partner reads a column nobody wrote (finite int16 values,
        // its results are discarded)
        const short *c0 = tile + 2 * el0 + (seat0 > 0), *c1 = tile + 2 * el1 + (seat1 > 0);
        auto pair = [](short lo, short hi) {
            const __nv_bfloat162 h = __floats2bfloat162_rn((float)lo, (float)hi);  // exact while |value| <= 256
            return *reinterpret_cast<const unsigned *>(&h);
        };
        float acc[8][4];
        first_layer64<KS2>(acc, w, g, t, [&](int s2, unsigned a_lo[4], unsigned a_hi[4]) {
            const int k = 32 * s2 + 8 * t;
            short x0[8], x1[8];
#pragma unroll
            for (int i = 0; i < 8; i++) x0[i] = c0[(k + i) * FEAT_LD], x1[i] = c1[(k + i) * FEAT_LD];
            a_lo[0] = pair(x0[0], x0[1]), a_lo[1] = pair(x1[0], x1[1]), a_lo[2] = pair(x0[2], x0[3]), a_lo[3] = pair(x1[2], x1[3]);
            a_hi[0] = pair(x0[4], x0[5]), a_hi[1] = pair(x1[4], x1[5]), a_hi[2] = pair(x0[6], x0[7]), a_hi[3] = pair(x1[6], x1[7]);
        });
        float out[1][4];
        tail_layers(out, acc, w, p.n_hidden, 0.f, g, t);
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const long long e = h ? e1 : e0;
            const int seat = h ? seat1 : seat0;
            float lp;
            const int best = draw_row<false>(out[0][2 * h], out[0][2 * h + 1], p.seed, step, 2 * e + (seat > 0), p.n_actions, lane, t, lp);
            if (seat >= 0) {
                if (t == 0) p.actions[2 * e + seat] = best;
                if (p.scores) *reinterpret_cast<float2 *>(p.scores + e * PT_NOUT + 2 * t) = make_float2(out[0][2 * h], out[0][2 * h + 1]);
            }
        }
    }
    advance_step(p.counter, step);
}

static int partner_policy_impl(const PartnerArgs &a, int n_features, int width, cudaStream_t st) {
    if (!a.f.lut || !a.partner_seat || !a.w_first || !a.b_first || !a.w_heads || !a.b_heads || !a.counter || !a.actions ||
        (a.n_hidden > 0 && (!a.w_hidden || !a.b_hidden)))
        return fail(OVC_E_BADARG, "null pointer argument");
    if (n_features != PP_F) return fail(OVC_E_UNSUPPORTED, "partner_policy: built for featurize_state at num_pots = 2 (96 features)", n_features);
    if (width != PT_H) return fail(OVC_E_UNSUPPORTED, "partner_policy: built for 64-wide layers", width);
    if (a.n_actions < 1 || a.n_actions > 7) return fail(OVC_E_UNSUPPORTED, "partner_policy: n_actions must be 1..7", a.n_actions);
    if (a.n_hidden < 0 || a.n_hidden > 8) return fail(OVC_E_BADARG, "n_hidden must be 0..8", a.n_hidden);
    if ((((uintptr_t)a.w_first | (uintptr_t)a.w_hidden | (uintptr_t)a.w_heads) & 15) != 0) return fail(OVC_E_BADARG, "weights must be 16-byte aligned");
    if ((((uintptr_t)a.b_first | (uintptr_t)a.b_hidden | (uintptr_t)a.b_heads | (uintptr_t)a.scores) & 7) != 0)
        return fail(OVC_E_BADARG, "biases and scores must be 8-byte aligned");
    if (a.f.n_envs == 0) return OVC_OK;
    int dev = 0, n_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    const size_t smem = tail_smem_bytes(PP_F, a.n_hidden) + PP_TILE_BYTES;
    cudaError_t e = cudaFuncSetAttribute(partner_policy_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return cuda_fail(e, "partner_policy kernel attribute");
    int per_sm = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, partner_policy_kernel, PP_THREADS, smem);
    if (e != cudaSuccess) return cuda_fail(e, "partner_policy occupancy");
    if (per_sm < 1) per_sm = 1;
    // persistent CTAs: each copies the weights into shared memory once and then walks its share of the tiles
    const long long n_tiles = (a.f.n_envs + FEAT_E - 1) / FEAT_E, cap = (long long)per_sm * n_sm;
    partner_policy_kernel<<<(unsigned)(n_tiles < cap ? n_tiles : cap), PP_THREADS, smem, st>>>(a);
    e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "partner_policy kernel launch");
    return OVC_OK;
}

// partner_seat[e] for every environment whose episode just ended (done[e] != 0; all with done == NULL): Philox4x32-10 with
// key = seed, counter = (e low, e high, step low, step high) -> words w0, w1;  seat = w0 < threshold ? w1 >> 31 : -1, where
// threshold = bc_factor * 2^32 saturated as the random-start draw saturates it (bc_factor >= 1: always a partner).
__global__ void __launch_bounds__(256) assign_partners_kernel(const int32_t *__restrict__ done, const float *__restrict__ bc_factor, long long n_envs,
                                                              unsigned long long seed, unsigned long long *counter, int32_t *__restrict__ partner_seat) {
    const unsigned long long step = *reinterpret_cast<volatile unsigned long long *>(counter);
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < n_envs && (!done || done[e] != 0)) {
        const float f = *bc_factor;
        const uint32_t thr = f >= 1.f ? 0xFFFFFFFFu : f > 0.f ? (uint32_t)((double)f * 4294967296.0) : 0u;
        const Philox4 P = philox4x32_10(seed, (uint32_t)e, (uint32_t)((unsigned long long)e >> 32), (uint32_t)step, (uint32_t)(step >> 32));
        partner_seat[e] = draw_below(P.v[0], thr) ? (int32_t)(P.v[1] >> 31) : -1;
    }
    advance_step(counter, step);
}

static int assign_partners_impl(const int32_t *done, const float *bc_factor, long long n_envs, unsigned long long seed,
                                unsigned long long *counter, int32_t *partner_seat, cudaStream_t st) {
    if (!bc_factor || !counter || !partner_seat) return fail(OVC_E_BADARG, "null pointer argument");
    if (n_envs < 0) return fail(OVC_E_BADARG, "negative env count");
    if (n_envs == 0) return OVC_OK;
    assign_partners_kernel<<<(unsigned)((n_envs + 255) / 256), 256, 0, st>>>(done, bc_factor, n_envs, seed, counter, partner_seat);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "assign_partners kernel launch");
    return OVC_OK;
}

// ---- a population of partners: environments grouped by member, the member drawn per episode ----
constexpr int GM_THREADS = 1024;  // one CTA: 32 warps, warp w owns the w-th contiguous segment of the environments
constexpr int MAX_MEMBERS = 64;

// Stable counting sort of the environments by member[e] in ONE CTA, so that nothing leaves the device between the count and
// the scatter: (1) every warp counts its segment per member (warp-private rows of a shared histogram), (2) 64 threads
// turn the histogram into each (warp, member) start: offsets[k] + the counts of member k in the earlier segments, (3) every
// warp walks its segment 32 environments at a time in order; lanes with the same member find each other with
// __match_any_sync and take consecutive slots in lane order.  Segments and chunks are visited in index order, so each group
// is ascending.
__global__ void __launch_bounds__(GM_THREADS, 1) group_members_kernel(const int32_t *__restrict__ member, int n_members, long long n_envs,
                                                                      int32_t *__restrict__ order, int32_t *__restrict__ offsets) {
    __shared__ int hist[GM_THREADS / 32][MAX_MEMBERS];
    __shared__ int tot[MAX_MEMBERS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < (GM_THREADS / 32) * MAX_MEMBERS; i += GM_THREADS) (&hist[0][0])[i] = 0;
    __syncthreads();
    const long long seg = (n_envs + GM_THREADS / 32 - 1) / (GM_THREADS / 32);
    const long long beg = warp * seg, end = beg + seg < n_envs ? beg + seg : n_envs;
    for (long long e = beg + lane; e < end; e += 32) atomicAdd(&hist[warp][__ldg(member + e)], 1);
    __syncthreads();
    if (threadIdx.x < MAX_MEMBERS) {  // thread k: member k's start in every segment, relative to the group's start
        const int k = threadIdx.x;
        int total = 0;
        for (int w = 0; w < GM_THREADS / 32; w++) {
            const int c = hist[w][k];
            hist[w][k] = total;
            total += c;
        }
        tot[k] = total;
    }
    __syncthreads();
    if (threadIdx.x == 0) {  // the group starts: an exclusive scan of the totals
        int run = 0;
        for (int k = 0; k < n_members; k++) {
            const int c = tot[k];
            tot[k] = run;
            run += c;
        }
        offsets[n_members] = run;
    }
    __syncthreads();
    if (threadIdx.x < n_members) {
        const int k = threadIdx.x, base = tot[k];
        offsets[k] = base;
        for (int w = 0; w < GM_THREADS / 32; w++) hist[w][k] += base;
    }
    __syncthreads();
    const unsigned lt = (1u << lane) - 1u;
    for (long long e0 = beg; e0 < end; e0 += 32) {
        const long long e = e0 + lane;
        const bool in = e < end;
        const int k = in ? __ldg(member + e) : -1 - lane;  // lanes past the end match nobody
        const unsigned peers = __match_any_sync(0xFFFFFFFFu, k);
        const int slot = in ? hist[warp][k] + __popc(peers & lt) : 0;
        __syncwarp();
        if (in) {
            order[slot] = (int32_t)e;
            if ((peers & lt) == 0) hist[warp][k] += __popc(peers);  // the group's first lane moves the start on
        }
        __syncwarp();
    }
}

static int group_members_impl(const int32_t *member, int n_members, long long n_envs, int32_t *order, int32_t *offsets, cudaStream_t st) {
    if (!member || !order || !offsets) return fail(OVC_E_BADARG, "null pointer argument");
    if (((uintptr_t)member | (uintptr_t)order | (uintptr_t)offsets) & 3) return fail(OVC_E_BADARG, "member, order and offsets must be 4-byte aligned");
    if (n_members < 1 || n_members > MAX_MEMBERS) return fail(OVC_E_BADARG, "n_members must be 1..64", n_members);
    if (n_envs < 0 || n_envs > 0x7FFFFFFFll) return fail(OVC_E_BADARG, "n_envs must be 0..2^31-1", n_envs);
    if (n_envs == 0) return OVC_OK;
    group_members_kernel<<<1, GM_THREADS, 0, st>>>(member, n_members, n_envs, order, offsets);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "group_members kernel launch");
    return OVC_OK;
}

// ---- self-play mixtures: the learner's rows of the joint [2 n_envs] rows ----
constexpr int LR_THREADS = 1024;  // one CTA: 32 warps, warp w owns the w-th contiguous segment of the environments
constexpr long long LR_MAX_ENVS = 1ll << 29;  // list entries pack e << 2 | mask into an int32

// A stable scan in ONE CTA, as group_members_kernel: (1) every warp counts its segment's learner views (2 where
// partner_seat[e] < 0, else 1), (2) one thread turns the warp totals into segment starts and writes range = {0, total},
// (3) every warp walks its segment 32 environments at a time in order, a warp-wide inclusive scan giving each environment
// its first compact row.  Environment e's views go to consecutive rows in ascending view order.
__global__ void __launch_bounds__(LR_THREADS, 1) learner_rows_kernel(const int32_t *__restrict__ partner_seat, long long n_envs,
                                                                     int32_t *__restrict__ list, int32_t *__restrict__ first,
                                                                     int32_t *__restrict__ jrow, int32_t *__restrict__ range) {
    __shared__ int start[LR_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long seg = (n_envs + LR_THREADS / 32 - 1) / (LR_THREADS / 32);
    const long long beg = warp * seg, end = beg + seg < n_envs ? beg + seg : n_envs;
    int cnt = 0;
    for (long long e = beg + lane; e < end; e += 32) cnt += __ldg(partner_seat + e) < 0 ? 2 : 1;
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) cnt += __shfl_xor_sync(0xFFFFFFFFu, cnt, d);
    if (lane == 0) start[warp] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
        int run = 0;
        for (int w = 0; w < LR_THREADS / 32; w++) {
            const int c = start[w];
            start[w] = run;
            run += c;
        }
        range[0] = 0;
        range[1] = run;
    }
    __syncthreads();
    int base = start[warp];
    for (long long e0 = beg; e0 < end; e0 += 32) {
        const long long e = e0 + lane;
        const bool in = e < end;
        const int s = in ? __ldg(partner_seat + e) : 0;
        const int mask = s < 0 ? 3 : (s == 0 ? 2 : 1);  // the learner's views: both in self-play, else view 1 - seat
        const int c = in ? (mask == 3 ? 2 : 1) : 0;
        int x = c;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int y = __shfl_up_sync(0xFFFFFFFFu, x, d);
            if (lane >= d) x += y;
        }
        if (in) {
            const int f = base + x - c;
            list[e] = (int32_t)(e << 2) | mask;
            first[e] = f;
            if (mask & 1) jrow[f] = (int32_t)(2 * e);
            if (mask & 2) jrow[f + (mask & 1)] = (int32_t)(2 * e + 1);
        }
        base += __shfl_sync(0xFFFFFFFFu, x, 31);
    }
}

static int learner_rows_impl(const int32_t *partner_seat, long long n_envs, int32_t *list, int32_t *first, int32_t *jrow, int32_t *range,
                             cudaStream_t st) {
    if (!partner_seat || !list || !first || !jrow || !range) return fail(OVC_E_BADARG, "null pointer argument");
    if (((uintptr_t)partner_seat | (uintptr_t)list | (uintptr_t)first | (uintptr_t)jrow | (uintptr_t)range) & 3)
        return fail(OVC_E_BADARG, "partner_seat, list, first, jrow and range must be 4-byte aligned");
    if (n_envs < 0 || n_envs >= LR_MAX_ENVS) return fail(OVC_E_BADARG, "n_envs must be 0..2^29-1", n_envs);
    if (n_envs == 0) return OVC_OK;
    learner_rows_kernel<<<1, LR_THREADS, 0, st>>>(partner_seat, n_envs, list, first, jrow, range);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "learner_rows kernel launch");
    return OVC_OK;
}

// Per environment e with done[e] (every e with done == NULL): the ending episode's member into the records' slot count[e]
// (when done is given, rec_member non-NULL and count[e] < capacity), then, with thresholds, a new member: Philox4x32-10,
// key = seed, counter = (e low, e high, step low, step high) -> w0;  member[e] = #{k < n_members - 1 : w0 >= thresholds[k]}.
__global__ void __launch_bounds__(256) assign_members_kernel(const int32_t *__restrict__ done, const long long *__restrict__ thresholds,
                                                             int n_members, long long n_envs, unsigned long long seed,
                                                             unsigned long long *counter, int32_t *__restrict__ member,
                                                             int32_t *__restrict__ rec_member, const int32_t *__restrict__ count, int capacity) {
    __shared__ long long thr[MAX_MEMBERS];
    const unsigned long long step = thresholds ? *reinterpret_cast<volatile unsigned long long *>(counter) : 0ull;
    if (thresholds)
        for (int i = threadIdx.x; i < n_members - 1; i += blockDim.x) thr[i] = thresholds[i];
    __syncthreads();
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < n_envs && (!done || done[e] != 0)) {
        if (done && rec_member) {
            const int k = count[e];
            if (k < capacity) rec_member[(long long)k * n_envs + e] = member[e];
        }
        if (thresholds) {
            const Philox4 P = philox4x32_10(seed, (uint32_t)e, (uint32_t)((unsigned long long)e >> 32), (uint32_t)step, (uint32_t)(step >> 32));
            const long long w0 = P.v[0];
            int m = 0;
            for (int k = 0; k < n_members - 1; k++) m += w0 >= thr[k];
            member[e] = m;
        }
    }
    if (thresholds) advance_step(counter, step);
}

static int assign_members_impl(const int32_t *done, const long long *thresholds, int n_members, long long n_envs, unsigned long long seed,
                               unsigned long long *counter, int32_t *member, int32_t *rec_member, const int32_t *count, int capacity,
                               cudaStream_t st) {
    if (!member || (thresholds && !counter) || (rec_member && !count)) return fail(OVC_E_BADARG, "null pointer argument");
    if (((uintptr_t)done | (uintptr_t)member | (uintptr_t)rec_member | (uintptr_t)count) & 3)
        return fail(OVC_E_BADARG, "done, member, rec_member and count must be 4-byte aligned");
    if (((uintptr_t)thresholds | (uintptr_t)counter) & 7) return fail(OVC_E_BADARG, "thresholds and counter must be 8-byte aligned");
    if (n_members < 1 || n_members > MAX_MEMBERS) return fail(OVC_E_BADARG, "n_members must be 1..64", n_members);
    if (capacity < 0) return fail(OVC_E_BADARG, "negative record capacity", capacity);
    if (n_envs < 0) return fail(OVC_E_BADARG, "negative env count");
    if (n_envs == 0) return OVC_OK;
    assign_members_kernel<<<(unsigned)((n_envs + 255) / 256), 256, 0, st>>>(done, thresholds, n_members, n_envs, seed, counter, member,
                                                                           rec_member, count, capacity);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "assign_members kernel launch");
    return OVC_OK;
}

// ---- population play: an ordered pair of learners per environment ----
constexpr int MAX_PAIR_THRESHOLDS = MAX_MEMBERS * MAX_MEMBERS - 1;

// assign_members_kernel for ordered pairs: the ending pair into rec_pair[count[e]][e], then, with thresholds, a new pair.
// The n_members^2 - 1 thresholds of the row-major pair weights are non-decreasing, so #{q : w0 >= thresholds[q]} is an
// upper bound found by binary search (at most 12 cached loads, for done environments only).
__global__ void __launch_bounds__(256) assign_pairs_kernel(const int32_t *__restrict__ done, const long long *__restrict__ thresholds,
                                                           int n_members, long long n_envs, unsigned long long seed,
                                                           unsigned long long *counter, int2 *__restrict__ pair, int2 *__restrict__ rec_pair,
                                                           const int32_t *__restrict__ count, int capacity) {
    const unsigned long long step = thresholds ? *reinterpret_cast<volatile unsigned long long *>(counter) : 0ull;
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < n_envs && (!done || done[e] != 0)) {
        if (done && rec_pair) {
            const int k = count[e];
            if (k < capacity) rec_pair[(long long)k * n_envs + e] = pair[e];
        }
        if (thresholds) {
            const Philox4 P = philox4x32_10(seed, (uint32_t)e, (uint32_t)((unsigned long long)e >> 32), (uint32_t)step, (uint32_t)(step >> 32));
            const long long w0 = P.v[0];
            int lo = 0, hi = n_members * n_members - 1;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (w0 >= __ldg(thresholds + mid)) lo = mid + 1;
                else hi = mid;
            }
            pair[e] = make_int2(lo / n_members, lo % n_members);
        }
    }
    if (thresholds) advance_step(counter, step);
}

static int assign_pairs_impl(const int32_t *done, const long long *thresholds, int n_members, long long n_envs, unsigned long long seed,
                             unsigned long long *counter, int32_t *pair, int32_t *rec_pair, const int32_t *count, int capacity, cudaStream_t st) {
    if (!pair || (thresholds && !counter) || (rec_pair && !count)) return fail(OVC_E_BADARG, "null pointer argument");
    if (((uintptr_t)done | (uintptr_t)count) & 3) return fail(OVC_E_BADARG, "done and count must be 4-byte aligned");
    if (((uintptr_t)pair | (uintptr_t)rec_pair | (uintptr_t)thresholds | (uintptr_t)counter) & 7)
        return fail(OVC_E_BADARG, "pair, rec_pair, thresholds and counter must be 8-byte aligned");
    if (n_members < 1 || n_members > MAX_MEMBERS) return fail(OVC_E_BADARG, "n_members must be 1..64", n_members);
    if (capacity < 0) return fail(OVC_E_BADARG, "negative record capacity", capacity);
    if (n_envs < 0) return fail(OVC_E_BADARG, "negative env count");
    if (n_envs == 0) return OVC_OK;
    assign_pairs_kernel<<<(unsigned)((n_envs + 255) / 256), 256, 0, st>>>(done, thresholds, n_members, n_envs, seed, counter, (int2 *)pair,
                                                                         (int2 *)rec_pair, count, capacity);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "assign_pairs kernel launch");
    return OVC_OK;
}

// The pairs grouped by member: group_members_kernel's stable counting sort in ONE CTA, over the 2 n_envs items (e, s) in
// index order 2 e + s.  Item (e, 0) is the entry of member pair[e][0]: e << 2 | 3 (two rows) where pair[e] = (i, i), else
// e << 2 | 1 (view 0); item (e, 1) is the entry e << 2 | 2 (view 1) of member pair[e][1], or nothing where the pair is a
// self-play one.  An environment has at most one entry per member, so each group is ascending in e.  Warps count entries
// and rows per member (warp-private histograms), 64 threads and then one thread turn them into starts, and every warp
// walks its segment 32 items at a time: lanes of one member find each other with __match_any_sync and take consecutive
// entries in lane order, their rows after the earlier lanes' rows (a self-play entry holds two).
__global__ void __launch_bounds__(GM_THREADS, 1) group_pairs_kernel(const int32_t *__restrict__ pair, int n_members, long long n_envs,
                                                                    int32_t *__restrict__ list, int32_t *__restrict__ first,
                                                                    int32_t *__restrict__ jrow, int32_t *__restrict__ entry_offsets,
                                                                    int32_t *__restrict__ row_offsets) {
    constexpr int NW = GM_THREADS / 32;
    __shared__ int hent[NW][MAX_MEMBERS], hrow[NW][MAX_MEMBERS];
    __shared__ int tent[MAX_MEMBERS], trow[MAX_MEMBERS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < NW * MAX_MEMBERS; i += GM_THREADS) (&hent[0][0])[i] = 0, (&hrow[0][0])[i] = 0;
    __syncthreads();
    const long long n_items = 2 * n_envs;
    const long long seg = (n_items + NW - 1) / NW;
    const long long beg = warp * seg, end = beg + seg < n_items ? beg + seg : n_items;
    // item v's member (-1: no entry) and its row count
    auto item = [&](long long v, int &rows) {
        const int2 p = __ldg(reinterpret_cast<const int2 *>(pair) + (v >> 1));
        rows = (v & 1) == 0 && p.x == p.y ? 2 : 1;
        return (v & 1) == 0 ? p.x : (p.x == p.y ? -1 : p.y);
    };
    for (long long v = beg + lane; v < end; v += 32) {
        int rows;
        const int k = item(v, rows);
        if (k >= 0) atomicAdd(&hent[warp][k], 1), atomicAdd(&hrow[warp][k], rows);
    }
    __syncthreads();
    if (threadIdx.x < MAX_MEMBERS) {  // thread k: member k's start in every segment, relative to the group's start
        const int k = threadIdx.x;
        int te = 0, tr = 0;
        for (int w = 0; w < NW; w++) {
            const int ce = hent[w][k], cr = hrow[w][k];
            hent[w][k] = te, hrow[w][k] = tr;
            te += ce, tr += cr;
        }
        tent[k] = te, trow[k] = tr;
    }
    __syncthreads();
    if (threadIdx.x == 0) {  // the group starts: exclusive scans of the totals
        int re = 0, rr = 0;
        for (int k = 0; k < n_members; k++) {
            const int ce = tent[k], cr = trow[k];
            tent[k] = re, trow[k] = rr;
            re += ce, rr += cr;
        }
        entry_offsets[n_members] = re, row_offsets[n_members] = rr;
    }
    __syncthreads();
    if (threadIdx.x < n_members) {
        const int k = threadIdx.x, be = tent[k], br = trow[k];
        entry_offsets[k] = be, row_offsets[k] = br;
        for (int w = 0; w < NW; w++) hent[w][k] += be, hrow[w][k] += br;
    }
    __syncthreads();
    const unsigned lt = (1u << lane) - 1u;
    for (long long v0 = beg; v0 < end; v0 += 32) {
        const long long v = v0 + lane;
        int rows = 0;
        int k = v < end ? item(v, rows) : -1;
        const bool in = k >= 0;
        if (!in) k = -1 - lane;  // lanes without an entry match nobody
        const unsigned peers = __match_any_sync(0xFFFFFFFFu, k);
        const unsigned twos = __ballot_sync(0xFFFFFFFFu, in && rows == 2);
        const int slot = in ? hent[warp][k] + __popc(peers & lt) : 0;
        const int row = in ? hrow[warp][k] + __popc(peers & lt) + __popc(peers & twos & lt) : 0;
        __syncwarp();
        if (in) {
            const long long e = v >> 1;
            const int mask = rows == 2 ? 3 : (v & 1) ? 2 : 1;
            list[slot] = (int32_t)(e << 2) | mask;
            first[slot] = row;
            jrow[row] = (int32_t)(2 * e + (mask == 2));
            if (mask == 3) jrow[row + 1] = (int32_t)(2 * e + 1);
            if ((peers & lt) == 0) hent[warp][k] += __popc(peers), hrow[warp][k] += __popc(peers) + __popc(peers & twos);
        }
        __syncwarp();
    }
}

static int group_pairs_impl(const int32_t *pair, int n_members, long long n_envs, int32_t *list, int32_t *first, int32_t *jrow,
                            int32_t *entry_offsets, int32_t *row_offsets, cudaStream_t st) {
    if (!pair || !list || !first || !jrow || !entry_offsets || !row_offsets) return fail(OVC_E_BADARG, "null pointer argument");
    if ((uintptr_t)pair & 7) return fail(OVC_E_BADARG, "pair must be 8-byte aligned");
    if (((uintptr_t)list | (uintptr_t)first | (uintptr_t)jrow | (uintptr_t)entry_offsets | (uintptr_t)row_offsets) & 3)
        return fail(OVC_E_BADARG, "list, first, jrow, entry_offsets and row_offsets must be 4-byte aligned");
    if (n_members < 1 || n_members > MAX_MEMBERS) return fail(OVC_E_BADARG, "n_members must be 1..64", n_members);
    if (n_envs < 0 || n_envs >= LR_MAX_ENVS) return fail(OVC_E_BADARG, "n_envs must be 0..2^29-1", n_envs);
    if (n_envs == 0) return OVC_OK;
    group_pairs_kernel<<<1, GM_THREADS, 0, st>>>(pair, n_members, n_envs, list, first, jrow, entry_offsets, row_offsets);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "group_pairs kernel launch");
    return OVC_OK;
}

}  // namespace ovc
