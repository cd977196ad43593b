// ovc_greedy.cu — the reference's GreedyHumanModel (agents/agent.py: action, ml_action, get_lowest_cost_action_and_goal,
// auto_unstuck) on the device, one thread per environment; the C ABI and the table format are in include/ovc_greedy.h.
// The motion plans are table lookups (overcooked_ai_b200/greedy.py builds them once per layout), so a step is the choice
// of a goal list from the pots and the held objects and an argmin over at most a few dozen plan entries.
#include <cuda_runtime.h>
#include <stdio.h>

#include "../../include/ovc_b200.h"
#include "../../include/ovc_greedy.h"
#include "ovc_rng.cuh"

namespace ovc {

static thread_local char g_greedy_err[512] = "";

static int greedy_fail(int code, const char *msg, long long value = 0) {
    snprintf(g_greedy_err, sizeof g_greedy_err, "%s (%lld)", msg, value);
    return code;
}

struct GreedyArgs {
    const ovc_layout_t *layouts;
    const ovc_greedy_layout_t *greedy;
    const uint16_t *plans;
    const int32_t *state, *player, *done;
    int32_t *prev;
    long long n_envs;
    int S;
    unsigned long long seed;
    unsigned long long *counter;
    int32_t *actions;
};

constexpr int GREEDY_THREADS = 128;

// The first cheapest goal of list [b, e) from node `start`: strict <, as get_lowest_cost_action_and_goal.  best / act carry
// the running minimum across calls, so consecutive lists act as one list.
__device__ __forceinline__ void argmin_goals(const ovc_greedy_layout_t &g, const uint16_t *plan_row, int b, int e, unsigned &best,
                                             int &act) {
    for (int i = b; i < e; i++) {
        const unsigned ent = __ldg(plan_row + g.goal[i]);
        if (ent != OVC_GREEDY_UNREACHABLE && (ent >> 3) < best) best = ent >> 3, act = (int)(ent & 7);
    }
}

__global__ void __launch_bounds__(GREEDY_THREADS) greedy_actions_kernel(GreedyArgs a) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long step = *(volatile unsigned long long *)a.counter;
    if (e < a.n_envs) {
        const int p = a.player[e];
        const int32_t *rec = a.state + e * a.S;
        const uint32_t w0 = (uint32_t)rec[1], w1 = (uint32_t)rec[2];
        const int32_t prev = a.prev[e];
        const bool valid = p >= 0 && (prev >> 20) == 1 && !(a.done && a.done[e]);
        const int32_t key = (int32_t)((w0 & 0x3FF) | ((w1 & 0x3FF) << 10) | (1u << 20));
        a.prev[e] = p >= 0 ? key : 0;
        if (p >= 0) {
            const int lid = rec[3] & 0xFF;
            const ovc_layout_t &L = a.layouts[lid];
            const ovc_greedy_layout_t &G = a.greedy[lid];
            const uint32_t me = p ? w1 : w0, other = p ? w0 : w1;
            int act = OVC_A_STAY;
            if (valid && key == prev) {  // stuck: a random move that unblocks, were the other player to stay
                const int x = me & 15, y = (me >> 4) & 15, opos = other & 0xFF;
                int moves[4], n = 0;
#pragma unroll
                for (int d = 0; d < 4; d++) {
                    const int nx = x + (d == 2) - (d == 3), ny = y + (d == 1) - (d == 0);
                    if (nx < 0 || ny < 0 || nx > 15 || ny > 15) continue;
                    const int q = (ny << 4) | nx;
                    if ((L.cell[q] & 7) == OVC_T_FLOOR && q != opos) moves[n++] = d;
                }
                if (n) {
                    const unsigned long long row = 2ull * (unsigned long long)e + (unsigned long long)p;
                    const Philox4 r = philox4x32_10(a.seed, (uint32_t)row, (uint32_t)(row >> 32), (uint32_t)step, (uint32_t)(step >> 32));
                    act = moves[mulhi32(r.v[0], (uint32_t)n)];
                }
            } else {
                // the pots: 0 empty, 1 / 2 / 3 idle with that many ingredients, 4 cooking, 5 ready
                int cls[OVC_MAX_POTS], partial_code = 0, pow3 = 1;
                bool any_hot = false, any_full = false;
                for (int k = 0; k < L.n_pots; k++, pow3 *= 3) {
                    const uint32_t code = (uint32_t)rec[4 + k] & OVC_OBJ_MASK;
                    int c = 0;
                    if ((code & 7) == OVC_O_SOUP) {
                        const int n = (code >> 3) & 3, n_tom = __popc((code >> 5) & ((1u << n) - 1u));
                        const int tick = (int)((code >> 8) & 0x3FFF) - 1;
                        c = tick < 0 ? n : (tick >= L.cook_time[(n - n_tom) * 4 + n_tom] ? 5 : 4);
                    }
                    cls[k] = c;
                    any_hot |= c >= 4;
                    any_full |= c == 3;
                    if (c == 1 || c == 2) partial_code += c * pow3;
                }
                const int start = 4 * G.free_index[me & 0xFF] + ((me >> 8) & 3);
                const uint16_t *row = a.plans + G.plan_offset + (long long)start * G.n_nodes;
                unsigned best = 0xFFFFFFFFu;
                const int held = (me >> 10) & 7;
                auto list = [&](int k) { argmin_goals(G, row, G.list_start[k], G.list_start[k + 1], best, act); };
                auto pots = [&](int c) {
                    for (int k = 0; k < L.n_pots; k++)
                        if (cls[k] == c) list(OVC_GREEDY_LIST_POT + k);
                };
                if (held == OVC_O_NONE) {
                    if (any_hot && ((other >> 10) & 7) != OVC_O_DISH) list(OVC_GREEDY_LIST_DISH);
                    else if (any_full) pots(3);
                    else list(OVC_GREEDY_LIST_ONION);
                } else if (held == OVC_O_ONION || held == OVC_O_TOMATO) {
                    for (int j = 0; j < OVC_MAX_POTS; j++) {
                        const int slot = G.partial_order[partial_code][j];
                        if (slot == OVC_NO_SLOT) break;
                        list(OVC_GREEDY_LIST_POT + slot);  // pots are slots 0 .. n_pots - 1
                    }
                    pots(0);
                } else if (held == OVC_O_DISH) {
                    pots(5), pots(4);
                } else {
                    list(OVC_GREEDY_LIST_SERVE);
                }
                if (best == 0xFFFFFFFFu) list(OVC_GREEDY_LIST_CLOSEST);
            }
            a.actions[2 * e + p] = act;
        }
    }
    // the last CTA to get here advances the step (every CTA has read it by then)
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned long long arrived = atomicAdd(a.counter + 1, 1ull);
        if (arrived == (unsigned long long)gridDim.x - 1) {
            a.counter[1] = 0;
            a.counter[0] = step + 1;
            __threadfence();
        }
    }
}

}  // namespace ovc

extern "C" {

int ovc_greedy_abi_version(void) { return OVC_GREEDY_ABI_VERSION; }

size_t ovc_greedy_layout_table_size(void) { return sizeof(ovc_greedy_layout_t); }

const char *ovc_greedy_last_error(void) { return ovc::g_greedy_err; }

int ovc_greedy_actions(const void *layouts, const void *greedy, const uint16_t *plans, int n_layouts, const int32_t *state,
                       const int32_t *player, const int32_t *done, int32_t *prev, int64_t n_envs, int state_words, uint64_t seed,
                       uint64_t *counter, int32_t *actions, void *stream) {
    using ovc::greedy_fail;
    if (!layouts || !greedy || !plans || !state || !player || !prev || !counter || !actions)
        return greedy_fail(OVC_E_BADARG, "null pointer argument");
    if (n_layouts <= 0 || n_layouts > 256) return greedy_fail(OVC_E_BADARG, "n_layouts must be 1..256", n_layouts);
    if (n_envs < 0) return greedy_fail(OVC_E_BADARG, "negative n_envs", (long long)n_envs);
    if (state_words != 16 && state_words != 32 && state_words != 64 && state_words != 128)
        return greedy_fail(OVC_E_BADARG, "state_words must be 16, 32, 64 or 128", state_words);
    if (((uintptr_t)state & 15) || ((uintptr_t)player & 3) || ((uintptr_t)prev & 3) || ((uintptr_t)actions & 3) ||
        ((uintptr_t)done & 3) || ((uintptr_t)counter & 7) || ((uintptr_t)plans & 1) || ((uintptr_t)greedy & 3))
        return greedy_fail(OVC_E_BADARG, "arrays must be aligned to their element size (state to 16 bytes)");
    if (n_envs == 0) return OVC_OK;
    const long long blocks = (n_envs + ovc::GREEDY_THREADS - 1) / ovc::GREEDY_THREADS;
    if (blocks > 0x7FFFFFFFLL) return greedy_fail(OVC_E_BADARG, "n_envs too large for one launch", (long long)n_envs);
    ovc::GreedyArgs a;
    a.layouts = (const ovc_layout_t *)layouts, a.greedy = (const ovc_greedy_layout_t *)greedy, a.plans = plans;
    a.state = state, a.player = player, a.done = done, a.prev = prev, a.n_envs = n_envs, a.S = state_words;
    a.seed = seed, a.counter = (unsigned long long *)counter, a.actions = actions;
    ovc::greedy_actions_kernel<<<(unsigned)blocks, ovc::GREEDY_THREADS, 0, (cudaStream_t)stream>>>(a);
    const cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) return greedy_fail(OVC_E_CUDA, cudaGetErrorString(err));
    return OVC_OK;
}

}  // extern "C"
