/*
 * ovc_greedy.h — C ABI of the greedy scripted partner (csrc/libovc_greedy.so): the reference's GreedyHumanModel
 * (src/overcooked_ai_py/agents/agent.py) with its defaults, under MediumLevelActionManager(mdp, NO_COUNTERS_PARAMS),
 * one thread per environment.
 *
 * The library reads the packed records and the layout tables of include/ovc_b200.h; its conventions are that header's:
 * `extern "C"`, device pointers owned by the caller, `stream` a cudaStream_t passed as void*, 0 on success or a negative
 * OVC_E_* code with a message from ovc_greedy_last_error().  Launches are asynchronous.
 *
 * Per layout, a table (ovc_greedy_layout_t, built by overcooked_ai_b200/greedy.py) and a plan block:
 *   node          4 * i + o: floor cell i (free_index[pos byte], row-major order) facing orientation o (N, S, E, W)
 *   plan          uint16 [n_nodes][n_nodes] at plans + plan_offset: entry [s][g] = (cost << 3) | first action of
 *                 MotionPlanner.get_plan(s, g), cost = path length + 1 (the final INTERACT), OVC_GREEDY_UNREACHABLE
 *                 where g is not reachable from s
 *   goal lists    goal[list_start[k] .. list_start[k + 1]): the motion goals (nodes) of list k's feature cells, features
 *                 in row-major order, each feature's goals in N, S, E, W order of the side they lie on
 *   partial_order the pots' slots in the order get_partially_full_pots lists them, per assignment of pots to classes
 *                 (row sum_k class_k * 3^k; class 1 / 2: one / two ingredients, idle), OVC_NO_SLOT after the last
 */
#ifndef OVC_GREEDY_H
#define OVC_GREEDY_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OVC_GREEDY_ABI_VERSION 1

#define OVC_GREEDY_UNREACHABLE 0xFFFF
#define OVC_GREEDY_MAX_GOALS 1024
/* goal lists */
#define OVC_GREEDY_LIST_ONION 0   /* onion dispensers */
#define OVC_GREEDY_LIST_DISH 1    /* dish dispensers */
#define OVC_GREEDY_LIST_SERVE 2   /* serving cells */
#define OVC_GREEDY_LIST_CLOSEST 3 /* go_to_closest_feature_actions: onion, tomato dispensers, pots, dish dispensers */
#define OVC_GREEDY_LIST_POT 4     /* + k: pot k */
#define OVC_GREEDY_LISTS 8

typedef struct ovc_greedy_layout {
    int32_t n_nodes;     /* 4 * floor cells, <= 512 */
    int32_t plan_offset; /* index of this layout's plan entry [0][0] in the plans array */
    uint16_t list_start[OVC_GREEDY_LISTS + 1];
    uint16_t reserved[3];
    uint8_t free_index[256];        /* pos byte -> floor cell index, 0xFF elsewhere */
    uint8_t partial_order[81][4];
    uint16_t goal[OVC_GREEDY_MAX_GOALS];
} ovc_greedy_layout_t;

int ovc_greedy_abi_version(void);
size_t ovc_greedy_layout_table_size(void);
const char *ovc_greedy_last_error(void);

/*
 * ovc_greedy_actions: for every environment e with player[e] in {0, 1} (int32 [n_envs]; -1 = the agent does not play e),
 * GreedyHumanModel.action of player player[e] on state[e], written to actions[e * 2 + player[e]] (int32 [n_envs, 2]);
 * other entries are left alone.
 *   ml_action        empty-handed: the dish dispensers when a pot is cooking or ready and the other player holds no dish,
 *                    else the idle pots with three ingredients, else the onion dispensers; holding an onion or a tomato:
 *                    the partially full pots (set order), then the empty pots; a dish: the ready, then the cooking pots;
 *                    a soup: the serving cells.  Goals not reachable from the player's node are dropped; with none left,
 *                    the goals of go_to_closest_feature_actions.  Counters are never goals (NO_COUNTERS_PARAMS).
 *   the action       the first action of the cheapest plan, the first goal of the list winning a tie; STAY if no goal.
 *   auto_unstuck     prev[e] (int32 [n_envs], read and written): bit 20 set = valid, bits 0-9 / 10-19 = player 0 / 1's
 *                    pos byte and orientation at the previous call.  It is invalid where done[e] != 0 (int32 [n_envs],
 *                    the previous ovc_step's done, nullable) and where player[e] < 0, like Agent.reset().  Where it is
 *                    valid and equals the current key, the step is stuck: the action is drawn uniformly from the moves
 *                    N, S, E, W into a floor cell the other player does not hold (STAY if none), with Philox4x32-10,
 *                    key = seed, counter (row lo, row hi, step lo, step hi) on the joint row 2 e + player[e] (two
 *                    greedy agents of one environment draw apart), index = mulhi(word 0, count).
 *   counter          uint64 [2]: counter[0] = the step, advanced by one per call (counter[1] is the launch's scratch,
 *                    zero between calls), so a captured CUDA graph draws fresh numbers at every replay.
 * layouts: ovc_layout_t [n_layouts] (include/ovc_b200.h), greedy: ovc_greedy_layout_t [n_layouts], plans: uint16.
 * The layout id of a record is word 3's low byte.  state 16-byte aligned, S in {16, 32, 64, 128}.
 */
int ovc_greedy_actions(const void *layouts, const void *greedy, const uint16_t *plans, int n_layouts, const int32_t *state,
                       const int32_t *player, const int32_t *done, int32_t *prev, int64_t n_envs, int state_words, uint64_t seed,
                       uint64_t *counter, int32_t *actions, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* OVC_GREEDY_H */
