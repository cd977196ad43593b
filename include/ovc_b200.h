/*
 * ovc_b200.h — C ABI of the H100-native (sm_90a) batched Overcooked MDP step engine.
 *
 * The reference (HumanCompatibleAI/overcooked_ai) is pure Python and has no FFI layer; the
 * boundary this library replaces is the Python call surface
 *
 *   OvercookedGridworld.get_state_transition   src/overcooked_ai_py/mdp/overcooked_mdp.py:1375-1430
 *   OvercookedEnv.step / reset / is_done       src/overcooked_ai_py/mdp/overcooked_env.py:244-325
 *   OvercookedGridworld.lossless_state_encoding  overcooked_mdp.py:2385-2561
 *   OvercookedGridworld.featurize_state          overcooked_mdp.py:2579-2898
 *
 * Every entry point is `extern "C"`, takes plain pointers and sizes, allocates nothing that
 * outlives the call and never throws.  All `state`, `actions`, output and table pointers are
 * DEVICE pointers owned by the caller (torch owns every buffer); `stream` is a cudaStream_t
 * passed as void*.  Return value: 0 on success, a negative OVC_E_* code otherwise, with a
 * human-readable message available from ovc_last_error().  Launches are asynchronous: device
 * faults surface at the caller's next synchronisation.
 *
 * ---------------------------------------------------------------------------------------------
 * Packed environment record (int32 words, `state_words` S in {16, 32, 64, 128} per record,
 * records contiguous: state[env * S + word]).
 *
 *   word 0        timestep                                   (OvercookedState.timestep, :814)
 *   word 1, 2     player 0 / player 1                        (PlayerState, :696-781)
 *                   bits 0-3  x      bits 4-7  y             (bits 0-7 = "pos byte" y<<4|x)
 *                   bits 8-9  orientation index  0 N, 1 S, 2 E, 3 W   (actions.py:12-17)
 *                   bits 10-31 held object, 22-bit object code (0 = empty hands)
 *   word 3        bits 0-7   layout id (index into the layout table)
 *                 bits 8-15  number of loose dishes on counters (derived cache, kept by every
 *                            kernel; pack() computes it)
 *                 bits 16-31 episode counter of the random-start generator (0 unless random starts are used);
 *                            it is part of the Philox counter and wraps after 65 536 episodes of an environment, after
 *                            which that environment's start-state sequence repeats (change the seed to move on)
 *   word 4+k      object on object-capable cell k, 22-bit object code (0 = empty).
 *                 Cells are ordered: the layout's pots (terrain row-major order, = the order of
 *                 get_pot_locations(), :1799) first, then its counters 'X' (row-major).
 *   remaining     zero padding up to S
 *
 * 22-bit object code (ObjectState :384-430, SoupState :433-693)
 *   bits 0-2   type: 0 none, 1 onion, 2 tomato, 3 dish, 4 soup
 *   bits 3-4   soup: number of ingredients (0..3)
 *   bits 5-7   soup: ingredient kinds in insertion order, bit (5+i) = 1 if slot i is a tomato
 *              (ordered, because SoupState.__eq__ :458-472 is order sensitive)
 *   bits 8-21  soup: _cooking_tick + 1   (0 = idle, i.e. _cooking_tick == -1)
 * ---------------------------------------------------------------------------------------------
 */
#ifndef OVC_B200_H
#define OVC_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OVC_ABI_VERSION 5

/* ---- action indices: Action.INDEX_TO_ACTION, actions.py:47-57 ---- */
#define OVC_A_NORTH 0
#define OVC_A_SOUTH 1
#define OVC_A_EAST 2
#define OVC_A_WEST 3
#define OVC_A_STAY 4
#define OVC_A_INTERACT 5
#define OVC_NUM_ACTIONS 6

/* ---- terrain codes (low 3 bits of ovc_layout_t.cell[]) ---- */
#define OVC_T_FLOOR 0   /* ' ' */
#define OVC_T_COUNTER 1 /* 'X' */
#define OVC_T_ONION 2   /* 'O' */
#define OVC_T_TOMATO 3  /* 'T' */
#define OVC_T_DISH 4    /* 'D' */
#define OVC_T_POT 5     /* 'P' */
#define OVC_T_SERVE 6   /* 'S' */
#define OVC_T_OUTSIDE 7 /* not part of the grid */

/* ---- object codes ---- */
#define OVC_O_NONE 0
#define OVC_O_ONION 1
#define OVC_O_TOMATO 2
#define OVC_O_DISH 3
#define OVC_O_SOUP 4

#define OVC_OBJ_BITS 22
#define OVC_OBJ_MASK 0x3FFFFF
#define OVC_MAX_TICK 16382 /* tick+1 must fit 14 bits */

/* ---- event bits: index = position in EVENT_TYPES, overcooked_mdp.py:1027-1058 ---- */
#define OVC_EV_TOMATO_PICKUP 0
#define OVC_EV_USEFUL_TOMATO_PICKUP 1
#define OVC_EV_TOMATO_DROP 2
#define OVC_EV_USEFUL_TOMATO_DROP 3
#define OVC_EV_POTTING_TOMATO 4
#define OVC_EV_ONION_PICKUP 5
#define OVC_EV_USEFUL_ONION_PICKUP 6
#define OVC_EV_ONION_DROP 7
#define OVC_EV_USEFUL_ONION_DROP 8
#define OVC_EV_POTTING_ONION 9
#define OVC_EV_DISH_PICKUP 10
#define OVC_EV_USEFUL_DISH_PICKUP 11
#define OVC_EV_DISH_DROP 12
#define OVC_EV_USEFUL_DISH_DROP 13
#define OVC_EV_SOUP_PICKUP 14
#define OVC_EV_SOUP_DELIVERY 15
#define OVC_EV_SOUP_DROP 16
#define OVC_EV_OPTIMAL_ONION_POTTING 17
#define OVC_EV_OPTIMAL_TOMATO_POTTING 18
#define OVC_EV_VIABLE_ONION_POTTING 19
#define OVC_EV_VIABLE_TOMATO_POTTING 20
#define OVC_EV_CATASTROPHIC_ONION_POTTING 21
#define OVC_EV_CATASTROPHIC_TOMATO_POTTING 22
#define OVC_EV_USELESS_ONION_POTTING 23
#define OVC_EV_USELESS_TOMATO_POTTING 24
#define OVC_NUM_EVENTS 25
/* events[env][agent] bits 25-28: recipe index (n_onion*4+n_tomato) of the soup this agent
 * delivered in this transition (0 if none) — lets the host attribute sparse reward per agent.
 * bit 30: OVC_EVF_STEPPED_DONE, the env was already done (timestep >= horizon) and was left
 * untouched (the reference raises AssertionError there, overcooked_env.py:255). */
#define OVC_EV_RECIPE_SHIFT 25
#define OVC_EVF_STEPPED_DONE (1 << 30)

/* ---- layout constant table: one record per layout, device resident, read only ---- */
#define OVC_LAYOUT_OLD_DYNAMICS 1 /* flags bit 0, overcooked_mdp.py:1121-1127,1515-1522,1696-1701 */
#define OVC_MAX_POTS 4
#define OVC_MAX_SLOTS 124
#define OVC_NO_SLOT 0xFF

typedef struct ovc_layout {
    int32_t width, height;
    int32_t n_pots;  /* <= OVC_MAX_POTS */
    int32_t n_slots; /* pots + counters, <= OVC_MAX_SLOTS */
    int32_t flags;
    int32_t rew_placement_in_pot; /* reward_shaping_params, overcooked_mdp.py:1018-1025,1136-1140 */
    int32_t rew_dish_pickup;
    int32_t rew_soup_pickup;
    int32_t state_words; /* smallest supported S that holds this layout */
    int32_t n_free;      /* number of floor cells (valid player positions) */
    int32_t reserved[6];
    /* recipe tables, index r = n_onion*4 + n_tomato (r == 0: empty pot) */
    int32_t cook_time[16];     /* Recipe.time, :163-188 */
    int32_t deliver_value[16]; /* get_recipe_value, :1581-1602 (bonus and all_orders applied) */
    int32_t best_value[16];    /* value of get_optimal_possible_recipe, :1976-2061 */
    /* cell[y<<4|x]: bits 0-2 terrain code, bits 8-15 object slot (OVC_NO_SLOT if none) */
    uint16_t cell[256];
    uint8_t slot_pos[128]; /* slot -> pos byte */
    uint8_t free_pos[128]; /* floor cells in terrain row-major order (get_valid_player_positions, :1733) */
} ovc_layout_t;           /* 1024 bytes */

/* ---- per-(layout, cell, orientation) lookup for featurize_state; see ovc_featurize ---- */
typedef struct ovc_feat_lut_entry {
    int8_t d_onion[2]; /* (dx,dy) to the closest onion dispenser by planner cost, (0,0) if none */
    int8_t d_tomato[2];
    int8_t d_dish[2];
    int8_t d_serve[2];
    uint8_t pot_order[OVC_MAX_POTS]; /* pot slots by increasing planner cost; 0xFF = unreachable */
} ovc_feat_lut_entry_t;              /* 12 bytes; table is [n_layouts][256][4] */

/* ---- potential_function constants (overcooked_mdp.py:2920-3250), one per layout, for ONE gamma ---- */
typedef struct ovc_potential {
    double steady;         /* steady-state term, :2985-2999 */
    double disc_value[16]; /* discounted value of the best recipe reachable from recipe r (r == 0: empty), :1976-2061 */
    int32_t opt_recipe[16]; /* that recipe's index (the DFS order of the reference decides ties) */
    int32_t max_delivery_steps, max_pickup_steps, pot_onion_steps, pot_tomato_steps; /* POTENTIAL_CONSTANTS :1060-1073 */
    int32_t onion_value, tomato_value;                                              /* :2975-2978 */
    int32_t reserved[2];
    /* iteration order of list(set().union(one_item_pots, two_item_pots)) (:1882-1890) for every assignment of
     * pots to {not partial, 1 item, 2 items}: index = sum class_k * 3^k, entries = pot slots, 0xFF ends */
    uint8_t partial_order[81][4];
    uint8_t pad[4];
} ovc_potential_t; /* 560 bytes */

/* planner costs per (layout, cell, orientation): MotionPlanner.min_cost_to_feature (planners.py:391-423) to
 * the serving cells and to each pot; 255 = unreachable.  Table is [n_layouts][256][4]. */
typedef struct ovc_cost_lut_entry {
    uint8_t serve;
    uint8_t pot[OVC_MAX_POTS];
    uint8_t pad[3];
} ovc_cost_lut_entry_t; /* 8 bytes */
#define OVC_COST_INF 255

/* ---- random start states: get_random_start_state_fn (overcooked_mdp.py:1307-1369) ----
 * The reference draws from numpy's global generator, which a device engine cannot reproduce; the engine
 * uses Philox4x32-10 keyed by `seed`, counter (env index, episode counter, draw block), mirrored bit for
 * bit by the CPU oracle.  Draw plan per reset: block 0 = {joint position, p0 holds?, p0 object, p0 n},
 * block 1 = {p0 m, p1 holds?, p1 object, p1 n}, block 2 = {p1 m, -, -, -}, block 3+k = pot k {filled?, n, m,
 * cooking?}.  "u < p" is `draw < threshold` with threshold = p * 2^32, saturated at 0xFFFFFFFF which means ALWAYS
 * (p = 1.0); randint(lo, hi) is lo + mulhi(draw, hi-lo);
 * the object is a dish / onion / soup with probability 0.2 / 0.6 / 0.2 (:1351-1353), a held soup is finished,
 * a pot soup has n in 1..3 onions then m in 0..3-n tomatoes and is cooking (tick 0) or idle.
 * Variable MDP (OvercookedEnv.reset(regen_mdp=True) with a generator over num_mdp > 1 layouts, overcooked_env.py:
 * 288-302): with `random_layout` every (auto-)reset first redraws the environment's layout uniformly from the
 * n_layouts of the table, id = mulhi(block 2 word 1, n_layouts) of the NEW episode, and then builds the start
 * state (standard or random, as the other fields say) on that layout.
 * Passed by HOST pointer (NULL = standard start states). */
typedef struct ovc_random_start {
    uint64_t seed;
    uint32_t obj_threshold;   /* rnd_obj_prob_thresh * 2^32 (0: no random objects, as :1325-1326) */
    int32_t random_start_pos; /* non-zero: a uniformly drawn ordered pair of distinct floor cells (:1311-1315) */
    int32_t random_layout;    /* non-zero: redraw the layout id at every reset (variable MDP) */
    int32_t reserved;
} ovc_random_start_t; /* 24 bytes */

/* ---- error codes ---- */
#define OVC_OK 0
#define OVC_E_BADARG (-1)
#define OVC_E_CUDA (-2)
#define OVC_E_UNSUPPORTED (-3)

/* flags for ovc_step / ovc_rollout */
#define OVC_F_AUTO_RESET 1 /* an env whose new timestep reaches horizon is set back to its start record */
/* launch the step kernel with programmatic dependent launch (stream serialization attribute): its
 * prologue (barrier init, layout-table fetch) overlaps the tail of the previous kernel in the stream;
 * every read of state / actions happens after griddepcontrol.wait, so results are unchanged. */
#define OVC_F_PDL 2
/* narrow host-transfer formats (same values, fewer bytes over PCIe: 15 instead of 32 per env-step):
 *   OVC_F_ACT_U8      `actions` is uint8[..][2] instead of int32[..][2]
 *   OVC_F_OUT_NARROW  `sparse` is int16[..], `shaped` is int8[..][2], `done` is uint8[..]; `events` stays
 *                     int32[..][2].  The host must make sure the layout's rewards fit (the Python layer
 *                     checks deliver_value <= 32767 and shaping rewards <= 127 before it sets the flag). */
#define OVC_F_ACT_U8 4
#define OVC_F_OUT_NARROW 8
/*   OVC_F_OUT_PACKED  (6 bytes per env-step) `sparse` int16[..], `shaped` int8[..][2], `events` is uint16[..]
 *                     holding both agents' event CODES, `done` is not written (may be NULL):
 *                       bits 0-4 agent 0 code, bits 5-9 agent 1 code, bit 10 done, bit 11 stepped-a-finished-env.
 *                     An agent produces at most one interaction per transition, so its 25 event bits + delivered
 *                     recipe take one of 32 values:
 *                       0 nothing | 1,2 onion_pickup (useful) | 3,4 tomato_pickup | 5,6 dish_pickup | 7 soup_pickup
 *                       8,9 onion_drop (useful) | 10,11 tomato_drop | 12,13 dish_drop | 14 soup_drop
 *                       15-18 potting_onion, 19-22 potting_tomato: + {0 optimal+viable, 1 viable, 2 catastrophic,
 *                       3 optimal+useless} | 23-31 soup_delivery of the recipe with rank 0..8 in the order
 *                       (n_onion,n_tomato) = (0,1),(0,2),(0,3),(1,0),(1,1),(1,2),(2,0),(2,1),(3,0)  [index n_onion*4+n_tomato ascending]
 *                     The host expands codes back to the int32 masks with a 32-entry table (wire.decode_event_codes). */
#define OVC_F_OUT_PACKED 16
/*   OVC_F_OUT_CODES   (2 bytes per env-step) only `events` is written, as uint16[..] (`sparse`, `shaped`, `done` may be
 *                     NULL): the OVC_F_OUT_PACKED word plus bit 12 / bit 13 = agent 0 / agent 1 received a shaped
 *                     reward in this transition.  Nothing is lost: an agent's rewards are functions of its code,
 *                     that bit and the layout — sparse = deliver_value[recipe of codes 23-31]; shaped =
 *                     PLACEMENT_IN_POT_REW for codes 15-22, DISH_PICKUP_REWARD for code 6 and SOUP_PICKUP_REWARD for
 *                     code 7 when the bit is set (a dish / soup taken from a COUNTER logs the same event without
 *                     the reward, hence the bit).  ovc_expand_codes_host rebuilds the dense arrays on the host.
 *   OVC_F_ACT_PACKED  `actions` is uint8[..]: agent 0's action index in bits 0-3, agent 1's in bits 4-7. */
#define OVC_F_OUT_CODES 32
#define OVC_F_ACT_PACKED 64
/*   OVC_F_OUT_STREAM  (ovc_rollout and the pipeline) the result as a SPARSE EVENT STREAM — what a rollout produces is mostly
 *                     zeros, so only the non-zero OVC_F_OUT_CODES words travel.  With G = ceil(n_envs / 32) groups of 32
 *                     consecutive environments (one warp each):
 *                       `events`  uint32[n_steps][G]  lane masks: bit l of [t][g] set = environment 32 g + l produced a
 *                                 non-zero code word in transition t (one __ballot_sync per warp and transition);
 *                       `sparse`  uint16[G][cap]      the group's non-zero words in (transition, lane) order; cap (words per
 *                                 group and launch) travels in flags bits 16-31 (OVC_F_STREAM_CAP_SHIFT).  Words beyond
 *                                 cap are dropped; the masks still count them, so the reader sees the overflow;
 *                       `done`    uint16[n_steps][n_envs] or NULL: the dense code words as well (device-side backup that
 *                                 makes an overflow recoverable; never copied to the host by the pipeline);
 *                       `shaped`  unused (may be NULL).
 *                     Lossless for every group whose word count stays within cap.  Combines with OVC_F_ACT_U8 / _PACKED.
 *                     ovc_expand_stream_host rebuilds dense arrays on the host. */
#define OVC_F_OUT_STREAM 128
#define OVC_F_STREAM_CAP_SHIFT 16
#define OVC_F_STREAM_CAP_MAX 0xFFFF
/* bits 8-11 select the record I/O strategy of the step kernel (0 = library default):
 *   1 = 2-D tensor-map TMA tile with hardware swizzle, 2 = 1-D bulk TMA (linear tile),
 *   3 = direct vectorised global loads/stores (no staging).  All produce identical results. */
#define OVC_F_IO_SHIFT 8
#define OVC_F_IO_MASK (0xF << OVC_F_IO_SHIFT)

/* element type of ovc_encode_lossless output */
#define OVC_DT_F32 0
#define OVC_DT_U8 1
#define OVC_DT_I32 2
#define OVC_DT_BF16 3 /* bfloat16: exact for the plane values up to 256 (cook times beyond that round) */

int ovc_abi_version(void);
size_t ovc_layout_table_size(void); /* sizeof(ovc_layout_t): the host packer checks it */
size_t ovc_feat_lut_entry_size(void);
const char *ovc_last_error(void);

/*
 * One joint transition of n_envs environments (replaces OvercookedGridworld.get_state_transition
 * :1375-1430 + the reward/done part of OvercookedEnv.step, overcooked_env.py:244-274).
 *   layouts        ovc_layout_t[n_layouts]
 *   start_records  int32[n_layouts][S], the packed standard start state per layout (auto reset)
 *   state          int32[n_envs][S], updated in place
 *   actions        int32[n_envs][2], values 0..5   (uint8[n_envs][2] with OVC_F_ACT_U8)
 *   sparse         int32[n_envs]      sum over both agents of the delivery reward (env.step's r)
 *   shaped         int32[n_envs][2]   shaped_reward_by_agent
 *   done           int32[n_envs]      1 iff new timestep >= horizon
 *   events         int32[n_envs][2]   event bit mask per agent (+ recipe / flag bits above)
 */
int ovc_step(const void *layouts, int n_layouts, const int32_t *start_records, int32_t *state,
             const int32_t *actions, int32_t *sparse, int32_t *shaped, int32_t *done,
             int32_t *events, int64_t n_envs, int state_words, int horizon, int flags,
             const ovc_random_start_t *random_start, void *stream);

/*
 * T consecutive transitions in ONE launch (the record stays on chip between transitions).
 * actions int32[T][n_envs][2]; sparse/done int32[T][n_envs]; shaped/events int32[T][n_envs][2] — or the narrower
 * element types the OVC_F_ACT_* / OVC_F_OUT_* flags select (pointers are then reinterpreted; outputs a format does
 * not produce may be NULL).  Every array must be aligned to its element type (OVC_E_BADARG otherwise).  Semantically
 * identical to T calls of ovc_step with the same flags.
 */
int ovc_rollout(const void *layouts, int n_layouts, const int32_t *start_records, int32_t *state,
                const int32_t *actions, int32_t *sparse, int32_t *shaped, int32_t *done,
                int32_t *events, int64_t n_envs, int n_steps, int state_words, int horizon,
                int flags, const ovc_random_start_t *random_start, void *stream);

/*
 * Rollout with HOST buffers: the native driver of the end-to-end path (what the reference's callers see is host
 * memory: actions come from a host policy, rewards / events go to a host learner, overcooked_env.py:449-462).
 * A pipeline object owns three CUDA streams and a few events, nothing else: the caller provides the device staging
 * buffers (two sets, for double buffering) and pinned host buffers.  ovc_pipeline_run cuts the n_steps transitions
 * into chunks of `chunk` and, per chunk, copies the actions host->device, runs ovc_rollout on them and copies the
 * outputs device->host, the three stages on their own streams and overlapped across chunks AND across successive
 * calls.  Element formats follow `flags` exactly as in ovc_rollout (OVC_F_ACT_U8 / OVC_F_ACT_PACKED,
 * OVC_F_OUT_NARROW / OVC_F_OUT_PACKED / OVC_F_OUT_CODES); output pointers a format does not use may be NULL.
 * One pipeline object is driven by one host thread at a time.
 */
typedef struct ovc_pipeline ovc_pipeline_t;
typedef struct ovc_pipeline_desc {
    const void *layouts;          /* as ovc_rollout */
    int32_t n_layouts;
    int32_t state_words;
    const int32_t *start_records;
    int32_t *state;
    int64_t n_envs;
    int32_t horizon;
    int32_t flags;
    int32_t chunk;                /* transitions per chunk, >= 1 */
    int32_t has_random_start;
    ovc_random_start_t random_start;
    void *d_actions[2];           /* device staging: chunk * n_envs joint actions each */
    void *d_sparse[2];            /* device staging of the outputs, chunk * n_envs env-steps each */
    void *d_shaped[2];            /*   (OVC_F_OUT_STREAM: d_events = lane masks uint32[chunk][G], d_sparse = values */
    void *d_done[2];              /*    uint16[G][stream_cap], d_shaped / d_done unused) */
    void *d_events[2];
    int32_t stream_cap;           /* OVC_F_OUT_STREAM: value words per group and CHUNK, 1..OVC_F_STREAM_CAP_MAX */
    int32_t reserved;
    void *d_codes_full[2];        /* OVC_F_OUT_STREAM, optional: dense code words uint16[n_steps][n_envs] of a whole pass, kept
                                     on the device (pass k writes set k & 1) so that the caller can recover an overflow */
} ovc_pipeline_desc_t;

int ovc_pipeline_create(const ovc_pipeline_desc_t *desc, ovc_pipeline_t **out);
/* Enqueues one pass over host buffers [n_steps][n_envs](..) and returns immediately (everything is asynchronous).
 * The pipeline first waits for the work already enqueued on `stream` (the caller's stream).  `join` != 0: `stream`
 * then waits for the pass, so later work on it sees the results (stream-ordered call); join == 0: successive passes
 * overlap, *ticket (nullable) identifies this pass for ovc_pipeline_wait. */
/* OVC_F_OUT_STREAM: h_events = lane masks uint32[n_steps][G], h_sparse = values uint16[n_chunks][G][stream_cap]
 * (n_chunks = ceil(n_steps / chunk); every chunk starts its groups' value slices afresh), h_shaped / h_done unused. */
int ovc_pipeline_run(ovc_pipeline_t *p, const void *h_actions, void *h_sparse, void *h_shaped, void *h_done,
                     void *h_events, int n_steps, void *stream, int join, int64_t *ticket);
int ovc_pipeline_wait(ovc_pipeline_t *p, int64_t ticket); /* blocks the HOST until that pass's last copy has landed */
int ovc_pipeline_join(ovc_pipeline_t *p, void *stream);   /* `stream` waits for everything enqueued so far */
void ovc_pipeline_destroy(ovc_pipeline_t *p);

/*
 * HOST function (no GPU work): expands OVC_F_OUT_CODES words into dense arrays, multi-threaded.
 *   codes        uint16[n_steps][n_envs] in host memory
 *   env_layout   int32[n_envs] layout of each environment, or NULL (every environment on layout 0)
 *   reward_tbl   int32[n_layouts][2][32]: [l][0][code] = delivery reward, [l][1][code] = shaped reward of the code
 *   sparse       int16[n_steps][n_envs] or NULL     shaped  int8[n_steps][n_envs][2] or NULL
 *   done         uint8[n_steps][n_envs] or NULL     events  int32[n_steps][n_envs][2] or NULL (masks, as ovc_step's)
 *   n_threads    <= 0: all online cores
 */
int ovc_expand_codes_host(const uint16_t *codes, int64_t n_steps, int64_t n_envs, const int32_t *env_layout,
                          const int32_t *reward_tbl, int n_layouts, int16_t *sparse, int8_t *shaped, uint8_t *done,
                          int32_t *events, int n_threads);

/*
 * HOST function (no GPU work): dense arrays from an OVC_F_OUT_STREAM result, multi-threaded (threads own ranges of
 * groups; zero fill + scatter of the non-zeros, so the cost is that of writing the arrays once).
 *   masks    uint32[n_steps][G]                    values  uint16[n_chunks][G][cap], n_chunks = ceil(n_steps / chunk)
 *   chunk    transitions per launch that produced the stream (n_steps for one ovc_rollout call)
 *   outputs / env_layout / reward_tbl / n_threads as ovc_expand_codes_host
 *   overflow (nullable) receives the number of (chunk, group) slices whose word count exceeded cap: their excess
 *            words read as zero and the caller must fall back to the dense code words of those chunks
 */
int ovc_expand_stream_host(const uint32_t *masks, const uint16_t *values, int64_t n_steps, int64_t chunk, int64_t cap,
                           int64_t n_envs, const int32_t *env_layout, const int32_t *reward_tbl, int n_layouts,
                           int16_t *sparse, int8_t *shaped, uint8_t *done, int32_t *events, int n_threads, int64_t *overflow);

/*
 * OvercookedEnv.reset (overcooked_env.py:288-319) for the envs whose mask[i] != 0 (all if mask
 * is NULL): state[i] = start_records[layout]; layout = env_layout[i] if env_layout != NULL, else
 * the id already stored in the record.  With `random_start` the record is drawn instead (see above) and the
 * episode counter of the record advances; auto-reset inside ovc_step / ovc_rollout does the same.
 */
int ovc_reset(const void *layouts, int n_layouts, const int32_t *start_records, int32_t *state,
              const int32_t *env_layout, const int32_t *mask, int64_t n_envs, int state_words,
              const ovc_random_start_t *random_start, void *stream);

/*
 * lossless_state_encoding (:2385-2561) for envs [0, n_envs) that all share one layout shape:
 * out[env][player][x][y][26] with element type `dtype` (OVC_DT_*).  `width`/`height` must equal
 * the layouts' own (all envs in the range must have equal-shape layouts).
 * view_swap (nullable, int32[n_envs]): where non-zero the two player views are written in swapped
 * order, out[env][0] = player 1's view — the "primary agent first" order of the gym wrapper
 * (overcooked_env.py:850-866) without a second pass over the observations.
 */
int ovc_encode_lossless(const void *layouts, int n_layouts, const int32_t *state, const int32_t *view_swap,
                        void *out, int dtype, int64_t n_envs, int state_words, int width, int height,
                        int horizon, void *stream);

/*
 * The first layer of a policy on lossless_state_encoding, evaluated from the packed record WITHOUT materialising the
 * observation (what the reference's rollout workers do per transition: lossless_state_encoding :2385-2561 feeding the
 * first convolution of the PPO model, human_aware_rl/ppo/ppo_rllib.py:43-79 — any first layer that is linear in the
 * observation, a 'same' convolution included, is one matrix over the flattened observation):
 *   out[2 env + view][:] = leaky_relu(W . obs[env][view].flatten() + bias, neg_slope)       bfloat16 [2 n_envs][n_out]
 *   wt    bfloat16 [width*height*26][n_out]: W TRANSPOSED, row index = the observation's element order
 *         (x*height + y)*26 + plane, 16-byte aligned;   bias  float32 [n_out];   n_out a multiple of 64;
 *   neg_slope in [0, 1] (0: ReLU, 1: no activation);   accumulation in float32;   view_swap / horizon as above.
 * The encoding is sparse (a few player / object entries per view; terrain planes are layout constants), so the kernel
 * gathers ~10 rows of `wt` per environment from shared memory instead of multiplying by width*height*26 inputs.
 * At most 8 layouts per call (one grid shape); OVC_E_UNSUPPORTED if the table of a grid does not fit shared memory.
 */
int ovc_encode_linear(const void *layouts, int n_layouts, const int32_t *state, const int32_t *view_swap,
                      const void *wt, const float *bias, void *out, int64_t n_envs, int state_words, int width,
                      int height, int horizon, int n_out, float neg_slope, void *stream);

/*
 * One view per environment (an agent pair: each agent's network sees its own seat only).  Common to every *_view entry
 * point: environment e's agent sits at player p(e) = seat ^ (swap[e] != 0), seat 0 or 1 (OVC_E_BADARG otherwise), swap
 * int32 [n] or NULL (no swap), 4-byte aligned; compact row r is environment r and its joint row is g(r) = 2 r + p(r).
 *
 * ovc_encode_linear_view: ovc_encode_linear for player p(e)'s view only, out bfloat16 [n_envs][n_out]; row e is bit for
 *   bit row g(e) of ovc_encode_linear (without view_swap) on the same operands.  Same limits as ovc_encode_linear.
 */
int ovc_encode_linear_view(const void *layouts, int n_layouts, const int32_t *state, const int32_t *swap, int seat,
                           const void *wt, const float *bias, void *out, int64_t n_envs, int state_words, int width,
                           int height, int horizon, int n_out, float neg_slope, void *stream);

/*
 * The two ends of a policy-in-the-loop transition around ovc_step (the reference's rollout worker samples the joint
 * action from the policy's action distribution and mixes the rewards, human_aware_rl/rllib/rllib.py:302-342):
 *
 * ovc_sample_actions: actions[r] ~ softmax(scores[r][0..n_actions)) for r in [0, n_rows) by the Gumbel-max rule,
 *   argmax_i (scores[r][i] - log(-log u_i)), u_i = ((draw_i >> 9) + 0.5) / 2^23 with draw_i word i of Philox4x32-10,
 *   key = seed, counter = (r low, r high, step low, 2 * step high + i / 4).  scores float32 [n_rows][ld], n_actions <= 8.
 *   `counter` is DEVICE memory uint64[2]: [0] = step (advanced by one per launch by the last CTA to finish, so a
 *   captured CUDA graph draws fresh numbers at every replay), [1] = scratch that must start at 0.  With rows ordered
 *   [env][agent] `actions` is the int32[n_envs][2] that ovc_step takes.
 * ovc_accumulate_returns: ret_sparse[e] += sparse[e] (int64);  ret_mixed[e] += sparse[e] + factor * shaped[e][0] +
 *   factor * shaped[e][1] (float32; rllib.py:328-329) from ovc_step's int32 outputs; either accumulator may be NULL.
 */
int ovc_sample_actions(const float *scores, int ld, int n_actions, int64_t n_rows, uint64_t seed, uint64_t *counter,
                       int32_t *actions, void *stream);
int ovc_accumulate_returns(const int32_t *sparse, const int32_t *shaped, float factor, int64_t n_envs, int64_t *ret_sparse,
                           float *ret_mixed, void *stream);
/* ovc_sample_actions_view: the ovc_sample_actions draw for one agent per environment (the *_view row map, see
 * ovc_encode_linear_view): scores row r, Philox counter row g(r), written to actions[g(r)] of the int32 [n_rows][2] joint
 * action (the other seat's entry untouched); logp[r] (nullable) as ovc_sample_actions_logp.  scores, actions, logp 4-byte
 * aligned. */
int ovc_sample_actions_view(const float *scores, int ld, int n_actions, int64_t n_rows, uint64_t seed, uint64_t *counter,
                            const int32_t *swap, int seat, int32_t *actions, float *logp, void *stream);

/*
 * What a PPO sample batch keeps of each transition (RLlib's SampleBatch: action_logp, rewards, dones; then its GAE
 * postprocessing into advantages and value_targets), produced on the device:
 *
 * ovc_sample_actions_logp: ovc_sample_actions, and logp[r] = s[a] - (m + log(sum_i exp(s[i] - m))) with s = scores[r],
 *   m = max_i s[i] over i < n_actions, a = the drawn action (float32): the log-probability of the draw.
 * ovc_record_transition: ovc_accumulate_returns with the factor read from DEVICE memory (`factor`: one float32, so a
 *   captured graph follows a factor changed between replays) and, each nullable,
 *     rewards[2 e + i] = (float)sparse[e] + factor * (float)shaped[e][i]   float32 [n_envs][2], the product rounded first
 *     dones[e] = done[e] != 0                                              uint8 [n_envs] from ovc_step's int32 done
 *   ret_sparse / ret_mixed are accumulated as ovc_accumulate_returns does when given.
 * ovc_gae: generalized advantage estimation over a window of n_steps transitions of n_rows = 2 n_envs agent rows:
 *     rewards, values, advantages, value_targets float32 [n_steps][n_rows];  dones uint8 [n_steps][n_rows / 2] (one flag
 *     per environment, shared by its two rows: done = terminal, the next value counts 0);  last_values float32 [n_rows]
 *   from t = n_steps - 1 down to 0, with A = 0 after the window, every operation rounded to float32 on its own:
 *     nt = 1 - dones[t][r / 2];  next_v = t < n_steps - 1 ? values[t + 1][r] : last_values[r]
 *     delta = (rewards[t][r] + (gamma * next_v) * nt) - values[t][r]
 *     A = delta + ((gamma * lambda) * nt) * A;   advantages[t][r] = A;   value_targets[t][r] = A + values[t][r]
 *   Float buffers 8-byte aligned.
 */
int ovc_sample_actions_logp(const float *scores, int ld, int n_actions, int64_t n_rows, uint64_t seed, uint64_t *counter,
                            int32_t *actions, float *logp, void *stream);
int ovc_record_transition(const int32_t *sparse, const int32_t *shaped, const int32_t *done, const float *factor, int64_t n_envs,
                          float *rewards, uint8_t *dones, int64_t *ret_sparse, float *ret_mixed, void *stream);
int ovc_gae(const float *rewards, const float *values, const uint8_t *dones, const float *last_values, int64_t n_steps, int64_t n_rows,
            float gamma, float lambda, float *advantages, float *value_targets, void *stream);

/*
 * Finished episodes on the device: the per-episode statistics the reference's env reports at an episode's end
 * (OvercookedEnv.game_stats and the info dict's "episode" entry, overcooked_env.py:363-401; logged by human_aware_rl's
 * TrainingCallbacks.on_episode_end, rllib.py:480-483), kept in the same kernel as ovc_record_transition.
 *
 * ovc_episode_stats_t: device pointers (the struct itself is passed by HOST pointer).  Running state, one entry per env:
 *   event_counts int32 [n_envs][2][25], sparse_by_agent / shaped_by_agent int64 [n_envs][2], reward_by_agent float32
 *   [n_envs][2] (nullable), ep_length int32 [n_envs], layout_id int32 [n_envs] (the running episode's layout; initialise it
 *   from word 3 of the records).  Records: slot k of env e is entry [k][e] of every rec_* array ([capacity][n_envs][...]);
 *   count / dropped int32 [n_envs] (zero them to clear the buffer).  capacity >= 0; the rec_* pointers may be NULL when it
 *   is 0, rec_reward_by_agent when reward_by_agent is.
 * ovc_record_transition_stats: ovc_record_transition, and per env e, in this order:
 *     d_i = events[e][i] bit 15 (soup_delivery) ? layouts[layout_id[e]].deliver_value[events[e][i] bits 25-28] : 0
 *     sparse_by_agent[e][i] += d_i;  shaped_by_agent[e][i] += shaped[e][i];  ep_length[e] += 1
 *     event_counts[e][i][b] += 1 for every set bit b < 25 of events[e][i]
 *     reward_by_agent[e][i] = reward_by_agent[e][i] + rewards_i (float32, rewards_i as ovc_record_transition defines them,
 *       with the factor of this call)
 *     L = layout_id[e];  layout_id[e] = state[e][3] & 0xFF   (the record after the step: a new episode's layout)
 *     if done[e]:  k = count[e];  if k < capacity: slot k <- (ep_length, L, partner_seat ? partner_seat[e] : -1, sparse,
 *                  shaped, event counts, reward), count[e] = k + 1;  else dropped[e] += 1;  then the running state is zeroed.
 *   One thread per env claims its slots without atomics, so the slot order is deterministic (the event counts, each
 *   owned by one thread, are updated with atomic adds only so that they do not wait for memory).  state: the records ovc_step left ([n_envs][state_words]), events: its
 *   int32 [n_envs][2] output; layouts: the table it ran on.
 */
typedef struct ovc_episode_stats {
    const void *layouts;
    const int32_t *state;
    const int32_t *events;
    const int32_t *partner_seat; /* nullable: the partner's seat in the ending episode, -1 = self-play */
    int32_t *event_counts;
    int64_t *sparse_by_agent;
    int64_t *shaped_by_agent;
    float *reward_by_agent; /* nullable */
    int32_t *ep_length;
    int32_t *layout_id;
    int32_t *count;
    int32_t *dropped;
    int32_t *rec_length;
    int32_t *rec_layout;
    int32_t *rec_partner_seat;
    int64_t *rec_sparse_by_agent;
    int64_t *rec_shaped_by_agent;
    int32_t *rec_event_counts;
    float *rec_reward_by_agent;
    int32_t capacity;
    int32_t state_words;
} ovc_episode_stats_t; /* 160 bytes */
int ovc_record_transition_stats(const int32_t *sparse, const int32_t *shaped, const int32_t *done, const float *factor, int64_t n_envs,
                                float *rewards, uint8_t *dones, int64_t *ret_sparse, float *ret_mixed, const ovc_episode_stats_t *stats,
                                void *stream);

/*
 * ovc_policy_tail: the narrow end of the rollout policy and the action draw in one kernel (reference model:
 * human_aware_rl/ppo/ppo_rllib.py:64-79 — dense layers of 64 after the convolutions, then the action / value heads):
 *   a = leaky_relu(x, in_slope)                          x bfloat16 [n_rows][k0], k0 a multiple of 32 in 32..256
 *   a = leaky_relu(a . w_first^T + b_first, slope)       w_first bfloat16 [64][k0], biases float32
 *   a = leaky_relu(a . w_hidden[l]^T + b_hidden[l], slope)   l < n_hidden, w_hidden bfloat16 [n_hidden][64][64]
 *   s = a . w_heads^T + b_heads                          w_heads bfloat16 [8][64]: heads 0..n_actions-1 are the logits,
 *                                                        head n_actions (<= 7) is the value
 *   actions[r] ~ softmax(s[r][0..n_actions)) exactly as ovc_sample_actions draws it (same seed / counter semantics);
 *   values[r] = s[r][n_actions] (nullable);  scores float32 [n_rows][8] = s (nullable).
 * Activations are rounded to bfloat16 between layers, accumulation is float32 (mma.sync m16n8k16).
 */
int ovc_policy_tail(const void *x, int64_t n_rows, int k0, float in_slope, const void *w_first, const float *b_first,
                    const void *w_hidden, const float *b_hidden, int n_hidden, const void *w_heads, const float *b_heads,
                    float slope, int n_actions, uint64_t seed, uint64_t *counter, int32_t *actions, float *values,
                    float *scores, void *stream);
/* ovc_policy_tail_logp: ovc_policy_tail, and logp[r] (nullable) = the log-probability of the drawn action under
 * softmax(s[r][0..n_actions)), as ovc_sample_actions_logp defines it on the float32 heads s. */
int ovc_policy_tail_logp(const void *x, int64_t n_rows, int k0, float in_slope, const void *w_first, const float *b_first,
                         const void *w_hidden, const float *b_hidden, int n_hidden, const void *w_heads, const float *b_heads,
                         float slope, int n_actions, uint64_t seed, uint64_t *counter, int32_t *actions, float *values,
                         float *scores, float *logp, void *stream);
/* ovc_policy_hidden: ovc_policy_tail's layers up to the last 64-wide one, without the heads and the draw:
 * hidden bfloat16 [n_rows][64] = that layer's activation a (rounded to bfloat16 as above).  The input of the LSTM policy
 * (ovc_lstm_head).  Arguments as ovc_policy_tail's; hidden 4-byte aligned. */
int ovc_policy_hidden(const void *x, int64_t n_rows, int k0, float in_slope, const void *w_first, const float *b_first,
                      const void *w_hidden, const float *b_hidden, int n_hidden, float slope, void *hidden, void *stream);
/* ovc_policy_tail_view: ovc_policy_tail_logp on one agent's rows (the *_view row map, see ovc_encode_linear_view): x row r
 * is environment r's agent; the draw uses the joint row g(r) with this call's seed and counter and writes actions[g(r)]
 * of the int32 [n_rows][2] joint action (the other seat's entry untouched); values[r], logp[r], scores[r] (each
 * nullable) as ovc_policy_tail_logp.  actions, values, logp 4-byte aligned, scores 8-byte aligned. */
int ovc_policy_tail_view(const void *x, int64_t n_rows, int k0, float in_slope, const void *w_first, const float *b_first,
                         const void *w_hidden, const float *b_hidden, int n_hidden, const void *w_heads, const float *b_heads,
                         float slope, int n_actions, uint64_t seed, uint64_t *counter, const int32_t *swap, int seat, int32_t *actions,
                         float *values, float *scores, float *logp, void *stream);

/*
 * ovc_lstm_head (K11): the recurrent end of the reference's LSTM PPO model (ppo_rllib.py:89-238, RllibLSTMPPOModel:
 * tf.keras.layers.LSTM(256) on the dense layers' output, the logits / value heads on its output) and the action draw:
 *   x bfloat16 [n_rows][64]; h_in bfloat16 [n_rows][256], c_in float32 [n_rows][256], both taken as zero for rows 2 e, 2 e + 1
 *     where reset[e] != 0 (reset int32 [ceil(n_rows / 2)], nullable: no reset)
 *   gates = [x | h_in] . w^T + b        w bfloat16 [1024][320] = [W_ih | W_hh], b float32 [1024] = b_ih + b_hh, gate rows
 *                                       permuted: row 64 j + 8 (4 half + gate) + n is gate (i, f, g, o) of hidden unit
 *                                       16 j + 8 half + n
 *   c_out = sigmoid(f) * c_in + sigmoid(i) * tanh(g);   h_out = bfloat16(sigmoid(o) * tanh(c_out))
 *   s = h_out . w_heads^T + b_heads     w_heads bfloat16 [8][256]: heads 0..n_actions-1 the logits, head n_actions the value
 *   actions / values / logp / scores as ovc_policy_tail_logp's (same seed / counter semantics; values, logp, scores nullable)
 *   snap_h bfloat16 / snap_c float32 [n_rows][256] (nullable): the state the row used, after the reset rule.
 * h_out / c_out may alias h_in / c_in (in-place update).  float32 accumulation (mma.sync m16n8k16), accurate expf / tanhf.
 * x, h_in, w, w_heads, snap_h 16-byte aligned; c_in, c_out, snap_c, b, b_heads, scores 8-byte aligned.
 */
int ovc_lstm_head(const void *x, const void *h_in, const float *c_in, const int32_t *reset, int64_t n_rows, const void *w,
                  const float *b, const void *w_heads, const float *b_heads, int n_actions, uint64_t seed, uint64_t *counter,
                  void *h_out, float *c_out, void *snap_h, float *snap_c, int32_t *actions, float *values, float *logp,
                  float *scores, void *stream);
/* ovc_lstm_head_view: ovc_lstm_head on one agent's rows (the *_view row map, see ovc_encode_linear_view): the state
 * h_in / c_in / h_out / c_out / snap_* is [n_rows][256], one row per environment for this agent; row r is zeroed where
 * reset[r] != 0 (reset int32 [n_rows], nullable, 4-byte aligned); the draw uses the joint row g(r) and writes
 * actions[g(r)] of the int32 [n_rows][2] joint action (the other seat's entry untouched); values / logp / scores row r.
 * actions, values, logp 4-byte aligned, the rest as ovc_lstm_head. */
int ovc_lstm_head_view(const void *x, const void *h_in, const float *c_in, const int32_t *reset, int64_t n_rows, const void *w,
                       const float *b, const void *w_heads, const float *b_heads, int n_actions, uint64_t seed, uint64_t *counter,
                       const int32_t *swap, int seat, void *h_out, float *c_out, void *snap_h, float *snap_c, int32_t *actions,
                       float *values, float *logp, float *scores, void *stream);
/* ovc_record_transition_view: ovc_record_transition (stats NULL) or ovc_record_transition_stats (stats given) for one
 * agent per environment (the *_view row map, see ovc_encode_linear_view): rewards float32 [n_envs] (required, 4-byte
 * aligned) with
 *     rewards[e] = (float)sparse[e] + factor * (float)shaped[e][p(e)]   the product rounded first
 *   bit for bit rewards[g(e)] of ovc_record_transition; dones, ret_sparse, ret_mixed and the episode statistics and
 *   records exactly as those calls write them. */
int ovc_record_transition_view(const int32_t *sparse, const int32_t *shaped, const int32_t *done, const float *factor, int64_t n_envs,
                               const int32_t *swap, int seat, float *rewards, uint8_t *dones, int64_t *ret_sparse, float *ret_mixed,
                               const ovc_episode_stats_t *stats, void *stream);
/* ovc_gae_view: ovc_gae over n_envs rows, one per environment (an agent pair's learner): rewards, values, advantages,
 * value_targets float32 [n_steps][n_envs], dones uint8 [n_steps][n_envs], last_values float32 [n_envs]; the recurrence
 * and rounding order are ovc_gae's, so the result is bit for bit ovc_gae's on those rows of a two-row layout.  Float
 * buffers 4-byte aligned. */
int ovc_gae_view(const float *rewards, const float *values, const uint8_t *dones, const float *last_values, int64_t n_steps,
                 int64_t n_envs, float gamma, float lambda, float *advantages, float *value_targets, void *stream);

/*
 * ovc_wide_layers (K9): the two wide layers of the rollout policy between ovc_encode_linear and ovc_policy_tail
 * (reference model: ppo_rllib.py:54-62, the two 3x3 convolutions, each folded into one matrix) as one wgmma kernel:
 *   a1 = leaky_relu(a0 . w1^T + b1, slope);   z2 = a1 . w2^T + b2
 *   a0 bfloat16 [m][k0], w1 bfloat16 [n1][k0], w2 bfloat16 [n2][n1], biases float32, z2 bfloat16 [m][n2] (pre-activation);
 *   built for k0 = 512, n1 = 512, n2 = 160 (OVC_E_UNSUPPORTED otherwise); operands 16-byte aligned, rows contiguous.
 * The activation tile a1 stays on chip (in registers, as the second layer's A operand); float32
 * accumulation, a1 rounded to bfloat16 as a materialised activation would be.
 */
int ovc_wide_layers(const void *a0, int64_t m, int k0, const void *w1, const float *b1, int n1, const void *w2, const float *b2,
                    int n2, float slope, void *z2, void *stream);

/*
 * A behaviour-cloned partner on the device (PPO_BC: human_aware_rl's OvercookedMultiAgent pairs the PPO agent with a fixed
 * BC agent in a seat drawn at every reset; the BC model, imitation/behavior_cloning_tf2.py, is featurize_state -> Dense 64
 * ReLU -> Dense 64 ReLU -> logits, its action sampled from the softmax).
 *
 * ovc_partner_policy (K10): for every environment e with partner_seat[e] in {0, 1} (int32 [n_envs]; -1 = self-play, nothing
 *   written), the BC policy on player seat's featurize_state view (as ovc_featurize computes it at num_pots = 2: 96 features,
 *   never materialised) and a draw from it:
 *     a = bf16(x)                                          x = the 96 features, exact in bfloat16 while |value| <= 256 (every
 *                                                          shipped layout; cook times above 256 round)
 *     a = bf16(relu(a . w_first^T + b_first))              w_first bfloat16 [64][96], biases float32
 *     a = bf16(relu(a . w_hidden[l]^T + b_hidden[l]))      l < n_hidden (0..8), w_hidden bfloat16 [n_hidden][64][64]
 *     s = a . w_heads^T + b_heads                          w_heads bfloat16 [8][64]: heads 0..n_actions-1 (<= 7) the logits
 *     actions[2 e + seat] ~ softmax(s[0..n_actions))       the ovc_sample_actions draw on row r = 2 e + seat with this call's
 *                                                          own seed and counter (uint64[2], same semantics)
 *   float32 accumulation (K8's mma.sync chain).  `actions` is the int32 [n_envs][2] joint action ovc_step takes: the
 *   partner's entry is overwritten, the other one is left alone.  scores (nullable) float32 [n_envs][8] = s of partnered
 *   environments.  n_features must be 96 and width 64 (OVC_E_UNSUPPORTED otherwise); weights 16-byte aligned.
 * ovc_assign_partners: partner_seat[e] for every e with done[e] != 0 (ovc_step's int32 done; NULL = every environment):
 *   Philox4x32-10, key = seed, counter = (e low, e high, step low, step high) -> words w0, w1;
 *   partner_seat[e] = w0 < thr ? w1 >> 31 : -1,  thr = floor(bc_factor * 2^32), saturated: bc_factor >= 1 always pairs,
 *   bc_factor <= 0 never.  bc_factor is one float32 in DEVICE memory (a captured graph follows an annealed value); counter
 *   uint64[2] as ovc_sample_actions' (one step per launch).
 */
int ovc_partner_policy(const void *layouts, int n_layouts, const void *lut, const int32_t *state, const int32_t *partner_seat,
                       int64_t n_envs, int state_words, int n_features, int width, const void *w_first, const float *b_first,
                       const void *w_hidden, const float *b_hidden, int n_hidden, const void *w_heads, const float *b_heads, int n_actions,
                       uint64_t seed, uint64_t *counter, int32_t *actions, float *scores, void *stream);
int ovc_assign_partners(const int32_t *done, const float *bc_factor, int64_t n_envs, uint64_t seed, uint64_t *counter, int32_t *partner_seat,
                        void *stream);

/*
 * A population of partners (fictitious co-play, training against a set of checkpoints, PPO_BC with several BC human
 * proxies): each environment plays one of n_members (1..64, OVC_E_BADARG otherwise) members in one seat, drawn per episode,
 * and each member's kernels run on its own environments only.
 *
 * ovc_group_members: a stable counting sort of the environments by member (int32 [n_envs], every value in
 *   [0, n_members); other values are undefined behaviour): order int32 [n_envs] = the environment indices grouped by member,
 *   ascending within a group; offsets int32 [n_members + 1] = the group starts (offsets[n_members] = n_envs), so member k's
 *   environments are order[offsets[k] .. offsets[k + 1]).  One CTA, no host synchronisation.  n_envs < 2^31; n_envs = 0
 *   writes nothing.  member, order, offsets 4-byte aligned.
 * ovc_assign_members: for every environment e with done[e] != 0 (ovc_step's int32 done; done = NULL: every environment),
 *   in this order:
 *     record  if done != NULL, rec_member != NULL and count[e] < capacity: rec_member[count[e]][e] = member[e]
 *             (rec_member int32 [capacity][n_envs]: the slot ovc_record_transition_stats writes the ending episode to when it
 *             runs after this call with the same count, int32 [n_envs]; at a full buffer nothing is written)
 *     draw    if thresholds != NULL: Philox4x32-10, key = seed, counter = (e low, e high, step low, step high) -> word w0;
 *             member[e] = #{k < n_members - 1 : w0 >= thresholds[k]}
 *   thresholds int64 [n_members - 1] in DEVICE memory (a captured graph follows a changed distribution), computed by the
 *   host as floor(cdf[k] * 2^32) with cdf[k] the float64 cumulative share of members 0..k: a member of weight 0 is never
 *   drawn.  counter uint64[2] as ovc_sample_actions' (one step per launch), used and advanced only with thresholds.
 *   done, member, rec_member, count 4-byte aligned, thresholds and counter 8-byte aligned; capacity >= 0.
 *
 * The rows map of the *_rows forms below (one member's share of one-view rows): compact row r in [range[0], range[1]) is
 * environment e = rows[r] (int32, in [0, n_envs)), whose agent sits at player p(e) = seat ^ (swap[e] != 0) (swap nullable,
 * seat 0 or 1); its joint row is 2 e + p(e).  range points to two int32 in DEVICE memory (e.g. offsets + k of
 * ovc_group_members, with rows = order), so one captured launch serves any group size; the range is clipped to
 * [0, n_rows).  rows, range, swap 4-byte aligned.  Each form computes on row r bit for bit what its one-view form computes
 * on the row of environment rows[r], and leaves every other row and the other seat's action entries untouched.
 *
 * ovc_encode_linear_rows: ovc_encode_linear_view on the rows map: out[r] (bfloat16 [n_envs][n_out]) = environment rows[r]'s
 *   row of ovc_encode_linear_view.  A CTA with no rows in the range exits before it loads its weight slice.
 * ovc_wide_layers_range: ovc_wide_layers on rows [range[0], range[1]) of a0 / z2 ([m][...], m < 2^31); other rows of z2 untouched.
 * ovc_policy_tail_rows: ovc_policy_tail_view on the rows map: x, values, scores, logp row r; the draw on the joint row of
 *   environment rows[r] into actions (int32 [n_rows][2]).  Every CTA advances the counter, also for an empty range.
 * ovc_sample_actions_rows: ovc_sample_actions_view on the rows map: scores / logp row r, the draw on the joint row of
 *   environment rows[r].  Every CTA advances the counter, also for an empty range.  counter 8-byte aligned.
 */
int ovc_group_members(const int32_t *member, int n_members, int64_t n_envs, int32_t *order, int32_t *offsets, void *stream);
int ovc_assign_members(const int32_t *done, const int64_t *thresholds, int n_members, int64_t n_envs, uint64_t seed, uint64_t *counter,
                       int32_t *member, int32_t *rec_member, const int32_t *count, int capacity, void *stream);
int ovc_encode_linear_rows(const void *layouts, int n_layouts, const int32_t *state, const int32_t *swap, int seat, const int32_t *rows,
                           const int32_t *range, const void *wt, const float *bias, void *out, int64_t n_envs, int state_words, int width,
                           int height, int horizon, int n_out, float neg_slope, void *stream);
int ovc_wide_layers_range(const void *a0, int64_t m, int k0, const void *w1, const float *b1, int n1, const void *w2, const float *b2,
                          int n2, float slope, const int32_t *range, void *z2, void *stream);
int ovc_policy_tail_rows(const void *x, int64_t n_rows, int k0, float in_slope, const void *w_first, const float *b_first,
                         const void *w_hidden, const float *b_hidden, int n_hidden, const void *w_heads, const float *b_heads,
                         float slope, int n_actions, uint64_t seed, uint64_t *counter, const int32_t *swap, int seat, const int32_t *rows,
                         const int32_t *range, int32_t *actions, float *values, float *scores, float *logp, void *stream);
int ovc_sample_actions_rows(const float *scores, int ld, int n_actions, int64_t n_rows, uint64_t seed, uint64_t *counter, const int32_t *swap,
                            int seat, const int32_t *rows, const int32_t *range, int32_t *actions, float *logp, void *stream);

/*
 * Self-play mixtures: each environment is self-play (partner_seat[e] = -1: the learner plays both views) or plays a frozen
 * partner in seat partner_seat[e] (0 or 1: the learner plays view 1 - partner_seat[e]).  The learner's policy runs on its
 * own rows of the joint [2 n_envs] rows only, with the object part of K7 computed once per environment.
 *
 * ovc_learner_rows: from partner_seat int32 [n_envs] (values -1, 0, 1), in ONE CTA without host synchronisation, for every
 *   environment e in ascending order: list[e] = e << 2 | mask (bit v: the learner plays view v; 3 for -1, 1 << (1 - seat)
 *   otherwise), first[e] = the compact row of its first view; the compact rows of e's views are consecutive, in ascending
 *   view order, so compact row r is joint row jrow[r] (int32 [2 n_envs]); range[0] = 0, range[1] = the row count (device
 *   memory: K9's and K8's range).  n_envs < 2^29; n_envs = 0 writes nothing.  All pointers 4-byte aligned.
 * ovc_encode_linear_masked: ovc_encode_linear for the views in a list: entry r < n_list is environment list[r] >> 2 with the
 *   views of mask list[r] & 3 (mask 0: nothing), written to out rows first[r], first[r] + 1, ... in ascending view order,
 *   each bit for bit row 2 e + v of ovc_encode_linear without view_swap.  The object part is computed once per entry.
 *   Environments index state; out holds at least as many rows as the list's views.  At most 8 layouts.  list, first 4-byte
 *   aligned.
 * ovc_policy_tail_joint: ovc_policy_tail_logp on compact rows r in [range[0], range[1]) of x ([n_rows][k0], the range
 *   clipped to [0, n_rows), n_rows < 2^31): row r is joint row jrow[r], drawn there with key seed and counter's step, and
 *   actions, values, logp (required) and scores ([.][8], nullable) are written at jrow[r]: bit for bit what
 *   ovc_policy_tail_logp writes at that joint row from the same x row.  Every other entry is untouched.  Every CTA
 *   advances the counter, also for an empty range.
 */
int ovc_learner_rows(const int32_t *partner_seat, int64_t n_envs, int32_t *list, int32_t *first, int32_t *jrow, int32_t *range, void *stream);
int ovc_encode_linear_masked(const void *layouts, int n_layouts, const int32_t *state, const int32_t *list, const int32_t *first,
                             const void *wt, const float *bias, void *out, int64_t n_list, int state_words, int width, int height,
                             int horizon, int n_out, float neg_slope, void *stream);
int ovc_policy_tail_joint(const void *x, int64_t n_rows, int k0, float in_slope, const void *w_first, const float *b_first,
                          const void *w_hidden, const float *b_hidden, int n_hidden, const void *w_heads, const float *b_heads,
                          float slope, int n_actions, uint64_t seed, uint64_t *counter, const int32_t *jrow, const int32_t *range,
                          int32_t *actions, float *values, float *scores, float *logp, void *stream);

/*
 * A population of self-play learners on one batch (fictitious co-play's first stage): member k of n_members (1..64,
 * OVC_E_BADARG otherwise) plays both views of the environments of its block, a contiguous range of rows.
 *
 * Each grouped form is ONE launch for every member: its tables are stacked with a leading member dimension, and offsets
 * (int32 [n_members + 1] in DEVICE memory, non-decreasing, clipped to the rows the call holds) gives the members' blocks.
 * A CTA (encode) or a tile (wide layers, tail) never spans two members.
 *
 * ovc_encode_linear_grouped: ovc_encode_linear (two views, no view_swap) with member k's table on environments
 *   [offsets[k], offsets[k + 1]) of state: wt bfloat16 [n_members][width*height*26][n_out], bias float32 [n_members][n_out].
 *   Output row 2 e + v is bit for bit row 2 e + v of ovc_encode_linear with member k's table; rows of environments outside
 *   every block are untouched.  The CTAs are split over (member, column slice, worker).  Same limits as ovc_encode_linear.
 * ovc_wide_layers_grouped: ovc_wide_layers with member k's weights on rows [offsets[k], offsets[k + 1]) of a0 / z2 ([m][...],
 *   m < 2^31): w1 bfloat16 [n_members * 512][512], w2 bfloat16 [n_members * 160][512] (one tensor map per operand serves
 *   every member through row coordinates), b1 float32 [n_members][512], b2 float32 [n_members][160] (8-byte aligned).  Each
 *   row is bit for bit ovc_wide_layers on that member's weights; rows outside every block are untouched.
 * ovc_policy_tail_grouped: ovc_policy_tail_logp for every member.  The tables are stacked with a leading
 *   member dimension: w_first bfloat16 [n_members][64][k0], b_first float32 [n_members][64], w_hidden bfloat16
 *   [n_members][n_hidden][64][64], b_hidden float32 [n_members][n_hidden][64], w_heads bfloat16 [n_members][8][64], b_heads
 *   float32 [n_members][8].  offsets int32 [n_members + 1] in DEVICE memory, non-decreasing: member k's rows are
 *   [offsets[k], offsets[k + 1]) of x ([n_rows][k0], n_rows < 2^31), clipped to [0, n_rows).  Row r of member k is drawn on
 *   row r with this call's seed and counter's step, and actions, values, scores ([.][8]) and logp (each but actions
 *   nullable) are written at row r: bit for bit what ovc_policy_tail_logp writes at row r with member k's tables.  Rows
 *   outside every block are untouched.  Every CTA advances the counter once per launch (one step per launch, as
 *   ovc_sample_actions').  x and the weight tables 16-byte aligned; biases, scores and counter 8-byte aligned; actions,
 *   values, logp and offsets 4-byte aligned.
 */
int ovc_encode_linear_grouped(const void *layouts, int n_layouts, const int32_t *state, const void *wt, const float *bias,
                              const int32_t *offsets, int n_members, void *out, int64_t n_envs, int state_words, int width, int height,
                              int horizon, int n_out, float neg_slope, void *stream);
int ovc_wide_layers_grouped(const void *a0, int64_t m, int k0, const void *w1, const float *b1, int n1, const void *w2, const float *b2,
                            int n2, float slope, const int32_t *offsets, int n_members, void *z2, void *stream);
int ovc_policy_tail_grouped(const void *x, int64_t n_rows, int k0, float in_slope, const void *w_first, const float *b_first,
                            const void *w_hidden, const float *b_hidden, int n_hidden, const void *w_heads, const float *b_heads,
                            float slope, int n_actions, uint64_t seed, uint64_t *counter, const int32_t *offsets, int n_members,
                            int32_t *actions, float *values, float *scores, float *logp, void *stream);

/*
 * Population play: member pair[e][0] of a population of n_members learners (1..64, OVC_E_BADARG otherwise) plays player 0
 * of environment e and member pair[e][1] player 1 (pair int32 [n_envs][2], 8-byte aligned, every value in [0, n_members);
 * other values are undefined behaviour).  Every row of the joint [2 n_envs] rows is a learner's row.
 *
 * ovc_assign_pairs: ovc_assign_members for ordered pairs.  For every environment e with done[e] != 0 (done = NULL: every
 *   environment), in this order:
 *     record  if done != NULL, rec_pair != NULL and count[e] < capacity: rec_pair[count[e]][e][0..1] = pair[e][0..1]
 *             (rec_pair int32 [capacity][n_envs][2], the slot the ending episode's record goes to, as rec_member)
 *     draw    if thresholds != NULL: Philox4x32-10, key = seed, counter = (e low, e high, step low, step high) -> word w0;
 *             p = #{q < n_members^2 - 1 : w0 >= thresholds[q]};  pair[e] = (p / n_members, p % n_members)
 *   thresholds int64 [n_members^2 - 1] in DEVICE memory: ovc_assign_members' table of the row-major flattened n_members x
 *   n_members weights (non-decreasing; a pair of weight 0 is never drawn).  counter uint64[2], one step per launch, used and
 *   advanced only with thresholds.  done and count 4-byte aligned; pair, rec_pair, thresholds and counter 8-byte aligned.
 * ovc_group_pairs: the compact layout of the pairs, in ONE CTA without host synchronisation.  Environment e contributes the
 *   list entry e << 2 | 3 (both views) to member i where pair[e] = (i, i), else e << 2 | 1 (view 0) to member pair[e][0]
 *   and e << 2 | 2 (view 1) to member pair[e][1].  list int32 [2 n_envs] holds the entries grouped by member, ascending in
 *   e within a member: member k's are list[entry_offsets[k] .. entry_offsets[k + 1]) (entry_offsets int32 [n_members + 1]).
 *   Each entry's views take consecutive compact rows in ascending view order, the members' rows in member order: first int32
 *   [2 n_envs] is the compact row of entry r's first view, jrow int32 [2 n_envs] maps compact row -> joint row 2 e + v, and
 *   member k's rows are [row_offsets[k], row_offsets[k + 1]) (row_offsets int32 [n_members + 1], row_offsets[n_members] =
 *   2 n_envs).  n_envs < 2^29; n_envs = 0 writes nothing.  The int32 outputs 4-byte aligned.
 * ovc_encode_linear_grouped_masked: ovc_encode_linear_masked with member k's table (wt / bias stacked as in
 *   ovc_encode_linear_grouped) on list entries [entry_offsets[k], entry_offsets[k + 1]) (device memory, clipped to
 *   [0, n_list)): each output row first[r] + i is bit for bit row 2 e + v of ovc_encode_linear with member k's table.  The
 *   object part is computed once per entry; the CTAs are split over (member, column slice, worker).  Same limits as
 *   ovc_encode_linear_masked.
 * ovc_policy_tail_grouped_joint: ovc_policy_tail_grouped on compact rows with ovc_policy_tail_joint's placement: member k's
 *   rows [row_offsets[k], row_offsets[k + 1]) of x ([n_rows][k0], n_rows < 2^31, clipped) use its stacked tables, row r is
 *   drawn on joint row jrow[r] with the call's step, and actions, values, logp (required) and scores ([.][8], nullable) are
 *   written at jrow[r]: bit for bit what ovc_policy_tail_logp writes at that joint row with member k's tables.  Every other
 *   entry is untouched.  Every CTA advances the counter once per launch.  Alignment as ovc_policy_tail_grouped; jrow 4-byte
 *   aligned.
 */
int ovc_assign_pairs(const int32_t *done, const int64_t *thresholds, int n_members, int64_t n_envs, uint64_t seed, uint64_t *counter,
                     int32_t *pair, int32_t *rec_pair, const int32_t *count, int capacity, void *stream);
int ovc_group_pairs(const int32_t *pair, int n_members, int64_t n_envs, int32_t *list, int32_t *first, int32_t *jrow, int32_t *entry_offsets,
                    int32_t *row_offsets, void *stream);
int ovc_encode_linear_grouped_masked(const void *layouts, int n_layouts, const int32_t *state, const int32_t *list, const int32_t *first,
                                     const void *wt, const float *bias, const int32_t *entry_offsets, int n_members, void *out, int64_t n_list,
                                     int state_words, int width, int height, int horizon, int n_out, float neg_slope, void *stream);
int ovc_policy_tail_grouped_joint(const void *x, int64_t n_rows, int k0, float in_slope, const void *w_first, const float *b_first,
                                  const void *w_hidden, const float *b_hidden, int n_hidden, const void *w_heads, const float *b_heads,
                                  float slope, int n_actions, uint64_t seed, uint64_t *counter, const int32_t *jrow, const int32_t *row_offsets,
                                  int n_members, int32_t *actions, float *values, float *scores, float *logp, void *stream);

/*
 * ovc_encode_linear_wgrad (K12): the weight gradient of ovc_encode_linear's layer, from the packed records,
 *     dwt[f][c] += sum over rows r of enc(r)[f] * dz[r][c]
 *   enc(r) = lossless_state_encoding of row r's record and view (never materialised), f in the observation's element order
 *   (x*height + y)*26 + plane, i.e. dwt has the layout of ovc_encode_linear's wt; dz float32 [rows][n_out] is the gradient
 *   at the layer's pre-activation (for a leaky ReLU layer: the output gradient times 1 or neg_slope).  Rows:
 *     seat -1: two views, rows = 2 n_records, row 2 m + v is view v of record m (ovc_encode_linear without view_swap);
 *     seat 0 / 1: one view, rows = n_records, row m is player seat ^ (swap[m] != 0) of record m (ovc_encode_linear_view).
 *   states int32 [n_records][state_words] (any records, e.g. a sample batch's, gathered); urgency from horizon minus the
 *   record's timestep, as in ovc_encode_linear.  dwt float32 [width*height*26][n_out] is added to, never overwritten; only
 *   rows < rows of dz are read.  Accumulation in float32, summation order unspecified (it varies between calls).
 *   dz and dwt 16-byte aligned, swap (nullable, one view only) 4-byte aligned, n_out a multiple of 64.  At most 8 layouts
 *   (OVC_E_UNSUPPORTED), one grid shape; OVC_E_UNSUPPORTED for a grid whose 32-column gradient table (width*height*19*128 B)
 *   does not fit 227 KB of shared memory.  n_records = 0 launches nothing.
 */
int ovc_encode_linear_wgrad(const void *layouts, int n_layouts, const int32_t *states, const int32_t *swap, int seat, const float *dz,
                            float *dwt, int64_t n_records, int state_words, int width, int height, int horizon, int n_out, void *stream);

/*
 * featurize_state (:2579-2898) with the default planner parameters (NO_COUNTERS_PARAMS,
 * planners.py:27-34): out float32[n_envs][2][F],
 * F = 2*(num_pots*10+28), lut = ovc_feat_lut_entry_t[n_layouts][256][4].  view_swap as above.
 */
int ovc_featurize(const void *layouts, int n_layouts, const void *lut, const int32_t *state,
                  const int32_t *view_swap, float *out, int64_t n_envs, int state_words, int num_pots,
                  void *stream);

/*
 * potential_function (:2920-3250): out double[n_envs] = phi(state) for the gamma the tables were built
 * for.  pot_tables = ovc_potential_t[n_layouts], cost_lut = ovc_cost_lut_entry_t[n_layouts][256][4],
 * gpow = double[n_pow] with gpow[k] = gamma**k as computed by the host (the reference evaluates
 * gamma ** integer in double precision; taking the powers from the host table and following the
 * reference's order of operations makes the result bit-identical, not merely close).
 */
int ovc_potential(const void *layouts, int n_layouts, const void *pot_tables, const void *cost_lut,
                  const double *gpow, int n_pow, const int32_t *state, double *out, int64_t n_envs,
                  int state_words, void *stream);
size_t ovc_potential_table_size(void);

/*
 * The potential-based dense reward (human_aware_rl's use_phi, rllib.py:314-329): both agents get
 *     reward = sparse + factor * dense,   dense = (float)(phi(s') - phi(s))
 * with phi = potential_function at gamma 0.99 (the value get_state_transition(display_phi=True) reports, MDP:1422-1429),
 * s the record before the transition and s' the record after it, BEFORE a finishing episode is reset.  A transition is
 *     ovc_potential (phi_s = phi(s)) -> ovc_step without OVC_F_AUTO_RESET -> ovc_potential_shaping -> ovc_record_transition_dense
 *
 * ovc_potential_shaping: per environment e, with the tables and gpow of ovc_potential and the records ovc_step left:
 *     dense[e] = (float)(phi(state[e]) - phi_s[e])     the float64 difference rounded once; float32 [n_envs]
 *   then, where done[e] != 0 (ovc_step's int32 done), state[e] is reset as OVC_F_AUTO_RESET inside ovc_step would reset it:
 *   the start record of its layout (word 3), or with random_start the random start of the next episode (layout drawn with
 *   random_layout, episode counter + 1, env index e).  phi_s float64 [n_envs] (8-byte aligned), done and dense 4-byte aligned;
 *   n_pow >= 2.
 * ovc_record_transition_dense: ovc_record_transition (stats NULL) or ovc_record_transition_stats (stats given) with the
 *   reward of both agents taken from dense (float32 [n_envs], 4-byte aligned) instead of shaped, each operation rounded
 *   to float32 on its own:
 *     r[e] = (float)sparse[e] + factor * dense[e];  rewards[2 e + i] = r[e] (one_view 0, [n_envs][2], 8-byte aligned) or
 *     rewards[e] = r[e] (one_view 1, [n_envs], 4-byte aligned; an agent pair's learner: no seat, both rewards are equal);
 *     ret_mixed[e] = ((ret_mixed[e] + (float)sparse[e]) + factor * dense[e]) + factor * dense[e]
 *   rewards nullable; reward_by_agent sums r[e] for both agents; shaped feeds shaped_by_agent, and dones, ret_sparse, the
 *   other statistics and the records are exactly what those calls write.
 */
int ovc_potential_shaping(const void *layouts, int n_layouts, const int32_t *start_records, const void *pot_tables, const void *cost_lut,
                          const double *gpow, int n_pow, int32_t *state, const int32_t *done, const double *phi_s, float *dense,
                          int64_t n_envs, int state_words, const ovc_random_start_t *random_start, void *stream);
int ovc_record_transition_dense(const int32_t *sparse, const int32_t *shaped, const float *dense, const int32_t *done, const float *factor,
                                int64_t n_envs, int one_view, float *rewards, uint8_t *dones, int64_t *ret_sparse, float *ret_mixed,
                                const ovc_episode_stats_t *stats, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* OVC_B200_H */
