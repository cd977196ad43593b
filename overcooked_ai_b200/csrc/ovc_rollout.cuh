// ovc_rollout.cuh — K5, the fused T-transition rollout kernel (ovc_rollout, and every chunk of the host-buffer
// pipeline).  Same transition as ovc_step.cuh (reference overcooked_mdp.py:1375-1430 + overcooked_env.py:244-274),
// restated for a kernel that keeps an environment on chip for many transitions:
//
//   * the record header (timestep, both players, misc word) lives in REGISTERS for the whole launch; the shared-memory
//     tile (one 2-D TMA load in, one TMA store out, hardware swizzle) is only touched for object slots, through
//     32-bit shared-window addresses;
//   * per-layout tables are DERIVED in the prologue from the ovc_layout_t records the CTA bulk-copied next to the
//     tile: face[(orientation, pos)] -> the faced cell, move[(action, pos)] -> position after the move (floor test
//     folded in), and the recipe tables re-keyed by the 5-bit (count, kinds) field of a soup code, so the hot loop
//     never does direction arithmetic, terrain tests or popcounts;
//   * NO per-transition pot work: while on chip a pot soup carries the index — on its environment's own clock of
//     transitions run in this launch — of the transition at which it becomes ready, instead of a tick that has to
//     be advanced (step_environment_effects :1691-1703 turns into a comparison made only when somebody holds a dish
//     against the pot), and the aggregates of get_pot_states (:1809-1838) that the usefulness predicates consume are
//     kept in a register that every pot change updates by its known effect; the external tick + 1 form is restored
//     on the way out;
//   * an agent produces at most one interaction per transition, so the interact logic (resolve_interacts
//     :1432-1579) computes the agent's 5-bit EVENT CODE (include/ovc_b200.h, OVC_F_OUT_PACKED) directly; the 25-bit
//     event masks of the int32 format are one shared-memory table lookup of that code, and the 2-byte host-transfer
//     word is the two codes side by side.
//
// One thread owns one environment; the interact body is emitted twice (first interacting player of an environment,
// then player 1 where both interact: most warps skip the second).  Results are bit-identical to step_kernel (tests
// replay every fixture through both).  Included by ovc_b200.cu after the PTX helpers and StepArgs.
#pragma once

// Action rows prefetched into L2 ahead of the transition loop.  The demand load of a transition's joint action is
// issued one transition ahead; on its own it is a DRAM read, and each transition starts by waiting for it.  With
// OVC_K5_PREFETCH = D >= 2 every thread also prefetches its own action D rows ahead (prefetch.global.L2: no register,
// no scoreboard), so the demand load hits L2.  0 (or 1): no prefetch, the kernel of the plain distance-1 load.  The
// host turns the prefetch off for a launch whose grid is resident in one wave at fewer than 12 or at least 24 warps per
// SM (launch_rollout).
#ifndef OVC_K5_PREFETCH
#define OVC_K5_PREFETCH 4
#endif

namespace ovc {

struct Derived {
    uint16_t face[1024];      // [(orientation << 8) | pos] -> ovc_layout_t.cell[] word of the cell the player faces
    uint8_t move[2048];       // [((action & 7) << 8) | pos] -> pos after the move; pos itself if blocked, STAY, INTERACT
    int32_t cook5[32];        // [(code >> 3) & 31] -> Recipe.time of a soup with that (count, kinds) field
    int32_t deliver5[32];     //                    -> its delivery reward (get_recipe_value :1581-1602)
    uint8_t potcode5[32][2];  //                    -> event code of potting an onion / a tomato INTO that soup
    uint8_t dcode5[32];       //                    -> event code of delivering that soup (23 + recipe rank)
    uint8_t pad[32];
};
static_assert(sizeof(Derived) == 4480, "Derived table size");
constexpr int DERIVED_ZERO_CHUNKS = (1024 * 2 + 2048) / 16;  // face + move, zero filled before the floor cells are written
#define OVC_DOFF(field) ((uint32_t)offsetof(Derived, field))
#define OVC_LOFF(field) ((uint32_t)offsetof(ovc_layout_t, field))

// On-chip pot word: bits 0-7 as in the record (type, count, kinds); bits 8-30 "clock": 0 = idle, else 1 + the index
// (environment clock: transitions the environment has run in this launch) of the first transition whose interacts
// see the soup ready; bit 31 "frozen": the soup was loaded with tick > cook time (ready; bits 8-21 keep its tick + 1).
constexpr unsigned POT_FROZEN = 1u << 31;
constexpr int ROLLOUT_MAX_STEPS = 1 << 22;  // clock field: n_steps + cook time + 1 < 2^23

// ---- shared memory through 32-bit window addresses ----
// tile words change during the launch: volatile + memory clobber keeps program order
__device__ __forceinline__ unsigned lds_tile(uint32_t a) {
    unsigned v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void sts_tile(uint32_t a, unsigned v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ int4 lds_tile4(uint32_t a) {
    int4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void sts_tile4(uint32_t a, int4 v) {
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
// tables are read-only once the prologue's barrier has passed (volatile keeps them behind it, nothing more)
__device__ __forceinline__ unsigned lds_tbl32(uint32_t a) {
    unsigned v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ unsigned lds_tbl16(uint32_t a) {
    unsigned short v;
    asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ unsigned lds_tbl8(uint32_t a) {
    unsigned v;
    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}

__device__ __forceinline__ int recipe_row5(unsigned k5) {  // (count, kinds) field -> n_onion*4 + n_tomato
    const int n = k5 & 3;
    const int nt = __popc((k5 >> 2) & ((1u << n) - 1u));
    return ((n - nt) << 2) | nt;
}

// 5-bit event code -> 25-bit event mask (+ delivered recipe in bits 25-28); inverse of event_code()
__device__ __forceinline__ unsigned code_mask_of(int c) {
    if (c == 0) return 0u;
    if (c <= 6) {
        const int b = (0x0A0005 >> (((c - 1) >> 1) * 8)) & 0xFF;  // onion / tomato / dish _pickup
        return (1u << b) | ((unsigned)((c - 1) & 1) << (b + 1));
    }
    if (c == 7) return 1u << OVC_EV_SOUP_PICKUP;
    if (c <= 13) {
        const int b = (0x0C0207 >> (((c - 8) >> 1) * 8)) & 0xFF;  // onion / tomato / dish _drop
        return (1u << b) | ((unsigned)((c - 8) & 1) << (b + 1));
    }
    if (c == 14) return 1u << OVC_EV_SOUP_DROP;
    if (c <= 22) {
        const int tom = (c - 15) >> 2, cls = (c - 15) & 3;
        const unsigned base = 1u << (tom ? OVC_EV_POTTING_TOMATO : OVC_EV_POTTING_ONION);
        const unsigned opt = 1u << (OVC_EV_OPTIMAL_ONION_POTTING + tom), via = 1u << (OVC_EV_VIABLE_ONION_POTTING + tom);
        const unsigned cat = 1u << (OVC_EV_CATASTROPHIC_ONION_POTTING + tom), usl = 1u << (OVC_EV_USELESS_ONION_POTTING + tom);
        return base | (cls == 0 ? (opt | via) : cls == 1 ? via : cls == 2 ? cat : (opt | usl));
    }
    const unsigned row = (unsigned)((0xC98654321ull >> ((c - 23) * 4)) & 15u);  // rank -> n_onion*4 + n_tomato
    return (1u << OVC_EV_SOUP_DELIVERY) | (row << OVC_EV_RECIPE_SHIFT);
}

// Shared-memory record of one thread.  The TMA swizzle XORs the 16-byte-chunk index with address bits 7.. ; for
// records of at most one 128-byte row that XOR term is a per-thread constant.
template <int S, int SWZ>
struct TileRec {
    uint32_t rec;  // shared-window address of the record: tile + tid * S * 4
    uint32_t xm;   // S <= 32: the thread's constant XOR term;  S > 32: row index of the record's first 128-byte row
    __device__ __forceinline__ TileRec(uint32_t tile, int tid) {
        rec = tile + (uint32_t)tid * S * 4;
        if (SWZ == 0) xm = 0;
        else if (S <= 32) xm = ((((uint32_t)tid * S * 4) >> 7) & ((1u << SWZ) - 1u)) << 4;
        else xm = (uint32_t)tid * (S / 32);
    }
    __device__ __forceinline__ uint32_t phys(uint32_t off) const {
        if (SWZ == 0) return off;
        if (S <= 32) return off ^ xm;
        return off ^ (((xm + (off >> 7)) & 7u) << 4);
    }
    __device__ __forceinline__ int4 ld4(int c) const { return lds_tile4(rec + phys((uint32_t)c * 16)); }
    __device__ __forceinline__ void st4(int c, int4 v) const { sts_tile4(rec + phys((uint32_t)c * 16), v); }
    __device__ __forceinline__ uint32_t addr(int w) const { return rec + phys((uint32_t)w * 4); }
    __device__ __forceinline__ unsigned ldw(int w) const { return lds_tile(addr(w)); }
    __device__ __forceinline__ void stw(int w, unsigned v) const { sts_tile(addr(w), v); }
};

// external pot word (tick + 1 in bits 8-21) <-> on-chip form; `clk` = index of the next transition of this launch
__device__ __forceinline__ unsigned pot_to_chip(unsigned w, uint32_t D, unsigned clk) {
    const unsigned tp1 = (w >> 8) & 0x3FFFu;
    if ((w & 7u) != OVC_O_SOUP || tp1 == 0) return w & 0x3FFFFFu;
    const unsigned cook = lds_tbl32(D + OVC_DOFF(cook5) + 4u * ((w >> 3) & 31u));
    if (tp1 - 1u > cook) return (w & 0x3FFFFFu) | POT_FROZEN;  // hand-built over-cooked soup: ready, keeps its tick
    return (w & 0xFFu) | ((clk + (cook - (tp1 - 1u)) + 1u) << 8);  // ready once `cook - tick` more transitions have run
}
__device__ __forceinline__ unsigned pot_to_ext(unsigned w, uint32_t D, unsigned clk) {
    if (w & POT_FROZEN) return w & 0x3FFFFFu;
    const unsigned g = w >> 8;
    if (g == 0) return w;
    const unsigned cook = lds_tbl32(D + OVC_DOFF(cook5) + 4u * ((w >> 3) & 31u));
    const unsigned left = g - 1u > clk ? g - 1u - clk : 0u;  // transitions still to run before it is ready
    return (w & 0xFFu) | ((cook - left + 1u) << 8);
}

struct RollOut {
    int sparse, sh0, sh1;
    unsigned c0, c1;  // event codes
};

// Aggregates of the pot snapshot (get_pot_states :1809-1838) that the usefulness predicates consume, in one register:
//   bits 0-3  n_full: pots that are full (cooking, ready, or idle with 3 ingredients; get_full_pots :1875-1880)
//   bits 4-7  n_dish: pots a dish is useful for (ready + cooking + idle with 1 or 2; is_dish_pickup_useful :2199-2203)
// Computed from the pot words when a record is loaded; afterwards every pot change updates it by its known effect:
//   ingredient into an empty pot / onto 1 ingredient / onto 2:  n_dish + 1 / nothing / n_full + 1, n_dish - 1
//   cooking starts on 1-2 ingredients / on 3:                    n_full + 1 / n_dish + 1
//   a ready soup is plated:                                      n_full - 1, n_dish - 1
constexpr unsigned PS_FULL = 1u, PS_DISH = 1u << 4;
template <class R>
__device__ __forceinline__ unsigned pot_summary(const R &r, int n_pots) {
    unsigned ps = 0;
#pragma unroll 1
    for (int k = 0; k < n_pots; k++) {
        const unsigned w = r.ldw(4 + k);
        const bool soup = (w & 7u) == OVC_O_SOUP;
        const bool idle = (w >> 8) == 0;
        const unsigned n = (w >> 3) & 3u;
        if (soup && (!idle || n == 3u)) ps += PS_FULL;
        if (soup && (!idle || n == 1u || n == 2u)) ps += PS_DISH;
    }
    return ps;
}

// One player's INTERACT (:1446-1577) -> the player's event code.  `ps`: pot_summary as it was before either player
// acted in this transition (quirk Q3); pot changes go to `psn`, which becomes the next transition's snapshot.
// `s` = the environment's clock: index of this transition among those it has run in this launch.
template <class R>
__device__ __forceinline__ unsigned interact_v2(const R &r, uint32_t L, uint32_t D, unsigned &me, const unsigned other_t,
                                                unsigned &misc, const unsigned ps, unsigned &psn, const int n_pots,
                                                const bool old_dyn, const unsigned s, int &sparse, int &shaped) {
    const unsigned cell = lds_tbl16(D + OVC_DOFF(face) + 2u * (me & 0x3FFu));
    const unsigned terr = cell & 7u;
    unsigned held = me >> 10;
    const unsigned ht = held & 7u;
    unsigned code = 0;
    if (terr - 1u < 4u) {  // counter 'X' (:1458-1485) or a dispenser 'O' 'T' 'D' (:1487-1513), which hands out object terr - 1
        const bool ctr = terr == OVC_T_COUNTER;
        const uint32_t wa = r.addr(4 + (int)(cell >> 8));
        unsigned cw = terr - 1u;
        if (ctr) cw = lds_tile(wa);
        const bool pick = held == 0 && cw != 0;
        const bool drop = ctr && held != 0 && cw == 0;
        if (pick || drop) {
            const unsigned ot = (held | cw) & 7u;  // the object that changes hands
            const unsigned n_full = ps & 15u;
            bool u;
            if (ot == OVC_O_DISH)  // is_dish_pickup_useful :2180-2204 / is_dish_drop_useful :2206-2221
                u = pick ? ((misc & 0xFF00u) == 0 && (other_t == OVC_O_DISH ? 1u : 0u) < (ps >> 4)) : (n_full == 0 && other_t != OVC_O_ONION);
            else  // is_ingredient_pickup_useful :2223-2237 / _drop_ :2239-2254 (a soup: never)
                u = ot <= OVC_O_TOMATO && pick != (n_full == (unsigned)n_pots && other_t != OVC_O_DISH);
            code = 2u * ot + (pick ? 0xFFFFFFFFu : 6u) + (unsigned)u;  // pickup codes 1-7, drop codes 8-14
            if (ctr) {
                sts_tile(wa, held);  // drop: the object; pickup: 0
                if (ot == OVC_O_DISH) misc += pick ? 0xFFFFFF00u : 0x100u;  // loose-dish count in bits 8-15
            } else {
                if (ot == OVC_O_TOMATO) code = 0;  // a tomato from the dispenser logs nothing (quirk Q5)
                if (ot == OVC_O_DISH && u) shaped += (int)lds_tbl32(L + OVC_LOFF(rew_dish_pickup));
            }
            held = pick ? cw : 0u;
        }
    } else if (terr == OVC_T_POT) {
        const uint32_t wa = r.addr(4 + (int)(cell >> 8));
        const unsigned w = lds_tile(wa);
        const unsigned k5 = (w >> 3) & 31u;
        const unsigned n = k5 & 3u;
        if (ht == 0) {  // :1515-1522 start cooking an idle, non-empty soup (new dynamics only): tick 0 now, ready `cook` transitions on
            if (!old_dyn && (w & ~0xF8u) == OVC_O_SOUP && n != 0) {
                sts_tile(wa, w | ((s + lds_tbl32(D + OVC_DOFF(cook5) + 4u * k5) + 1u) << 8));
                psn += n == 3u ? PS_DISH : PS_FULL;
            }
        } else if (ht == OVC_O_DISH) {  // :1525-1539 plate a ready soup
            const unsigned g = w >> 8;
            if ((int)w < 0 || g - 1u <= s) {  // frozen, or its clock has run out (g == 0, idle, wraps to "never")
                code = 7;
                held = pot_to_ext(w, D, s);   // a ready soup leaves the pot with tick == cook time (or its frozen tick)
                sts_tile(wa, 0u);
                shaped += (int)lds_tbl32(L + OVC_LOFF(rew_soup_pickup));
                psn -= PS_FULL + PS_DISH;
            }
        } else if (ht <= OVC_O_TOMATO) {  // :1541-1568 add an ingredient (an empty pot gets a fresh soup first)
            if ((w >> 8) == 0 && n < 3u) {
                const unsigned tom = ht == OVC_O_TOMATO;
                code = lds_tbl8(D + OVC_DOFF(potcode5) + 2u * k5 + tom);
                sts_tile(wa, ((w ? w : (unsigned)OVC_O_SOUP) + 8u) | (tom << (5 + n)));
                shaped += (int)lds_tbl32(L + OVC_LOFF(rew_placement_in_pot));
                held = 0;
                psn += n == 0 ? PS_DISH : n == 2u ? PS_FULL - PS_DISH : 0u;
            }
        }
    } else if (terr == OVC_T_SERVE && ht == OVC_O_SOUP) {  // :1570-1577, deliver_soup :1631-1642
        const unsigned k5 = (held >> 3) & 31u;
        sparse += (int)lds_tbl32(D + OVC_DOFF(deliver5) + 4u * k5);
        code = lds_tbl8(D + OVC_DOFF(dcode5) + k5);
        held = 0;
    }
    me = (me & 0x3FFu) | (held << 10);
    return code;
}

// Kernel instantiations by transfer format: the device-resident int32 formats carry none of the format tests
// (3 % of a transition when they sat in every instantiation), the sparse event stream carries the warp votes.
constexpr int FMT_WIDE = 0, FMT_HOST = 1, FMT_STREAM = 2;

// A flags bit the host sets per launch (launch_rollout; the ABI's flags leave bits 12-15 free): skip the action prefetch.
constexpr int F_K5_NO_PREFETCH = 1 << 12;

// Output / action addressing of one thread: ONE 32-bit element index per stream (outputs, actions), advanced by n_envs
// per transition; every array address is then a single IMAD.WIDE of that index onto the array's base pointer.  (The
// host keeps n_steps * n_envs below 2^32 per launch by cutting longer rollouts into several launches.)
template <int FMT>
struct RollIO {
    static constexpr bool WIDE = FMT == FMT_WIDE;
    const StepArgs &a;
    unsigned oi, ai;  // element index of this transition's outputs / of the action row loaded last
    const unsigned n;
    // FMT_STREAM: lane-mask rows uint32[n_steps][n_groups] (index mi), the group's slice of uint16[n_groups][cap]
    unsigned live_mask, cnt, cap, lane_lt, mi, n_groups;
    unsigned short *vals;
    bool leader;
    __device__ __forceinline__ RollIO(const StepArgs &args, long long env, unsigned live) : a(args), n((unsigned)args.n_envs) {
        oi = ai = (unsigned)env;
        live_mask = live, cnt = 0, cap = 0, lane_lt = 0, mi = 0, n_groups = 0, vals = nullptr, leader = false;
        if (FMT == FMT_STREAM) {
            n_groups = (unsigned)((a.n_envs + 31) >> 5);
            mi = (unsigned)(env >> 5);
            cap = ((unsigned)a.flags >> OVC_F_STREAM_CAP_SHIFT) & 0xFFFFu;
            const unsigned lane = (unsigned)env & 31u;
            lane_lt = (1u << lane) - 1u, leader = lane == 0;
            vals = reinterpret_cast<unsigned short *>(a.sparse) + (size_t)mi * cap;
        }
    }
    __device__ __forceinline__ int2 load_action() const { return ovc::load_action<WIDE>(a, ai); }
    __device__ __forceinline__ void next_action() { ai += n; }
    // L2 prefetch of the action `rows` rows after the one loaded last (the caller keeps that row below n_steps)
    __device__ __forceinline__ void prefetch_action(unsigned rows) const { prefetch_l2(action_addr<WIDE>(a, ai + rows * n)); }
    // Writes this transition's outputs and advances to the next transition.  FMT_STREAM: called at ONE program point by
    // every live thread of the warp, once per transition (it votes across the warp).
    __device__ __forceinline__ void write(const RollOut &o, int done_v, bool stepped, uint32_t mask) {
        const unsigned i = oi;
        oi += n;
        if (FMT == FMT_STREAM) {
            // What a rollout produces is mostly zeros.  Per warp (32 consecutive environments) and transition: ONE
            // 32-bit lane mask of the non-zero code words (__ballot_sync), and the non-zero words compacted behind the
            // group's earlier ones (rank among the voters = popcount of the lower lanes).
            const unsigned w = o.c0 | (o.c1 << 5) | ((unsigned)done_v << 10) | (stepped ? 1u << 11 : 0u) |
                               (o.sh0 != 0 ? 1u << 12 : 0u) | (o.sh1 != 0 ? 1u << 13 : 0u);
            const unsigned m = __ballot_sync(live_mask, w != 0);
            if (leader) reinterpret_cast<unsigned *>(a.events)[mi] = m;
            mi += n_groups;
            if (w != 0) {
                const unsigned pos = cnt + __popc(m & lane_lt);
                if (pos < cap) vals[pos] = (unsigned short)w;  // beyond cap: dropped, the masks tell
            }
            cnt += __popc(m);
            if (a.done) reinterpret_cast<unsigned short *>(a.done)[i] = (unsigned short)w;  // dense backup
            return;
        }
        if (!WIDE && (a.flags & (OVC_F_OUT_CODES | OVC_F_OUT_PACKED))) {
            unsigned w = o.c0 | (o.c1 << 5) | ((unsigned)done_v << 10) | (stepped ? 1u << 11 : 0u);
            if (a.flags & OVC_F_OUT_CODES) {
                w |= (o.sh0 != 0 ? 1u << 12 : 0u) | (o.sh1 != 0 ? 1u << 13 : 0u);
            } else {
                reinterpret_cast<short *>(a.sparse)[i] = (short)o.sparse;
                reinterpret_cast<char2 *>(a.shaped)[i] = make_char2((signed char)o.sh0, (signed char)o.sh1);
            }
            reinterpret_cast<unsigned short *>(a.events)[i] = (unsigned short)w;
            return;
        }
        const unsigned e0 = stepped ? (unsigned)OVC_EVF_STEPPED_DONE : lds_tbl32(mask + 4u * o.c0);
        const unsigned e1 = stepped ? (unsigned)OVC_EVF_STEPPED_DONE : lds_tbl32(mask + 4u * o.c1);
        if (!WIDE && (a.flags & OVC_F_OUT_NARROW)) {
            reinterpret_cast<short *>(a.sparse)[i] = (short)o.sparse;
            reinterpret_cast<unsigned char *>(a.done)[i] = (unsigned char)done_v;
            reinterpret_cast<char2 *>(a.shaped)[i] = make_char2((signed char)o.sh0, (signed char)o.sh1);
        } else {
            a.sparse[i] = o.sparse;
            a.done[i] = done_v;
            reinterpret_cast<int2 *>(a.shaped)[i] = make_int2(o.sh0, o.sh1);
        }
        reinterpret_cast<int2 *>(a.events)[i] = make_int2((int)e0, (int)e1);
    }
};

// Shared-memory plan (1024-byte aligned): [ tile TILE*S*4 ][ ovc_layout_t x n_layouts ][ Derived x n_layouts ]
//                                         [ event-mask table 128 B ][ mbarrier 8 B ]
template <int S, int TILE>
struct RollCfg {
    static constexpr int ROW_WORDS = S == 16 ? 16 : 32;
    static constexpr int ROWS_PER_ENV = S / ROW_WORDS;
    static constexpr int BOX_ROWS = TILE * ROWS_PER_ENV;
    static constexpr int SWZ = S == 16 ? 2 : 3;
    static constexpr int TILE_BYTES = TILE * S * 4;
    static_assert(BOX_ROWS <= 256, "TMA box rows");
    static_assert(TILE_BYTES % 1024 == 0, "tile must keep the swizzle alignment of what follows");
    static size_t smem_bytes(int n_layouts) { return (size_t)TILE_BYTES + (size_t)n_layouts * (sizeof(ovc_layout_t) + sizeof(Derived)) + 128 + 16; }
};

template <int S, int TILE, bool RS, int FMT>
__global__ void __launch_bounds__(TILE)
rollout_kernel(const __grid_constant__ CUtensorMap tmap, const StepArgs a) {
    using C = RollCfg<S, TILE>;
    constexpr bool WIDE = FMT == FMT_WIDE;
    const int tid = threadIdx.x;
    const long long env0 = (long long)blockIdx.x * TILE;
    const long long env = env0 + tid;
    const bool live = env < a.n_envs;
    const int T = a.n_steps;
    const int n_tbl = a.n_layouts;  // host guarantees n_layouts <= MAX_SMEM_LAYOUTS for this kernel

    extern __shared__ __align__(1024) char smem[];
    char *tile = smem;
    ovc_layout_t *tbl = reinterpret_cast<ovc_layout_t *>(smem + C::TILE_BYTES);
    Derived *der = reinterpret_cast<Derived *>(smem + C::TILE_BYTES + (size_t)n_tbl * sizeof(ovc_layout_t));
    unsigned *mask = reinterpret_cast<unsigned *>(reinterpret_cast<char *>(der) + (size_t)n_tbl * sizeof(Derived));
    uint64_t *bar = reinterpret_cast<uint64_t *>(mask + 32);
    const uint32_t tbl_bytes = (uint32_t)n_tbl * (uint32_t)sizeof(ovc_layout_t);

    if (tid == 0) {
        mbar_init(bar, 1);
        mbar_expect_tx(bar, (uint32_t)C::TILE_BYTES + tbl_bytes);
        prefetch_tmap(&tmap);
        bulk_load_1d(tbl, a.layouts, tbl_bytes, bar);
    }
    // zero the derived move / face tables and build the code -> mask table while the copies fly (constants only:
    // legal before the programmatic-dependent-launch wait)
    for (int l = 0; l < n_tbl; l++)
        for (int i = tid; i < DERIVED_ZERO_CHUNKS; i += TILE) reinterpret_cast<int4 *>(der + l)[i] = make_int4(0, 0, 0, 0);
    if (tid < 32) mask[tid] = code_mask_of(tid);
    asm volatile("griddepcontrol.wait;" ::: "memory");
    if (tid == 0) tma_load_2d(tile, &tmap, 0, (int)(env0 * C::ROWS_PER_ENV), bar);  // rows past the end: zero fill, still counted
    int2 act = make_int2(OVC_A_STAY, OVC_A_STAY);
    if (live) act = load_action<WIDE>(a, env);
#if OVC_K5_PREFETCH > 1
    // rows 1 .. D-1; the transition loop prefetches row s + D in transition s
    const bool prefetch = !(a.flags & F_K5_NO_PREFETCH);
    if (live && prefetch)
        for (int k = 1; k < OVC_K5_PREFETCH && k < T; k++) prefetch_l2(action_addr<WIDE>(a, (unsigned)env + (unsigned)k * (unsigned)a.n_envs));
#endif
    __syncthreads();  // barrier initialised + zero fill complete
    mbar_wait(bar, 0);
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

    // ---- derive the per-layout tables from the records that just landed ----
    for (int l = 0; l < n_tbl; l++) {
        const ovc_layout_t *L = tbl + l;
        Derived *D = der + l;
        if (tid < 32) {
            const unsigned k5 = tid;
            const int n = k5 & 3, row = recipe_row5(k5);
            D->cook5[k5] = L->cook_time[row];
            D->deliver5[k5] = L->deliver_value[row];
            D->dcode5[k5] = (uint8_t)(23u + (unsigned)((0x0008007605432100ull >> (row * 4)) & 15u));
            const int old_val = L->best_value[n ? row : 0];
#pragma unroll
            for (int tom = 0; tom < 2; tom++) {  // log_object_potting :2121-2140 + is_potting_* :2256-2308
                int cls = 0;
                if (n < 3) {
                    const int new_val = L->best_value[recipe_row5((k5 + 1u) | ((unsigned)tom << (2 + n)))];
                    cls = new_val > 0 ? (old_val == new_val ? 0 : 1) : (old_val > 0 ? 2 : 3);
                }
                D->potcode5[k5][tom] = (uint8_t)(15 + 4 * tom + cls);
            }
        }
        const int n_free = L->n_free;
        for (int i = tid; i < n_free * 12; i += TILE) {  // only floor cells can hold a player
            const int f = i / 12, d = i - f * 12;
            const int pos = L->free_pos[f];
            if (d < 4) {
                D->face[(d << 8) | pos] = L->cell[(pos + dir_delta(d)) & 0xFF];
            } else {
                const int act_i = d - 4;
                int np = pos;
                if (act_i < 4) {
                    const int tp = (pos + dir_delta(act_i)) & 0xFF;
                    if ((L->cell[tp] & 7) == OVC_T_FLOOR) np = tp;
                }
                D->move[(act_i << 8) | pos] = (uint8_t)np;
            }
        }
    }
    __syncthreads();

    const unsigned live_mask = __ballot_sync(0xFFFFFFFFu, live);  // the warp's live lanes (a partial last tile)
    if (live) {
        const TileRec<S, C::SWZ> r(smem_u32(tile), tid);
        const uint32_t tbl_s = smem_u32(tbl), der_s = smem_u32(der), mask_s = smem_u32(mask);
        // ---- register-resident part of the record + the thread's layout ----
        int t;
        unsigned toff;  // environment clock = t + toff: transitions this environment has RUN in this launch (a finished,
                        // un-reset environment stands still, and so do its soups)
        unsigned p0, p1, misc, ps, psn;  // ps: pot snapshot of this transition, psn: what the next one will see
        uint32_t L, D;  // shared-window addresses of the thread's ovc_layout_t / Derived
        int n_pots;
        bool old_dyn;
        auto load_regs = [&](unsigned clk) {  // after the tile landed and after every (auto) reset
            const int4 h = r.ld4(0);
            t = h.x, p0 = (unsigned)h.y, p1 = (unsigned)h.z, misc = (unsigned)h.w;
            toff = clk - (unsigned)t;
            unsigned lid = misc & 0xFFu;
            if (lid >= (unsigned)n_tbl) lid = 0;
            L = tbl_s + lid * (uint32_t)sizeof(ovc_layout_t), D = der_s + lid * (uint32_t)sizeof(Derived);
            n_pots = (int)lds_tbl32(L + OVC_LOFF(n_pots));
            old_dyn = (lds_tbl32(L + OVC_LOFF(flags)) & OVC_LAYOUT_OLD_DYNAMICS) != 0;
#pragma unroll 1
            for (int k = 0; k < n_pots; k++) r.stw(4 + k, pot_to_chip(r.ldw(4 + k), D, clk));
            ps = psn = pot_summary(r, n_pots);
        };
        load_regs(0u);

        RollIO<FMT> io(a, env, live_mask);

        // one player's interact on the live record (:1446-1577); `second`: the acting player is player 1
        auto interact = [&](bool second, RollOut &o) {
            unsigned pa = second ? p1 : p0;
            const unsigned pb = second ? p0 : p1;
            int sh = 0;
            const unsigned c = interact_v2(r, L, D, pa, (pb >> 10) & 7u, misc, ps, psn, n_pots, old_dyn, (unsigned)t + toff, o.sparse, sh);
            if (second) p1 = pa, o.sh1 = sh, o.c1 = c;
            else p0 = pa, o.sh0 = sh, o.c0 = c;
        };
        // everything of a transition after the interacts: movement, environment effects, outputs, episode end
        auto finish = [&](int a0, int a1, const RollOut &o, bool stepped) {
            int done = 1;
            if (!stepped) {
                // ---- resolve_movement :1644-1727; a blocked or collided player still turns (quirk Q8) ----
                const unsigned o0 = p0 & 0xFFu, o1 = p1 & 0xFFu;
                unsigned n0 = lds_tbl8(D + OVC_DOFF(move) + ((((unsigned)a0 & 7u) << 8) | o0));
                unsigned n1 = lds_tbl8(D + OVC_DOFF(move) + ((((unsigned)a1 & 7u) << 8) | o1));
                const bool collide = n0 == n1 || (n0 == o1 && n1 == o0);  // :1673-1683
                if (collide) n0 = o0, n1 = o1;
                if ((unsigned)a0 < 4u) p0 = (p0 & ~0x3FFu) | ((unsigned)a0 << 8) | n0;
                if ((unsigned)a1 < 4u) p1 = (p1 & ~0x3FFu) | ((unsigned)a1 << 8) | n1;
                // ---- step_environment_effects :1691-1703: cooking soups carry their ready clock, nothing to advance.
                //      Old dynamics: an idle soup with 3 ingredients starts by itself (:1696-1701), tick 0 -> 1 in this
                //      transition, i.e. the same clock as a soup started by an interact of this transition ----
                if (old_dyn) {
#pragma unroll 1
                    for (int k = 0; k < n_pots; k++) {
                        const unsigned w = r.ldw(4 + k);
                        if ((w & ~0xE0u) == (OVC_O_SOUP | (3u << 3))) {
                            r.stw(4 + k, w | (((unsigned)t + toff + lds_tbl32(D + OVC_DOFF(cook5) + 4u * ((w >> 3) & 31u)) + 1u) << 8));
                            psn += PS_DISH;  // idle with 3 (full, no dish wanted) -> cooking (full, a dish will be wanted)
                        }
                    }
                }
                ps = psn;  // next transition's snapshot
                done = a.horizon > 0 && t + 1 >= a.horizon;  // is_done overcooked_env.py:321-325
            }
            io.write(o, done, stepped, mask_s);
            if (stepped) return;
            if (done && (a.flags & OVC_F_AUTO_RESET)) {
                const unsigned lid0 = misc & 0xFFu;
                if (RS && a.has_rs) {
                    const unsigned episode = ((misc >> 16) + 1u) & 0xFFFFu;
                    int lid = (int)lid0;
                    if (a.rs.random_layout) lid = random_layout_id(a.rs, (uint64_t)env, episode, a.n_layouts);  // variable MDP
                    const ovc_layout_t *Ln = tbl + lid;
                    random_start_record([&](int w, int32_t v) { r.stw(w, (unsigned)v); }, S, a.start_records + (size_t)lid * S,
                                        Ln->cook_time, Ln->free_pos, Ln->n_free, Ln->n_pots, lid, a.rs, (uint64_t)env, episode);
                } else {
                    const int4 *__restrict__ src = reinterpret_cast<const int4 *>(a.start_records + (size_t)lid0 * S);
#pragma unroll 4
                    for (int c = 0; c < S / 4; c++) r.st4(c, __ldg(src + c));
                }
                load_regs((unsigned)t + toff + 1u);
            } else {
                t = t + 1;
            }
        };

        for (int s = 0; s < T; s++) {
            int2 nxt = act;
            io.next_action();
            if (s + 1 < T) nxt = io.load_action();  // prefetch
#if OVC_K5_PREFETCH > 1
            if (prefetch && s + OVC_K5_PREFETCH < T) io.prefetch_action(OVC_K5_PREFETCH - 1);  // row s + D into L2
#endif
            const int a0 = act.x, a1 = act.y;
            act = nxt;
            RollOut o{0, 0, 0, 0u, 0u};
            bool stepped = a.horizon > 0 && t >= a.horizon;  // a finished env: untouched + flagged (overcooked_env.py:255)
            if (FMT != FMT_STREAM) {  // its own exit: the common path below then carries no "stepped" selects
                if (stepped) {
                    io.write(o, 1, true, mask_s);
                    continue;
                }
                stepped = false;
            }
            if (!stepped) {
                // two emissions of the interact body: the first serves, per environment, the first interacting player,
                // the second player 1 where BOTH interact (1 environment in 36 under a uniform policy)
                const bool i0 = a0 == OVC_A_INTERACT, i1 = a1 == OVC_A_INTERACT;
                if (i0 || i1) interact(!i0, o);
                if (i0 && i1) interact(true, o);
            }
            // FMT_STREAM: ONE program point for the warp votes, so finished environments go through it as well
            finish(a0, a1, o, FMT == FMT_STREAM && stepped);
        }
        // ---- registers and pot clocks back into the tile in the external format ----
#pragma unroll 1
        for (int k = 0; k < n_pots; k++) r.stw(4 + k, pot_to_ext(r.ldw(4 + k), D, (unsigned)t + toff));
        r.st4(0, make_int4(t, (int)p0, (int)p1, (int)misc));
    }
    fence_async_smem();  // generic-proxy writes -> visible to the async proxy (TMA store)
    __syncthreads();
    if (tid == 0) {
        tma_store_2d(&tmap, 0, (int)(env0 * C::ROWS_PER_ENV), tile);  // rows past the end are clipped
        bulk_commit();
        bulk_wait_read<0>();
    }
}

}  // namespace ovc
