/* mp_oracle.c -- CPU restatement of the Melting Pot hot path (TEST INFRASTRUCTURE ONLY).
 *
 * PARITY UNPINNED: the arithmetic of this path lives in the third-party engine
 * dmlab2d==1.0.0 (requirements.txt:339), which is neither vendored nor
 * installable here, and the reference's tests hold no golden pixels / reward traces / RNG
 * known-answers for it (SURVEY.md section 8c). This file restates
 *   (1) the Melting Pot Lua scheduling + components, citing file:line for every function, and
 *   (2) the engine rules they rely on, as the named policies of DESIGN.md "Engine policy ledger"
 *       (SURVEY.md Appendix A), each implemented in exactly one function below.
 * What IS pinned: Philox4x32-10 known answers (Random123), and the behaviours the reference's
 * Lua tests state (game_object_test.lua:252-411) -- see tests/test_oracle_semantics.py.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's CPU legs (cpu_baseline, --impl reference) may load this library.
 * The product (meltingpot_b200/csrc) shares no code with it except include/mpb_format.h
 * (the blob layout).
 *
 * Structure mirrors the reference: an engine core (pieces on a layered grid, a deferred action
 * queue, contact/hit/state callbacks -- docs/advanced.md:7-56) and components dispatched by type.
 */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../include/mpb_format.h"

#define OR_MAX_PLAYERS 16
#define OR_MAX_LAYERS 16
#define OR_MAX_ROUNDS 128 /* policy A.4: grid:update flushCount */

/* ------------------------------------------------------------------------------------------
 * RNG: Philox4x32-10 (Salmon et al., SC'11), counter-based so that the CUDA engine can draw
 * the same numbers in any schedule. Policy A.16: the reference's mt19937_64 stream is out of
 * reach; every draw is addressed by (seed, episode, frame, stream, index).
 * ---------------------------------------------------------------------------------------- */
enum { RS_SCENE = 0, RS_AVATAR = 1, RS_OBJECT = 2, RS_AVATAR_RESET = 3, RS_OBJECT_RESET = 4, RS_CHOICE = 5 };
enum { SCENE_DRAW_DIRT = 0, SCENE_DRAW_EPISODE_END = 1 };

static void philox4x32_10(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4]) {
  uint32_t c0 = ctr[0], c1 = ctr[1], c2 = ctr[2], c3 = ctr[3], k0 = key[0], k1 = key[1];
  for (int r = 0; r < 10; ++r) {
    uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;
    uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0, n1 = (uint32_t)p1;
    uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1, n3 = (uint32_t)p0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

void oracle_philox(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4]) { philox4x32_10(ctr, key, out); }

static inline double u01(uint32_t a, uint32_t b) { /* 53-bit uniform in [0,1) */
  return ((double)(a >> 5) * 67108864.0 + (double)(b >> 6)) / 9007199254740992.0;
}
static inline uint32_t pick(uint32_t w, uint32_t n) { return (uint32_t)(((uint64_t)w * n) >> 32); }

/* ------------------------------------------------------------------------------------------ */
typedef struct { int layer, sprite, contact; uint32_t groups; } StateDef;
typedef struct { int type; int ip[MPB_COMP_NI]; double dp[MPB_COMP_ND]; } CompDef;
typedef struct { int state0, n_states, comp0, n_comps, is_avatar; } KindDef;

typedef struct {
  int kind, state, x, y, orient;
  int layer;       /* current layer, -1 = off grid (policy A.1) */
  int state_frame; /* grid frame at which the current state was entered */
  int prev_state;
  /* component variables */
  int act[4];
  double reward;
  int movement_allowed, freeze, removal;              /* Avatar */
  int spawn_group;
  int zap_cool;                                      /* Zapper */
  int clean_cool, player_cleaned;                    /* Cleaner */
  int player_ate;                                    /* Taste */
  int num_others_cleaned, num_others_ate;            /* AllNonselfCumulants */
  int num_neighbors, dr_started, grass_obj;          /* DensityRegrow */
  int disallow_zapping, no_zap_counter;              /* Zapper (timed zapping prevention) */
  int n_connected, connected[4];                     /* Avatar:connect (pieces that move / turn with it) */
  int health, rewarding_active, claimed_by, never_claimed, destroyed, frames_since_zapped; /* Resource */
  int absent; /* a 'choice' prefab that was not drawn into this episode's map: the piece does not exist */
  int texture_obj, damage_obj;                       /* Resource:postStart */
  int paired_resource;                               /* RewardIndicator */
  int claim_cool;                                    /* ResourceClaimer */
  int level, time_not_initial, marking_avatar;       /* GraduatedSanctionsMarking */
  int partner_match, partner_mismatch;               /* PartnerTracker (coins) */
  int coins_cumulative;                              /* GlobalCoinCollectionTracker.cumulativeCoinsCollected(player) */
  int ore_miners[2], ore_cd[2];                      /* Ore._miners (bit per player), Ore._miningCountdown -- one pair per Ore component */
  int mine_cool;                                     /* MineBeam._coolingTimer */
} Obj;

enum { ACT_SET_STATE, ACT_TURN, ACT_MOVE_REL, ACT_TELEPORT_GROUP, ACT_BEAM, ACT_TELEPORT, ACT_SET_ORIENT };
typedef struct { int type, obj, a, b, c; } Action;

enum { EV_ZAP = 1, EV_EDIBLE_CONSUMED = 2, EV_PLAYER_CLEANED = 3, EV_CLAIMED_RESOURCE = 4, EV_DESTROYED_RESOURCE = 5, EV_SANCTIONING = 6, EV_REMOVAL = 7,
       EV_COIN_CONSUMED = 8 /* a = player, b = 1 match / 0 mismatch */,
       EV_MINING = 9 /* a = player, b = ore type */, EV_EXTRACTION = 10 /* a = player, b = ore type */,
       EV_EXTRACTION_PAIR = 11 /* a = player_a, b = player_b | ore type << 8 */ };
typedef struct { int type, a, b; } Event;

enum { /* updater function ids */
  UF_AVATAR_MOVE, UF_ZAP, UF_RESPAWN, UF_CLEAN, UF_CLEANER_RESET, UF_TASTE_RESET, UF_NONSELF_GET,
  UF_NONSELF_RESET, UF_GLOBAL_RESET, UF_EPISODE_END, UF_ANIMATION, UF_SPROUT,
  UF_PAINTBRUSH, UF_CLAIM, UF_PROVIDE_REWARDS, UF_RELEASE_CLAIM, UF_MARKING_RECOVERY, UF_COIN_REGROW,
  UF_ORE_REGROW_0, UF_ORE_REGROW_1
};
typedef struct { int priority, comp_type, fn, seq; } Updater;

typedef struct OrEnv {
  /* static tables */
  int W, H, L, P, S, topology, max_frames, n_obj, n_kinds, n_sprites, n_hits, n_groups;
  int view_l, view_r, view_f, view_b, n_actions, oob_sprite, oov_sprite, n_scalar;
  StateDef* states; KindDef* kinds; CompDef* comps; int* objdef; int* hits; int* action_table;
  int* sprite_map; int* scalar_obs; uint8_t* atlas; uint8_t* sprite_opaque;
  int avatar_obj[OR_MAX_PLAYERS];
  Updater* updaters; int n_updaters;
  /* dynamic */
  uint32_t key[2];
  int episode, frame, step, cont, done, step_type;
  Obj* obj;
  int* grid;   /* [L][cells] obj id + 1 */
  uint16_t* beam; /* [L][cells] temporary hit sprites (MPB_CELL) */
  Action* q; int qn, qcap; Action* qnext; int qnn, qncap;
  Event* ev; int evn, evcap;
  int order[OR_MAX_PLAYERS]; /* avatar processing order this frame */
  /* scene component variables */
  int dirt_count, clean_count, spawner_t, ending_t;
  int cleaned_flag[OR_MAX_PLAYERS], ate_flag[OR_MAX_PLAYERS];
  uint8_t hit_class[64]; /* 1 = directionHit*, 2 = claimBeam_* */
  int n_choice; int* choice_n; int* obj_choice; /* 'choice' prefabs drawn per env and episode: options per group; per object (group or -1, ticket mask) */
} OrEnv;

static const int DX[4] = {0, 1, 0, -1}, DY[4] = {-1, 0, 1, 0}; /* N E S W (component_library.lua:38-43) */

static void rng(const OrEnv* e, int stream, int index, uint32_t out[4]) {
  uint32_t ctr[4] = {(uint32_t)e->frame, (uint32_t)e->episode, (uint32_t)index, (uint32_t)stream};
  philox4x32_10(ctr, e->key, out);
}

static inline const KindDef* kind_of(const OrEnv* e, const Obj* o) { return &e->kinds[o->kind]; }
static inline const StateDef* state_def(const OrEnv* e, const Obj* o, int s) { return &e->states[kind_of(e, o)->state0 + s]; }
static const CompDef* find_comp(const OrEnv* e, const Obj* o, int type) {
  const KindDef* k = kind_of(e, o);
  for (int i = 0; i < k->n_comps; ++i) if (e->comps[k->comp0 + i].type == type) return &e->comps[k->comp0 + i];
  return 0;
}
static inline int cell_of(const OrEnv* e, int x, int y) { return y * e->W + x; }
static int wrap_or_reject(const OrEnv* e, int* x, int* y);

static void enqueue(OrEnv* e, int type, int obj, int a, int b, int c) {
  if (e->qnn == e->qncap) { e->qncap = e->qncap ? e->qncap * 2 : 256; e->qnext = (Action*)realloc(e->qnext, sizeof(Action) * e->qncap); }
  Action act = {type, obj, a, b, c};
  e->qnext[e->qnn++] = act;
}
static void add_event(OrEnv* e, int type, int a, int b) {
  if (e->evn == e->evcap) { e->evcap = e->evcap ? e->evcap * 2 : 64; e->ev = (Event*)realloc(e->ev, sizeof(Event) * e->evcap); }
  Event ev = {type, a, b};
  e->ev[e->evn++] = ev;
}

/* ------------------------------------------------------------------------------------------
 * Components: callbacks. Each cites the Lua it restates.
 * ---------------------------------------------------------------------------------------- */
/* Avatar:addReward -- avatar_library.lua:364-378 */
static void avatar_add_reward(OrEnv* e, Obj* av, double amount) {
  const CompDef* c = find_comp(e, av, MPB_C_AVATAR);
  if (c->ip[9] /* skipWaitStateRewards */ && av->state == c->ip[2]) return;
  av->reward += amount;
}
static int avatar_is_alive(const OrEnv* e, const Obj* av) { /* avatar_library.lua:493-495 */
  return av->state == find_comp(e, av, MPB_C_AVATAR)->ip[1];
}

/* GameObject:_onEnter -> component onEnter (game_object.lua:316-318). */
static void on_enter(OrEnv* e, int target, int initiator) {
  Obj* t = &e->obj[target]; Obj* ini = &e->obj[initiator];
  const CompDef* ed = find_comp(e, t, MPB_C_EDIBLE);
  if (ed) { /* Edible:onEnter -- clean_up/components.lua:390-408 ; component_library.lua:990-1002 */
    if (t->state == ed->ip[0]) {
      const CompDef* taste = find_comp(e, ini, MPB_C_TASTE);
      const CompDef* avc = find_comp(e, ini, MPB_C_AVATAR);
      if (taste) { /* Taste:consumed -- clean_up/components.lua:446-455 */
        if (taste->ip[0] == 1) avatar_add_reward(e, ini, 0.0);
        else if (taste->ip[0] == 2) avatar_add_reward(e, ini, taste->dp[0]);
        else avatar_add_reward(e, ini, ed->dp[0]);
        ini->player_ate += 1;                 /* Taste:setCumulant :457-464 */
        e->ate_flag[avc->ip[0]] = 1;          /* GlobalData:setAteThisStep :498-500 */
      } else {
        avatar_add_reward(e, ini, ed->dp[0]);
      }
      add_event(e, EV_EDIBLE_CONSUMED, avc->ip[0] + 1, 0);
      enqueue(e, ACT_SET_STATE, target, ed->ip[1], 0, 0);
    }
  }
  const CompDef* coin = find_comp(e, t, MPB_C_COIN);
  if (coin && t->state != coin->ip[0]) { /* Coin:onEnter -- coins/components.lua:87-160 */
    const CompDef* avc = find_comp(e, ini, MPB_C_AVATAR);
    const CompDef* role = find_comp(e, ini, MPB_C_COINS_ROLE);
    const CompDef* regrow = find_comp(e, t, MPB_C_CHOICE_COIN_REGROW);
    const int me = avc->ip[0], partner = 1 - me;
    const int my_type_state = find_comp(e, ini, MPB_C_PLAYER_COIN_TYPE)->ip[0] == 0 ? regrow->ip[0] : regrow->ip[1];
    const int match = t->state == my_type_state;
    Obj* other = &e->obj[e->avatar_obj[partner]];
    if (match) {
      avatar_add_reward(e, ini, coin->dp[0] * role->dp[0]);  /* Role:getRewardSelfForMatch :231-235 */
      avatar_add_reward(e, other, coin->dp[2] * role->dp[2]); /* Coin:rewardOthers :74-85 (two players) */
      other->partner_match = 1;                               /* PartnerTracker:reportMatch :324-326 */
    } else {
      avatar_add_reward(e, ini, coin->dp[1] * role->dp[1]);
      avatar_add_reward(e, other, coin->dp[3] * role->dp[3]);
      other->partner_mismatch = 1;                            /* PartnerTracker:reportMismatch :328-330 */
    }
    add_event(e, EV_COIN_CONSUMED, me + 1, match);
    enqueue(e, ACT_SET_STATE, target, coin->ip[0], 0, 0);
    ini->coins_cumulative += 1;
    if (coin->ip[1] && ini->coins_cumulative >= coin->ip[2]) e->cont = 0; /* simulation:endEpisode() */
  }
}

/* ---- territory (lua/levels/territory/components.lua, avatar_library.lua:948-1121) ---------------- */
static int hit_is_direction(const OrEnv* e, int hit); /* 'directionHit*' */
static int hit_is_claim(const OrEnv* e, int hit);     /* 'claimBeam_*' */

/* Avatar:disallowMovementUntil (avatar_library.lua:475-480), Zapper:disallowZappingUntil (:755-758). */
static void avatar_disallow_movement_until(Obj* av, int frames) { if (frames > 0) { av->movement_allowed = 0; av->freeze = frames; } }
static void zapper_disallow_zapping_until(Obj* av, int frames) { av->disallow_zapping = 1; av->no_zap_counter = frames; }

/* Resource:_claim (components.lua:114-131). */
static void resource_claim(OrEnv* e, int ri, int shooter, const CompDef* c) {
  Obj* r = &e->obj[ri]; Obj* sh = &e->obj[shooter];
  const CompDef* av = find_comp(e, sh, MPB_C_AVATAR);
  r->claimed_by = shooter;
  int claimed_state = c->ip[4] + av->ip[0];
  if (r->state != claimed_state && !r->destroyed) {
    enqueue(e, ACT_SET_STATE, ri, claimed_state, 0, 0);
    r->rewarding_active = 0;
    const CompDef* taste = find_comp(e, sh, MPB_C_TERRITORY_TASTE);
    if (taste && taste->ip[0] != 0) { /* Taste:addRewardIfApplicable :337-346 */
      double amount = taste->dp[0];
      if (r->never_claimed) amount = amount * taste->dp[1];
      avatar_add_reward(e, sh, amount);
    }
    r->never_claimed = 0;
    add_event(e, EV_CLAIMED_RESOURCE, av->ip[0] + 1, 0);
  }
}
/* Resource:onHit (components.lua:133-175). */
static int resource_on_hit(OrEnv* e, int ri, int shooter, int hit, const CompDef* c) {
  Obj* r = &e->obj[ri];
  if (hit_is_direction(e, hit)) resource_claim(e, ri, shooter, c);
  if (hit_is_claim(e, hit)) { resource_claim(e, ri, shooter, c); return 0; } /* claims pass through resources */
  const CompDef* z = find_comp(e, &e->obj[shooter], MPB_C_ZAPPER);
  if (z && hit == z->ip[5]) {
    r->health -= 1; r->frames_since_zapped = 0;
    if (r->health == 0) {
      r->health = c->ip[0];
      enqueue(e, ACT_SET_STATE, ri, c->ip[1], 0, 0);
      r->rewarding_active = 0;
      if (r->texture_obj >= 0) enqueue(e, ACT_SET_STATE, r->texture_obj, c->ip[9], 0, 0);
      if (r->damage_obj >= 0) enqueue(e, ACT_SET_STATE, r->damage_obj, c->ip[10], 0, 0);
      add_event(e, EV_DESTROYED_RESOURCE, find_comp(e, &e->obj[shooter], MPB_C_AVATAR)->ip[0] + 1, 0);
      r->destroyed = 1;
      return 0; /* zaps pass through a destroyed resource */
    }
    return 1;
  }
  return 0;
}
/* GraduatedSanctionsMarking:onHit (avatar_library.lua:1049-1093). */
static void marking_on_hit(OrEnv* e, int mi, int shooter, int hit, const CompDef* c) {
  if (hit != c->ip[4]) return;
  Obj* mk = &e->obj[mi]; Obj* sh = &e->obj[shooter]; Obj* me = &e->obj[mk->marking_avatar];
  if (me->layer < 0) return; /* policy A.19: the marking of an avatar that left the grid this frame ignores hits */
  int l = mk->level - 1;
  if (l < 0 || l >= c->ip[5]) return;
  avatar_add_reward(e, sh, c->dp[2 * l]);
  avatar_add_reward(e, me, c->dp[2 * l + 1]);
  mk->level += c->ip[7 + 3 * l];
  const CompDef* sav = find_comp(e, sh, MPB_C_AVATAR); const CompDef* mav = find_comp(e, me, MPB_C_AVATAR);
  if (c->ip[8 + 3 * l]) { /* remove one frame later (:1058-1069) */
    me->removal = 1;
    avatar_disallow_movement_until(me, 1);
    zapper_disallow_zapping_until(me, 1);
    add_event(e, EV_REMOVAL, sav->ip[0] + 1, mav->ip[0] + 1);
  } else {
    enqueue(e, ACT_SET_STATE, mi, c->ip[6] + mk->level - 1, 0, 0); /* _setLevel */
    if (c->ip[9 + 3 * l]) { avatar_disallow_movement_until(me, c->ip[9 + 3 * l]); zapper_disallow_zapping_until(me, c->ip[9 + 3 * l]); }
  }
  mk->time_not_initial = 0;
  add_event(e, EV_SANCTIONING, sav->ip[0] + 1, mav->ip[0] + 1);
}

static int hit_is_direction(const OrEnv* e, int hit) { return hit >= 0 && hit < 64 && e->hit_class[hit] == 1; }
static int hit_is_claim(const OrEnv* e, int hit) { return hit >= 0 && hit < 64 && e->hit_class[hit] == 2; }

/* GameObject:_onHit: any component returning true blocks the beam (game_object.lua:305-314). */
static int on_hit(OrEnv* e, int target, int shooter, int hit) {
  Obj* t = &e->obj[target]; Obj* sh = &e->obj[shooter];
  const KindDef* k = kind_of(e, t);
  int blocked = 0;
  for (int i = 0; i < k->n_comps; ++i) {
    const CompDef* c = &e->comps[k->comp0 + i];
    switch (c->type) {
      case MPB_C_BEAM_BLOCKER: /* component_library.lua:678-685 */
        if (c->ip[0] == hit) blocked = 1;
        break;
      case MPB_C_ZAPPER: /* Zapper:onHit -- avatar_library.lua:652-681 */
        if (hit == c->ip[5]) {
          const CompDef* tav = find_comp(e, t, MPB_C_AVATAR);
          const CompDef* sav = find_comp(e, sh, MPB_C_AVATAR);
          add_event(e, EV_ZAP, sav->ip[0] + 1, tav->ip[0] + 1);
          avatar_add_reward(e, t, c->dp[0]);
          avatar_add_reward(e, sh, c->dp[1]);
          if (c->ip[4]) enqueue(e, ACT_SET_STATE, target, tav->ip[2], 0, 0);
          blocked = 1;
        }
        break;
      case MPB_C_DIRT_CLEANING: /* DirtCleaning:onHit -- clean_up/components.lua:141-157 */
        if (t->state == c->ip[0] && hit == c->ip[2]) {
          enqueue(e, ACT_SET_STATE, target, c->ip[1], 0, 0);
          const CompDef* taste = find_comp(e, sh, MPB_C_TASTE);
          if (taste) { /* Taste:cleaned :437-444 */
            if (taste->ip[0] == 1) avatar_add_reward(e, sh, taste->dp[0]);
            if (taste->ip[0] == 2) avatar_add_reward(e, sh, 0.0);
          }
          const CompDef* sav = find_comp(e, sh, MPB_C_AVATAR);
          if (find_comp(e, sh, MPB_C_CLEANER)) { /* Cleaner:setCumulant :248-255 */
            sh->player_cleaned += 1;
            e->cleaned_flag[sav->ip[0]] = 1;
          }
          add_event(e, EV_PLAYER_CLEANED, sav->ip[0] + 1, 0);
          blocked = 1;
        }
        break;
      case MPB_C_ORE: { /* Ore:onHit -- coop_mining/components.lua:118-150 (an ore object carries one Ore component per ore type) */
        const CompDef* mb = find_comp(e, sh, MPB_C_MINE_BEAM);
        if (!mb || hit != mb->ip[3] || (t->state != c->ip[1] && t->state != c->ip[2])) break;
        int k = 0; /* which of the object's Ore components this is */
        for (int j = 0; j < i; ++j) if (e->comps[kind_of(e, t)->comp0 + j].type == MPB_C_ORE) ++k;
        const int me = find_comp(e, sh, MPB_C_AVATAR)->ip[0], type = c->ip[3];
        t->ore_cd[k] = c->ip[4]; t->ore_miners[k] |= 1 << me;             /* Ore:addMiner :110-114 */
        enqueue(e, ACT_SET_STATE, target, c->ip[2], 0, 0);
        avatar_add_reward(e, sh, mb->dp[type - 1]);                        /* MineBeam:processRoleMineEvent :203-212 */
        add_event(e, EV_MINING, me + 1, type);
        int count = 0;
        for (int p = 0; p < e->P; ++p) count += (t->ore_miners[k] >> p) & 1;
        if (count == c->ip[3]) {
          for (int p = 0; p < e->P; ++p) if ((t->ore_miners[k] >> p) & 1) {
            Obj* av = &e->obj[e->avatar_obj[p]];
            avatar_add_reward(e, av, find_comp(e, av, MPB_C_MINE_BEAM)->dp[2 + type - 1]); /* processRoleExtractEvent :214-224 */
            add_event(e, EV_EXTRACTION, p + 1, type);
            for (int q = 0; q < e->P; ++q) if (q != p && ((t->ore_miners[k] >> q) & 1)) add_event(e, EV_EXTRACTION_PAIR, p + 1, (q + 1) | (type << 8));
          }
          t->ore_miners[k] = 0; t->ore_cd[k] = 0;                          /* Ore:reset :96-103 */
          if (t->state != c->ip[0]) enqueue(e, ACT_SET_STATE, target, c->ip[1], 0, 0);
          enqueue(e, ACT_SET_STATE, target, c->ip[0], 0, 0);
        }
        blocked = 1;
      } break;
      case MPB_C_ALL_BEAM_BLOCKER: blocked = 1; break; /* territory/components.lua:46-49 */
      case MPB_C_RESOURCE: if (resource_on_hit(e, target, shooter, hit, c)) blocked = 1; break;
      case MPB_C_GRADUATED_SANCTIONS_MARKING: marking_on_hit(e, target, shooter, hit, c); break; /* never blocks */
      default: break;
    }
  }
  return blocked;
}

/* DensityRegrow:_getNeighbors (commons_harvest/components.lua:195-204): pieces on the wait layer
 * ('logic') and on the live layer ('lowerPhysical') inside the disc transform:queryDisc(layer, radius). */
static int in_disc(double radius, int dx, int dy) { return (double)(dx * dx + dy * dy) <= radius * radius; }
static void density_begin_live(OrEnv* e, int oi, const CompDef* c) { /* :206-219 */
  Obj* o = &e->obj[oi];
  int cells = e->W * e->H, r = (int)c->dp[0];
  for (int dy = -r; dy <= r; ++dy) for (int dx = -r; dx <= r; ++dx) {
    if (!in_disc(c->dp[0], dx, dy)) continue;
    int x = o->x + dx, y = o->y + dy;
    if (!wrap_or_reject(e, &x, &y)) continue;
    int q = e->grid[c->ip[6] * cells + cell_of(e, x, y)] - 1;
    if (q >= 0 && q != oi) e->obj[q].num_neighbors += 1;
  }
}
static void density_end_live(OrEnv* e, int oi, const CompDef* c) { /* :221-240 */
  Obj* o = &e->obj[oi];
  int cells = e->W * e->H, r = (int)c->dp[0], live = 0;
  for (int dy = -r; dy <= r; ++dy) for (int dx = -r; dx <= r; ++dx) {
    if (!in_disc(c->dp[0], dx, dy)) continue;
    int x = o->x + dx, y = o->y + dy;
    if (!wrap_or_reject(e, &x, &y)) continue;
    if (e->grid[c->ip[7] * cells + cell_of(e, x, y)]) ++live;
  }
  for (int dy = -r; dy <= r; ++dy) for (int dx = -r; dx <= r; ++dx) {
    if (!in_disc(c->dp[0], dx, dy)) continue;
    int x = o->x + dx, y = o->y + dy;
    if (!wrap_or_reject(e, &x, &y)) continue;
    int q = e->grid[c->ip[6] * cells + cell_of(e, x, y)] - 1;
    if (q < 0) continue;
    if (q != oi) e->obj[q].num_neighbors -= 1; else e->obj[q].num_neighbors = live;
  }
}

/* GameObject:_onAdd -> component onStateChange(previousState) (game_object.lua:273-285). */
static void on_state_change(OrEnv* e, int oi, int old_state) {
  Obj* o = &e->obj[oi];
  const KindDef* k = kind_of(e, o);
  for (int i = 0; i < k->n_comps; ++i) {
    const CompDef* c = &e->comps[k->comp0 + i];
    switch (c->type) {
      case MPB_C_DIRT_TRACKER: /* clean_up/components.lua:118-129 */
        if (old_state == c->ip[1] && o->state == c->ip[0]) { e->dirt_count++; e->clean_count--; }
        else if (old_state == c->ip[0] && o->state == c->ip[1]) { e->dirt_count--; e->clean_count++; }
        break;
      case MPB_C_AVATAR: /* avatar_library.lua:430-453 */
        if (old_state == c->ip[2] && o->state == c->ip[1]) {
          o->freeze = 0; o->removal = 0;
          for (int k = 0; k < o->n_connected; ++k) { /* avatarStateChange('respawn') :1099-1107 */
            int mi = o->connected[k]; const CompDef* mc = find_comp(e, &e->obj[mi], MPB_C_GRADUATED_SANCTIONS_MARKING);
            if (!mc) continue;
            enqueue(e, ACT_SET_STATE, mi, mc->ip[6] + e->obj[mi].level - 1, 0, 0);
            enqueue(e, ACT_TELEPORT, mi, o->x, o->y, 0);
            enqueue(e, ACT_SET_ORIENT, mi, o->orient, 0, 0);
          }
        } else if (old_state == c->ip[1] && o->state == c->ip[2]) {
          for (int k = 0; k < o->n_connected; ++k) { /* avatarStateChange('die') :1108-1110 */
            int mi = o->connected[k]; const CompDef* mc = find_comp(e, &e->obj[mi], MPB_C_GRADUATED_SANCTIONS_MARKING);
            if (mc) enqueue(e, ACT_SET_STATE, mi, mc->ip[1], 0, 0);
          }
        }
        break;
      case MPB_C_DENSITY_REGROW: /* commons_harvest/components.lua:153-163 */
        if (o->dr_started) {
          if (o->state == c->ip[0]) density_begin_live(e, oi, c);
          else if (old_state == c->ip[0]) density_end_live(e, oi, c);
        }
        break;
      default: break;
    }
  }
}

/* ------------------------------------------------------------------------------------------
 * Engine core (policies A.1-A.9 of the ledger).
 * ---------------------------------------------------------------------------------------- */
static void lift(OrEnv* e, int oi) {
  Obj* o = &e->obj[oi];
  if (o->layer >= 0) { e->grid[o->layer * e->W * e->H + cell_of(e, o->x, o->y)] = 0; }
}
static void place(OrEnv* e, int oi) {
  Obj* o = &e->obj[oi];
  if (o->layer >= 0) e->grid[o->layer * e->W * e->H + cell_of(e, o->x, o->y)] = oi + 1;
}
/* Policy A.5: placing a piece fires contact `enter` both ways with every other piece on the cell. */
static void trigger_enter(OrEnv* e, int oi) {
  Obj* o = &e->obj[oi];
  if (o->layer < 0) return;
  int cell = cell_of(e, o->x, o->y), cells = e->W * e->H;
  int my_contact = state_def(e, o, o->state)->contact;
  for (int l = 0; l < e->L; ++l) {
    int q = e->grid[l * cells + cell] - 1;
    if (q < 0 || q == oi) continue;
    if (my_contact >= 0) on_enter(e, q, oi);
    if (state_def(e, &e->obj[q], e->obj[q].state)->contact >= 0) on_enter(e, oi, q);
  }
}
/* grid:setState (component_library.lua:194-198). Policy A.18: same-state is a no-op; policy A.2. */
static void do_set_state(OrEnv* e, int oi, int ns) {
  Obj* o = &e->obj[oi];
  if (ns == o->state) return;
  int nl = state_def(e, o, ns)->layer;
  if (nl >= 0) {
    int occ = e->grid[nl * e->W * e->H + cell_of(e, o->x, o->y)] - 1;
    if (occ >= 0 && occ != oi) return; /* blocked: stays as it was (onBlocked has no listeners) */
  }
  int old = o->state;
  lift(e, oi);
  o->prev_state = old; o->state = ns; o->layer = nl; o->state_frame = e->frame;
  place(e, oi);
  on_state_change(e, oi, old);
  trigger_enter(e, oi);
}
static void do_turn(OrEnv* e, int oi, int k) { /* policy A.6 */
  Obj* o = &e->obj[oi];
  if (o->layer < 0) return;
  o->orient = (o->orient + k) & 3;
}
static int wrap_or_reject(const OrEnv* e, int* x, int* y) {
  if (e->topology == 1) { *x = ((*x % e->W) + e->W) % e->W; *y = ((*y % e->H) + e->H) % e->H; return 1; }
  return *x >= 0 && *x < e->W && *y >= 0 && *y < e->H;
}
/* grid:moveRel (component_library.lua:320-322): lift, attempt, place (docs/advanced.md:45-52). */
static void do_move_rel(OrEnv* e, int oi, int rel) {
  Obj* o = &e->obj[oi];
  if (o->layer < 0) return;
  int d = (o->orient + rel) & 3;
  int nx = o->x + DX[d], ny = o->y + DY[d];
  lift(e, oi);
  int ok = wrap_or_reject(e, &nx, &ny) && e->grid[o->layer * e->W * e->H + cell_of(e, nx, ny)] == 0;
  for (int k = 0; ok && k < o->n_connected; ++k) { /* grid:connect: the group moves only if every member can (policy A.5b) */
    const Obj* c = &e->obj[o->connected[k]];
    if (c->layer < 0) continue;
    int occ = e->grid[c->layer * e->W * e->H + cell_of(e, nx, ny)] - 1;
    if (occ >= 0 && occ != o->connected[k]) ok = 0;
  }
  if (ok) { o->x = nx; o->y = ny; }
  place(e, oi);
  for (int k = 0; k < o->n_connected; ++k) { /* grid:connect: connected pieces are carried along */
    Obj* c = &e->obj[o->connected[k]];
    if (c->layer < 0) continue;
    lift(e, o->connected[k]); c->x = o->x; c->y = o->y; place(e, o->connected[k]);
  }
  trigger_enter(e, oi); /* fires even when the move was blocked */
}
/* grid:teleport / grid:setOrientation (component_library.lua:331-334). Off-grid pieces have no position. */
static void do_teleport(OrEnv* e, int oi, int x, int y) {
  Obj* o = &e->obj[oi];
  if (o->layer < 0) return;
  int occ = e->grid[o->layer * e->W * e->H + cell_of(e, x, y)] - 1;
  if (occ >= 0 && occ != oi) return;
  lift(e, oi); o->x = x; o->y = y; place(e, oi);
  trigger_enter(e, oi);
}
static void do_set_orient(OrEnv* e, int oi, int orient) { if (e->obj[oi].layer >= 0) e->obj[oi].orient = orient & 3; }
/* grid:teleportToGroup (component_library.lua:351-354). Policy A.9. */
static void do_teleport_group(OrEnv* e, int oi, int group, int ns) {
  Obj* o = &e->obj[oi];
  const CompDef* av = find_comp(e, o, MPB_C_AVATAR);
  uint32_t w[4];
  rng(e, RS_AVATAR, av ? av->ip[0] : oi, w);
  int n = 0;
  for (int i = 0; i < e->n_obj; ++i) {
    const Obj* c = &e->obj[i];
    if (c->layer >= 0 && (state_def(e, c, c->state)->groups & (1u << group))) ++n;
  }
  if (n == 0) return;
  int k = (int)pick(w[1], (uint32_t)n), target = -1;
  for (int i = 0; i < e->n_obj; ++i) {
    const Obj* c = &e->obj[i];
    if (c->layer >= 0 && (state_def(e, c, c->state)->groups & (1u << group))) { if (k-- == 0) { target = i; break; } }
  }
  int tx = e->obj[target].x, ty = e->obj[target].y;
  int nl = state_def(e, o, ns)->layer;
  if (nl >= 0) {
    int occ = e->grid[nl * e->W * e->H + cell_of(e, tx, ty)] - 1;
    if (occ >= 0 && occ != oi) return; /* blocked; the respawn updater fires again next frame */
  }
  int old = o->state;
  lift(e, oi);
  o->x = tx; o->y = ty; o->orient = (int)(w[2] & 3u); /* TELEPORT_ORIENTATION.PICK_RANDOM */
  o->prev_state = old; o->state = ns; o->layer = nl; o->state_frame = e->frame;
  place(e, oi);
  if (old != ns) on_state_change(e, oi, old);
  trigger_enter(e, oi);
}
/* One beam cell: onHit on every piece of the cell, then the hit sprite if not blocked.
 * Returns 1 if the ray stops here. Policy A.8. */
static int beam_cell(OrEnv* e, int shooter, int hit, int x, int y) {
  if (!wrap_or_reject(e, &x, &y)) return 1;
  int cells = e->W * e->H, cell = cell_of(e, x, y), blocked = 0;
  for (int l = 0; l < e->L; ++l) {
    int q = e->grid[l * cells + cell] - 1;
    if (q < 0 || q == shooter) continue;
    if (on_hit(e, q, shooter, hit)) blocked = 1;
  }
  if (blocked) return 1;
  int hl = e->hits[hit * 2 + MPB_HIT_LAYER], hs = e->hits[hit * 2 + MPB_HIT_SPRITE];
  if (e->beam[hl * cells + cell] == 0 && e->grid[hl * cells + cell] == 0) /* only where the hit's layer is free */
    e->beam[hl * cells + cell] = MPB_CELL(hs, e->obj[shooter].orient);
  return 0;
}
/* grid:hitBeam(piece, hit, length, radius) (game_object.lua:253-258); geometry mirrors
 * Zapper:getWhoZappable (avatar_library.lua:785-821). Policy A.8. */
static void do_beam(OrEnv* e, int oi, int hit, int length, int radius) {
  Obj* o = &e->obj[oi];
  if (o->layer < 0) return;
  int f = o->orient, fx = DX[f], fy = DY[f];
  for (int i = 1; i <= length; ++i) if (beam_cell(e, oi, hit, o->x + fx * i, o->y + fy * i)) break;
  for (int side = 0; side < 2; ++side) {
    int s = side == 0 ? (f + 3) & 3 : (f + 1) & 3; /* left, then right */
    for (int k = 1; k <= radius; ++k) {
      int bx = o->x + DX[s] * k, by = o->y + DY[s] * k;
      if (beam_cell(e, oi, hit, bx, by)) break;
      for (int i = 1; i <= length - k; ++i) if (beam_cell(e, oi, hit, bx + fx * i, by + fy * i)) break;
    }
  }
}

static void process_queue(OrEnv* e) { /* policy A.4: rounds until empty, at most flushCount */
  for (int round = 0; round < OR_MAX_ROUNDS && e->qnn > 0; ++round) {
    Action* tmp = e->q; e->q = e->qnext; e->qnext = tmp;
    int tcap = e->qcap; e->qcap = e->qncap; e->qncap = tcap;
    e->qn = e->qnn; e->qnn = 0;
    for (int i = 0; i < e->qn; ++i) {
      Action a = e->q[i];
      switch (a.type) {
        case ACT_SET_STATE: do_set_state(e, a.obj, a.a); break;
        case ACT_TURN: do_turn(e, a.obj, a.a); break;
        case ACT_MOVE_REL: do_move_rel(e, a.obj, a.a); break;
        case ACT_TELEPORT_GROUP: do_teleport_group(e, a.obj, a.a, a.b); break;
        case ACT_BEAM: do_beam(e, a.obj, a.a, a.b, a.c); break;
        case ACT_TELEPORT: do_teleport(e, a.obj, a.a, a.b); break;
        case ACT_SET_ORIENT: do_set_orient(e, a.obj, a.a); break;
      }
    }
  }
}

/* ------------------------------------------------------------------------------------------
 * Updaters (updater_registry.lua:114-159; priorities in SURVEY.md section 3.3).
 * ---------------------------------------------------------------------------------------- */
static void run_updater(OrEnv* e, const Updater* u, int oi) {
  Obj* o = &e->obj[oi];
  const CompDef* c = find_comp(e, o, u->comp_type);
  int age = e->frame - o->state_frame;
  switch (u->fn) {
    case UF_AVATAR_MOVE: { /* avatar_library.lua:156-171 */
      if (!o->movement_allowed) break;
      if (o->act[MPB_ACT_TURN] != 0) {
        enqueue(e, ACT_TURN, oi, o->act[MPB_ACT_TURN], 0, 0);
        for (int k = 0; k < o->n_connected; ++k) enqueue(e, ACT_TURN, o->connected[k], o->act[MPB_ACT_TURN], 0, 0);
      }
      if (o->act[MPB_ACT_MOVE] != 0) enqueue(e, ACT_MOVE_REL, oi, o->act[MPB_ACT_MOVE] - 1, 0, 0);
    } break;
    case UF_ZAP: { /* avatar_library.lua:613-631 */
      if (!avatar_is_alive(e, o) || c->ip[0] < 0) break;
      if (o->zap_cool > 0) o->zap_cool--;
      else if (o->act[MPB_ACT_FIRE_ZAP] == 1) { o->zap_cool = c->ip[0]; enqueue(e, ACT_BEAM, oi, c->ip[5], c->ip[1], c->ip[2]); }
    } break;
    case UF_RESPAWN: { /* avatar_library.lua:638-649: state = waitState, startFrame = framesTillRespawn */
      const CompDef* av = find_comp(e, o, MPB_C_AVATAR);
      if (o->state != av->ip[2] || age < c->ip[3]) break;
      enqueue(e, ACT_TELEPORT_GROUP, oi, o->spawn_group, av->ip[1], 0);
    } break;
    case UF_CLEAN: { /* clean_up/components.lua:201-219 */
      if (!avatar_is_alive(e, o) || c->ip[0] < 0) break;
      if (o->clean_cool > 0) o->clean_cool--;
      else if (o->act[MPB_ACT_FIRE_2] == 1) { o->clean_cool = c->ip[0]; enqueue(e, ACT_BEAM, oi, c->ip[3], c->ip[1], c->ip[2]); }
    } break;
    case UF_CLEANER_RESET: o->player_cleaned = 0; break;   /* clean_up/components.lua:226-232 */
    case UF_TASTE_RESET: o->player_ate = 0; break;          /* :428-434 */
    case UF_NONSELF_GET: { /* :535-545, sumNonself :524-531 */
      int me = find_comp(e, o, MPB_C_AVATAR)->ip[0], sc = 0, sa = 0;
      for (int p = 0; p < e->P; ++p) if (p != me) { sc += e->cleaned_flag[p]; sa += e->ate_flag[p]; }
      o->num_others_cleaned = sc; o->num_others_ate = sa;
    } break;
    case UF_NONSELF_RESET: o->num_others_cleaned = 0; o->num_others_ate = 0; break; /* :547-556 */
    case UF_GLOBAL_RESET: /* :484-491 */
      for (int p = 0; p < e->P; ++p) { e->cleaned_flag[p] = 0; e->ate_flag[p] = 0; }
      break;
    case UF_EPISODE_END: { /* component_library.lua:927-940 */
      if (age < c->ip[0]) break;
      if (e->ending_t % c->ip[1] == 0) {
        uint32_t w[4]; rng(e, RS_SCENE, SCENE_DRAW_EPISODE_END, w);
        if (u01(w[0], w[1]) < c->dp[0]) e->cont = 0; /* simulation:endEpisode() */
      }
    } break;
    case UF_PAINTBRUSH: enqueue(e, ACT_BEAM, oi, c->ip[1], 1, 0); break; /* territory/components.lua:401-410 */
    case UF_CLAIM: { /* ResourceClaimer (components.lua:249-269): no alive check */
      if (c->ip[3] < 0) break;
      if (o->claim_cool > 0) o->claim_cool--;
      else if (o->act[MPB_ACT_FIRE_2] == 1) { o->claim_cool = c->ip[3]; enqueue(e, ACT_BEAM, oi, c->ip[4], c->ip[1], c->ip[2]); }
    } break;
    case UF_PROVIDE_REWARDS: { /* components.lua:82-99: group claimedResources, probability rewardRate, startFrame rewardDelay */
      if (!(state_def(e, o, o->state)->groups & (1u << c->ip[6])) || age < c->ip[2]) break;
      uint32_t w[4]; rng(e, RS_OBJECT, oi, w);
      if (!(u01(w[2], w[3]) < c->dp[1])) break;
      if (o->state != c->ip[1] && o->claimed_by >= 0) {
        Obj* av = &e->obj[o->claimed_by];
        const CompDef* taste = find_comp(e, av, MPB_C_TERRITORY_TASTE);
        if (taste && taste->ip[0] == 2) avatar_add_reward(e, av, 0.0); else avatar_add_reward(e, av, c->dp[0]);
        o->rewarding_active = 1;
      }
    } break;
    case UF_RELEASE_CLAIM: { /* components.lua:100-112: priority 2, startFrame 5 */
      if (!(state_def(e, o, o->state)->groups & (1u << c->ip[6])) || age < 5 || o->claimed_by < 0) break;
      Obj* av = &e->obj[o->claimed_by];
      if (av->state == find_comp(e, av, MPB_C_AVATAR)->ip[2] && !o->destroyed) {
        enqueue(e, ACT_SET_STATE, oi, c->ip[5], 0, 0);
        o->rewarding_active = 0; o->claimed_by = -1;
      }
    } break;
    case UF_MARKING_RECOVERY: { /* avatar_library.lua:1009-1026 */
      Obj* av = &e->obj[o->marking_avatar];
      if (o->level != c->ip[2] && avatar_is_alive(e, av)) {
        o->time_not_initial += 1;
        if (o->time_not_initial == c->ip[3]) {
          o->level = c->ip[2];
          enqueue(e, ACT_SET_STATE, oi, c->ip[6] + o->level - 1, 0, 0);
          o->time_not_initial = 0;
        }
      }
    } break;
    case UF_SPROUT: { /* commons_harvest/components.lua:92-123: one updater per wait_k state, priority 10 */
      int k = o->state - c->ip[1];
      if (k < 0 || k >= c->ip[2]) break;
      int idx = k < c->ip[4] ? k : c->ip[4] - 1;
      uint32_t w[4]; rng(e, RS_OBJECT, oi, w);
      if (u01(w[0], w[1]) < c->dp[1 + idx]) enqueue(e, ACT_SET_STATE, oi, c->ip[0], 0, 0); /* canRegrowIfOccupied */
    } break;
    case UF_COIN_REGROW: { /* ChoiceCoinRegrow (coins/components.lua:183-194): state = waitState, probability = regrowRate */
      if (o->state != c->ip[2]) break;
      uint32_t w[4]; rng(e, RS_OBJECT, oi, w);
      if (u01(w[0], w[1]) < c->dp[0]) enqueue(e, ACT_SET_STATE, oi, c->ip[pick(w[2], 2u)], 0, 0); /* random:choice(liveStates) */
    } break;
    case UF_ORE_REGROW_0: case UF_ORE_REGROW_1: { /* FixedRateRegrow (coop_mining/components.lua:41-57): priority 200, one updater per live state */
      const int i = u->fn - UF_ORE_REGROW_0;
      if (o->state != c->ip[5] || i >= c->ip[0]) break;
      uint32_t w[4]; rng(e, RS_OBJECT, oi, w);
      if (!(u01(w[2 * i], w[2 * i + 1]) < c->dp[i])) break;
      const Obj* a0 = &e->obj[e->avatar_obj[0]]; /* transform:queryPosition('upperPhysical'): the avatars' layer */
      const int layer = state_def(e, a0, find_comp(e, a0, MPB_C_AVATAR)->ip[1])->layer;
      if (e->grid[layer * e->W * e->H + cell_of(e, o->x, o->y)] == 0) enqueue(e, ACT_SET_STATE, oi, c->ip[1 + i], 0, 0);
    } break;
    case UF_ANIMATION: { /* component_library.lua:1070-1094: one updater per state, startFrame */
      if (age < c->ip[9]) break;
      int n = c->ip[0];
      for (int i = 0; i < n; ++i) if (c->ip[1 + i] == o->state) {
        if (i + 1 < n) enqueue(e, ACT_SET_STATE, oi, c->ip[2 + i], 0, 0);
        else if (c->ip[10]) enqueue(e, ACT_SET_STATE, oi, c->ip[1], 0, 0);
        break;
      }
    } break;
  }
}

static void add_updater(OrEnv* e, int priority, int comp_type, int fn) {
  for (int i = 0; i < e->n_updaters; ++i) if (e->updaters[i].comp_type == comp_type && e->updaters[i].fn == fn) return;
  e->updaters = (Updater*)realloc(e->updaters, sizeof(Updater) * (e->n_updaters + 1));
  Updater u = {priority, comp_type, fn, e->n_updaters};
  e->updaters[e->n_updaters++] = u;
}
static int cmp_updater(const void* a, const void* b) {
  const Updater* x = (const Updater*)a; const Updater* y = (const Updater*)b;
  if (x->priority != y->priority) return y->priority - x->priority; /* descending (updater_registry.lua:163-170) */
  return x->seq - y->seq; /* policy A.7: ties in first-registration order */
}
static void build_updaters(OrEnv* e) {
  for (int oi = 0; oi < e->n_obj; ++oi) {
    const KindDef* k = &e->kinds[e->objdef[oi * MPB_OBJ_COLS + MPB_OBJ_KIND]];
    for (int i = 0; i < k->n_comps; ++i) {
      switch (e->comps[k->comp0 + i].type) {
        case MPB_C_AVATAR: add_updater(e, 150, MPB_C_AVATAR, UF_AVATAR_MOVE); break;
        case MPB_C_ZAPPER: add_updater(e, 140, MPB_C_ZAPPER, UF_ZAP); add_updater(e, 135, MPB_C_ZAPPER, UF_RESPAWN); break;
        case MPB_C_CLEANER: add_updater(e, 140, MPB_C_CLEANER, UF_CLEAN); add_updater(e, 400, MPB_C_CLEANER, UF_CLEANER_RESET); break;
        case MPB_C_TASTE: add_updater(e, 400, MPB_C_TASTE, UF_TASTE_RESET); break;
        case MPB_C_ALL_NONSELF_CUMULANTS: add_updater(e, 4, MPB_C_ALL_NONSELF_CUMULANTS, UF_NONSELF_GET); add_updater(e, 400, MPB_C_ALL_NONSELF_CUMULANTS, UF_NONSELF_RESET); break;
        case MPB_C_GLOBAL_DATA: add_updater(e, 2, MPB_C_GLOBAL_DATA, UF_GLOBAL_RESET); break;
        case MPB_C_STOCHASTIC_INTERVAL_EPISODE_ENDING: add_updater(e, 100, MPB_C_STOCHASTIC_INTERVAL_EPISODE_ENDING, UF_EPISODE_END); break;
        case MPB_C_ANIMATION: add_updater(e, 100, MPB_C_ANIMATION, UF_ANIMATION); break;
        case MPB_C_DENSITY_REGROW: add_updater(e, 10, MPB_C_DENSITY_REGROW, UF_SPROUT); break;
        case MPB_C_CHOICE_COIN_REGROW: add_updater(e, 100, MPB_C_CHOICE_COIN_REGROW, UF_COIN_REGROW); break; /* default priority (updater_registry.lua:47) */
        case MPB_C_FIXED_RATE_REGROW: add_updater(e, 200, MPB_C_FIXED_RATE_REGROW, UF_ORE_REGROW_0); add_updater(e, 200, MPB_C_FIXED_RATE_REGROW, UF_ORE_REGROW_1); break;
        case MPB_C_PAINTBRUSH: add_updater(e, 130, MPB_C_PAINTBRUSH, UF_PAINTBRUSH); break;
        case MPB_C_RESOURCE_CLAIMER: add_updater(e, 100, MPB_C_RESOURCE_CLAIMER, UF_CLAIM); break;
        case MPB_C_RESOURCE: add_updater(e, 100, MPB_C_RESOURCE, UF_PROVIDE_REWARDS); add_updater(e, 2, MPB_C_RESOURCE, UF_RELEASE_CLAIM); break;
        case MPB_C_GRADUATED_SANCTIONS_MARKING: add_updater(e, 3, MPB_C_GRADUATED_SANCTIONS_MARKING, UF_MARKING_RECOVERY); break;
        default: break;
      }
    }
  }
  qsort(e->updaters, e->n_updaters, sizeof(Updater), cmp_updater);
}

/* Policy A.7: avatars are visited in a fresh random order every frame (the engine shuffles group
 * members); all other objects in creation order. Order = ascending (philox word 0, index). */
static void draw_avatar_order(OrEnv* e) {
  uint32_t keyv[OR_MAX_PLAYERS];
  for (int p = 0; p < e->P; ++p) { uint32_t w[4]; rng(e, RS_AVATAR, p, w); keyv[p] = w[0]; e->order[p] = p; }
  for (int i = 1; i < e->P; ++i) { /* insertion sort by (key, index) */
    int v = e->order[i], j = i - 1;
    while (j >= 0 && (keyv[e->order[j]] > keyv[v] || (keyv[e->order[j]] == keyv[v] && e->order[j] > v))) { e->order[j + 1] = e->order[j]; --j; }
    e->order[j + 1] = v;
  }
}

/* grid:update(random) -- api_factory.lua:101,106; docs/advanced.md:33-56. */
static void grid_update(OrEnv* e) {
  memset(e->beam, 0, sizeof(uint16_t) * e->L * e->W * e->H); /* hit sprites last one frame (A.8) */
  draw_avatar_order(e);
  for (int ui = 0; ui < e->n_updaters; ++ui) {
    const Updater* u = &e->updaters[ui];
    int avatar_comp = 0;
    for (int p = 0; p < e->P && !avatar_comp; ++p) if (find_comp(e, &e->obj[e->avatar_obj[p]], u->comp_type)) avatar_comp = 1;
    if (avatar_comp) {
      for (int i = 0; i < e->P; ++i) run_updater(e, u, e->avatar_obj[e->order[i]]);
    } else {
      for (int oi = 0; oi < e->n_obj; ++oi) if (!e->obj[oi].absent && find_comp(e, &e->obj[oi], u->comp_type)) run_updater(e, u, oi);
    }
  }
  process_queue(e);
  e->frame++;
}

/* BaseSimulation:update -- base_simulation.lua:476-486 (preUpdate all, then update all). */
static void simulation_update(OrEnv* e) {
  for (int p = 0; p < e->P; ++p) e->obj[e->avatar_obj[p]].reward = 0.0; /* Avatar:preUpdate :330-332 */
  for (int p = 0; p < e->P; ++p) { Obj* a = &e->obj[e->avatar_obj[p]]; a->partner_match = 0; a->partner_mismatch = 0; } /* PartnerTracker:preUpdate (coins/components.lua:303-306) */
  for (int oi = 0; oi < e->n_obj; ++oi) {
    Obj* o = &e->obj[oi];
    if (o->absent) continue;
    const KindDef* k = kind_of(e, o);
    for (int i = 0; i < k->n_comps; ++i) {
      const CompDef* c = &e->comps[k->comp0 + i];
      switch (c->type) {
        case MPB_C_DIRT_SPAWNER: { /* clean_up/components.lua:329-340 */
          if (e->spawner_t > c->ip[0]) {
            uint32_t w[4]; rng(e, RS_SCENE, SCENE_DRAW_DIRT, w);
            if (u01(w[0], w[1]) < c->dp[0]) {
              int n = 0; /* set.toSortedList(potentialDirts): inactive dirt pieces in piece order */
              for (int j = 0; j < e->n_obj; ++j) { const CompDef* dt = find_comp(e, &e->obj[j], MPB_C_DIRT_TRACKER); if (dt && e->obj[j].state == dt->ip[1]) ++n; }
              if (n > 0) {
                int kk = (int)pick(w[2], (uint32_t)n);
                for (int j = 0; j < e->n_obj; ++j) { const CompDef* dt = find_comp(e, &e->obj[j], MPB_C_DIRT_TRACKER); if (dt && e->obj[j].state == dt->ip[1]) { if (kk-- == 0) { enqueue(e, ACT_SET_STATE, j, dt->ip[0], 0, 0); break; } } }
              }
            }
          }
          e->spawner_t++;
        } break;
        case MPB_C_STOCHASTIC_INTERVAL_EPISODE_ENDING: e->ending_t++; break; /* component_library.lua:946-948 */
        case MPB_C_ORE: { /* Ore:update -- coop_mining/components.lua:104-109 */
          int kk = 0; /* which of the object's Ore components this is */
          for (int j = 0; j < i; ++j) if (e->comps[k->comp0 + j].type == MPB_C_ORE) ++kk;
          o->ore_cd[kk] -= 1;
          if (o->ore_cd[kk] == 0) { /* Ore:reset :96-103 */
            o->ore_miners[kk] = 0;
            if (o->state != c->ip[0]) enqueue(e, ACT_SET_STATE, oi, c->ip[1], 0, 0);
          }
        } break;
        case MPB_C_MINE_BEAM: { /* MineBeam:update -- coop_mining/components.lua:236-252 */
          if (o->mine_cool > 0) o->mine_cool--;
          if (o->act[MPB_ACT_FIRE_ZAP] == 1 && o->mine_cool == 0) { o->mine_cool = c->ip[0]; enqueue(e, ACT_BEAM, oi, c->ip[3], c->ip[1], c->ip[2]); }
        } break;
        case MPB_C_AVATAR: { /* Avatar:update -- avatar_library.lua:334-354 */
          if (o->freeze == 1) o->movement_allowed = 1;
          o->freeze = o->freeze > 0 ? o->freeze - 1 : 0;
          if (o->removal == 1) enqueue(e, ACT_SET_STATE, oi, c->ip[2], 0, 0);
          o->removal = o->removal > 0 ? o->removal - 1 : 0;
        } break;
        case MPB_C_ZAPPER: { /* Zapper:update -- avatar_library.lua:713-724 */
          if (o->disallow_zapping) o->zap_cool = c->ip[0] + 1;
          int old_counter = o->no_zap_counter;
          o->no_zap_counter = o->no_zap_counter > 0 ? o->no_zap_counter - 1 : 0;
          if (old_counter == 1) o->disallow_zapping = 0;
        } break;
        case MPB_C_RESOURCE: { /* Resource:update -- territory/components.lua:184-197 */
          if (o->health < c->ip[0]) {
            if (o->damage_obj >= 0) enqueue(e, ACT_SET_STATE, o->damage_obj, c->ip[11], 0, 0);
            if (o->frames_since_zapped >= c->ip[3]) {
              uint32_t w[4]; rng(e, RS_OBJECT, oi, w);
              if (u01(w[0], w[1]) < c->dp[2]) {
                o->health += 1;
                if (o->health == c->ip[0] && o->damage_obj >= 0) enqueue(e, ACT_SET_STATE, o->damage_obj, c->ip[10], 0, 0);
              }
            }
            o->frames_since_zapped += 1;
          }
        } break;
        case MPB_C_REWARD_INDICATOR: { /* RewardIndicator:update -- components.lua:303-312 */
          const Obj* r = &e->obj[o->paired_resource];
          const CompDef* rc = find_comp(e, r, MPB_C_RESOURCE);
          if (r->rewarding_active && r->state >= rc->ip[4]) enqueue(e, ACT_SET_STATE, oi, c->ip[1] + (r->state - rc->ip[4]), 0, 0);
          else enqueue(e, ACT_SET_STATE, oi, c->ip[0], 0, 0);
        } break;
        case MPB_C_DENSITY_REGROW: { /* DensityRegrow:update -> _updateWaitState (commons_harvest/components.lua:147-151,170-193) */
          if (o->layer != c->ip[6] || o->state == c->ip[0]) break;
          int kk = o->num_neighbors;
          if (kk >= c->ip[2]) kk = c->ip[2] - 1;
          enqueue(e, ACT_SET_STATE, oi, c->ip[1] + kk, 0, 0);
          if (o->grass_obj >= 0) enqueue(e, ACT_SET_STATE, o->grass_obj, kk == 0 ? c->ip[10] : c->ip[9], 0, 0);
        } break;
        case MPB_C_APPLE_GROW: { /* clean_up/components.lua:64-80 */
          double dirt = (double)e->dirt_count, clean = (double)e->clean_count;
          double fraction = dirt / (dirt + clean);
          double interpolation = (fraction - c->dp[1]) / (c->dp[2] - c->dp[1]);
          interpolation = 1.0 < interpolation ? 1.0 : interpolation; /* math.min keeps a NaN (policy A.22) */
          double probability = c->dp[0] * interpolation;
          uint32_t w[4]; rng(e, RS_OBJECT, oi, w);
          if (u01(w[0], w[1]) < probability) enqueue(e, ACT_SET_STATE, oi, c->ip[0], 0, 0);
        } break;
        default: break;
      }
    }
  }
}

/* ------------------------------------------------------------------------------------------
 * Episode start: api:start (api_factory.lua:85-102), BaseSimulation:start/_avatarStart
 * (base_simulation.lua:396-471).
 * ---------------------------------------------------------------------------------------- */
static void episode_start(OrEnv* e) {
  int cells = e->W * e->H;
  e->frame = 0; e->step = 0; e->cont = 1; e->done = 0; e->qn = e->qnn = 0; e->evn = 0;
  memset(e->grid, 0, sizeof(int) * e->L * cells);
  memset(e->beam, 0, sizeof(uint16_t) * e->L * cells);
  e->dirt_count = e->clean_count = 0; e->spawner_t = 1; e->ending_t = 1; /* reset(): :271-274,:324-327, component_library.lua:942-944 */
  memset(e->cleaned_flag, 0, sizeof e->cleaned_flag); memset(e->ate_flag, 0, sizeof e->ate_flag);
  for (int oi = 0; oi < e->n_obj; ++oi) {
    const int* d = &e->objdef[oi * MPB_OBJ_COLS];
    Obj* o = &e->obj[oi];
    memset(o, 0, sizeof *o);
    o->kind = d[MPB_OBJ_KIND]; o->x = d[MPB_OBJ_X]; o->y = d[MPB_OBJ_Y]; o->orient = d[MPB_OBJ_ORIENT];
    o->state = d[MPB_OBJ_STATE]; o->prev_state = -1; o->layer = -1; o->state_frame = 0; o->movement_allowed = 1;
    if (e->obj_choice && e->obj_choice[oi * 2] >= 0) { /* prefab_utils.lua:63-65: random:choice(prefab.list), once per group */
      uint32_t w[4]; rng(e, RS_CHOICE, e->obj_choice[oi * 2], w);
      const uint32_t ticket = pick(w[0], (uint32_t)e->choice_n[e->obj_choice[oi * 2]]);
      if (!(((uint32_t)e->obj_choice[oi * 2 + 1] >> ticket) & 1u)) { o->absent = 1; o->destroyed = 1; continue; }
    }
    if (!kind_of(e, o)->is_avatar) { /* Transform:start -> createPiece (component_library.lua:236-254) */
      o->layer = state_def(e, o, o->state)->layer;
      place(e, oi);
    }
  }
  /* _avatarStart: groupShuffledWithCount per spawn group, sampled without replacement. */
  for (int g = 0; g < e->n_groups; ++g) {
    int members[1024], n = 0, k = 0;
    for (int p = 0; p < e->P; ++p) if (find_comp(e, &e->obj[e->avatar_obj[p]], MPB_C_AVATAR)->ip[3] == g) ++k;
    if (k == 0) continue;
    for (int i = 0; i < e->n_obj && n < 1024; ++i) { const Obj* c = &e->obj[i]; if (c->layer >= 0 && (state_def(e, c, c->state)->groups & (1u << g))) members[n++] = i; }
    int j = 0;
    for (int p = 0; p < e->P; ++p) {
      int oi = e->avatar_obj[p]; Obj* o = &e->obj[oi];
      const CompDef* av = find_comp(e, o, MPB_C_AVATAR);
      if (av->ip[3] != g) continue;
      uint32_t w[4]; rng(e, RS_AVATAR_RESET, p, w);
      int r = j + (int)pick(w[0], (uint32_t)(n - j)); /* partial Fisher-Yates */
      int t = members[j]; members[j] = members[r]; members[r] = t;
      o->x = e->obj[members[j]].x; o->y = e->obj[members[j]].y;
      o->orient = av->ip[10] ? (int)(w[1] & 3u) : 0;          /* Avatar:start :299-304 */
      o->layer = state_def(e, o, o->state)->layer;
      place(e, oi);
      o->spawn_group = av->ip[4] >= 0 ? av->ip[4] : av->ip[3]; /* Avatar:postStart :322-328 */
      for (int a = 0; a < 4; ++a) o->act[a] = 0;
      ++j;
    }
  }
  /* postStart on all objects. */
  for (int oi = 0; oi < e->n_obj; ++oi) {
    Obj* o = &e->obj[oi];
    if (o->absent) continue;
    const KindDef* k = kind_of(e, o);
    for (int i = 0; i < k->n_comps; ++i) {
      const CompDef* c = &e->comps[k->comp0 + i];
      if (c->type == MPB_C_ANIMATION && c->ip[11]) { /* component_library.lua:1064-1068 */
        uint32_t w[4]; rng(e, RS_OBJECT_RESET, oi, w);
        enqueue(e, ACT_SET_STATE, oi, c->ip[1 + pick(w[0], (uint32_t)c->ip[0])], 0, 0);
      } else if (c->type == MPB_C_RESOURCE) { /* Resource:reset / postStart -- components.lua:73-80,177-182 */
        o->health = c->ip[0]; o->rewarding_active = 0; o->claimed_by = -1; o->never_claimed = 1; o->destroyed = 0; o->frames_since_zapped = 0;
        o->texture_obj = e->grid[c->ip[7] * (e->W * e->H) + cell_of(e, o->x, o->y)] - 1;
        o->damage_obj = e->grid[c->ip[8] * (e->W * e->H) + cell_of(e, o->x, o->y)] - 1;
      } else if (c->type == MPB_C_REWARD_INDICATOR) { /* postStart :288-301 */
        o->paired_resource = e->grid[c->ip[2] * (e->W * e->H) + cell_of(e, o->x, o->y)] - 1;
      } else if (c->type == MPB_C_GRADUATED_SANCTIONS_MARKING) { /* reset :985-998, postStart :1033-1047 */
        o->level = c->ip[2]; o->time_not_initial = 0;
        o->marking_avatar = e->avatar_obj[c->ip[0]];
        Obj* av = &e->obj[o->marking_avatar];
        enqueue(e, ACT_SET_STATE, oi, c->ip[6] + o->level - 1, 0, 0);
        enqueue(e, ACT_TELEPORT, oi, av->x, av->y, 0);
        enqueue(e, ACT_SET_ORIENT, oi, av->orient, 0, 0);
        if (av->n_connected < 4) av->connected[av->n_connected++] = oi;
      } else if (c->type == MPB_C_DENSITY_REGROW) { /* start :139-145, postStart :147-152 */
        o->num_neighbors = 0;
        density_begin_live(e, oi, c);
        o->dr_started = 1;
        o->grass_obj = e->grid[c->ip[8] * (e->W * e->H) + cell_of(e, o->x, o->y)] - 1;
      } else if (c->type == MPB_C_DIRT_TRACKER) {    /* clean_up/components.lua:103-116 */
        if (o->state == c->ip[1]) e->clean_count++; else if (o->state == c->ip[0]) e->dirt_count++;
      }
    }
  }
  grid_update(e); /* api:start ends with one grid:update (api_factory.lua:101) */
  e->step_type = 0;
}

/* ------------------------------------------------------------------------------------------
 * Rendering: world:createView + tile.Scene:render (avatar_library.lua:225-277,
 * base_simulation.lua:347-368). Policies A.11-A.14.
 * ---------------------------------------------------------------------------------------- */
static inline void blend_px(uint8_t* dst, const uint8_t* src) {
  unsigned a = src[3];
  if (a == 255) { dst[0] = src[0]; dst[1] = src[1]; dst[2] = src[2]; }
  else if (a != 0) for (int c = 0; c < 3; ++c) dst[c] = (uint8_t)((src[c] * a + dst[c] * (255u - a)) / 255u); /* A.14: truncate */
}
static void draw_sprite(const OrEnv* e, uint8_t* img, int stride, int px, int py, int sprite, int facing) {
  int S = e->S;
  const uint8_t* t = e->atlas + ((size_t)sprite * 4 + facing) * S * S * 4;
  for (int y = 0; y < S; ++y) for (int x = 0; x < S; ++x) blend_px(img + (size_t)(py + y) * stride + (px + x) * 3, t + (y * S + x) * 4);
}
static void draw_cell(const OrEnv* e, uint8_t* img, int stride, int px, int py, int cell, int viewer, int viewer_orient) {
  int cells = e->W * e->H;
  const int* map = e->sprite_map + (size_t)viewer * e->n_sprites;
  for (int l = 0; l < e->L; ++l) {
    int q = e->grid[l * cells + cell] - 1;
    if (q >= 0) {
      const Obj* o = &e->obj[q];
      int sp = state_def(e, o, o->state)->sprite;
      if (sp >= 0) draw_sprite(e, img, stride, px, py, map[sp], (o->orient - viewer_orient) & 3);
    }
    uint16_t b = e->beam[l * cells + cell];
    if (b) draw_sprite(e, img, stride, px, py, map[(b - 1) >> 2], (((b - 1) & 3) - viewer_orient) & 3);
  }
}
void oracle_render_player(const OrEnv* e, int p, uint8_t* img) {
  int S = e->S, vw = e->view_l + e->view_r + 1, vh = e->view_f + e->view_b + 1, stride = vw * S * 3;
  memset(img, 0, (size_t)vh * S * stride);
  const Obj* a = &e->obj[e->avatar_obj[p]];
  for (int vy = 0; vy < vh; ++vy) for (int vx = 0; vx < vw; ++vx) {
    if (a->layer < 0) { draw_sprite(e, img, stride, vx * S, vy * S, e->oov_sprite, 0); continue; } /* A.13 */
    int r = (a->orient + 1) & 3, f = a->orient; /* A.11 */
    int dxr = vx - e->view_l, dyf = e->view_f - vy;
    int x = a->x + DX[r] * dxr + DX[f] * dyf, y = a->y + DY[r] * dxr + DY[f] * dyf;
    if (!wrap_or_reject(e, &x, &y)) { draw_sprite(e, img, stride, vx * S, vy * S, e->oob_sprite, 0); continue; }
    draw_cell(e, img, stride, vx * S, vy * S, cell_of(e, x, y), p, a->orient);
  }
}
void oracle_render_world(const OrEnv* e, uint8_t* img) {
  int S = e->S, stride = e->W * S * 3;
  memset(img, 0, (size_t)e->H * S * stride);
  for (int y = 0; y < e->H; ++y) for (int x = 0; x < e->W; ++x) draw_cell(e, img, stride, x * S, y * S, cell_of(e, x, y), e->P, 0);
}

/* ------------------------------------------------------------------------------------------
 * Public C API (host pointers only).
 * ---------------------------------------------------------------------------------------- */
#define SEC(name) const MpbSection* s_##name = mpb_find(blob, n, #name); if (!s_##name) { fprintf(stderr, "oracle: missing section %s\n", #name); oracle_destroy(e); return 0; }
void oracle_destroy(OrEnv* e);

OrEnv* oracle_create(const void* blob, size_t n, uint64_t seed) {
  OrEnv* e = (OrEnv*)calloc(1, sizeof(OrEnv));
  SEC(meta) SEC(atlas) SEC(sprite_opaque) SEC(states) SEC(kinds) SEC(comps) SEC(comps_f) SEC(objects) SEC(hits) SEC(action_table) SEC(sprite_map) SEC(scalar_obs)
  const int32_t* m = (const int32_t*)mpb_data(blob, s_meta);
  e->W = m[MPB_META_W]; e->H = m[MPB_META_H]; e->L = m[MPB_META_L]; e->P = m[MPB_META_P]; e->S = m[MPB_META_SPRITE_SIZE];
  e->topology = m[MPB_META_TOPOLOGY]; e->max_frames = m[MPB_META_MAX_FRAMES]; e->n_obj = m[MPB_META_N_OBJECTS];
  e->n_kinds = m[MPB_META_N_KINDS]; e->n_sprites = m[MPB_META_N_SPRITES]; e->n_hits = m[MPB_META_N_HITS]; e->n_groups = m[MPB_META_N_GROUPS];
  e->view_l = m[MPB_META_VIEW_LEFT]; e->view_r = m[MPB_META_VIEW_RIGHT]; e->view_f = m[MPB_META_VIEW_FORWARD]; e->view_b = m[MPB_META_VIEW_BACKWARD];
  e->n_actions = m[MPB_META_N_ACTIONS]; e->oob_sprite = m[MPB_META_OOB_SPRITE]; e->oov_sprite = m[MPB_META_OOV_SPRITE]; e->n_scalar = m[MPB_META_N_SCALAR_OBS];
  if (e->P > OR_MAX_PLAYERS || e->L > OR_MAX_LAYERS) { oracle_destroy(e); return 0; }
  int n_states = m[MPB_META_N_STATES], n_comps = m[MPB_META_N_COMPS];
  e->states = (StateDef*)calloc(n_states, sizeof(StateDef));
  const int32_t* st = (const int32_t*)mpb_data(blob, s_states);
  for (int i = 0; i < n_states; ++i) { e->states[i].layer = st[i * 4]; e->states[i].sprite = st[i * 4 + 1]; e->states[i].contact = st[i * 4 + 2]; e->states[i].groups = (uint32_t)st[i * 4 + 3]; }
  e->kinds = (KindDef*)calloc(e->n_kinds, sizeof(KindDef));
  const int32_t* kd = (const int32_t*)mpb_data(blob, s_kinds);
  for (int i = 0; i < e->n_kinds; ++i) { e->kinds[i].state0 = kd[i * 6]; e->kinds[i].n_states = kd[i * 6 + 1]; e->kinds[i].comp0 = kd[i * 6 + 2]; e->kinds[i].n_comps = kd[i * 6 + 3]; e->kinds[i].is_avatar = kd[i * 6 + 4]; }
  e->comps = (CompDef*)calloc(n_comps, sizeof(CompDef));
  const int32_t* ci = (const int32_t*)mpb_data(blob, s_comps); const double* cd = (const double*)mpb_data(blob, s_comps_f);
  for (int i = 0; i < n_comps; ++i) { e->comps[i].type = ci[i * (MPB_COMP_NI + 1)]; for (int j = 0; j < MPB_COMP_NI; ++j) e->comps[i].ip[j] = ci[i * (MPB_COMP_NI + 1) + 1 + j]; for (int j = 0; j < MPB_COMP_ND; ++j) e->comps[i].dp[j] = cd[i * MPB_COMP_ND + j]; }
#define DUP(dst, sec, type) e->dst = (type*)malloc(s_##sec->nbytes); memcpy(e->dst, mpb_data(blob, s_##sec), s_##sec->nbytes);
  DUP(objdef, objects, int) DUP(hits, hits, int) DUP(action_table, action_table, int) DUP(sprite_map, sprite_map, int) DUP(scalar_obs, scalar_obs, int)
  DUP(atlas, atlas, uint8_t) DUP(sprite_opaque, sprite_opaque, uint8_t)
  e->obj = (Obj*)calloc(e->n_obj, sizeof(Obj));
  e->grid = (int*)calloc((size_t)e->L * e->W * e->H, sizeof(int));
  e->beam = (uint16_t*)calloc((size_t)e->L * e->W * e->H, sizeof(uint16_t));
  for (int oi = 0; oi < e->n_obj; ++oi) {
    const KindDef* k = &e->kinds[e->objdef[oi * MPB_OBJ_COLS]];
    if (!k->is_avatar) continue;
    for (int i = 0; i < k->n_comps; ++i) if (e->comps[k->comp0 + i].type == MPB_C_AVATAR) e->avatar_obj[e->comps[k->comp0 + i].ip[0]] = oi;
  }
  for (int i = 0; i < n_comps; ++i) { /* hit names -> classes (Resource:onHit matches on the name) */
    if (e->comps[i].type == MPB_C_PAINTBRUSH && e->comps[i].ip[1] < 64) e->hit_class[e->comps[i].ip[1]] = 1;
    if (e->comps[i].type == MPB_C_RESOURCE_CLAIMER && e->comps[i].ip[4] < 64) e->hit_class[e->comps[i].ip[4]] = 2;
  }
  { const MpbSection* cg = mpb_find(blob, n, "choice_groups"); const MpbSection* oc = mpb_find(blob, n, "obj_choice");
    if (cg && oc) { e->n_choice = (int)(cg->nbytes / 4); e->choice_n = (int*)malloc(cg->nbytes); memcpy(e->choice_n, mpb_data(blob, cg), cg->nbytes);
                    e->obj_choice = (int*)malloc(oc->nbytes); memcpy(e->obj_choice, mpb_data(blob, oc), oc->nbytes); } }
  build_updaters(e);
  e->key[0] = (uint32_t)seed; e->key[1] = (uint32_t)(seed >> 32);
  e->episode = -1; e->done = 1;
  return e;
}
void oracle_destroy(OrEnv* e) {
  if (!e) return;
  free(e->states); free(e->kinds); free(e->comps); free(e->objdef); free(e->hits); free(e->action_table); free(e->sprite_map);
  free(e->scalar_obs); free(e->atlas); free(e->sprite_opaque); free(e->obj); free(e->grid); free(e->beam); free(e->q); free(e->qnext);
  free(e->ev); free(e->updaters); free(e->choice_n); free(e->obj_choice); free(e);
}
/* Starts the next episode; returns StepType.FIRST (0). */
int oracle_reset(OrEnv* e) { e->episode++; episode_start(e); return 0; }
void oracle_set_episode(OrEnv* e, int episode) { e->episode = episode - 1; }

/* One env step (api:advance, api_factory.lua:104-111). `actions[P]` are discrete action ids
 * (discrete_action_wrapper.py:97-100). Returns the step type: 0 FIRST, 1 MID, 2 LAST.
 * Policy A.17: a step after LAST ignores the action and starts a new episode. */
int oracle_step(OrEnv* e, const int32_t* actions) {
  if (e->done) return oracle_reset(e);
  e->step++;
  e->evn = 0;
  for (int p = 0; p < e->P; ++p) { /* Avatar:discreteActions -- avatar_library.lua:218-223 */
    int a = actions[p];
    if (a < 0 || a >= e->n_actions) a = 0;
    for (int f = 0; f < 4; ++f) e->obj[e->avatar_obj[p]].act[f] = e->action_table[a * 4 + f];
  }
  simulation_update(e);
  grid_update(e);
  int cont = e->cont && e->step < e->max_frames;
  e->step_type = cont ? 1 : 2;
  e->done = !cont;
  return e->step_type;
}

void oracle_get_rewards(const OrEnv* e, double* out) { for (int p = 0; p < e->P; ++p) out[p] = e->step_type == 0 ? 0.0 : e->obj[e->avatar_obj[p]].reward; }
double oracle_get_discount(const OrEnv* e) { return e->step_type == 1 ? 1.0 : 0.0; }
int oracle_get_step_type(const OrEnv* e) { return e->step_type; }
/* out[P][n_scalar] in the order of section "scalar_obs". */
void oracle_get_scalar_obs(const OrEnv* e, double* out) {
  for (int p = 0; p < e->P; ++p) {
    const Obj* o = &e->obj[e->avatar_obj[p]];
    for (int k = 0; k < e->n_scalar; ++k) {
      double v = 0.0;
      if (e->scalar_obs[k] == MPB_OBS_READY_TO_SHOOT) { /* Zapper:readyToShoot -- avatar_library.lua:737-744 */
        const CompDef* z = find_comp(e, o, MPB_C_ZAPPER);
        const CompDef* mb = find_comp(e, o, MPB_C_MINE_BEAM);
        if (mb) v = 1.0 - (double)o->mine_cool / (double)mb->ip[0]; /* MineBeam:readyToShoot -- coop_mining/components.lua:186-189 */
        else if (avatar_is_alive(e, o)) v = fmax(1.0 - (double)o->zap_cool / (double)z->ip[0], 0.0);
      } else if (e->scalar_obs[k] == MPB_OBS_NUM_OTHERS_WHO_CLEANED) v = (double)o->num_others_cleaned;
      else if (e->scalar_obs[k] == MPB_OBS_MISMATCHED_COIN_BY_PARTNER) v = (double)o->partner_mismatch;
      out[p * e->n_scalar + k] = v;
    }
  }
}
/* out[P][4] = x, y, orientation, alive. */
void oracle_get_avatars(const OrEnv* e, int32_t* out) {
  for (int p = 0; p < e->P; ++p) { const Obj* o = &e->obj[e->avatar_obj[p]]; out[p * 4] = o->x; out[p * 4 + 1] = o->y; out[p * 4 + 2] = o->orient; out[p * 4 + 3] = o->layer >= 0; }
}
/* Sprite grid in the engine's encoding: out[L][cells] uint16 (beams merged in). */
void oracle_get_grid(const OrEnv* e, uint16_t* out);
void oracle_get_grid(const OrEnv* e, uint16_t* out) {
  int cells = e->W * e->H;
  for (int l = 0; l < e->L; ++l) for (int c = 0; c < cells; ++c) {
    int q = e->grid[l * cells + c] - 1; uint16_t v = 0;
    if (q >= 0) { const Obj* o = &e->obj[q]; int sp = state_def(e, o, o->state)->sprite; if (sp >= 0) v = MPB_CELL(sp, o->orient); }
    if (e->beam[l * cells + c]) v = e->beam[l * cells + c];
    out[l * cells + c] = v;
  }
}
/* {p}.LAYER (avatar_library.lua:247-257: playerLayerView:observation{grid, piece, orientation = 'N'}): the avatar's view
 * window, NOT rotated, as sprite id + 1 per layer; 0 empty, -1 outside a BOUNDED map (policy A.21). out[view_h][view_w][L]. */
void oracle_layer_view(const OrEnv* e, int p, int32_t* out) {
  const Obj* a = &e->obj[e->avatar_obj[p]];
  const int vw = e->view_l + e->view_r + 1, vh = e->view_f + e->view_b + 1, cells = e->W * e->H;
  uint16_t* g = (uint16_t*)malloc(sizeof(uint16_t) * (size_t)e->L * cells);
  oracle_get_grid(e, g);
  for (int vy = 0; vy < vh; ++vy) for (int vx = 0; vx < vw; ++vx) {
    int x = a->x - e->view_l + vx, y = a->y - e->view_f + vy;
    const int inside = wrap_or_reject(e, &x, &y);
    for (int l = 0; l < e->L; ++l) {
      int32_t v = -1;
      if (inside) { const uint16_t q = g[(size_t)l * cells + y * e->W + x]; v = q ? ((q - 1) >> 2) + 1 : 0; }
      out[((size_t)vy * vw + vx) * e->L + l] = v;
    }
  }
  free(g);
}
int oracle_get_events(const OrEnv* e, int32_t* out, int max_events) {
  int n = e->evn < max_events ? e->evn : max_events;
  for (int i = 0; i < n; ++i) { out[i * 3] = e->ev[i].type; out[i * 3 + 1] = e->ev[i].a; out[i * 3 + 2] = e->ev[i].b; }
  return e->evn;
}
int oracle_get_object_state(const OrEnv* e, int oi) { return e->obj[oi].state; }
void oracle_get_counters(const OrEnv* e, int32_t* out) { out[0] = e->dirt_count; out[1] = e->clean_count; out[2] = e->frame; out[3] = e->step; out[4] = e->episode; }

/* Test hooks: place an avatar / set an object state directly (bypassing the queue). */
void oracle_debug_set_avatar(OrEnv* e, int p, int x, int y, int orient) {
  int oi = e->avatar_obj[p]; Obj* o = &e->obj[oi];
  lift(e, oi); o->x = x; o->y = y; o->orient = orient & 3;
  if (o->layer < 0) { o->state = find_comp(e, o, MPB_C_AVATAR)->ip[1]; o->layer = state_def(e, o, o->state)->layer; }
  place(e, oi);
  for (int k = 0; k < o->n_connected; ++k) { /* connected pieces (markings) travel with the avatar */
    Obj* c = &e->obj[o->connected[k]];
    if (c->layer < 0) continue;
    lift(e, o->connected[k]); c->x = o->x; c->y = o->y; c->orient = o->orient; place(e, o->connected[k]);
  }
}
void oracle_debug_set_object_state(OrEnv* e, int oi, int state) { do_set_state(e, oi, state); process_queue(e); }

/* CPU baseline: `n_envs` independent envs stepped `n_steps` times with uniform-random actions
 * (splitmix64 stream; not part of parity), rendering every observation each step like the
 * reference does. Envs are split over `n_threads` pthreads. Returns env-steps executed. */
static inline uint64_t splitmix64(uint64_t* s) { uint64_t z = (*s += 0x9E3779B97F4A7C15ull); z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull; z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; return z ^ (z >> 31); }
typedef struct { const void* blob; size_t n; int b0, b1, n_steps, render; uint64_t seed; long total; uint64_t sum; } RunArgs;
static void* run_worker(void* argp) {
  RunArgs* a = (RunArgs*)argp;
  for (int b = a->b0; b < a->b1; ++b) {
    OrEnv* e = oracle_create(a->blob, a->n, a->seed + (uint64_t)b);
    if (!e) continue;
    int vw = e->view_l + e->view_r + 1, vh = e->view_f + e->view_b + 1;
    uint8_t* rgb = (uint8_t*)malloc((size_t)vw * vh * e->S * e->S * 3);
    uint8_t* world = (uint8_t*)malloc((size_t)e->W * e->H * e->S * e->S * 3);
    uint64_t s = a->seed * 0x2545F4914F6CDD1Dull + (uint64_t)b; int32_t act[OR_MAX_PLAYERS]; double rew[OR_MAX_PLAYERS];
    oracle_reset(e);
    for (int t = 0; t < a->n_steps; ++t) {
      for (int p = 0; p < e->P; ++p) act[p] = (int32_t)(splitmix64(&s) % (uint64_t)e->n_actions);
      oracle_step(e, act);
      oracle_get_rewards(e, rew);
      for (int p = 0; p < e->P; ++p) a->sum += (uint64_t)rew[p];
      if (a->render) { for (int p = 0; p < e->P; ++p) { oracle_render_player(e, p, rgb); a->sum += rgb[1000]; } oracle_render_world(e, world); a->sum += world[5000]; }
      ++a->total;
    }
    free(rgb); free(world); oracle_destroy(e);
  }
  return 0;
}
long oracle_run_random(const void* blob, size_t n, int n_envs, int n_steps, int n_threads, uint64_t seed, int render, uint64_t* checksum) {
  if (n_threads < 1) n_threads = 1;
  if (n_threads > n_envs) n_threads = n_envs;
  pthread_t* th = (pthread_t*)calloc(n_threads, sizeof(pthread_t));
  RunArgs* args = (RunArgs*)calloc(n_threads, sizeof(RunArgs));
  for (int t = 0; t < n_threads; ++t) {
    RunArgs a = {blob, n, (int)((long)n_envs * t / n_threads), (int)((long)n_envs * (t + 1) / n_threads), n_steps, render, seed, 0, 0};
    args[t] = a;
    pthread_create(&th[t], 0, run_worker, &args[t]);
  }
  long total = 0; uint64_t sum = 0;
  for (int t = 0; t < n_threads; ++t) { pthread_join(th[t], 0); total += args[t].total; sum += args[t].sum; }
  free(th); free(args);
  if (checksum) *checksum = sum;
  return total;
}

/* Persistent batch for the CPU baseline / reference arm: envs live across calls. */
typedef struct OrBatch { int n_envs; OrEnv** envs; uint64_t* rng; uint8_t** rgb; uint8_t** world; uint64_t sum; } OrBatch;
OrBatch* oracle_batch_create(const void* blob, size_t n, int n_envs, uint64_t seed) {
  OrBatch* bt = (OrBatch*)calloc(1, sizeof(OrBatch));
  bt->n_envs = n_envs;
  bt->envs = (OrEnv**)calloc(n_envs, sizeof(OrEnv*)); bt->rng = (uint64_t*)calloc(n_envs, sizeof(uint64_t));
  bt->rgb = (uint8_t**)calloc(n_envs, sizeof(uint8_t*)); bt->world = (uint8_t**)calloc(n_envs, sizeof(uint8_t*));
  for (int b = 0; b < n_envs; ++b) {
    OrEnv* e = oracle_create(blob, n, seed + (uint64_t)b);
    if (!e) return 0;
    bt->envs[b] = e; bt->rng[b] = seed * 0x2545F4914F6CDD1Dull + (uint64_t)b;
    int vw = e->view_l + e->view_r + 1, vh = e->view_f + e->view_b + 1;
    bt->rgb[b] = (uint8_t*)malloc((size_t)vw * vh * e->S * e->S * 3);
    bt->world[b] = (uint8_t*)malloc((size_t)e->W * e->H * e->S * e->S * 3);
    oracle_reset(e);
  }
  return bt;
}
void oracle_batch_destroy(OrBatch* bt) {
  if (!bt) return;
  for (int b = 0; b < bt->n_envs; ++b) { oracle_destroy(bt->envs[b]); free(bt->rgb[b]); free(bt->world[b]); }
  free(bt->envs); free(bt->rng); free(bt->rgb); free(bt->world); free(bt);
}
typedef struct { OrBatch* bt; int b0, b1, n_steps, render; long total; uint64_t sum; } BatchArgs;
static void* batch_worker(void* argp) {
  BatchArgs* a = (BatchArgs*)argp;
  int32_t act[OR_MAX_PLAYERS]; double rew[OR_MAX_PLAYERS];
  for (int b = a->b0; b < a->b1; ++b) {
    OrEnv* e = a->bt->envs[b];
    for (int t = 0; t < a->n_steps; ++t) {
      for (int p = 0; p < e->P; ++p) act[p] = (int32_t)(splitmix64(&a->bt->rng[b]) % (uint64_t)e->n_actions);
      oracle_step(e, act);
      oracle_get_rewards(e, rew);
      for (int p = 0; p < e->P; ++p) a->sum += (uint64_t)rew[p];
      if (a->render) { for (int p = 0; p < e->P; ++p) { oracle_render_player(e, p, a->bt->rgb[b]); a->sum += a->bt->rgb[b][1000]; } oracle_render_world(e, a->bt->world[b]); a->sum += a->bt->world[b][5000]; }
      ++a->total;
    }
  }
  return 0;
}
/* Steps every env `n_steps` times with uniform-random actions on `n_threads` threads. */
long oracle_batch_step_random(OrBatch* bt, int n_steps, int n_threads, int render) {
  if (n_threads < 1) n_threads = 1;
  if (n_threads > bt->n_envs) n_threads = bt->n_envs;
  pthread_t* th = (pthread_t*)calloc(n_threads, sizeof(pthread_t));
  BatchArgs* args = (BatchArgs*)calloc(n_threads, sizeof(BatchArgs));
  for (int t = 0; t < n_threads; ++t) {
    BatchArgs a = {bt, (int)((long)bt->n_envs * t / n_threads), (int)((long)bt->n_envs * (t + 1) / n_threads), n_steps, render, 0, 0};
    args[t] = a;
    pthread_create(&th[t], 0, batch_worker, &args[t]);
  }
  long total = 0;
  for (int t = 0; t < n_threads; ++t) { pthread_join(th[t], 0); total += args[t].total; bt->sum += args[t].sum; }
  free(th); free(args);
  return total;
}
uint64_t oracle_batch_checksum(const OrBatch* bt) { return bt->sum; }

/* Whole-batch checking (tests only): step every env with caller-given actions on host threads, then dump every
 * output of every env into caller-owned arrays laid out like the engine's device buffers (include/mp_engine.h), so
 * a parity test compares whole batches with one array comparison per field instead of sampling envs. */
typedef struct { OrBatch* bt; int b0, b1; const int32_t* actions; } StepArgs;
static void* step_actions_worker(void* argp) {
  StepArgs* a = (StepArgs*)argp;
  for (int b = a->b0; b < a->b1; ++b) { OrEnv* e = a->bt->envs[b]; oracle_step(e, a->actions + (size_t)b * e->P); }
  return 0;
}
void oracle_batch_step_actions(OrBatch* bt, const int32_t* actions, int n_threads) {
  if (n_threads < 1) n_threads = 1;
  if (n_threads > bt->n_envs) n_threads = bt->n_envs;
  pthread_t* th = (pthread_t*)calloc(n_threads, sizeof(pthread_t));
  StepArgs* args = (StepArgs*)calloc(n_threads, sizeof(StepArgs));
  for (int t = 0; t < n_threads; ++t) {
    StepArgs a = {bt, (int)((long)bt->n_envs * t / n_threads), (int)((long)bt->n_envs * (t + 1) / n_threads), actions};
    args[t] = a;
    pthread_create(&th[t], 0, step_actions_worker, &args[t]);
  }
  for (int t = 0; t < n_threads; ++t) pthread_join(th[t], 0);
  free(th); free(args);
}
typedef struct {
  OrBatch* bt; int b0, b1, max_ev;
  double* reward; double* discount; int64_t* step_type; double* scalar_obs; int32_t* avatars; uint16_t* grid;
  int32_t* events; int32_t* n_events; uint8_t* rgb; uint8_t* world;
} DumpArgs;
static int cmp_event(const void* pa, const void* pb) {
  const int32_t* a = (const int32_t*)pa; const int32_t* b = (const int32_t*)pb;
  for (int i = 0; i < 3; ++i) if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
  return 0;
}
static void* dump_worker(void* argp) {
  DumpArgs* a = (DumpArgs*)argp;
  const int B = a->bt->n_envs;
  double tmp[OR_MAX_PLAYERS * 8];
  for (int b = a->b0; b < a->b1; ++b) {
    OrEnv* e = a->bt->envs[b];
    const int P = e->P, cells = e->W * e->H;
    if (a->reward) oracle_get_rewards(e, a->reward + (size_t)b * P);
    if (a->discount) a->discount[b] = oracle_get_discount(e);
    if (a->step_type) a->step_type[b] = oracle_get_step_type(e);
    if (a->scalar_obs && e->n_scalar) {
      oracle_get_scalar_obs(e, tmp);
      for (int k = 0; k < e->n_scalar; ++k) for (int p = 0; p < P; ++p) a->scalar_obs[((size_t)k * B + b) * P + p] = tmp[p * e->n_scalar + k];
    }
    if (a->avatars) oracle_get_avatars(e, a->avatars + (size_t)b * P * 4);
    if (a->grid) oracle_get_grid(e, a->grid + (size_t)b * e->L * cells);
    if (a->events) {
      int32_t* ev = a->events + (size_t)b * a->max_ev * 3;
      int n = oracle_get_events(e, ev, a->max_ev);
      a->n_events[b] = n;
      qsort(ev, n < a->max_ev ? n : a->max_ev, 3 * sizeof(int32_t), cmp_event);
    }
    if (a->rgb) {
      const size_t pb = (size_t)(e->view_l + e->view_r + 1) * (e->view_f + e->view_b + 1) * e->S * e->S * 3;
      for (int p = 0; p < P; ++p) oracle_render_player(e, p, a->rgb + ((size_t)b * P + p) * pb);
    }
    if (a->world) oracle_render_world(e, a->world + (size_t)b * cells * e->S * e->S * 3);
  }
  return 0;
}
/* Any output pointer may be NULL. events rows are sorted per env; n_events holds the true count. */
void oracle_batch_dump(OrBatch* bt, int n_threads, double* reward, double* discount, int64_t* step_type, double* scalar_obs,
                       int32_t* avatars, uint16_t* grid, int32_t* events, int32_t* n_events, int max_ev, uint8_t* rgb, uint8_t* world) {
  if (n_threads < 1) n_threads = 1;
  if (n_threads > bt->n_envs) n_threads = bt->n_envs;
  pthread_t* th = (pthread_t*)calloc(n_threads, sizeof(pthread_t));
  DumpArgs* args = (DumpArgs*)calloc(n_threads, sizeof(DumpArgs));
  for (int t = 0; t < n_threads; ++t) {
    DumpArgs a = {bt, (int)((long)bt->n_envs * t / n_threads), (int)((long)bt->n_envs * (t + 1) / n_threads), max_ev,
                  reward, discount, step_type, scalar_obs, avatars, grid, events, n_events, rgb, world};
    args[t] = a;
    pthread_create(&th[t], 0, dump_worker, &args[t]);
  }
  for (int t = 0; t < n_threads; ++t) pthread_join(th[t], 0);
  free(th); free(args);
}
