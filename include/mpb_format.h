/* mpb_format.h -- layout of a compiled-substrate blob ("MPB1").
 *
 * A blob is what the Python substrate compiler (meltingpot_b200/compiler.py)
 * emits from a reference lab2d settings dict -- the value that
 * meltingpot/utils/substrates/builder.py:142-187 would hand to
 * dmlab2d.Lab2d(...). It replaces the {str:str} settings flattening
 * (builder.py:55-67) + Lua world construction (base_simulation.lua:77-148,
 * 253-320; prefab_utils.lua:163-176) with flat numeric tables.
 *
 * File = MpbHeader, n_sections x MpbSection, then 16-byte aligned payloads.
 * Plain C99; shared by the CUDA engine (meltingpot_b200/csrc) and by the CPU
 * oracle (oracle/), which otherwise share no code.
 *
 * The meta fields, ids, table columns and every slot of the family parameter
 * blocks "<fam>_ip" / "<fam>_dp" are named here. The compiler mirrors these
 * enums by name (META, FAMILY, FP, CU_I, ... in compiler.py) and
 * tests/test_blob_layout_cpu.py checks the mirrors against this file; the
 * engine decodes a family's blocks in that family's step_<family>.cuh.
 */
#ifndef MPB_FORMAT_H_
#define MPB_FORMAT_H_

#include <stdint.h>
#include <string.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MPB_MAGIC "MPB1"
#define MPB_VERSION 4u
#define MPB_NAME_LEN 32

enum MpbDtype { MPB_U8 = 0, MPB_U16 = 1, MPB_I32 = 2, MPB_F64 = 3, MPB_I64 = 4, MPB_CHAR = 5 };

typedef struct MpbHeader {
  char magic[4];
  uint32_t version;
  uint32_t n_sections;
  uint32_t reserved;
} MpbHeader;

typedef struct MpbSection {
  char name[MPB_NAME_LEN];
  uint32_t dtype;
  uint32_t ndim;
  uint32_t shape[4];
  uint64_t offset; /* from start of blob */
  uint64_t nbytes;
} MpbSection;

/* Indices into section "meta" (int32[MPB_META_COUNT]). */
enum MpbMeta {
  MPB_META_FAMILY = 0,       /* MpbFamily */
  MPB_META_W = 1,            /* map width in cells */
  MPB_META_H = 2,            /* map height in cells */
  MPB_META_L = 3,            /* number of layers == render order length */
  MPB_META_P = 4,            /* number of players */
  MPB_META_SPRITE_SIZE = 5,  /* pixels per cell edge (8) */
  MPB_META_TOPOLOGY = 6,     /* 0 BOUNDED, 1 TORUS */
  MPB_META_MAX_FRAMES = 7,   /* maxEpisodeLengthFrames */
  MPB_META_N_OBJECTS = 8,
  MPB_META_N_KINDS = 9,
  MPB_META_N_STATES = 10,
  MPB_META_N_COMPS = 11,
  MPB_META_N_SPRITES = 12,
  MPB_META_N_HITS = 13,
  MPB_META_N_GROUPS = 14,
  MPB_META_VIEW_LEFT = 15,
  MPB_META_VIEW_RIGHT = 16,
  MPB_META_VIEW_FORWARD = 17,
  MPB_META_VIEW_BACKWARD = 18,
  MPB_META_N_ACTIONS = 19,
  MPB_META_N_ACTION_FIELDS = 20,
  MPB_META_OOB_SPRITE = 21,  /* 'OutOfBounds' sprite id */
  MPB_META_OOV_SPRITE = 22,  /* 'OutOfView' sprite id */
  MPB_META_N_SCALAR_OBS = 23, /* per-player f64 observations besides REWARD */
  MPB_META_COUNT = 32
};

enum MpbFamily { MPB_FAMILY_CLEAN_UP = 1, MPB_FAMILY_COMMONS_HARVEST = 2, MPB_FAMILY_TERRITORY = 3, MPB_FAMILY_COINS = 4, MPB_FAMILY_COOP_MINING = 5 };

/* Family parameter blocks. The blob of family <fam> carries its scalar parameters in two sections, "<fam>_ip"
 * (int32[MPB_<FAM>_I_COUNT]) and "<fam>_dp" (f64[MPB_<FAM>_D_COUNT]), with <fam> one of cu (clean_up), ch
 * (commons_harvest), tr (territory), co (coins) and cm (coop_mining). Every slot the compiler writes has a name below;
 * the others are 0. A run of slots ending in _0, _1, ... is an array and is read as first slot + index. */

/* Zapper and StochasticIntervalEpisodeEnding slots the int32 blocks of clean_up, commons_harvest and territory share. */
enum MpbFamilyShared {
  MPB_FP_ZAP_COOLDOWN = 12, MPB_FP_ZAP_LENGTH = 13, MPB_FP_ZAP_RADIUS = 14, MPB_FP_ZAP_RESPAWN = 15 /* framesTillRespawn */,
  MPB_FP_ZAP_REMOVE = 16 /* removeHitPlayer */, MPB_FP_ZAP_LAYER = 21, MPB_FP_ZAP_SPRITE = 22,
  MPB_FP_END_MIN_FRAMES = 26, MPB_FP_END_INTERVAL = 27
};

enum MpbCleanUpI {
  MPB_CU_I_N_APPLES = 0, MPB_CU_I_N_DIRT = 1, MPB_CU_I_N_WATER = 2, MPB_CU_I_APPLE_LAYER = 3, MPB_CU_I_APPLE_SPRITE = 4,
  MPB_CU_I_DIRT_LAYER = 5, MPB_CU_I_DIRT_SPRITE = 6, MPB_CU_I_DIRT_WAIT_LAYER = 7, MPB_CU_I_WATER_LAYER = 8,
  MPB_CU_I_N_ANIM = 9, MPB_CU_I_ANIM_FRAMES = 10 /* gameFramesPerAnimationFrame */, MPB_CU_I_ANIM_RANDOM = 11,
  MPB_CU_I_CLEAN_COOLDOWN = 18, MPB_CU_I_CLEAN_LENGTH = 19, MPB_CU_I_CLEAN_RADIUS = 20, MPB_CU_I_CLEAN_LAYER = 23,
  MPB_CU_I_CLEAN_SPRITE = 24, MPB_CU_I_DIRT_DELAY = 25, MPB_CU_I_TASTE_ROLE = 28,
  MPB_CU_I_COUNT = 48
};
enum MpbCleanUpD {
  MPB_CU_D_GROW_RATE = 0, MPB_CU_D_GROW_DEPLETION = 1, MPB_CU_D_GROW_RESTORATION = 2, MPB_CU_D_EAT_REWARD = 3,
  MPB_CU_D_ZAP_PENALTY = 4, MPB_CU_D_ZAP_REWARD = 5, MPB_CU_D_DIRT_PROB = 6, MPB_CU_D_END_PROB = 7,
  MPB_CU_D_TASTE_AMOUNT = 8,
  MPB_CU_D_COUNT = 16
};

enum MpbCommonsI {
  MPB_CH_I_N_APPLES = 0, MPB_CH_I_APPLE_LAYER = 1, MPB_CH_I_APPLE_SPRITE = 2, MPB_CH_I_WAIT_LAYER = 3,
  MPB_CH_I_WAIT_SPRITE = 4, MPB_CH_I_N_WAIT = 5 /* appleWait_<k> states */, MPB_CH_I_N_PROBS = 6,
  MPB_CH_I_GRASS_LAYER = 7, MPB_CH_I_GRASS_SPRITE = 8, MPB_CH_I_DESS_SPRITE = 9,
  MPB_CH_I_COUNT = 48
};
enum MpbCommonsD {
  MPB_CH_D_PROB_0 = 0, MPB_CH_D_PROB_1 = 1, MPB_CH_D_PROB_2 = 2, MPB_CH_D_PROB_3 = 3 /* regrowthProbabilities */,
  MPB_CH_D_EAT_REWARD = 4, MPB_CH_D_ZAP_PENALTY = 5, MPB_CH_D_ZAP_REWARD = 6, MPB_CH_D_END_PROB = 7,
  MPB_CH_D_COUNT = 16
};

/* Marking level l (0-based) of territory: int32 slots MPB_TR_I_MARK_*_0 + 4 l, f64 slots MPB_TR_D_MARK_*_0 + 2 l. */
enum MpbTerritoryI {
  MPB_TR_I_N_RES = 0, MPB_TR_I_RES_LAYER = 1, MPB_TR_I_UNCLAIMED_SPRITE = 2, MPB_TR_I_TEX_LAYER = 3,
  MPB_TR_I_TEX_SPRITE = 4, MPB_TR_I_IND_LAYER = 5, MPB_TR_I_DMG_LAYER = 6, MPB_TR_I_DMG_SPRITE = 7,
  MPB_TR_I_MARK_LAYER = 8, MPB_TR_I_MARK_INITIAL_LEVEL = 9, MPB_TR_I_MARK_RECOVERY = 10, MPB_TR_I_MARK_N_LEVELS = 11,
  MPB_TR_I_CLAIM_LENGTH = 18, MPB_TR_I_CLAIM_RADIUS = 19, MPB_TR_I_CLAIM_WAIT = 20, MPB_TR_I_BRUSH_LAYER = 23,
  MPB_TR_I_CLAIM_LAYER = 24, MPB_TR_I_RES_HEALTH = 28, MPB_TR_I_RES_REWARD_DELAY = 29, MPB_TR_I_RES_REPAIR_DELAY = 30,
  MPB_TR_I_TASTE_ROLE = 31,
  MPB_TR_I_MARK_INC_0 = 32, MPB_TR_I_MARK_REMOVE_0 = 33, MPB_TR_I_MARK_FREEZE_0 = 34, MPB_TR_I_MARK_SPRITE_0 = 35,
  MPB_TR_I_MARK_INC_1 = 36, MPB_TR_I_MARK_REMOVE_1 = 37, MPB_TR_I_MARK_FREEZE_1 = 38, MPB_TR_I_MARK_SPRITE_1 = 39,
  MPB_TR_I_MARK_INC_2 = 40, MPB_TR_I_MARK_REMOVE_2 = 41, MPB_TR_I_MARK_FREEZE_2 = 42, MPB_TR_I_MARK_SPRITE_2 = 43,
  MPB_TR_I_COUNT = 64
};
enum MpbTerritoryD {
  MPB_TR_D_RES_REWARD = 0, MPB_TR_D_RES_RATE = 1, MPB_TR_D_RES_REPAIR_PROB = 2, MPB_TR_D_ZAP_PENALTY = 3,
  MPB_TR_D_ZAP_REWARD = 4, MPB_TR_D_END_PROB = 5, MPB_TR_D_TASTE_AMOUNT = 6, MPB_TR_D_TASTE_MULT = 7,
  MPB_TR_D_MARK_SRC_REWARD_0 = 8, MPB_TR_D_MARK_TGT_REWARD_0 = 9, MPB_TR_D_MARK_SRC_REWARD_1 = 10,
  MPB_TR_D_MARK_TGT_REWARD_1 = 11, MPB_TR_D_MARK_SRC_REWARD_2 = 12, MPB_TR_D_MARK_TGT_REWARD_2 = 13,
  MPB_TR_D_COUNT = 16
};

enum MpbCoinsI {
  MPB_CO_I_N_COINS = 0, MPB_CO_I_COIN_LAYER = 1, MPB_CO_I_COIN_SPRITE_0 = 2, MPB_CO_I_COIN_SPRITE_1 = 3 /* liveStateA, B */,
  MPB_CO_I_TERMINATE = 4, MPB_CO_I_TERMINATE_N = 5, MPB_CO_I_END_MIN_FRAMES = 6, MPB_CO_I_END_INTERVAL = 7,
  MPB_CO_I_COIN_TYPE_0 = 8, MPB_CO_I_COIN_TYPE_1 = 9 /* PlayerCoinType of each player */,
  MPB_CO_I_COUNT = 48
};
/* Coin rewards as collecting player p pays them (base reward x p's Role multiplier): slots MPB_CO_D_REWARD_0_* + 4 p. */
enum MpbCoinsD {
  MPB_CO_D_REGROW_RATE = 0, MPB_CO_D_END_PROB = 1,
  MPB_CO_D_REWARD_0_SELF_MATCH = 4, MPB_CO_D_REWARD_0_SELF_MISMATCH = 5, MPB_CO_D_REWARD_0_OTHER_MATCH = 6,
  MPB_CO_D_REWARD_0_OTHER_MISMATCH = 7, MPB_CO_D_REWARD_1_SELF_MATCH = 8, MPB_CO_D_REWARD_1_SELF_MISMATCH = 9,
  MPB_CO_D_REWARD_1_OTHER_MATCH = 10, MPB_CO_D_REWARD_1_OTHER_MISMATCH = 11,
  MPB_CO_D_COUNT = 16
};

/* Ore sprites 0..3: wait, single-miner raw, two-miner raw, two-miner partial. Ore types 0 / 1: one miner / two miners. */
enum MpbMiningI {
  MPB_CM_I_N_ORES = 0, MPB_CM_I_ORE_LAYER = 1, MPB_CM_I_ORE_SPRITE_0 = 2, MPB_CM_I_ORE_SPRITE_1 = 3,
  MPB_CM_I_ORE_SPRITE_2 = 4, MPB_CM_I_ORE_SPRITE_3 = 5, MPB_CM_I_MINE_WINDOW = 6, MPB_CM_I_MINE_COOLDOWN = 7,
  MPB_CM_I_MINE_LENGTH = 8, MPB_CM_I_MINE_LAYER = 9, MPB_CM_I_MINE_SPRITE = 10, MPB_CM_I_END_MIN_FRAMES = 11,
  MPB_CM_I_END_INTERVAL = 12, MPB_CM_I_MINE_HIT = 13,
  MPB_CM_I_COUNT = 48
};
enum MpbMiningD {
  MPB_CM_D_RATE_0 = 0, MPB_CM_D_RATE_1 = 1 /* FixedRateRegrow liveRates */, MPB_CM_D_END_PROB = 2,
  MPB_CM_D_MINE_REWARD_0 = 4, MPB_CM_D_MINE_REWARD_1 = 5, MPB_CM_D_EXTRACT_REWARD_0 = 6, MPB_CM_D_EXTRACT_REWARD_1 = 7,
  MPB_CM_D_COUNT = 16
};

/* Primitive action fields (columns of section "action_table"). */
enum MpbActionField { MPB_ACT_MOVE = 0, MPB_ACT_TURN = 1, MPB_ACT_FIRE_ZAP = 2 /* fireZap | mine */, MPB_ACT_FIRE_2 = 3 /* fireClean | fireClaim */ };

/* Per-player scalar observation ids (section "scalar_obs", int32[N_SCALAR_OBS]). */
enum MpbScalarObs { MPB_OBS_READY_TO_SHOOT = 0, MPB_OBS_NUM_OTHERS_WHO_CLEANED = 1, MPB_OBS_MISMATCHED_COIN_BY_PARTNER = 2 };

/* Component type ids (section "comps", column 0). */
enum MpbComp {
  MPB_C_STATE_MANAGER = 1,
  MPB_C_TRANSFORM = 2,
  MPB_C_APPEARANCE = 3,
  MPB_C_BEAM_BLOCKER = 4,      /* ip0 hit id */
  MPB_C_EDIBLE = 5,            /* ip0 live state, ip1 wait state; dp0 reward */
  MPB_C_APPLE_GROW = 6,        /* ip0 apple state; dp0 max rate, dp1 depletion, dp2 restoration */
  MPB_C_DIRT_TRACKER = 7,      /* ip0 active state, ip1 inactive state */
  MPB_C_DIRT_CLEANING = 8,     /* ip0 dirt state, ip1 dirtWait state, ip2 cleanHit id */
  MPB_C_AVATAR = 9,            /* ip0 index0, ip1 alive, ip2 wait, ip3 spawn group, ip4 post-initial group|-1,
                                  ip5..8 view l r f b, ip9 skipWaitStateRewards, ip10 randomizeInitialOrientation; dp0 speed */
  MPB_C_ZAPPER = 10,           /* ip0 cooldown, ip1 length, ip2 radius, ip3 framesTillRespawn, ip4 removeHitPlayer, ip5 zapHit id;
                                  dp0 penaltyForBeingZapped, dp1 rewardForZapping */
  MPB_C_READY_TO_SHOOT = 11,
  MPB_C_CLEANER = 12,          /* ip0 cooldown, ip1 length, ip2 radius, ip3 cleanHit id */
  MPB_C_TASTE = 13,            /* ip0 role (0 free, 1 cleaner, 2 consumer); dp0 rewardAmount */
  MPB_C_ALL_NONSELF_CUMULANTS = 14,
  MPB_C_AVATAR_METRIC_REPORTER = 15,
  MPB_C_RIVER_MONITOR = 16,
  MPB_C_DIRT_SPAWNER = 17,     /* ip0 delayStartOfDirtSpawning; dp0 dirtSpawnProbability */
  MPB_C_STOCHASTIC_INTERVAL_EPISODE_ENDING = 18, /* ip0 minimumFramesPerEpisode, ip1 intervalLength; dp0 probability */
  MPB_C_GLOBAL_DATA = 19,
  MPB_C_ANIMATION = 20,        /* ip0 n states, ip1..ip8 states, ip9 gameFramesPerAnimationFrame, ip10 loop, ip11 randomStartFrame */
  MPB_C_ADDITIONAL_SPRITES = 21,
  MPB_C_NEIGHBORHOODS = 22,
  MPB_C_DENSITY_REGROW = 23,   /* ip0 live state, ip1 first wait_k state, ip2 n wait_k states, ip3 plain wait state,
                                  ip4 n probabilities, ip5 canRegrowIfOccupied; dp0 radius, dp1.. probabilities */
  MPB_C_LOCATION_OBSERVER = 24,
  MPB_C_ALL_BEAM_BLOCKER = 25,
  MPB_C_RESOURCE = 26,         /* ip0 initialHealth, ip1 destroyed state, ip2 rewardDelay, ip3 delayTillSelfRepair, ip4 claimed_by_1 state,
                                  ip5 initial state, ip6 claimedResources group, ip7 texture layer, ip8 damage-indicator layer,
                                  ip9 texture 'destroyed' state, ip10 damage 'inactive' state, ip11 damage 'damaged' state;
                                  dp0 reward, dp1 rewardRate, dp2 selfRepairProbability */
  MPB_C_RESOURCE_CLAIMER = 27, /* ip0 player index0, ip1 beamLength, ip2 beamRadius, ip3 beamWait, ip4 claimBeam hit id */
  MPB_C_REWARD_INDICATOR = 28, /* ip0 'inactive' state, ip1 dry_claimed_by_1 state, ip2 resource layer */
  MPB_C_PAINTBRUSH = 29,       /* ip0 player index0, ip1 directionHit id */
  MPB_C_GRADUATED_SANCTIONS_MARKING = 30, /* ip0 player index0, ip1 wait state, ip2 initialLevel, ip3 recoveryTime|-1, ip4 hit id,
                                  ip5 n levels, ip6 level_1 state, ip(7+3l) levelIncrement, ip(8+3l) remove, ip(9+3l) freeze;
                                  dp(2l) sourceReward, dp(2l+1) targetReward */
  MPB_C_TERRITORY_TASTE = 31,  /* ip0 role (0 none, 1 rewarded_per_claim, 2 rewarded_per_claim_only); dp0 rewardAmount, dp1 firstClaimRewardMultiplier */
  MPB_C_ROLE = 32,             /* inert: the role string only matters to RoleBasedRewardTile */
  MPB_C_ROLE_BASED_REWARD_TILE = 33, /* inert: the compiler rejects configs in which an avatar's role is rewarded */
  MPB_C_COIN = 34,             /* ip0 wait state, ip1 terminateEpisode, ip2 coinsToTerminateEpisode;
                                  dp0 rewardSelfForMatch, dp1 rewardSelfForMismatch, dp2 rewardOtherForMatch, dp3 rewardOtherForMismatch */
  MPB_C_CHOICE_COIN_REGROW = 35, /* ip0 liveStateA, ip1 liveStateB, ip2 wait state; dp0 regrowRate */
  MPB_C_GLOBAL_COIN_COLLECTION_TRACKER = 36,
  MPB_C_PLAYER_COIN_TYPE = 37, /* ip0 0 / 1: the player's coin type is the coin's liveStateA / liveStateB */
  MPB_C_COINS_ROLE = 38,       /* dp0..3 multipliers of the four Coin rewards (self match, self mismatch, other match, other mismatch) */
  MPB_C_PARTNER_TRACKER = 39,
  MPB_C_FIXED_RATE_REGROW = 40, /* ip0 n live states (<= 4), ip1..4 live states, ip5 wait state; dp0..3 rates */
  MPB_C_ORE = 41,              /* ip0 wait state, ip1 raw state, ip2 partial state, ip3 minNumMiners, ip4 miningWindow */
  MPB_C_MINE_BEAM = 42,        /* ip0 cooldownTime, ip1 beamLength, ip2 beamRadius, ip3 'mine' hit id;
                                  dp0..1 roleRewardForMining[role][1..2], dp2..3 roleRewardForExtracting[role][1..2] */
  MPB_C_MINING_TRACKER = 43,
  MPB_C_COUNT
};

#define MPB_COMP_NI 16
#define MPB_COMP_ND 6

/* Columns of int32 tables. */
enum { MPB_STATE_LAYER = 0, MPB_STATE_SPRITE = 1, MPB_STATE_CONTACT = 2, MPB_STATE_GROUPS = 3, MPB_STATE_COLS = 4 };
enum { MPB_KIND_STATE0 = 0, MPB_KIND_NSTATES = 1, MPB_KIND_COMP0 = 2, MPB_KIND_NCOMPS = 3, MPB_KIND_IS_AVATAR = 4, MPB_KIND_COLS = 6 };
enum { MPB_OBJ_KIND = 0, MPB_OBJ_X = 1, MPB_OBJ_Y = 2, MPB_OBJ_ORIENT = 3, MPB_OBJ_STATE = 4, MPB_OBJ_COLS = 5 };
enum { MPB_HIT_LAYER = 0, MPB_HIT_SPRITE = 1, MPB_HIT_COLS = 2 };

/* Grid cell encoding used by engine and oracle: 0 = empty, else 1 + sprite*4 + orientation. */
#define MPB_CELL_EMPTY 0
#define MPB_CELL(sprite, orient) ((uint16_t)(1 + (sprite) * 4 + ((orient) & 3)))

/* Returns the section named `name`, or NULL. `blob` must hold `n` valid bytes. */
static inline const MpbSection* mpb_find(const void* blob, size_t n, const char* name) {
  const MpbHeader* h = (const MpbHeader*)blob;
  if (n < sizeof(MpbHeader) || memcmp(h->magic, MPB_MAGIC, 4) != 0 || h->version != MPB_VERSION) return 0;
  if (n < sizeof(MpbHeader) + (size_t)h->n_sections * sizeof(MpbSection)) return 0;
  const MpbSection* s = (const MpbSection*)((const char*)blob + sizeof(MpbHeader));
  for (uint32_t i = 0; i < h->n_sections; ++i) {
    if (strncmp(s[i].name, name, MPB_NAME_LEN) == 0) {
      if (s[i].offset + s[i].nbytes > n) return 0;
      return &s[i];
    }
  }
  return 0;
}

static inline const void* mpb_data(const void* blob, const MpbSection* s) {
  return (const char*)blob + s->offset;
}

#ifdef __cplusplus
}
#endif
#endif /* MPB_FORMAT_H_ */
