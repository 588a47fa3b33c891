/* oracle_keys.c -- the CPU oracle with one more entry point (TEST INFRASTRUCTURE ONLY, built by tests/oracle_keys.py).
 *
 * oracle_set_key switches an oracle env's Philox key, which the oracle otherwise fixes at oracle_create. A state-bank
 * restore with MP_RESTORE_REKEY keeps an env's state but gives it another key; switching the key of the stored env's
 * oracle env at the store point is what that restore is checked against. Compiled from the oracle's own source, so
 * OrEnv has the oracle's layout and the function applies to envs made by liboracle.so. */
#include "../oracle/mp_oracle.c"

void oracle_set_key(OrEnv* e, uint64_t key) {
  e->key[0] = (uint32_t)key;
  e->key[1] = (uint32_t)(key >> 32);
}
