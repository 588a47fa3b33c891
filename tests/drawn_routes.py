"""The draw rule of drawn routes (mp_run's draw), on the host, for the tests.

Player slot p of an env with Philox key `key` plays, in episode `episode`, choice
pick(philox4x32_10(counter {0, episode, p, RS_ROUTE}, key {key low, key high}).x, n) of its n choices, where
pick(w, n) = w * n >> 32 and RS_ROUTE = 6 (common.cuh). Built on the CPU oracle's Philox (oracle_philox), which every
other draw of the oracle uses too.
"""

from oracle import binding as oracle

RS_ROUTE = 6


def route_draw(key: int, episode: int, p: int, n: int) -> int:
  """The choice slot p plays in `episode` under `key`, or -1 for a slot without choices (n == 0)."""
  if n <= 0:
    return -1
  w = oracle.philox([0, episode & 0xffffffff, p, RS_ROUTE], [key & 0xffffffff, (key >> 32) & 0xffffffff])[0]
  return (w * n) >> 32
