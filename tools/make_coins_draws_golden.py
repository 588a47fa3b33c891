"""Records a set of coins draws: the lab2d settings the reference's coins builder returns for each of DRAW_SEEDS.

coins' builder draws its map interior (width and height each in 10..15, padded to 15x15 inside the walls) and an
ordered pair of coin colours out of five on every build. The seeds below cover the smallest (10x10) and the largest
(15x15) interior and eleven colour pairs, five of them in both orders. The record, in
tests/golden/settings_coins_draws__2p.json.gz, has the layout of tools/make_settings_golden.py's files, so the GPU
tests compile the draw set (compiler.compile_settings_set) without a reference checkout. Each stored draw is checked
to compile to the blob the checkout's config gives for its seed, alone and inside the set.

  MELTINGPOT_REFERENCE_ROOT=<checkout> python tools/make_coins_draws_golden.py
"""
import gzip
import json
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from meltingpot_b200 import compiler  # noqa: E402
from make_settings_golden import config_record  # noqa: E402

DRAW_SEEDS = (93, 179, 13, 91, 173, 0, 1, 2, 5, 6, 7, 8, 14, 17, 19, 21)
PATH = os.path.join(ROOT, 'tests', 'golden', 'settings_coins_draws__2p.json.gz')


def main():
  if compiler.reference_root() is None:
    raise SystemExit('set MELTINGPOT_REFERENCE_ROOT to a Melting Pot checkout')
  config = compiler.load_reference_config('coins')
  roles = ('default',) * 2
  by_seed = {}
  for seed in DRAW_SEEDS:
    state = random.getstate()
    try:
      random.seed(seed)
      by_seed[str(seed)] = compiler._plain(config.lab2d_settings_builder(roles=roles, config=config))  # pylint: disable=protected-access
    finally:
      random.setstate(state)
  rec = json.loads(json.dumps({'substrate': 'coins', 'players': 2, 'seeds': list(DRAW_SEEDS), 'config': config_record(config),
                               'settings': by_seed}))
  with gzip.open(PATH, 'wt') as f:
    json.dump(rec, f, separators=(',', ':'))
  stored = [compiler.compile_settings(rec['settings'][str(s)], config, s) for s in DRAW_SEEDS]
  for seed, blob in zip(DRAW_SEEDS, stored):
    assert blob == compiler.compile_substrate('coins', roles, build_seed=seed), seed
  assert compiler.compile_settings_set([rec['settings'][str(s)] for s in DRAW_SEEDS], config, DRAW_SEEDS) == \
      compiler.compile_substrate_set('coins', roles, DRAW_SEEDS)
  print(PATH, os.path.getsize(PATH))


if __name__ == '__main__':
  main()
