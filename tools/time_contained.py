"""Positions inside sprites on one GPU: kernel time of swb_sample_contained.

    python tools/time_contained.py [--seconds 1.0] [--out results.json]

For the COBRA exploration (2 to 6 sprites per scene) and sorting (2 sprites) configs, at 4096 and
16384 envs drawn by the device scene sampler, after a reset and a few steps, Engine.sample_contained
of the live envs with n_samples 1, 16 and 256, each between CUDA events over many launches, warmed
up and repeated for at least --seconds.  Reports microseconds per launch and samples per second.
Prints one JSON line per case, headed by the card's name and power limit read in the same run.
Needs a CUDA device.
"""
import argparse
import importlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from time_rollout import _card, _time_alternating  # noqa: E402  (tools/ is this script's path)


def _env(name, E):
  from spriteworld_b200 import environment, renderers
  cfg = importlib.import_module('spriteworld_b200.configs.cobra.' + name).get_config('train')
  cfg['renderers'] = {'factors': renderers.SpriteFactors()}
  return environment.BatchedEnvironment(n_envs=E, pool_depth=4, rng=np.random.RandomState(0), sampler='device',
                                        seed=3, **cfg)


def run(name, E, seconds):
  import torch
  env = _env(name, E)
  env.reset()
  rng = np.random.RandomState(1)
  for _ in range(3):
    env.step(rng.uniform(0, 1, (E, 4)).astype(np.float32))
  torch.cuda.synchronize()
  eng = env.engine
  out = []
  for ns in (1, 16, 256):
    us, = _time_alternating([lambda: eng.sample_contained(12345, ns)], seconds)
    _, _, status = eng.sample_contained(12345, ns)
    out.append(dict(config=name, n_envs=E, n_samples=ns, us_per_launch=us, samples_per_s=E * ns / (us * 1e-6),
                    failed=int((status != 0).sum().item())))
  env.close()
  return out


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--seconds', type=float, default=1.0)
  p.add_argument('--out')
  args = p.parse_args()
  rows = [_card()]
  print(json.dumps(rows[0]), flush=True)
  for name in ('exploration', 'sorting'):
    for E in (4096, 16384):
      for r in run(name, E, args.seconds):
        rows.append(r)
        print(json.dumps(r), flush=True)
  if args.out:
    with open(args.out, 'w') as f:
      json.dump(rows, f, indent=1)


if __name__ == '__main__':
  main()
