"""Whole-run checkpoints on one GPU: size, BatchedEnvironment.state_dict() and load_state_dict().

    python tools/time_checkpoint.py [--repeats 5] [--out results.json]

Two shapes of goal_finding_more_targets with the device sampler (SelectMove, 64x64 at
anti_aliasing 5, 5 sprite slots as bench.py's C2): E = 4096 envs with pool_depth K = 14 (C2), and
E = 16384 with K = 32.  Each env
steps a few times, then state_dict() and load_state_dict() of that dict (a rewind) run --repeats
times, each timed on the host clock and ended by a device synchronise; the median is printed.
Before timing, a save after the load is checked to be the same bytes as the save before it.
Prints one JSON line per shape, headed by the card's name and power limit read in the same run.
Needs a CUDA device.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from time_rollout import _card  # noqa: E402  (tools/ is this script's path)


def run(E, K, repeats):
  import torch
  from spriteworld_b200 import environment
  from spriteworld_b200.configs.cobra import goal_finding_more_targets
  cfg = dict(goal_finding_more_targets.get_config('train'))
  cfg.pop('metadata', None)
  env = environment.BatchedEnvironment(n_envs=E, pool_depth=K, n_slots=5, sampler='device', seed=1,
                                       rng=np.random.RandomState(0), **cfg)
  rng = np.random.RandomState(2)
  env.reset()
  for _ in range(5):
    env.step(torch.from_numpy(rng.uniform(0, 1, (E, 4)).astype(np.float32)).cuda())
  sd = env.state_dict()
  env.load_state_dict(sd)
  assert torch.equal(env.state_dict()['engine'], sd['engine'])
  save, load = [], []
  for _ in range(repeats):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sd = env.state_dict()
    t1 = time.perf_counter()
    env.load_state_dict(sd)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    save.append(t1 - t0)
    load.append(t2 - t1)
  out = dict(n_envs=E, pool_depth=K, n_slots=env.engine.n_slots, engine_bytes=int(sd['engine'].numel()),
             state_dict_ms=round(1e3 * float(np.median(save)), 2),
             load_state_dict_ms=round(1e3 * float(np.median(load)), 2))
  env.close()
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--repeats', type=int, default=5)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  rows = [dict(_card(), tool='time_checkpoint')]
  print(json.dumps(rows[0]), flush=True)
  for E, K in ((4096, 14), (16384, 32)):
    rows.append(run(E, K, args.repeats))
    print(json.dumps(rows[-1]), flush=True)
  if args.out:
    with open(args.out, 'w') as f:
      json.dump(rows, f, indent=1)


if __name__ == '__main__':
  main()
