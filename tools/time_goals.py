"""Step rate of configs/examples/goal_finding_random_goal (goals drawn per scene) against its
constant-goal twin (cobra/goal_finding_new_position's scene and task) at C2 size (4096 envs), with
and without its GoalPositions observation, and
the throughput of BatchedEnvironment.evaluate (relabelling env records with new goals).

  python tools/time_goals.py [--envs 4096] [--steps 400]

Prints one JSON line.  Rates are env-steps/s and records/s, timed with CUDA events around work that
ends in a device synchronise; the GPU's name and power limit are printed beside them."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from spriteworld_b200 import environment  # noqa: E402
from spriteworld_b200.configs.cobra import goal_finding_new_position  # noqa: E402
from spriteworld_b200.configs.examples import goal_finding_random_goal  # noqa: E402


def _rate(env, steps, n_envs):
  acts = torch.rand((steps, n_envs, 4), dtype=torch.float32, device=env.engine.device)
  env.reset()
  for t in range(20):
    env.step(acts[t])
  torch.cuda.synchronize()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for t in range(steps):
    env.step(acts[t])
  b.record()
  torch.cuda.synchronize()
  return steps * n_envs / (a.elapsed_time(b) / 1e3)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--envs', type=int, default=4096)
  ap.add_argument('--steps', type=int, default=400)
  args = ap.parse_args()
  out = {}
  variants = (('constant_goal', goal_finding_new_position, True),
              ('random_goal_unobserved', goal_finding_random_goal, False),   # no GoalPositions
              ('random_goal', goal_finding_random_goal, True))
  for name, mod, observe_goals in variants:
    cfg = dict(mod.get_config('train'))
    cfg.pop('metadata')
    if not observe_goals:
      cfg['renderers'] = {k: r for k, r in cfg['renderers'].items() if k != 'goal'}
    env = environment.BatchedEnvironment(n_envs=args.envs, pool_depth=14, rng=np.random.RandomState(0), **cfg)
    out[name + '_env_steps_per_s'] = _rate(env, args.steps, args.envs)
    if name == 'random_goal':
      states = env.save_envs()
      reps = 50
      goals = torch.rand((len(states), 1, 2), dtype=torch.float64, device=env.engine.device)
      env.evaluate(states, goals)
      torch.cuda.synchronize()
      a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      a.record()
      for _ in range(reps):
        env.evaluate(states, goals)
      b.record()
      torch.cuda.synchronize()
      out['evaluate_records_per_s'] = reps * len(states) / (a.elapsed_time(b) / 1e3)
    env.close()
  try:
    out['gpu'] = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                                capture_output=True, text=True, check=True).stdout.strip()
  except Exception as ex:  # pragma: no cover
    out['gpu'] = 'unknown (%s)' % ex
  print(json.dumps(out))


if __name__ == '__main__':
  main()
