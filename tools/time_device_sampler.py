"""Host vs device scene sampler at C2's plugin config, on one GPU.

    python tools/time_device_sampler.py [--rounds 3] [--steps 800] [--out DIR]

Measures, in one process:
  * the `api` rate (BatchedEnvironment.step with device actions, 4096 envs, ring 32 deep, every env
    resetting each 20 steps) with sampler='host' and sampler='device', alternately, `rounds` times;
  * the refill kernel's time from CUDA events around swb_refill_device launches that each refill
    every env's whole ring (K - 1 scenes per env), and around launches that refill what one
    episode's worth of steps consumed;
  * the GPU's name and power limit (nvidia-smi), read in the same run.
Prints one JSON line (and writes it to DIR/time_device_sampler.json with --out).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from spriteworld_b200 import environment, workloads  # noqa: E402


def api_rate(wl, E, steps, sampler):
  kw = dict(sampler='device', seed=4242) if sampler == 'device' else {}
  env = environment.BatchedEnvironment(n_envs=E, rng=np.random.RandomState(4242), pool_depth=32,
                                       **dict(wl.plugin_config(), **kw))
  acts = torch.from_numpy(wl.sample_actions(np.random.RandomState(5), 16, E)).to(env.engine.device)
  for i in range(4 * wl.max_episode_length + 3):
    env.step(acts[i % 16])
  torch.cuda.synchronize()
  ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  t0 = time.perf_counter()
  ev0.record()
  for i in range(steps):
    env.step(acts[i % 16])
  ev1.record()
  torch.cuda.synchronize()
  ms = max(ev0.elapsed_time(ev1), 1e3 * (time.perf_counter() - t0))
  stats = env.refill_stats()
  env.close()
  return dict(env_steps_per_sec=E * steps / (ms * 1e-3), ms_per_step=ms / steps, refill=stats)


def refill_kernel_ms(wl, E, reps=50):
  """ms per swb_refill_device launch: (whole ring of K - 1 scenes per env, one scene per env)."""
  env = environment.BatchedEnvironment(n_envs=E, rng=np.random.RandomState(1), pool_depth=32,
                                       sampler='device', seed=1, **wl.plugin_config())
  eng = env.engine
  upto = eng.refilled_upto()
  out = {}
  for name, back in (('whole_ring', eng.pool_depth - 1), ('one_scene', 1)):
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    total = 0.0
    for r in range(reps + 3):
      upto.sub_(back)          # pretend the last `back` scenes of every ring were consumed
      ev0.record()
      eng.refill_device()
      ev1.record()
      torch.cuda.synchronize()
      if r >= 3:
        total += ev0.elapsed_time(ev1)
    out[name] = dict(ms=total / reps, scenes_per_launch=E * back,
                     scenes_per_sec=E * back / (total / reps * 1e-3))
  env.close()
  return out


def gpu_info():
  try:
    return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                          stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError) as ex:
    return 'unavailable: %s' % ex


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--steps', type=int, default=800)
  ap.add_argument('--envs', type=int, default=4096)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('time_device_sampler: no CUDA device (the numbers are GPU measurements)')
  wl = workloads.WORKLOADS['c2']()
  runs = {'host': [], 'device': []}
  for _ in range(args.rounds):
    for sampler in ('host', 'device'):
      runs[sampler].append(api_rate(wl, args.envs, args.steps, sampler))
  line = dict(
      gpu=gpu_info(), torch_device=torch.cuda.get_device_name(0), envs=args.envs, pool_depth=32,
      max_episode_length=wl.max_episode_length, steps=args.steps,
      api={k: dict(env_steps_per_sec=[r['env_steps_per_sec'] for r in v],
                   median=float(np.median([r['env_steps_per_sec'] for r in v])), refill=v[-1]['refill'])
           for k, v in runs.items()},
      refill_kernel=refill_kernel_ms(wl, args.envs))
  text = json.dumps(line)
  print(text)
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'time_device_sampler.json'), 'w') as f:
      f.write(text + '\n')


if __name__ == '__main__':
  main()
