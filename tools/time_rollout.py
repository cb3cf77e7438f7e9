"""Scoring C plans of T steps per env on one GPU: Engine.rollout beside the clone-and-step path.

    python tools/time_rollout.py [--seconds 1.0] [--out results.json]

Per shape, in one process and alternating, between CUDA events, each warmed up and repeated for at
least --seconds:
  rollout   Engine.rollout of (T, E, C) plans: one launch, no second engine
  clone     what the same question costs without it: a second engine of E x C envs, save_envs of the
            E envs, the records repeated C times (a device gather), load_envs into the second
            engine, then T Engine.step calls without a raster
Before anything is timed the two are compared: wherever the rollout is not padding, it must equal
the clone path bit for bit.  Shapes: C2 (goal finding, 5 slots) with 4096 envs, C in {16, 64},
T in {5, 20}; C3 (clustering, 9 slots) with 1024 envs, C = 16, T = 10.  Envs are two steps into
their episodes.  Rates are plan-steps/s = T x E x C / time, padding included.  Prints one JSON line
per shape, headed by the card's name and power limit read in the same run.  Needs a CUDA device.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = [('c2', 4096, 16, 5), ('c2', 4096, 16, 20), ('c2', 4096, 64, 5), ('c2', 4096, 64, 20),
          ('c3', 1024, 16, 10)]


def _card():
  import torch
  name = torch.cuda.get_device_name(0)
  try:
    q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader',
                        '-i', '0'], capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError) as ex:
    q = 'unavailable (%s)' % ex
  return dict(card=name, power_limit_and_max_sm_clock=q)


def _ms(fn, n):
  import torch
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(n):
    fn()
  b.record()
  b.synchronize()
  return a.elapsed_time(b)


def _time_alternating(fns, seconds):
  """Mean microseconds per call of each of `fns`, measured in alternating batches until each has
  run for at least `seconds`."""
  import torch
  for fn in fns:
    for _ in range(3):
      fn()
  torch.cuda.synchronize()
  n = [max(1, int(50.0 / max(_ms(fn, 2) / 2, 1e-3))) for fn in fns]     # batches of about 50 ms
  total, calls = [0.0] * len(fns), [0] * len(fns)
  while min(total) < 1e3 * seconds:
    for i, fn in enumerate(fns):
      total[i] += _ms(fn, n[i])
      calls[i] += n[i]
  return [1e3 * t / c for t, c in zip(total, calls)]


def run(key, E, C, T, seconds):
  import torch
  from spriteworld_b200 import _native, constants, engine, workloads
  wl = workloads.WORKLOADS[key]()
  eng, _, _ = workloads.build_engine(wl, E, 4)
  rng = np.random.RandomState(7)
  for a in wl.sample_actions(rng, 3, E):
    eng.step(torch.from_numpy(a).to(eng.device))
  plans = torch.from_numpy(rng.uniform(0, 1, (T, E, C, 4)).astype(np.float32)).to(eng.device)
  flat = plans.reshape(T, E * C, 4)
  big = engine.Engine(E * C, wl.n_slots, 1, wl.action, wl.nodes, constants.SHAPES,
                      max_episode_length=wl.max_episode_length)
  repeat = torch.arange(E, device=eng.device).repeat_interleave(C)
  out = torch.empty(T * E * C * engine.OUT_BYTES_PER_ENV, dtype=torch.uint8, device=eng.device)
  cloned = {k: torch.empty((T, E * C), dtype=d, device=eng.device) for k, d in (
      ('reward', torch.float64), ('step_type', torch.int8), ('success', torch.uint8), ('status', torch.uint8))}

  def rollout():
    return eng.rollout(plans, out=out)

  def clone(keep=False):
    saved = eng.save_envs()
    big.load_envs(engine.EnvStates(saved.data[repeat], saved.span_class, saved.signature, saved.n_slots))
    for t in range(T):
      res = big.step(flat[t])
      if keep:
        for k, v in cloned.items():
          v[t].copy_(getattr(res, k))

  got = rollout()
  clone(keep=True)
  live = got.step_type.reshape(T, E * C) != _native.STEP_NONE
  for k, v in cloned.items():
    a, b = getattr(got, k).reshape(T, E * C)[live], v[live]
    if k == 'reward':
      a, b = a.view(torch.int64), b.view(torch.int64)
    if not torch.equal(a, b):
      raise SystemExit('%s: rollout and clone-and-step disagree on %s' % (key, k))
  us = _time_alternating([rollout, clone], seconds)
  n = T * E * C
  res = dict(workload=key, n_envs=E, n_candidates=C, n_steps=T, live_share=float(live.float().mean().item()),
             rollout_us=us[0], clone_us=us[1], rollout_plan_steps_per_s=n / us[0] * 1e6,
             clone_plan_steps_per_s=n / us[1] * 1e6, speedup=us[1] / us[0])
  big.close()
  eng.close()
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--seconds', type=float, default=1.0)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  import torch
  if not torch.cuda.is_available():
    raise SystemExit('time_rollout.py measures on a CUDA device; there is none')
  from spriteworld_b200 import build
  build.build()
  lines = [_card()]
  print(json.dumps(lines[0]), flush=True)
  for key, E, C, T in SHAPES:
    lines.append(run(key, E, C, T, args.seconds))
    print(json.dumps(lines[-1]), flush=True)
  if args.out:
    with open(args.out, 'w') as f:
      json.dump(lines, f, indent=1)


if __name__ == '__main__':
  main()
