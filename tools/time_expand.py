"""One level of a search tree on one GPU: rollouts that write leaves, beside the paths without them.

    python tools/time_expand.py [--seconds 1.0] [--out results.json]

Per shape, in one process and alternating, between CUDA events, each warmed up and repeated for at
least --seconds:
  (a) rollout          Engine.rollout of (T, E, C) plans from the live envs, no leaves
      rollout_leaves   the same with leaves=True: the E x C end states written as env records
  (b) expand           Engine.rollout from E saved records (states=) with leaves=True
      clone            the same question without it: the records repeated C times (a device
                       gather), load_envs into a second engine of E x C envs, T Engine.step calls
                       without a raster, save_envs of the E x C envs
Before anything is timed the paths are compared bit for bit: (a) the outputs with and without
leaves, and the leaves of live and record roots; (b) wherever the rollout is not padding, its
outputs against the clone path's steps, and the leaves of plans that ran all T steps without a LAST
against the clone path's saved records (a plan that ended earlier has no leaf on the clone path:
its env has moved on to another scene).  Shapes: C2 (goal finding, 5 slots) with 4096 envs, C in
{16, 64}, T in {5, 20}; C3 (clustering, 9 slots) with 1024 envs, C = 16, T = 10.  Envs are two
steps into their episodes.  Rates are plan-steps/s = T x E x C / time, padding included.  Prints
one JSON line per shape, headed by the card's name and power limit read in the same run.  Needs a
CUDA device.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from time_rollout import SHAPES, _card, _time_alternating  # noqa: E402  (tools/ is this script's path)


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
  roots = eng.save_envs()
  big = engine.Engine(E * C, wl.n_slots, 1, wl.action, wl.nodes, constants.SHAPES,
                      max_episode_length=wl.max_episode_length)
  repeat = torch.arange(E, device=eng.device).repeat_interleave(C)
  out = torch.empty(T * E * C * engine.OUT_BYTES_PER_ENV, dtype=torch.uint8, device=eng.device)
  leaves = engine.EnvStates(torch.empty((E * C, eng.record_bytes), dtype=torch.uint8, device=eng.device),
                            1, eng.signature, eng.n_slots)
  cloned = {k: torch.empty((T, E * C), dtype=d, device=eng.device) for k, d in (
      ('reward', torch.float64), ('step_type', torch.int8), ('success', torch.uint8), ('status', torch.uint8))}
  names = tuple(cloned)

  def rollout():
    return eng.rollout(plans, out=out)

  def rollout_leaves():
    return eng.rollout(plans, out=out, leaves=leaves)

  def expand():
    return eng.rollout(plans, out=out, states=roots, leaves=leaves)

  def clone(keep=False):
    big.load_envs(engine.EnvStates(roots.data[repeat], roots.span_class, roots.signature, roots.n_slots))
    for t in range(T):
      res = big.step(flat[t])
      if keep:
        for k, v in cloned.items():
          v[t].copy_(getattr(res, k))
    return big.save_envs()

  def host(res):
    return {k: getattr(res, k).reshape(T, E * C).clone() for k in names}

  def same(a, b):
    return torch.equal(a.view(torch.int64), b.view(torch.int64)) if a.dtype == torch.float64 else torch.equal(a, b)

  plain = host(rollout())
  with_leaves = host(rollout_leaves())
  live_leaves = leaves.data.clone()
  from_records = host(expand())
  for k in names:
    if not (same(plain[k], with_leaves[k]) and same(plain[k], from_records[k])):
      raise SystemExit('%s: rollouts with and without leaves or from records disagree on %s' % (key, k))
  if not torch.equal(live_leaves, leaves.data):
    raise SystemExit('%s: leaves of live and record roots disagree' % key)
  saved = clone(keep=True)
  live = from_records['step_type'] != _native.STEP_NONE
  for k, v in cloned.items():
    if not same(from_records[k][live], v[live]):
      raise SystemExit('%s: expand and clone-and-step disagree on %s' % (key, k))
  through = live.all(0) & (from_records['step_type'] == _native.STEP_MID).all(0)
  if not torch.equal(leaves.data[through], saved.data[through]):
    raise SystemExit('%s: leaves and the clone path\'s saved records disagree' % key)
  us = _time_alternating([rollout, rollout_leaves, expand, clone], seconds)
  n = T * E * C
  res = dict(workload=key, n_envs=E, n_candidates=C, n_steps=T, record_bytes=eng.record_bytes,
             leaf_mb=E * C * eng.record_bytes / 1e6, live_share=float(live.float().mean().item()),
             ran_through_share=float(through.float().mean().item()),
             rollout_us=us[0], rollout_leaves_us=us[1], expand_us=us[2], clone_us=us[3],
             rollout_plan_steps_per_s=n / us[0] * 1e6, rollout_leaves_plan_steps_per_s=n / us[1] * 1e6,
             expand_plan_steps_per_s=n / us[2] * 1e6, clone_plan_steps_per_s=n / us[3] * 1e6,
             leaves_cost=us[1] / us[0], expand_speedup_over_clone=us[3] / us[2])
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
    raise SystemExit('time_expand.py measures on a CUDA device; there is none')
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
