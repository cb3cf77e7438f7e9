"""Rollout trajectories on one GPU: every step's state as env records, beside the paths without them.

    python tools/time_trajectory.py [--seconds 1.0] [--out results.json]

Per shape, in one process and alternating, between CUDA events, each warmed up and repeated for at
least --seconds:
  rollout      Engine.rollout of (T, E, C) plans from E saved records, no records written
  trajectory   the same with trajectory=: the T x E x C states after every step, one launch
  expand_loop  the same trajectory from T expand levels: the first from the E roots with C plans,
               then T - 1 levels of one step and one plan from the previous level's leaves, each
               level's leaves written into its slice of the trajectory buffer (T launches)
Before anything is timed the three are compared bit for bit: the outputs of all three, and the
trajectory against the expand loop's records.  Shapes: C2 (goal finding, 5 slots) and C3
(clustering, 9 slots), E = 1024 roots two steps into their episodes, C = 32, T = 16.  Reports the
bytes each call writes (outputs, and records for the two trajectory paths) and the write bandwidth
they make at the measured time.  Prints one JSON line per shape, headed by the card's name and power
limit read in the same run.  Needs a CUDA device.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from time_rollout import _card, _time_alternating  # noqa: E402  (tools/ is this script's path)

SHAPES = [('c2', 1024, 32, 16), ('c3', 1024, 32, 16)]


def run(key, E, C, T, seconds):
  import torch
  from spriteworld_b200 import engine, workloads
  wl = workloads.WORKLOADS[key]()
  eng, _, _ = workloads.build_engine(wl, E, 4)
  rng = np.random.RandomState(7)
  for a in wl.sample_actions(rng, 2, E):
    eng.step(torch.from_numpy(a).to(eng.device))
  plans = torch.from_numpy(rng.uniform(0, 1, (T, E, C, 4)).astype(np.float32)).to(eng.device)
  step_plans = [plans[t].reshape(1, E * C, 1, 4) for t in range(T)]
  roots = eng.save_envs()
  rb, EC = eng.record_bytes, E * C
  out_bytes = T * EC * engine.OUT_BYTES_PER_ENV
  out = torch.empty(out_bytes, dtype=torch.uint8, device=eng.device)
  level_out = [torch.empty(EC * engine.OUT_BYTES_PER_ENV, dtype=torch.uint8, device=eng.device) for _ in range(T)]

  def states(data):
    return engine.EnvStates(data, roots.span_class, roots.signature, roots.n_slots, roots.n_goals)

  traj = states(torch.empty((T * EC, rb), dtype=torch.uint8, device=eng.device))
  loop = states(torch.empty((T * EC, rb), dtype=torch.uint8, device=eng.device))
  slices = [loop[t * EC:(t + 1) * EC] for t in range(T)]

  def rollout():
    return eng.rollout(plans, out=out, states=roots)

  def trajectory():
    return eng.rollout(plans, out=out, states=roots, trajectory=traj)

  def expand_loop():
    res = [eng.rollout(plans[:1], out=level_out[0], states=roots, leaves=slices[0])]
    for t in range(1, T):
      res.append(eng.rollout(step_plans[t], out=level_out[t], states=slices[t - 1], leaves=slices[t]))
    return res

  names = ('reward', 'step_type', 'success', 'status')

  def host(res):
    return {k: getattr(res, k).reshape(T, EC).clone() for k in names}

  def same(a, b):
    return torch.equal(a.view(torch.int64), b.view(torch.int64)) if a.dtype == torch.float64 else torch.equal(a, b)

  plain = host(rollout())
  traced = host(trajectory())
  levels = expand_loop()
  looped = {k: torch.cat([getattr(r, k).reshape(1, EC) for r in levels]) for k in names}
  for k in names:
    if not (same(plain[k], traced[k]) and same(plain[k], looped[k])):
      raise SystemExit('%s: rollout, trajectory and the expand loop disagree on %s' % (key, k))
  if not torch.equal(traj.data, loop.data):
    raise SystemExit('%s: the trajectory and the expand loop\'s records disagree' % key)
  live = plain['step_type'] >= 0
  us = _time_alternating([rollout, trajectory, expand_loop], seconds)
  rec_bytes = T * EC * rb
  written = (out_bytes, out_bytes + rec_bytes, out_bytes + rec_bytes)
  res = dict(workload=key, n_roots=E, n_candidates=C, n_steps=T, record_bytes=rb,
             live_share=float(live.float().mean().item()),
             rollout_us=us[0], trajectory_us=us[1], expand_loop_us=us[2],
             rollout_bytes=written[0], trajectory_bytes=written[1], expand_loop_bytes=written[2],
             rollout_write_gb_per_s=written[0] / us[0] / 1e3, trajectory_write_gb_per_s=written[1] / us[1] / 1e3,
             expand_loop_write_gb_per_s=written[2] / us[2] / 1e3,
             trajectory_cost_over_rollout=us[1] / us[0], expand_loop_over_trajectory=us[2] / us[1])
  eng.close()
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--seconds', type=float, default=1.0)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  import torch
  if not torch.cuda.is_available():
    raise SystemExit('time_trajectory.py measures on a CUDA device; there is none')
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
