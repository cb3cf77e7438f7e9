"""Frames of env records on one GPU: render_states beside the live render and the clone path.

    python tools/time_render_states.py [--seconds 1.0] [--out results.json]

C2 (goal finding, 5 slots, 64x64 at anti_aliasing 5) with n records, n = E = 4096 and n = 16 E
(leaves of expand() with C = 16).  In one process and alternating, between CUDA events, each warmed
up and repeated for at least --seconds:
  render_states   Engine.render_states of the n records, one launch
  render          Engine.render of an engine of n live envs loaded from the same records
  clone           the same question without render_states: load_envs of the n records into that
                  engine, then Engine.render
Before anything is timed the three are compared bit for bit, frames and status.  Rates are
frames/s.  Prints one JSON line per shape, headed by the card's name and power limit read in the
same run.  Needs a CUDA device.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from time_rollout import _card, _time_alternating  # noqa: E402  (tools/ is this script's path)


def run(E, C, seconds):
  import torch
  from spriteworld_b200 import constants, engine, workloads
  wl = workloads.WORKLOADS['c2']()
  eng, raster, _ = workloads.build_engine(wl, E, 4)
  rng = np.random.RandomState(7)
  for a in wl.sample_actions(rng, 3, E):
    eng.step(torch.from_numpy(a).to(eng.device))
  states = eng.save_envs()
  if C > 1:
    plans = torch.from_numpy(rng.uniform(0, 1, (5, E, C, 4)).astype(np.float32)).to(eng.device)
    states = eng.rollout(plans, states=states, leaves=True).leaves
  n = len(states)
  big = engine.Engine(n, wl.n_slots, 1, wl.action, wl.nodes, constants.SHAPES,
                      max_episode_length=wl.max_episode_length)
  big_raster = engine.Raster(big, wl.image_size[0], wl.image_size[1], wl.anti_aliasing)
  frames = torch.empty((n, big_raster.height, big_raster.width, 3), dtype=torch.uint8, device=eng.device)
  status = torch.empty(n, dtype=torch.uint8, device=eng.device)
  live = torch.empty_like(frames)

  def render_states():
    return eng.render_states(raster, states, frames, status)

  def render():
    return big.render(big_raster, live)

  def clone():
    big.load_envs(states)
    return big.render(big_raster, live)

  clone()
  want, want_status = live.clone(), big.render_status().clone()
  render_states()
  render()
  torch.cuda.synchronize()
  checked = (torch.equal(frames, want) and torch.equal(status, want_status) and torch.equal(live, want))
  if not checked:
    raise SystemExit('render_states, render and clone disagree at n = %d' % n)
  us = _time_alternating([render_states, render, clone], seconds)
  big_raster.close()
  big.close()
  raster.close()
  eng.close()
  return dict(workload='C2', n_envs=E, records=n, frames_per_s={
      k: n / (u * 1e-6) for k, u in zip(('render_states', 'render', 'clone'), us)},
      us_per_call=dict(zip(('render_states', 'render', 'clone'), us)), bit_exact=checked)


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--seconds', type=float, default=1.0)
  p.add_argument('--out')
  args = p.parse_args()
  rows = [_card()]
  print(json.dumps(rows[0]), flush=True)
  for E, C in ((4096, 1), (4096, 16)):
    rows.append(run(E, C, args.seconds))
    print(json.dumps(rows[-1]), flush=True)
  if args.out:
    with open(args.out, 'w') as f:
      json.dump(rows, f, indent=1)


if __name__ == '__main__':
  main()
