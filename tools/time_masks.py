"""Sprite instance masks on one GPU: the mask launch beside the render launch on the same state.

    python tools/time_masks.py [--seconds 1.0] [--out results.json]

For each workload C2..C5 of spriteworld_b200/workloads.py at its n_envs (C4 and C5: one GPU's
share), slots and frame size, after a few steps, in one process and alternating, between CUDA
events, each warmed up and repeated for at least --seconds:
  masks    Engine.render_masks at the workload's frame size and anti_aliasing, one launch
  render   Engine.render of the same state into frames (PILRenderer), one launch
A mask scans one canvas row per mask row and filters nothing; a frame scans every canvas row and
runs the LANCZOS passes.  Rates are frames (or masks) per second.  Prints one JSON line per
workload, headed by the card's name and power limit read in the same run.  Needs a CUDA device.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from time_rollout import _card, _time_alternating  # noqa: E402  (tools/ is this script's path)


def run(key, seconds):
  import torch
  from spriteworld_b200 import workloads
  wl = workloads.WORKLOADS[key]()
  E = wl.n_envs
  eng, raster, _ = workloads.build_engine(wl, E, 4)
  rng = np.random.RandomState(7)
  for a in wl.sample_actions(rng, 3, E):
    eng.step(torch.from_numpy(a).to(eng.device))
  W, H, aa = raster.width, raster.height, raster.anti_aliasing
  masks = torch.empty((E, H, W), dtype=torch.uint8, device=eng.device)
  frames = raster.new_frames()

  def render_masks():
    return eng.render_masks(W, H, aa, out=masks)

  def render():
    return eng.render(raster, frames)

  us = _time_alternating([render_masks, render], seconds)
  raster.close()
  eng.close()
  names = ('masks', 'render')
  return dict(workload=key.upper(), n_envs=E, n_slots=wl.n_slots, image_size=[W, H], anti_aliasing=aa,
              per_s={k: E / (u * 1e-6) for k, u in zip(names, us)},
              us_per_call=dict(zip(names, us)), masks_over_render=us[0] / us[1])


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--seconds', type=float, default=1.0)
  p.add_argument('--out')
  args = p.parse_args()
  rows = [_card()]
  print(json.dumps(rows[0]), flush=True)
  for key in ('c2', 'c3', 'c4', 'c5'):
    rows.append(run(key, args.seconds))
    print(json.dumps(rows[-1]), flush=True)
  if args.out:
    with open(args.out, 'w') as f:
      json.dump(rows, f, indent=1)


if __name__ == '__main__':
  main()
