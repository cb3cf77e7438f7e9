"""Amodal sprite coverage on one GPU: the coverage launch beside the mask launch on the same state.

    python tools/time_coverage.py [--seconds 1.0] [--out results.json]

For workloads C2 and C3 of spriteworld_b200/workloads.py at their n_envs and slots, after a few
steps, at 64 x 64 with anti_aliasing 1 and 5, in one process and alternating, between CUDA events,
each warmed up and repeated for at least --seconds:
  masks     Engine.render_masks, one launch (uint8 (n, 64, 64))
  coverage  Engine.render_coverage, two memsets of the counts and one launch (int32 (n, 64, 64) and
            the per-slot visible and area counts)
Both scan the same canvas rows; the coverage stages and writes four bytes a pixel instead of one
and counts every slot in the kernel.  Rates are envs per second.  Prints one JSON line per row,
headed by the card's name and power limit read in the same run.  Needs a CUDA device.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from time_rollout import _card, _time_alternating  # noqa: E402  (tools/ is this script's path)


def run(key, seconds, W=64, H=64, aa_values=(1, 5)):
  import torch
  from spriteworld_b200 import workloads
  wl = workloads.WORKLOADS[key]()
  E, S = wl.n_envs, wl.n_slots
  eng, raster, _ = workloads.build_engine(wl, E, 4)
  rng = np.random.RandomState(7)
  for a in wl.sample_actions(rng, 3, E):
    eng.step(torch.from_numpy(a).to(eng.device))
  masks = torch.empty((E, H, W), dtype=torch.uint8, device=eng.device)
  cover = (torch.empty((E, H, W), dtype=torch.int32, device=eng.device),
           torch.empty((E, S), dtype=torch.int32, device=eng.device),
           torch.empty((E, S), dtype=torch.int32, device=eng.device))
  rows = []
  for aa in aa_values:
    def render_masks():
      return eng.render_masks(W, H, aa, out=masks)

    def render_coverage():
      return eng.render_coverage(W, H, aa, out=cover)

    us = _time_alternating([render_masks, render_coverage], seconds)
    names = ('masks', 'coverage')
    rows.append(dict(workload=key.upper(), n_envs=E, n_slots=S, image_size=[W, H], anti_aliasing=aa,
                     per_s={k: E / (u * 1e-6) for k, u in zip(names, us)},
                     us_per_call=dict(zip(names, us)), coverage_over_masks=us[1] / us[0]))
  raster.close()
  eng.close()
  return rows


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--seconds', type=float, default=1.0)
  p.add_argument('--out')
  args = p.parse_args()
  rows = [_card()]
  print(json.dumps(rows[0]), flush=True)
  for key in ('c2', 'c3'):
    for row in run(key, args.seconds):
      rows.append(row)
      print(json.dumps(row), flush=True)
  if args.out:
    with open(args.out, 'w') as f:
      json.dump(rows, f, indent=1)


if __name__ == '__main__':
  main()
