"""Soft sprite masks on one GPU: the soft-mask launch beside the mask launch on the same state.

    python tools/time_soft_masks.py [--seconds 1.0] [--out results.json]

For workloads C2 to C5 of spriteworld_b200/workloads.py at their per-GPU n_envs, slots and image
size with anti_aliasing 5, and for C2 at 64 x 64 with anti_aliasing 10, after a few steps, in one
process and alternating, between CUDA events, each warmed up and repeated for at least --seconds:
  masks  Engine.render_masks, one launch (uint8 (n, H, W)): one canvas row per mask row
  soft   Engine.render_soft_masks, one launch (uint8 (n, S, H, W)): all aa canvas rows per mask
         row, and S bytes out per pixel
The write rate is the soft masks' n * S * H * W bytes over the soft launch's time.  Prints one JSON
line per row, headed by the card's name and power limit read in the same run.  Needs a CUDA device.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from time_rollout import _card, _time_alternating  # noqa: E402  (tools/ is this script's path)

ROWS = (('c2', 5), ('c3', 5), ('c4', 5), ('c5', 5), ('c2', 10))


def run(key, aa, seconds):
  import torch
  from spriteworld_b200 import workloads
  wl = workloads.WORKLOADS[key]()
  E, S = wl.n_envs, wl.n_slots
  W, H = wl.image_size
  eng, raster, _ = workloads.build_engine(wl, E, 4)
  rng = np.random.RandomState(7)
  for a in wl.sample_actions(rng, 3, E):
    eng.step(torch.from_numpy(a).to(eng.device))
  masks = torch.empty((E, H, W), dtype=torch.uint8, device=eng.device)
  soft = torch.empty((E, S, H, W), dtype=torch.uint8, device=eng.device)

  def render_masks():
    return eng.render_masks(W, H, aa, out=masks)

  def render_soft():
    return eng.render_soft_masks(W, H, aa, out=soft)

  us = _time_alternating([render_masks, render_soft], seconds)
  # the soft masks' samples are the mask's at aa // 2: where the mask names slot k, slot k owns one
  torch.cuda.synchronize()
  m = masks.long()
  owned = soft.gather(1, (m - 1).clamp(min=0).unsqueeze(1)).squeeze(1)
  assert bool((owned[m > 0] >= 1).all()) and int(soft.sum(1, dtype=torch.int32).max()) <= aa * aa
  nbytes = E * S * H * W
  row = dict(workload=key.upper(), n_envs=E, n_slots=S, image_size=[W, H], anti_aliasing=aa,
             us_per_call=dict(masks=us[0], soft=us[1]), soft_over_masks=us[1] / us[0],
             soft_bytes=nbytes, soft_write_GB_per_s=nbytes / (us[1] * 1e-6) / 1e9)
  del masks, soft
  raster.close()
  eng.close()
  return row


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--seconds', type=float, default=1.0)
  p.add_argument('--out')
  args = p.parse_args()
  rows = [_card()]
  print(json.dumps(rows[0]), flush=True)
  for key, aa in ROWS:
    rows.append(run(key, aa, args.seconds))
    print(json.dumps(rows[-1]), flush=True)
  if args.out:
    with open(args.out, 'w') as f:
      json.dump(rows, f, indent=1)


if __name__ == '__main__':
  main()
