"""Sprite bounding boxes on one GPU: the boxes call beside the coverage call of the same state and
beside the torch derivation a user would otherwise write.

    python tools/time_boxes.py [--seconds 1.0] [--out results.json]

For workloads C2 to C5 of spriteworld_b200/workloads.py at their per-GPU n_envs, slots and image
size, after a few steps, with anti_aliasing 1 and 5, in one process and alternating, between CUDA
events, each warmed up and repeated for at least --seconds:
  boxes     Engine.render_boxes: four memsets, the mask kernel's box mode and the decoding kernel
            (int32 (n, S, 4) twice and the per-slot visible and area counts)
  coverage  Engine.render_coverage: two memsets of the counts and one launch (int32 (n, H, W) and
            the counts)
  torch     what the same boxes cost without the box mode: Engine.render_masks and
            Engine.render_coverage, then the visible boxes by four scatter_reduce passes over the
            mask, and the amodal boxes from each slot's bit plane of the coverage
Before timing, the torch path's boxes and the coverage's counts are checked equal to the boxes
call's.  Prints one JSON line per row, headed by the card's name and power limit read in the same
run.  Needs a CUDA device.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from time_rollout import _card, _time_alternating  # noqa: E402  (tools/ is this script's path)


def _extent(plane, axis_len):
  """(first, last + 1) of the True entries of (n, axis_len) `plane` per row, (0, 0) where none."""
  import torch
  any_ = plane.any(1)
  first = plane.to(torch.uint8).argmax(1)
  end = axis_len - plane.flip(1).to(torch.uint8).argmax(1)
  return torch.where(any_, first, 0), torch.where(any_, end, 0)


def torch_boxes(masks, cover, n_slots):
  """(visible_box, amodal_box) int32 (n, n_slots, 4) of a mask (n, H, W) uint8 and its coverage
  (n, H, W) int32, in torch."""
  import torch
  n, H, W = masks.shape
  dev = masks.device
  idx = masks.view(n, -1).long()
  xs = torch.arange(W, device=dev).repeat(H).expand(n, -1)
  ys = torch.arange(H, device=dev).repeat_interleave(W).expand(n, -1)

  def reduce(src, init, how):
    t = torch.full((n, n_slots + 1), init, dtype=torch.int64, device=dev)
    return t.scatter_reduce(1, idx, src, how)[:, 1:]
  x0, y0 = reduce(xs, W, 'amin'), reduce(ys, H, 'amin')
  x1, y1 = reduce(xs, -1, 'amax') + 1, reduce(ys, -1, 'amax') + 1
  visible_box = torch.stack([x0, y0, x1, y1], 2)
  visible_box[x1 == 0] = 0
  amodal = []
  for k in range(n_slots):
    plane = ((cover >> k) & 1).bool()
    ax0, ax1 = _extent(plane.any(1), W)
    ay0, ay1 = _extent(plane.any(2), H)
    amodal.append(torch.stack([ax0, ay0, ax1, ay1], 1))
  return visible_box.int(), torch.stack(amodal, 1).int()


def run(key, seconds, aa_values=(1, 5)):
  import torch
  from spriteworld_b200 import workloads
  wl = workloads.WORKLOADS[key]()
  E, S = wl.n_envs, wl.n_slots
  W, H = wl.image_size
  eng, raster, _ = workloads.build_engine(wl, E, 4)
  rng = np.random.RandomState(7)
  for a in wl.sample_actions(rng, 3, E):
    eng.step(torch.from_numpy(a).to(eng.device))
  i32 = dict(dtype=torch.int32, device=eng.device)
  boxes = (torch.empty((E, S, 4), **i32), torch.empty((E, S, 4), **i32), torch.empty((E, S), **i32),
           torch.empty((E, S), **i32))
  cover = (torch.empty((E, H, W), **i32), torch.empty((E, S), **i32), torch.empty((E, S), **i32))
  masks = torch.empty((E, H, W), dtype=torch.uint8, device=eng.device)
  rows = []
  for aa in aa_values:
    def render_boxes():
      return eng.render_boxes(W, H, aa, out=boxes)

    def render_coverage():
      return eng.render_coverage(W, H, aa, out=cover)

    def derive_in_torch():
      eng.render_masks(W, H, aa, out=masks)
      eng.render_coverage(W, H, aa, out=cover)
      return torch_boxes(masks, cover[0], S)

    got = render_boxes()
    vb, ab = derive_in_torch()
    assert torch.equal(vb, got[0]) and torch.equal(ab, got[1]), (key, aa)
    assert torch.equal(cover[1], got[2]) and torch.equal(cover[2], got[3]), (key, aa)
    us = _time_alternating([render_boxes, render_coverage, derive_in_torch], seconds)
    names = ('boxes', 'coverage', 'torch')
    rows.append(dict(workload=key.upper(), n_envs=E, n_slots=S, image_size=[W, H], anti_aliasing=aa,
                     us_per_call=dict(zip(names, us)), boxes_over_coverage=us[0] / us[1],
                     torch_over_boxes=us[2] / us[0]))
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
  for key in ('c2', 'c3', 'c4', 'c5'):
    for row in run(key, args.seconds):
      rows.append(row)
      print(json.dumps(row), flush=True)
  if args.out:
    with open(args.out, 'w') as f:
      json.dump(rows, f, indent=1)


if __name__ == '__main__':
  main()
