"""Views with chosen sprites drawn on one GPU: Engine.render_windows(draw=...) beside render_states of
as many full frames.

    python tools/time_layers.py [--seconds 1.0] [--out results.json]

  layers   C2's scenes (goal finding, 5 slots), 4096 envs: SpriteLayers, each slot drawn alone in a
           64x64 frame at anti_aliasing 5 (V = 5)
  removed  C5's scenes (Embodied, 8 slots), 4096 envs: every slot removed in turn, the rest of the
           scene drawn in a 64x64 frame at anti_aliasing 5 (V = 8)
Beside each, render_states of as many full frames of the same raster (n = envs x V records).  In one
process and alternating, between CUDA events, each warmed up and repeated for at least --seconds.
Rates are frames/s.  Prints one JSON line per row, headed by the card's name and power limit read in
the same run.  Needs a CUDA device.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from time_rollout import _card, _time_alternating  # noqa: E402  (tools/ is this script's path)


def run(name, wl_name, E, size, aa, seconds):
  import torch
  from spriteworld_b200 import engine, renderers, workloads
  wl = workloads.WORKLOADS[wl_name]()
  eng, _, _ = workloads.build_engine(wl, E, 4)
  rng = np.random.RandomState(7)
  for a in wl.sample_actions(rng, 3, E):
    eng.step(torch.from_numpy(a).to(eng.device))
  raster = engine.Raster(eng, size, size, aa)
  pos = eng.state_tensors()
  windows, draw = renderers.SpriteLayers(image_size=(size, size), anti_aliasing=aa).views(pos['pos_x'], pos['pos_y'])
  if name == 'removed':
    draw = ~draw
  V = windows.shape[1]
  states = eng.save_envs()
  full = states.take(torch.arange(E * V, device=eng.device) % E)
  frames = torch.empty((E, V, size, size, 3), dtype=torch.uint8, device=eng.device)
  status = torch.empty((E, V), dtype=torch.uint8, device=eng.device)
  full_frames = torch.empty((E * V, size, size, 3), dtype=torch.uint8, device=eng.device)
  full_status = torch.empty(E * V, dtype=torch.uint8, device=eng.device)

  def views():
    return eng.render_windows(raster, windows, None, frames, status, draw)

  def render_states():
    return eng.render_states(raster, full, full_frames, full_status)

  views()
  render_states()
  torch.cuda.synchronize()
  flagged = int((status != 0).sum().item())
  us = _time_alternating([views, render_states], seconds)
  n = E * V
  return dict(row=name, workload=wl_name, envs=E, views=V, image=size, anti_aliasing=aa, frames=n,
              frames_per_s=dict(render_views=n / (us[0] * 1e-6), render_states=n / (us[1] * 1e-6)),
              us_per_call=dict(render_views=us[0], render_states=us[1]), flagged_views=flagged)


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--seconds', type=float, default=1.0)
  p.add_argument('--out', default=None)
  args = p.parse_args()
  rows = [_card()]
  print(json.dumps(rows[0]), flush=True)
  for spec in (('layers', 'c2', 4096, 64, 5), ('removed', 'c5', 4096, 64, 5)):
    rows.append(run(*spec, seconds=args.seconds))
    print(json.dumps(rows[-1]), flush=True)
  if args.out:
    with open(args.out, 'w') as f:
      json.dump(rows, f, indent=1)


if __name__ == '__main__':
  main()
