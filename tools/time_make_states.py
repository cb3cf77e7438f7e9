"""Env records from factor tensors (Engine.make_states) on one GPU: time per call and bandwidth.

    python tools/time_make_states.py [--seconds 1.0] [--out results.json]

For 2^20 records at S = 5 and 9 slots and G = 0 and 1 sampled goals, the call with a given span
class (one launch, no host synchronisation) is timed between CUDA events, warmed up and repeated for
at least --seconds.  The columns are every factor: x, y, scale, c0, c1, c2, x_vel, y_vel float32,
shape uint8 and angle int16, under hsv_to_rgb with one task filter; step_count and, for G = 1, the
goals are given.  Reports the bytes read (columns, goals, step counts) and written (records,
status), and the bandwidth that makes against the H100 SXM data sheet's 3.35 TB/s.

One end-to-end row: n = 2^14 scenes sampled in torch on the device (positions, shapes, angles,
scales and colours), make_states, then the frames of the C2 raster (64 x 64, anti_aliasing 5) of
the records (Engine.render_states), in frames per second.  Prints one JSON line per row, headed by
the card's name and power limit read in the same run.  Needs a CUDA device.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from time_rollout import _card, _time_alternating  # noqa: E402  (tools/ is this script's path)

HBM_TB_PER_S = 3.35   # H100 SXM data sheet


def _engine(S, G):
  from spriteworld_b200 import constants, engine, scene_program, workloads
  from spriteworld_b200 import factor_distributions as distribs
  from spriteworld_b200.renderers import color_maps
  wl = workloads.WORKLOADS['c2']()
  nodes = [dict(wl.nodes[0], goal_slot=0)] if G else wl.nodes
  eng = engine.Engine(16, S, 2, wl.action, nodes, constants.SHAPES)
  eng.load_packer(scene_program.compile_packer([distribs.Continuous('c0', 0.0, 0.25)], color_maps.hsv_to_rgb))
  return eng, wl


def _factors(torch, n, S, device, gen):
  def u(lo, hi):
    return torch.rand((n, S), generator=gen, device=device) * (hi - lo) + lo
  return {'x': u(0.1, 0.9), 'y': u(0.1, 0.9), 'scale': u(0.05, 0.2), 'c0': u(0, 1), 'c1': u(0.3, 1), 'c2': u(0.3, 1),
          'x_vel': u(-0.01, 0.01), 'y_vel': u(-0.01, 0.01),
          'shape': torch.randint(1, 7, (n, S), generator=gen, device=device, dtype=torch.uint8),
          'angle': torch.randint(-180, 181, (n, S), generator=gen, device=device, dtype=torch.int16)}


def run(S, G, n, seconds):
  import torch
  eng, _ = _engine(S, G)
  gen = torch.Generator(device=eng.device)
  gen.manual_seed(S * 10 + G)
  factors = _factors(torch, n, S, eng.device, gen)
  goals = torch.rand((n, G, 2), dtype=torch.float64, device=eng.device) if G else None
  step = torch.zeros(n, dtype=torch.int32, device=eng.device)
  out, status = eng.make_states(factors, goals, step, span_class=1)
  torch.cuda.synchronize()
  if status.any():
    raise SystemExit('S=%d G=%d: records refused' % (S, G))

  def call():
    eng.make_states(factors, goals, step, span_class=1, out=out)

  us = _time_alternating([call], seconds)[0]
  rb = eng.record_bytes
  read = sum(t.numel() * t.element_size() for t in factors.values()) + n * (4 + 16 * G)
  written = n * (rb + 1)
  eng.close()
  return dict(slots=S, goals=G, records=n, record_bytes=rb, make_states_us=us,
              bytes_read=read, bytes_written=written, gb_per_s=(read + written) / us / 1e3,
              share_of_hbm=(read + written) / us / 1e6 / HBM_TB_PER_S)


def end_to_end(n, seconds):
  import torch
  from spriteworld_b200 import engine
  eng, wl = _engine(5, 0)
  raster = engine.Raster(eng, wl.image_size[0], wl.image_size[1], wl.anti_aliasing)
  gen = torch.Generator(device=eng.device)
  gen.manual_seed(1)
  frames = torch.empty((n, raster.height, raster.width, 3), dtype=torch.uint8, device=eng.device)
  status = torch.empty(n, dtype=torch.uint8, device=eng.device)

  def once():
    states, _ = eng.make_states(_factors(torch, n, 5, eng.device, gen), span_class=1)
    eng.render_states(raster, states, frames, status)

  us = _time_alternating([once], seconds)[0]
  raster.close()
  eng.close()
  return dict(end_to_end='torch factor sampling + make_states + C2 render_states', records=n,
              us_per_batch=us, frames_per_s=n / us * 1e6)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--seconds', type=float, default=1.0)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  import torch
  if not torch.cuda.is_available():
    raise SystemExit('time_make_states.py measures on a CUDA device; there is none')
  lines = [_card()]
  print(json.dumps(lines[0]), flush=True)
  for S in (5, 9):
    for G in (0, 1):
      lines.append(run(S, G, 1 << 20, args.seconds))
      print(json.dumps(lines[-1]), flush=True)
  lines.append(end_to_end(1 << 14, args.seconds))
  print(json.dumps(lines[-1]), flush=True)
  if args.out:
    with open(args.out, 'w') as f:
      json.dump(lines, f, indent=1)


if __name__ == '__main__':
  main()
