"""Render kernel time and env-steps/s at anti_aliasing 5, 10 and 13 on one GPU.

    python tools/time_render_aa.py [--seconds 1.0] [--out results.json]

Workloads (defined here; bench.py's are all anti_aliasing 5):
  c2_aa5 / c2_aa10 / c2_aa13   C2's goal-finding scenes, 4096 envs x 5 slots, 64x64
  c3_aa10                      C3's clustering scenes, 16384 envs x 9 slots, 64x64
  demo_256_aa10                the demo's renderer: 256x256 at anti_aliasing 10, hsv_to_rgb, on
                               scenes of the cobra clustering config, 1024 envs

Per workload: Engine.render alone between CUDA events (the render kernel) and Engine.step with
the render (step kernel + render kernel) between CUDA events, each warmed up and repeated for
at least --seconds.  Prints one JSON line per workload, headed by the card's name and power
limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
  import torch
  name = torch.cuda.get_device_name(0)
  try:
    q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader',
                        '-i', '0'], capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError) as ex:
    q = 'unavailable (%s)' % ex
  return dict(card=name, power_limit_and_max_sm_clock=q)


def _workload_engine(key, aa, n_envs):
  from spriteworld_b200 import workloads
  base = workloads.WORKLOADS[key]
  wl = type(base.__name__ + '_aa%d' % aa, (base,), dict(anti_aliasing=aa))()
  eng, raster, _ = workloads.build_engine(wl, n_envs, 4)
  return eng, raster, wl.sample_actions(np.random.RandomState(7), 16, n_envs)


def _demo_engine(n_envs):
  from spriteworld_b200 import constants, engine, scene, sprite_generators
  from spriteworld_b200.configs.cobra import clustering
  from spriteworld_b200.renderers import color_maps
  cfg = clustering.get_config('train')
  nodes, filters = cfg['task'].compile()
  K, S = 4, 4
  eng = engine.Engine(n_envs, S, K, cfg['action_space'].compile(), nodes, constants.SHAPES,
                      keep_in_frame=True, max_episode_length=cfg['max_episode_length'])
  lay = sprite_generators.batch_of(cfg['init_sprites'], n_envs * K, np.random.RandomState(3))
  eng.upload_scenes(scene.arrays_from_layout(lay, S, filters, color_maps.hsv_to_rgb),
                    np.repeat(np.arange(n_envs), K), np.tile(np.arange(K), n_envs))
  raster = engine.Raster(eng, 256, 256, 10)
  actions = np.random.RandomState(7).uniform(0, 1, (16, n_envs, 4)).astype(np.float32)
  return eng, raster, actions


def _timed(fn, seconds):
  """ms per call between CUDA events, over at least `seconds` of calls after a warm-up."""
  import torch
  for _ in range(3):
    fn(0)
  torch.cuda.synchronize()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  fn(0)
  b.record()
  b.synchronize()
  n = max(10, int(seconds * 1e3 / max(a.elapsed_time(b), 1e-3)))
  a.record()
  for i in range(n):
    fn(i)
  b.record()
  b.synchronize()
  return a.elapsed_time(b) / n, n


def measure(name, eng, raster, actions, seconds):
  import torch
  E = eng.n_envs
  frames = raster.new_frames()
  dev_actions = torch.from_numpy(actions).to(eng.device)
  eng.step(dev_actions[0])                       # every env past its first reset
  render_ms, n_render = _timed(lambda i: eng.render(raster, frames), seconds)
  step_ms, n_step = _timed(lambda i: eng.step(dev_actions[i % len(dev_actions)], raster, frames),
                           seconds)
  eng.check_render()                             # no env overflowed its span tables
  return dict(workload=name, n_envs=E, n_slots=eng.n_slots, image=[raster.height, raster.width],
              anti_aliasing=raster.anti_aliasing, render_ms=round(render_ms, 4),
              render_frames_per_s=round(E / render_ms * 1e3),
              step_render_ms=round(step_ms, 4), env_steps_per_s=round(E / step_ms * 1e3),
              calls=[n_render, n_step])


def main():
  ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
  ap.add_argument('--seconds', type=float, default=1.0, help='least timed time per measurement')
  ap.add_argument('--only', default=None, help='comma-separated workload names')
  ap.add_argument('--out', default=None, help='also write the JSON lines to this file')
  args = ap.parse_args()
  import torch
  if not torch.cuda.is_available():
    sys.exit('time_render_aa.py measures on a GPU; none is visible')
  plan = [('c2_aa5', lambda: _workload_engine('c2', 5, 4096)),
          ('c2_aa10', lambda: _workload_engine('c2', 10, 4096)),
          ('c2_aa13', lambda: _workload_engine('c2', 13, 4096)),
          ('c3_aa10', lambda: _workload_engine('c3', 10, 16384)),
          ('demo_256_aa10', lambda: _demo_engine(1024))]
  if args.only:
    keep = set(args.only.split(','))
    plan = [p for p in plan if p[0] in keep]
  lines = [dict(_card())]
  print(json.dumps(lines[0]), flush=True)
  for name, make in plan:
    eng, raster, actions = make()
    lines.append(measure(name, eng, raster, actions, args.seconds))
    print(json.dumps(lines[-1]), flush=True)
    raster.close()
    eng.close()
  if args.out:
    with open(args.out, 'w') as f:
      for line in lines:
        f.write(json.dumps(line) + '\n')


if __name__ == '__main__':
  main()
