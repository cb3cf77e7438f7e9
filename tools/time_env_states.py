"""Cost of env records on one GPU: copy_envs, save_envs and load_envs of every env, beside a step.

    python tools/time_env_states.py [--seconds 1.0] [--out results.json]

Workloads: C2 (goal finding, 4096 envs x 5 slots) and C3 (clustering, 16384 envs x 9 slots),
64x64 at anti_aliasing 5, pool depth 4, as bench.py builds them.

Per workload, each between CUDA events, warmed up and repeated for at least --seconds:
  step          Engine.step with the render (step kernel + render kernel)
  copy_shift    copy_envs(all, all shifted by one): the id sets overlap, so two kernels through
                engine scratch
  copy_half     copy_envs(first half, second half): disjoint sets, one kernel
  save_load     save_envs() then load_envs() of all envs
  *_dev         the same three calls with check='device': int64 id tensors on the device,
                checked there (a copy always goes through engine scratch: three kernels)
The calls include their host work (id checks, pinned staging), as a user pays it; the events
measure the stream, so a call that the host cannot enqueue as fast as the device runs it shows
its host time.  GB/s counts the record bytes read and written on the device: 2 x records for a
direct copy, 4 x for a copy through scratch and for a save plus a load.

Then a branching loop, timed on the host clock and ending in a synchronise: per step one
Engine.step with the render and a torch.multinomial resample of all envs (weights drawn on the
device), copied into place with copy_envs.  `resample_host` passes the draw as host-checked ids,
which copies it to the host and so waits for the step; `resample_dev` passes it with
check='device'.  Both in env-steps/s.  Prints one JSON line per workload, headed by the card's
name and power limit read in the same run.
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


def _time(fn, seconds):
  """Mean microseconds per call of fn() between CUDA events, over at least `seconds`."""
  import torch
  for _ in range(5):
    fn()
  torch.cuda.synchronize()
  n, total = 10, 0.0
  while True:
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
      fn()
    b.record()
    b.synchronize()
    ms = a.elapsed_time(b)
    if ms >= 1e3 * seconds:
      return 1e3 * ms / n
    total = ms
    n = max(2 * n, int(n * 1e3 * seconds / max(total, 1e-3)) + 1)


def run(key, seconds):
  import torch
  from spriteworld_b200 import workloads
  wl = workloads.WORKLOADS[key]()
  E = wl.n_envs
  eng, raster, _ = workloads.build_engine(wl, E, 4)
  acts = [torch.from_numpy(a).to(eng.device) for a in wl.sample_actions(np.random.RandomState(7), 16, E)]
  frames = raster.new_frames()
  it = iter(range(1 << 62))

  def step():
    eng.step(acts[next(it) % len(acts)], raster, frames)

  step_us = _time(step, seconds)
  ids = np.arange(E, dtype=np.int32)
  shifted = np.roll(ids, 1)
  half = E // 2
  rb = eng.record_bytes
  out = dict(workload=key, n_envs=E, n_slots=wl.n_slots, record_bytes=rb, step_us=step_us)

  def save_load():
    eng.load_envs(eng.save_envs(ids), ids)

  for name, fn, moved in (('copy_shift', lambda: eng.copy_envs(ids, shifted), 4 * E * rb),
                          ('copy_half', lambda: eng.copy_envs(ids[:half], ids[half:2 * half]), 2 * half * rb),
                          ('save_load', save_load, 4 * E * rb)):
    us = _time(fn, seconds)
    out[name + '_us'] = us
    out[name + '_GBps'] = moved / us / 1e3
    out[name + '_share_of_step'] = us / step_us
  dev = torch.arange(E, device=eng.device)
  dev_shifted, dev_lo, dev_hi = torch.roll(dev, 1), dev[:half].clone(), dev[half:2 * half].clone()

  def save_load_dev():
    eng.load_envs(eng.save_envs(dev, check='device'), dev, check='device')

  for name, fn, moved in (('copy_shift_dev', lambda: eng.copy_envs(dev, dev_shifted, check='device'), 4 * E * rb),
                          ('copy_half_dev', lambda: eng.copy_envs(dev_lo, dev_hi, check='device'), 4 * half * rb),
                          ('save_load_dev', save_load_dev, 4 * E * rb)):
    us = _time(fn, seconds)
    out[name + '_us'] = us
    out[name + '_GBps'] = moved / us / 1e3
    out[name + '_share_of_step'] = us / step_us
  eng.check_env_ids()
  gen = torch.Generator(device=eng.device)
  gen.manual_seed(0)

  def resample(check):
    eng.step(acts[next(it) % len(acts)], raster, frames)
    src = torch.multinomial(torch.rand(E, device=eng.device, generator=gen), E, replacement=True, generator=gen)
    if check == 'device':
      eng.copy_envs(src, dev, check='device')
    else:
      eng.copy_envs(src, np.arange(E))

  for check in ('host', 'device'):
    out['resample_%s_env_steps_per_s' % check] = E / _loop_seconds(lambda: resample(check), seconds)
  eng.check_env_ids()
  return out


def _loop_seconds(fn, seconds):
  """Seconds per call of fn(), host clock around calls that end in a synchronise."""
  import time
  import torch
  for _ in range(5):
    fn()
  torch.cuda.synchronize()
  n = 10
  while True:
    t0 = time.perf_counter()
    for _ in range(n):
      fn()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    if dt >= seconds:
      return dt / n
    n = max(2 * n, int(n * seconds / max(dt, 1e-6)) + 1)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--seconds', type=float, default=1.0)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  import torch
  if not torch.cuda.is_available():
    raise SystemExit('time_env_states.py measures on a CUDA device; there is none')
  from spriteworld_b200 import build
  build.build()
  lines = [dict(_card())]
  print(json.dumps(lines[0]), flush=True)
  for key in ('c2', 'c3'):
    lines.append(run(key, args.seconds))
    print(json.dumps(lines[-1]), flush=True)
  if args.out:
    with open(args.out, 'w') as f:
      json.dump(lines, f, indent=1)


if __name__ == '__main__':
  main()
