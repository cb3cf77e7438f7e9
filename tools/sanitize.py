"""Workload run for compute-sanitizer (memcheck / racecheck / initcheck / synccheck).

  compute-sanitizer --tool racecheck python tools/sanitize.py

Small batches of the BASELINE workloads (C2 5 sprites, C3 9 sprites, C5 128x128 with two
bands per frame and the Embodied action space) stepped past an auto-reset through the three
launch paths: swb_step_render (device buffers), swb_step_host (host buffers, chunked
renders) and swb_step_render_gather with two targets (render_kernel<true>, the variant that
also stores every frame into a second buffer: here a second buffer of the same device stands in
for a peer's).  The render kernel aliases its scratch area between phases and hands the staged
frame to the bulk-copy engine while the next frame's set-up runs: what racecheck is for.

The last run renders 70-row frames (bands of 64 and 6 rows) for three times as many (env, band)
items as there are resident render CTAs, so every CTA claims several items of unequal bands,
some written out by the bulk copy and some by the per-byte loop, one after the other.

Between those, device-checked env records: saves, loads and copies with int32 and int64 device
ids, valid and refused (out of range either way, 2^32 + 1, repeated destinations), so that memcheck
sees that a refused id never indexes engine memory.
"""
import ctypes
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
  import torch
  from spriteworld_b200 import _native, workloads
  E = int(os.environ.get('SWB_SAN_ENVS', '24'))
  for key in ('c2', 'c3', 'c5'):
    wl = workloads.WORKLOADS[key]()
    T = 6
    eng, raster, _ = workloads.build_engine(wl, E, 4, device=0, seed=3, max_episode_length=3)
    acts = wl.sample_actions(np.random.RandomState(1), T, E)
    frames = raster.new_frames()
    for t in range(T):
      eng.step(torch.from_numpy(acts[t]).cuda(), raster, frames)
    for t in range(2):
      eng.step_host(acts[t], raster)
    # two targets on one device: the peer-store variant of the kernel
    H, W = wl.image_size[1], wl.image_size[0]
    bufs = [torch.zeros((2 * E, H, W, 3), dtype=torch.uint8, device='cuda') for _ in range(2)]
    ptrs = (ctypes.c_void_p * 2)(bufs[0].data_ptr(), bufs[1].data_ptr())
    for t in range(3):
      eng.step_gather(torch.from_numpy(acts[t]).cuda(), raster, (ptrs, 2, 0, bufs[0]))
    torch.cuda.synchronize()
    assert torch.equal(bufs[0][:E], bufs[1][:E]) and bufs[0][:E].any()
    print('%s: %d envs, %d kernel launches' % (wl.name, E, eng.launch_count()), flush=True)
    raster.close()
    eng.close()
  device_checked_records(torch)
  persistent_mixed(torch)


def device_checked_records(torch):
  from spriteworld_b200 import workloads
  wl = workloads.WORKLOADS['c2']()
  E = 40
  eng, raster, _ = workloads.build_engine(wl, E, 4, device=0, seed=4, max_episode_length=3)
  eng.step(torch.from_numpy(wl.sample_actions(np.random.RandomState(2), 1, E)[0]).cuda(), raster)
  ids = torch.arange(E, device='cuda')
  refused = 0
  for dt in (torch.int32, torch.int64):
    good = ids.flip(0).to(dt)
    s = eng.save_envs(good, check='device')
    eng.load_envs(s, ids.to(dt), check='device')
    eng.copy_envs(good, torch.roll(ids, 3).to(dt), check='device')
    for bad in ([-1, 3], [E, 3], [5, 5]) + (([2 ** 32 + 1, 3],) if dt == torch.int64 else ()):
      b = torch.tensor(bad, device='cuda', dtype=dt)
      for call in (lambda: eng.save_envs(b, check='device'), lambda: eng.load_envs(s[:2], b, check='device'),
                   lambda: eng.copy_envs(b, ids[:2].to(dt), check='device'),
                   lambda: eng.copy_envs(ids[:2].to(dt), b, check='device')):
        call()
        try:
          eng.check_env_ids()
        except ValueError:
          refused += 1
  torch.cuda.synchronize()
  eng.check_env_ids()
  assert refused == 24, refused   # every call but a save or a copy source with a repeat
  print('device-checked records: %d envs, %d refused reports, %d kernel launches'
        % (E, refused, eng.launch_count()), flush=True)
  raster.close()
  eng.close()


def persistent_mixed(torch):
  from spriteworld_b200 import constants, engine, scene
  n_sms = torch.cuda.get_device_properties(0).multi_processor_count
  W, H, aa, S = 36, 70, 3, 9
  E = 3 * n_sms * 5 // 2 + 1   # 2 bands per frame, 5 resident render CTAs per SM
  rng = np.random.RandomState(5)
  z = np.zeros((E, S))
  b = scene.batch_from_factor_arrays(
      rng.uniform(-0.1, 1.1, (E, S)), rng.uniform(-0.1, 1.1, (E, S)), np.zeros((E, S), np.uint8),
      rng.randint(1, 13, (E, S)), rng.randint(0, 360, (E, S)), rng.uniform(0.02, 1.2, (E, S)),
      z, z, z, z, z, np.zeros((E, S), np.uint32), rng.randint(0, 256, (E, S, 3)))
  eng = engine.Engine(E, S, 1, dict(kind='select_move', scale=1.0), [dict(kind='no_reward')],
                      constants.SHAPES, keep_in_frame=False)
  eng.upload_scenes(b, np.arange(E), np.zeros(E, int))
  eng.upload_state(pos_x=b['x'], pos_y=b['y'], cursor=np.zeros(E), step_count=np.zeros(E),
                   reset_next=np.zeros(E))
  raster = engine.Raster(eng, W, H, aa, (30, 60, 90))
  frames = raster.new_frames()
  for _ in range(2):
    eng.render(raster, frames)
  acts = torch.full((E, 4), 0.5, device=eng.device)
  eng.step(acts, raster, frames)
  eng.step_host(acts.cpu().numpy(), raster)
  torch.cuda.synchronize()
  print('persistent %dx%d: %d envs, %d kernel launches' % (W, H, E, eng.launch_count()), flush=True)
  raster.close()
  eng.close()


if __name__ == '__main__':
  main()
