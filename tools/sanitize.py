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
  persistent_mixed(torch)


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
