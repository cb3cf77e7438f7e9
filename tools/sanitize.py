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

Between those, env records: host-checked saves, loads and copies (disjoint and overlapping), which
run the device-checked calls' save and load kernels on int32 ids, and device-checked ones with int32
and int64 device ids, valid and refused (out of range either way, 2^32 + 1, repeated destinations),
so that memcheck sees that a refused id never indexes engine memory.  Then rollouts from records
into leaves, from those leaves, and from the live envs into leaves, renders of records, windows of
live envs and records (swb_render_windows, flagged windows among them) on a narrow and a wide
raster, and the same with random subsets of the sprites drawn (swb_render_views), the sprite
coverage (swb_render_coverage) of live envs and records into buffers that are not 16-byte aligned,
their soft masks (swb_render_soft_masks) into buffers at odd byte offsets, their boxes
(swb_render_boxes) at 4-byte offsets that are not 16-byte aligned, and an engine
checkpoint saved, loaded and rendered, with a corrupt one refused.  Records are then made from
factor columns (swb_make_states) of every column dtype, with refused records among them, into a
record buffer one record past the start of its allocation, and rendered.
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
  made_records(torch)
  persistent_mixed(torch)


def device_checked_records(torch):
  from spriteworld_b200 import engine, workloads
  wl = workloads.WORKLOADS['c2']()
  E = 40
  eng, raster, _ = workloads.build_engine(wl, E, 4, device=0, seed=4, max_episode_length=3)
  eng.step(torch.from_numpy(wl.sample_actions(np.random.RandomState(2), 1, E)[0]).cuda(), raster)
  host = np.arange(E)
  eng.load_envs(eng.save_envs(host[::-1].copy()), host)
  eng.copy_envs(host, np.roll(host, 3))          # overlapping: through engine scratch
  eng.copy_envs(host[:10], host[20:30])          # disjoint: one kernel
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
  # rollouts from records (an odd count, some about to reset) into leaves, and from the leaves
  roots = eng.save_envs(np.arange(E - 3))
  T, C = 4, 3
  plans = torch.rand((T, len(roots), C, 4), device='cuda')
  res = eng.rollout(plans, states=roots, leaves=True)
  eng.rollout(torch.rand((T, len(res.leaves), 1, 4), device='cuda'), states=res.leaves, leaves=True)
  eng.rollout(torch.rand((T, E, 2, 4), device='cuda'), leaves=True)
  torch.cuda.synchronize()
  print('record rollouts: %d roots, %d leaves, %d kernel launches'
        % (len(roots), len(res.leaves), eng.launch_count()), flush=True)
  # frames of those leaves (more records than envs) and of zero records
  frames, status = eng.render_states(raster, res.leaves)
  eng.render_states(raster, res.leaves.take(torch.tensor([-1, 0, len(res.leaves)], device='cuda')))
  torch.cuda.synchronize()
  print('record renders: %d frames, %d overflowed, %d kernel launches'
        % (len(frames), int(status.bool().sum()), eng.launch_count()), flush=True)
  # windows of the live envs and of the leaves: zoomed, off-scene and flagged (empty, NaN) windows
  pos = eng.state_tensors()
  win = torch.stack([pos['pos_x'] - 0.1, pos['pos_y'] - 0.05, pos['pos_x'] + 0.1, pos['pos_y'] + 0.15], -1)
  win[0, 0] = torch.tensor([0.5, 0.0, 0.5, 1.0], dtype=torch.float64)
  win[-1, -1] = torch.tensor([float('nan'), 0.0, 1.0, 1.0], dtype=torch.float64)
  lwin = torch.tensor([-2.0, -2.0, 3.0, 3.0], dtype=torch.float64, device='cuda').repeat(len(res.leaves), 2, 1)
  # the workload's raster and a wide one (anti_aliasing 7: render_kernel<false, true, *, true>)
  wide = engine.Raster(eng, 64, 64, 7, (40, 40, 40))
  # views with random subsets drawn (swb_render_views), the flagged windows among them, and a
  # draw that leaves the NaN window's row empty
  draw = torch.rand(win.shape[:2] + (eng.n_slots,), device='cuda') < 0.5
  draw[-1] = False
  ldraw = torch.rand((len(res.leaves), 2, eng.n_slots), device='cuda') < 0.5
  for r in (raster, wide):
    _, wstatus = eng.render_windows(r, win.contiguous())
    eng.render_windows(r, lwin, res.leaves)
    _, vstatus = eng.render_windows(r, win.contiguous(), draw=draw)
    eng.render_windows(r, lwin, res.leaves, draw=ldraw)
  torch.cuda.synchronize()
  wide.close()
  print('window renders: %d views on 2 rasters, %d flagged, %d kernel launches'
        % (2 * (wstatus.numel() + lwin.shape[0] * 2), int(wstatus.bool().sum()), eng.launch_count()), flush=True)
  print('view renders: %d views on 2 rasters, %d flagged'
        % (2 * (vstatus.numel() + lwin.shape[0] * 2), int(vstatus.bool().sum())), flush=True)
  # coverage of the live envs and of the leaves: odd widths at 4-byte offsets that are not
  # 16-byte aligned (the write-out's head and tail), bands of one and many rows, and zero records
  S = eng.n_slots
  for W, H, aa, skew in ((wl.image_size[0], wl.image_size[1], 1, 0), (13, 7, 5, 1), (1023, 3, 4, 3)):
    for states in (None, res.leaves, res.leaves[:0]):
      n = E if states is None else len(states)
      flat = torch.zeros(n * (H * W + 2 * S) + 4, dtype=torch.int32, device='cuda')
      cover = flat[skew:skew + n * H * W].view(n, H, W)
      visible = flat[skew + n * H * W:skew + n * (H * W + S)].view(n, S)
      area = flat[skew + n * (H * W + S):skew + n * (H * W + 2 * S)].view(n, S)
      eng.render_coverage(W, H, aa, states=states, out=(cover, visible, area))
  torch.cuda.synchronize()
  print('coverage: live envs and %d leaves, %d kernel launches' % (len(res.leaves), eng.launch_count()),
        flush=True)
  # soft masks of the live envs and of the leaves at odd byte offsets: bands of one mask row (a
  # 4095-wide canvas at aa 15) and of many, and zero records
  for W, H, aa, skew in ((wl.image_size[0], wl.image_size[1], 5, 1), (13, 7, 15, 3), (273, 2, 15, 7),
                         (1023, 3, 4, 5)):
    for states in (None, res.leaves, res.leaves[:0]):
      n = E if states is None else len(states)
      flat = torch.zeros(n * S * H * W + 16, dtype=torch.uint8, device='cuda')
      eng.render_soft_masks(W, H, aa, states=states, out=flat[skew:skew + n * S * H * W].view(n, S, H, W))
  torch.cuda.synchronize()
  print('soft masks: live envs and %d leaves, %d kernel launches' % (len(res.leaves), eng.launch_count()),
        flush=True)
  # boxes of the live envs and of the leaves at 4-byte offsets that are not 16-byte aligned: bands
  # of one row (4095 wide) and of many, and zero records
  for W, H, aa, skew in ((wl.image_size[0], wl.image_size[1], 5, 1), (13, 7, 5, 3), (4095, 2, 1, 2)):
    for states in (None, res.leaves, res.leaves[:0]):
      n = E if states is None else len(states)
      flat = torch.zeros(n * 10 * S + 4, dtype=torch.int32, device='cuda')
      views = [flat[skew + o * n * S:skew + (o + k) * n * S] for o, k in ((0, 4), (4, 4), (8, 1), (9, 1))]
      eng.render_boxes(W, H, aa, states=states, out=tuple(v.view(n, S, 4) if i < 2 else v.view(n, S)
                                                          for i, v in enumerate(views)))
  torch.cuda.synchronize()
  print('boxes: live envs and %d leaves, %d kernel launches' % (len(res.leaves), eng.launch_count()),
        flush=True)
  # an engine checkpoint round trip, and a corrupt one refused before anything is enqueued
  from spriteworld_b200 import _native
  state = eng.save_state()
  eng.load_state(state)
  eng.render(raster)
  bad = state.clone()
  bad[12] ^= 1                                   # E
  try:
    eng.load_state(bad)
    raise AssertionError('a corrupt checkpoint was loaded')
  except _native.NativeError:
    pass
  torch.cuda.synchronize()
  assert torch.equal(eng.save_state(), state)
  print('checkpoint: %d bytes saved and loaded, a corrupt one refused' % state.numel(), flush=True)
  raster.close()
  eng.close()


def made_records(torch):
  from spriteworld_b200 import engine, scene_program, workloads
  from spriteworld_b200 import factor_distributions as distribs
  from spriteworld_b200.renderers import color_maps
  wl = workloads.WORKLOADS['c3']()
  eng, raster, _ = workloads.build_engine(wl, 8, 2, device=0, seed=3)
  eng.load_packer(scene_program.compile_packer([distribs.Continuous('c0', 0.0, 0.5)], color_maps.hsv_to_rgb))
  n, S, rb = 37, eng.n_slots, eng.record_bytes
  rng = np.random.RandomState(5)
  buf = torch.zeros((n + 1, rb), dtype=torch.uint8, device='cuda')
  out = engine.EnvStates(buf[1:], 1, eng.signature, S)
  for dt in (torch.float32, torch.float64, torch.int8, torch.int16, torch.int32, torch.int64, torch.uint8):
    shape = torch.from_numpy(rng.randint(0, 13, (n, S))).cuda().to(dt)
    shape[:, -1] = 8
    factors = {'shape': shape, 'x': torch.rand(n, S, device='cuda').to(dt), 'angle': torch.zeros(n, 1, device='cuda').to(dt),
               'c0': torch.rand(n, S, device='cuda'), 'c1': torch.rand(1, S, device='cuda'), 'c2': torch.rand(n, 1, device='cuda')}
    states, status = eng.make_states(factors, out=out)
    eng.render_states(raster, states)
    eng.make_states({'shape': shape[:0]}, span_class=1)
  torch.cuda.synchronize()
  print('made records: %d per dtype, %d refused in the last, %d kernel launches'
        % (n, int((status != 0).sum()), eng.launch_count()), flush=True)
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
