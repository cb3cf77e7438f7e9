"""Generates tests/golden/wide_aa/render_cases_wide_aa.npz by RUNNING THE UNMODIFIED REFERENCE.

Run in the build container only (needs /root/reference):

    python tests/golden/make_golden_wide_aa.py

Frames of PILRenderer at anti_aliasing 6 to 20 (the reference's demo renders 256x256 at 10),
laid out like render_cases.npz: per case its meta data (name, size, anti_aliasing, background,
colour map), the sprite factor arrays and the frame.  The reference is imported through
oracle/refshim by make_golden.py, whose helpers this script shares.  SWB_GOLDEN_OUT redirects the
output directory (tests/test_golden_wide_aa_reproducible.py).
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402  (loads the reference)

OUT = os.environ.get('SWB_GOLDEN_OUT') or os.path.join(os.path.dirname(os.path.abspath(__file__)),
                                                       'wide_aa')


def render_cases_wide_aa():
  cases = []
  hsv = mg.sw_renderers.color_maps.hsv_to_rgb

  def add(name, sprites, size, aa, ctr=None, bg=None):
    r = mg.sw_renderers.PILRenderer(image_size=size, anti_aliasing=aa, bg_color=bg,
                                    color_to_rgb=ctr)
    cases.append(dict(
        name=name, width=int(size[0]), height=int(size[1]), aa=int(aa),
        bg=[int(c) for c in (bg or (0, 0, 0))], color_map='hsv' if ctr is not None else 'none',
        frame=r.render(sprites), **mg.sprites_to_arrays(sprites, len(sprites), [], ctr)))

  def fixture():  # tests/renderers/pil_renderer_test.py:31-43
    return [
        mg.sprite_lib.Sprite(x=0.75, y=0.95, shape='spoke_6', scale=0.2, c0=20, c1=50, c2=80),
        mg.sprite_lib.Sprite(x=0.2, y=0.3, shape='triangle', scale=0.1, c0=150, c1=255, c2=100),
        mg.sprite_lib.Sprite(x=0.7, y=0.5, shape='square', scale=0.3, c0=0, c1=255, c2=0),
        mg.sprite_lib.Sprite(x=0.5, y=0.5, shape='square', scale=0.3, c0=255, c1=0, c2=0),
    ]

  for aa in (6, 7, 8, 9, 10, 13):
    add('fixture_aa%d_64' % aa, fixture(), (64, 64), aa)
  # all 12 shapes at 64x64 aa 10: six per scene, random angle / scale / colour, partly off frame
  rng = np.random.RandomState(17)
  names = sorted(mg.constants.SHAPES)

  def random_sprites(shapes):
    return [mg.sprite_lib.Sprite(
        x=np.float32(rng.uniform(-0.05, 1.05)), y=np.float32(rng.uniform(-0.05, 1.05)),
        shape=str(shape), angle=int(rng.randint(0, 360)), scale=float(rng.uniform(0.03, 0.4)),
        c0=int(rng.randint(256)), c1=int(rng.randint(256)), c2=int(rng.randint(256)))
        for shape in shapes]

  for i in range(4):
    shapes = names[6 * (i % 2):6 * (i % 2) + 6] if i < 2 else rng.permutation(names)[:6]
    add('allshapes_aa10_%d' % i, random_sprites(shapes), (64, 64), 10)
  # the demo's renderer (256x256, aa 10, hsv_to_rgb) on scenes of the cobra clustering config
  np.random.seed(23)
  cfg = mg.clustering.get_config('train')
  for i in range(3):
    add('clustering256_aa10_%d' % i, cfg['init_sprites'](), (256, 256), 10, ctr=hsv)
  # a non-square frame with a background, and a short frame above aa 13 whose one-block tiles
  # still fit the render kernel's H tile
  add('nonsquare_72x40_aa9', random_sprites(rng.permutation(names)[:8]), (72, 40), 9,
      bg=(30, 60, 90))
  add('short_64x8_aa20', random_sprites(rng.permutation(names)[:5]), (64, 8), 20)

  blob = dict(names=np.array([c['name'] for c in cases]))
  for i, c in enumerate(cases):
    blob['meta_%d' % i] = np.array(json.dumps(
        {k: c[k] for k in ('name', 'width', 'height', 'aa', 'bg', 'color_map')}))
    blob['frame_%d' % i] = c['frame']
    for f in mg.FIELDS:
      blob['%s_%d' % (f, i)] = c[f]
  blob.update(mg.shapes_blob())
  os.makedirs(OUT, exist_ok=True)
  np.savez_compressed(os.path.join(OUT, 'render_cases_wide_aa.npz'), **blob)
  print('render_cases_wide_aa.npz: %d cases' % len(cases))


if __name__ == '__main__':
  render_cases_wide_aa()
