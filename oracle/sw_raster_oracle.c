/*
 * ORACLE (test infrastructure, not product code) -- CPU restatement of the two
 * Pillow stages the reference's PILRenderer runs per frame:
 *
 *   ImageDraw.polygon(xy, fill)          /root/reference/spriteworld/renderers/pil_renderer.py:83
 *   Image.resize(size, Image.ANTIALIAS)  /root/reference/spriteworld/renderers/pil_renderer.py:84
 *
 * The arithmetic lives in Pillow's C core (libImaging Draw.c / Resample.c), a
 * third-party dependency whose source is NOT under /root/reference and which
 * setup.py:44-54 does not pin; this image has Pillow 12.2.0.  The algorithms are
 * restated from Pillow's published implementation and pinned bit-exact against the
 * installed Pillow by tests/test_oracle_raster.py (random polygons of every
 * Spriteworld shape; random/blocky images through LANCZOS) and against the golden
 * frames generated from the reference itself (tests/golden/make_golden.py).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline/reference arm may
 * load this library.  The product (spriteworld_b200/) never links or imports it.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define SWO_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------- */
/* Polygon fill -- Pillow Draw.c: ImagingDrawPolygon -> polygon_generic        */
/* ------------------------------------------------------------------------- */

typedef struct {
  int d;
  int x0, y0;
  int xmin, ymin, xmax, ymax;
  float dx;
} swo_edge;

static void add_edge(swo_edge *e, int x0, int y0, int x1, int y1) {
  if (x0 <= x1) { e->xmin = x0; e->xmax = x1; } else { e->xmin = x1; e->xmax = x0; }
  if (y0 <= y1) { e->ymin = y0; e->ymax = y1; } else { e->ymin = y1; e->ymax = y0; }
  if (y0 == y1) {
    e->d = 0;
    e->dx = 0.0f;
  } else {
    e->dx = ((float)(x1 - x0)) / (y1 - y0);
    e->d = (y0 == e->ymin) ? 1 : -1;
  }
  e->x0 = x0;
  e->y0 = y0;
}

static int round_up_i(float f) {
  return (int)(f >= 0.0 ? floor(f + 0.5F) : -floor(fabs(f) + 0.5F));
}
static int round_down_i(float f) {
  return (int)(f >= 0.0 ? ceil(f - 0.5F) : -ceil(fabs(f) - 0.5F));
}

/* canvas: H rows x W pixels x 3 bytes (RGB, row-major, top row first) */
static void hline(uint8_t *canvas, int W, int H, int x0, int y, int x1, const uint8_t *rgb) {
  if (y < 0 || y >= H) return;
  if (x0 < 0) x0 = 0; else if (x0 >= W) return;
  if (x1 < 0) return; else if (x1 >= W) x1 = W - 1;
  uint8_t *p = canvas + ((size_t)y * W + x0) * 3;
  for (; x0 <= x1; x0++, p += 3) { p[0] = rgb[0]; p[1] = rgb[1]; p[2] = rgb[2]; }
}

static int cmp_float(const void *a, const void *b) {
  float fa = *(const float *)a, fb = *(const float *)b;
  return (fa > fb) - (fa < fb);
}

static float edge_x_at(const swo_edge *e, int y) {
  /* float32 multiply then float32 add; volatile blocks FMA contraction */
  volatile float prod = (float)(y - e->y0) * e->dx;
  return prod + (float)e->x0;
}

/*
 * xy: n vertices as doubles (x0,y0,x1,y1,...).  Each coordinate is truncated with a C
 * (int) cast exactly as Pillow's _draw_polygon does before ImagingDrawPolygon.
 * corner_join: 1 = include Pillow's "connect discontiguous corners" refinement (what the
 * installed Pillow does); 0 = plain scanline rule (kept so tests can show the refinement
 * matters: 135 of 30000 random Spriteworld-shape instances differ without it).
 */
SWO_API void swo_polygon_fill(uint8_t *canvas, int W, int H, const double *xy, int n,
                              const uint8_t *rgb, int corner_join) {
  if (n <= 0) return;
  int *ixy = (int *)malloc(sizeof(int) * 2 * (size_t)n);
  for (int i = 0; i < 2 * n; i++) ixy[i] = (int)xy[i];

  swo_edge *e = (swo_edge *)calloc((size_t)n + 1, sizeof(swo_edge));
  int ne = 0;
  int i;
  for (i = 0; i < n - 1; i++) {
    int x0 = ixy[i * 2], y0 = ixy[i * 2 + 1], x1 = ixy[i * 2 + 2], y1 = ixy[i * 2 + 3];
    if (y0 == y1 && i != 0 && y0 == ixy[i * 2 - 1]) {
      /* horizontal edge directly after another horizontal edge: merge when both run the same way */
      swo_edge *last = &e[ne - 1];
      if (x1 > x0 && x0 > ixy[i * 2 - 2]) { last->xmax = x1; continue; }
      if (x1 < x0 && x0 < ixy[i * 2 - 2]) { last->xmin = x1; continue; }
    }
    add_edge(&e[ne++], x0, y0, x1, y1);
  }
  if (ixy[i * 2] != ixy[0] || ixy[i * 2 + 1] != ixy[1]) {
    add_edge(&e[ne++], ixy[i * 2], ixy[i * 2 + 1], ixy[0], ixy[1]);
  }

  /* polygon_generic */
  swo_edge **table = (swo_edge **)calloc((size_t)ne + 1, sizeof(swo_edge *));
  int count = 0;
  int ymin = H - 1, ymax = 0;
  for (i = 0; i < ne; i++) {
    if (ymin > e[i].ymin) ymin = e[i].ymin;
    if (ymax < e[i].ymax) ymax = e[i].ymax;
    if (e[i].ymin == e[i].ymax) {
      hline(canvas, W, H, e[i].xmin, e[i].ymin, e[i].xmax, rgb);
      continue;
    }
    table[count++] = &e[i];
  }
  if (ymin < 0) ymin = 0;
  if (ymax > H) ymax = H;

  float *xx = (float *)calloc((size_t)count * 2 + 2, sizeof(float));
  int *xk = (int *)calloc((size_t)count + 1, sizeof(int));
  for (; ymin <= ymax; ymin++) {
    int j = 0;
    for (i = 0; i < count; i++) {
      swo_edge *cur = table[i];
      xk[i] = 2 * count + 1;
      if (ymin >= cur->ymin && ymin <= cur->ymax) {
        xk[i] = j;
        xx[j++] = edge_x_at(cur, ymin);
        if (ymin == cur->ymax && ymin < ymax) {
          /* "needed to draw consistent polygons": an edge ending on an interior row counts twice */
          xx[j] = xx[j - 1];
          j++;
        } else if (corner_join && cur->dx != 0) {
          /*
           * "Connect discontiguous corners".  Behavioural model fitted to the installed
           * Pillow 12.2.0 (source not available here): when this edge and an EARLIER table
           * edge leave the same corner in the same x direction -- both start on this row,
           * or both end on the polygon's last row -- the earlier edge's crossing is moved
           * towards where the adjacent row's span begins (min of the two edges one row on,
           * minus 1, for a corner opening to the right; max plus 1 to the left), rounded
           * half-up and never pulled back across the corner itself.
           */
          for (int k = 0; k < i; k++) {
            swo_edge *other = table[k];
            if ((cur->dx > 0 && other->dx <= 0) || (cur->dx < 0 && other->dx >= 0)) continue;
            int both_start = (ymin == other->ymin && ymin == cur->ymin);
            int both_end_last = (ymin == ymax && ymin == other->ymax && ymin == cur->ymax);
            if (!both_start && !both_end_last) continue;
            if (roundf(xx[j - 1]) != roundf(edge_x_at(other, ymin))) continue;
            int offset = (ymin == ymax) ? -1 : 1;
            float adj = edge_x_at(cur, ymin + offset);
            float adj_other = edge_x_at(other, ymin + offset);
            int right = (ymin == cur->ymax) ? (cur->dx < 0) : (cur->dx > 0);
            float nv = right ? fminf(adj, adj_other) - 1 : fmaxf(adj, adj_other) + 1;
            nv = floorf(nv + 0.5f);
            nv = right ? fmaxf(nv, xx[j - 1]) : fminf(nv, xx[j - 1]);
            xx[xk[k]] = nv;
            break;
          }
        }
      }
    }
    qsort(xx, (size_t)j, sizeof(float), cmp_float);
    int x_pos = (j == 0) ? -1 : 0;
    for (i = 1; i < j; i += 2) {
      int x_end = round_down_i(xx[i]);
      if (x_end < x_pos) continue; /* span would lie before the current position */
      if (xx[i - 1] > (float)x_pos) {
        x_pos = round_up_i(xx[i - 1]);
        if (x_end < x_pos) continue;
      }
      hline(canvas, W, H, x_pos, ymin, x_end, rgb);
      x_pos = x_end + 1;
    }
  }
  free(xx);
  free(xk);
  free(table);
  free(e);
  free(ixy);
}

/* ------------------------------------------------------------------------- */
/* LANCZOS resize, 8 bits per channel -- Pillow Resample.c                     */
/* ------------------------------------------------------------------------- */

#define SWO_PRECISION_BITS (32 - 8 - 2) /* 22 */

static double sinc_filter(double x) {
  if (x == 0.0) return 1.0;
  x = x * M_PI;
  return sin(x) / x;
}
static double lanczos_filter(double x) {
  if (-3.0 <= x && x < 3.0) return sinc_filter(x) * sinc_filter(x / 3);
  return 0.0;
}

/* ksize for one axis (precompute_coeffs) */
SWO_API int swo_lanczos_ksize(int in_size, int out_size) {
  double scale = (double)in_size / out_size;
  double filterscale = scale < 1.0 ? 1.0 : scale;
  double support = 3.0 * filterscale;
  return (int)ceil(support) * 2 + 1;
}

/*
 * bounds: out_size pairs (xmin, count); kk: out_size * ksize int32 fixed-point taps.
 * precompute_coeffs + normalize_coeffs_8bpc.
 */
SWO_API void swo_lanczos_coeffs(int in_size, int out_size, int *bounds, int32_t *kk) {
  double scale = (double)in_size / out_size;
  double filterscale = scale < 1.0 ? 1.0 : scale;
  double support = 3.0 * filterscale;
  int ksize = (int)ceil(support) * 2 + 1;
  double *k = (double *)malloc(sizeof(double) * (size_t)ksize);
  for (int xx = 0; xx < out_size; xx++) {
    double center = (xx + 0.5) * scale;
    double ww = 0.0;
    double ss = 1.0 / filterscale;
    int xmin = (int)(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)(center + support + 0.5);
    if (xmax > in_size) xmax = in_size;
    xmax -= xmin;
    int x;
    for (x = 0; x < xmax; x++) {
      double w = lanczos_filter((x + xmin - center + 0.5) * ss);
      k[x] = w;
      ww += w;
    }
    for (x = 0; x < xmax; x++) {
      if (ww != 0.0) k[x] /= ww;
    }
    for (; x < ksize; x++) k[x] = 0;
    bounds[xx * 2 + 0] = xmin;
    bounds[xx * 2 + 1] = xmax;
    for (x = 0; x < ksize; x++) {
      double v = k[x] * (1 << SWO_PRECISION_BITS);
      kk[xx * ksize + x] = (v < 0) ? (int)(-0.5 + v) : (int)(0.5 + v);
    }
  }
  free(k);
}

static inline uint8_t clip8(int in) {
  int v = in >> SWO_PRECISION_BITS;
  return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

/* One LANCZOS pass of ImagingResample over an RGB image: horizontal (inW -> outW columns of
 * H rows) or vertical (inH -> outH rows of W columns), each output clip8'ed to uint8. */
static void hpass(const uint8_t *in, int inW, int H, uint8_t *out, int outW) {
  int ks = swo_lanczos_ksize(inW, outW);
  int *bounds = (int *)malloc(sizeof(int) * 2 * (size_t)outW);
  int32_t *kk = (int32_t *)malloc(sizeof(int32_t) * (size_t)ks * outW);
  swo_lanczos_coeffs(inW, outW, bounds, kk);
  for (int y = 0; y < H; y++) {
    const uint8_t *line = in + (size_t)y * inW * 3;
    for (int xx = 0; xx < outW; xx++) {
      int xmin = bounds[xx * 2], cnt = bounds[xx * 2 + 1];
      const int32_t *k = kk + (size_t)xx * ks;
      int s0 = 1 << (SWO_PRECISION_BITS - 1), s1 = s0, s2 = s0;
      for (int x = 0; x < cnt; x++) {
        const uint8_t *p = line + (size_t)(x + xmin) * 3;
        s0 += p[0] * k[x];
        s1 += p[1] * k[x];
        s2 += p[2] * k[x];
      }
      uint8_t *o = out + ((size_t)y * outW + xx) * 3;
      o[0] = clip8(s0); o[1] = clip8(s1); o[2] = clip8(s2);
    }
  }
  free(bounds);
  free(kk);
}

static void vpass(const uint8_t *in, int W, int inH, uint8_t *out, int outH) {
  int ks = swo_lanczos_ksize(inH, outH);
  int *bounds = (int *)malloc(sizeof(int) * 2 * (size_t)outH);
  int32_t *kk = (int32_t *)malloc(sizeof(int32_t) * (size_t)ks * outH);
  swo_lanczos_coeffs(inH, outH, bounds, kk);
  for (int yy = 0; yy < outH; yy++) {
    int ymin = bounds[yy * 2], cnt = bounds[yy * 2 + 1];
    const int32_t *k = kk + (size_t)yy * ks;
    for (int xx = 0; xx < W; xx++) {
      int s0 = 1 << (SWO_PRECISION_BITS - 1), s1 = s0, s2 = s0;
      for (int y = 0; y < cnt; y++) {
        const uint8_t *p = in + ((size_t)(y + ymin) * W + xx) * 3;
        s0 += p[0] * k[y];
        s1 += p[1] * k[y];
        s2 += p[2] * k[y];
      }
      uint8_t *o = out + ((size_t)yy * W + xx) * 3;
      o[0] = clip8(s0); o[1] = clip8(s1); o[2] = clip8(s2);
    }
  }
  free(bounds);
  free(kk);
}

/*
 * in: inH x inW x 3, out: outH x outW x 3 (RGB row-major).  Image.resize: a plain copy if the
 * sizes are equal; otherwise ImagingResample, one pass per axis whose size changes, each into a
 * uint8 image.  The horizontal pass comes first, except that Image.resize (Pillow 12.2.0)
 * resizes an image more than 100 times taller than wide vertically first when it shrinks its
 * height (`self.size[1] > self.size[0] * 100 and size[1] < self.size[1]`).
 * tmp (optional, may be NULL): receives the first pass's image when both axes change, inH x outW
 * x 3 (horizontal first) or outH x inW x 3 (vertical first) -- the same number of bytes when
 * both sizes shrink by the same factor.
 */
static int vertical_first(int inW, int inH, int outH) {
  return (int64_t)inH > (int64_t)inW * 100 && outH < inH;
}

SWO_API void swo_lanczos_resize(const uint8_t *in, int inW, int inH, uint8_t *out, int outW,
                                int outH, uint8_t *tmp) {
  if (inW == outW && inH == outH) {
    memcpy(out, in, (size_t)inW * inH * 3);
    return;
  }
  if (inW == outW) {
    vpass(in, inW, inH, out, outH);
    return;
  }
  if (inH == outH) {
    hpass(in, inW, inH, out, outW);
    return;
  }
  const int vfirst = vertical_first(inW, inH, outH);
  const size_t mid_bytes = vfirst ? (size_t)outH * inW * 3 : (size_t)inH * outW * 3;
  uint8_t *mid = tmp ? tmp : (uint8_t *)malloc(mid_bytes);
  if (vfirst) {
    vpass(in, inW, inH, mid, outH);
    hpass(mid, inW, outH, out, outW);
  } else {
    hpass(in, inW, inH, mid, outW);
    vpass(mid, outW, inH, out, outH);
  }
  if (mid != tmp) free(mid);
}
