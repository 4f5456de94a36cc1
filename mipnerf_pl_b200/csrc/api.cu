// api.cu — the extern "C" surface declared in include/mipnerf_b200.h and the level loop of
// MipNerf.forward (models/mip_nerf.py:172-248) expressed as kernel launches on one stream.
#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>

#include "../../include/mipnerf_b200.h"
#include "kernels.h"
#include "mlp_tc.h"
#include "profile.h"

namespace {

thread_local std::string g_last_error;

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
  return code;
}

#define CUDA_TRY(expr)                                                                           \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess)                                                                       \
      return fail(MIPNERF_B200_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),    \
                  __FILE__, __LINE__);                                                           \
  } while (0)

constexpr int64_t kChunkRaysFp32 = 4096;  // bounds the fp32 path's activation scratch (~1.8 GB)
// the bf16x3 training step carries every tile image twice (hi, lo): half the chunk keeps its scratch at the 16-bit
// step's (5.7 GiB instead of 11 GiB at the default architecture)
constexpr int64_t kChunkRaysX3 = 2048;
// Largest histogram the stand-alone resampler entries take.  Its row sum restates torch.sum's fp32 order, which CPU
// torch keeps for rows of up to 544 floats and changes above that; 512 also keeps the kernel's 4 x (3 nb + 2) floats of
// shared memory inside the 48 KiB default.  The model itself resamples at most 256 bins.
constexpr int kMaxResampleBins = 512;

using mipnerf::align_up;
using mipnerf::Carver;

struct Dims {
  int xyz_dim, view_dim, n_lin;
};

// The per-ray sample counts the compositing kernel is instantiated for (launch_composite: P = N/32 in 1,2,3,4,6,8).
int check_num_samples(int n) {
  if (n <= 0 || n % 32 != 0 || n > 256 || n / 32 == 5 || n / 32 == 7)
    return fail(MIPNERF_B200_EUNSUPPORTED, "num_samples=%d: need a multiple of 32 in {32,64,96,128,192,256}", n);
  return MIPNERF_B200_OK;
}

int check_config(const mipnerf_b200_config* c, Dims* d) {
  if (!c) return fail(MIPNERF_B200_EINVAL, "config is NULL");
  if (int rc = check_num_samples(c->num_samples)) return rc;
  if (c->num_levels < 1) return fail(MIPNERF_B200_EINVAL, "num_levels=%d", c->num_levels);
  if (c->max_deg_point <= c->min_deg_point || c->min_deg_point < -60 || c->max_deg_point > 60)
    return fail(MIPNERF_B200_EINVAL, "bad point degrees [%d,%d)", c->min_deg_point, c->max_deg_point);
  if (c->deg_view < 0 || c->deg_view > 60) return fail(MIPNERF_B200_EINVAL, "deg_view=%d", c->deg_view);
  if (c->net_depth < 1 || c->net_width < 1 || c->skip_index < 1 || c->net_depth_condition < 0 ||
      c->net_width_condition < 1)
    return fail(MIPNERF_B200_EINVAL, "bad MLP shape");
  if (c->num_rgb_channels != 3 || c->num_density_channels != 1)
    return fail(MIPNERF_B200_EUNSUPPORTED, "only 3 rgb / 1 density channels (volumetric_rendering assumes it)");
  const int last = c->net_depth - 1;
  if (last > 0 && last % c->skip_index == 0)
    return fail(MIPNERF_B200_EUNSUPPORTED,
                "skip connection after the last trunk layer: the reference's density_layer cannot take it");
  if (!c->use_viewdirs && c->net_width != c->net_width_condition)
    return fail(MIPNERF_B200_EUNSUPPORTED,
                "use_viewdirs=False needs net_width == net_width_condition (reference color_layer shape)");
  // view_layers is then an empty Sequential: the colour head would see net_width + view_dim inputs, which the
  // reference's color_layer (net_width_condition inputs) cannot take
  if (c->use_viewdirs && c->net_depth_condition == 0)
    return fail(MIPNERF_B200_EUNSUPPORTED, "net_depth_condition=0 with use_viewdirs");
  if (!(c->density_noise >= 0.f) || c->density_noise > 3.0e38f)
    return fail(MIPNERF_B200_EINVAL, "density_noise=%g: need a finite standard deviation >= 0", (double)c->density_noise);
  d->xyz_dim = (c->max_deg_point - c->min_deg_point) * 6;
  d->view_dim = c->deg_view * 6 + 3;
  d->n_lin = c->net_depth + 2 + c->net_depth_condition + 1;
  return MIPNERF_B200_OK;
}

int check_weights(const mipnerf_b200_config* c, const Dims& d, const mipnerf_b200_weights* w) {
  if (!w || !w->linears) return fail(MIPNERF_B200_EINVAL, "weights are NULL");
  if (w->num_linears != d.n_lin)
    return fail(MIPNERF_B200_EINVAL, "expected %d linears (state_dict order), got %d", d.n_lin, w->num_linears);
  auto expect = [&](int idx, int in, int out, const char* name) {
    const mipnerf_b200_linear& l = w->linears[idx];
    if (!l.weight || !l.bias) return fail(MIPNERF_B200_EINVAL, "%s has a NULL tensor", name);
    if (l.in_features != in || l.out_features != out)
      return fail(MIPNERF_B200_EINVAL, "%s is [%d,%d], expected [%d,%d]", name, l.out_features, l.in_features,
                  out, in);
    return MIPNERF_B200_OK;
  };
  int rc;
  for (int i = 0; i < c->net_depth; ++i) {
    int in = i == 0 ? d.xyz_dim : c->net_width;
    if (i > 1 && (i - 1) % c->skip_index == 0) in = c->net_width + d.xyz_dim;  // models/mip_nerf.py:40-42
    if ((rc = expect(i, in, c->net_width, "layers[i]"))) return rc;
  }
  if ((rc = expect(c->net_depth, c->net_width, 1, "density_layer"))) return rc;
  if ((rc = expect(c->net_depth + 1, c->net_width, c->net_width, "extra_layer"))) return rc;
  for (int i = 0; i < c->net_depth_condition; ++i) {
    const int in = i == 0 ? c->net_width + d.view_dim : c->net_width_condition;
    if ((rc = expect(c->net_depth + 2 + i, in, c->net_width_condition, "view_layers[i]"))) return rc;
  }
  return expect(d.n_lin - 1, c->net_width_condition, 3, "color_layer");
}

// The precondition of the entry points that run the level kernels: `precision` runs on the tensor cores for this
// config, and w->packed is an image of that precision, at least tc_packed_bytes long.
int check_tc(const mipnerf_b200_config* c, const mipnerf_b200_weights* w, int precision, const char* what) {
  if (!mipnerf::tc_supported(c, precision))
    return fail(MIPNERF_B200_EUNSUPPORTED,
                "tensor-core %s: the 8x256 / 1x128 model with num_samples 128 or 256, min_deg_point 0, max_deg_point "
                "1..16, deg_view 1..4 and precision bf16|fp16|fp16x3|bf16x3 only; use MIPNERF_B200_FP32",
                what);
  const size_t need = mipnerf::tc_packed_bytes(c, precision);
  if (!w->packed || w->packed_precision != precision || w->packed_bytes < need)
    return fail(MIPNERF_B200_EINVAL, "weights->packed missing, packed for another precision or shorter than %zu bytes",
                need);
  return MIPNERF_B200_OK;
}

// Floats of the wgrad partial sums: kWgradMaxSlices slices of [n, k + 1] for the widest layer of the MLP
size_t wgrad_part_floats(const mipnerf_b200_config* c, const Dims& d) {
  const size_t max_n = std::max(c->net_width, c->net_width_condition);
  const size_t max_k = (size_t)c->net_width + std::max(d.xyz_dim, d.view_dim) + 1;
  return (size_t)mipnerf::kWgradMaxSlices * max_n * max_k;
}

int check_rays(const mipnerf_b200_rays* r) {
  if (!r) return fail(MIPNERF_B200_EINVAL, "rays is NULL");
  if (r->num_rays < 0) return fail(MIPNERF_B200_EINVAL, "num_rays=%lld", (long long)r->num_rays);
  if (r->num_rays > 0 && (!r->origins || !r->directions || !r->radii || !r->near || !r->far))
    return fail(MIPNERF_B200_EINVAL, "a ray field is NULL");
  return MIPNERF_B200_OK;
}

// The grid description of mipnerf_b200_grid_render, its backward, mipnerf_b200_grid_visibility and
// mipnerf_b200_grid_tv (`g` checked
// non-NULL by the caller).  With `bricks` (mipnerf_b200_grid_render_bricks and mipnerf_b200_grid_visibility_bricks,
// checked non-NULL by the caller) the
// cells are the bricks: every levels[l].cells must be NULL and every bricks->table[l] set.
int check_grid(const mipnerf_b200_grid* g, const mipnerf_b200_grid_bricks* bricks = nullptr) {
  if (g->num_levels < 1 || g->num_levels > MIPNERF_B200_GRID_MAX_LEVELS)
    return fail(MIPNERF_B200_EINVAL, "num_levels=%d: need 1..%d", g->num_levels, MIPNERF_B200_GRID_MAX_LEVELS);
  if (g->degree < 0 || g->degree > 3) return fail(MIPNERF_B200_EINVAL, "degree=%d: need 0..3", g->degree);
  const int scale = 1 << (g->num_levels - 1);
  if (g->block < 1 || g->block % scale != 0)
    return fail(MIPNERF_B200_EINVAL, "block=%d: need a positive multiple of 2^(num_levels - 1) = %d", g->block, scale);
  if (!g->occupancy) return fail(MIPNERF_B200_EINVAL, "occupancy is NULL");
  if (!std::isfinite(g->rgb_padding)) return fail(MIPNERF_B200_EINVAL, "rgb_padding=%g", g->rgb_padding);
  for (int a = 0; a < 3; ++a)
    if (!(g->hi[a] > g->lo[a]) || !std::isfinite(g->lo[a]) || !std::isfinite(g->hi[a]))
      return fail(MIPNERF_B200_EINVAL, "bounds axis %d: [%g, %g], need lo < hi, finite", a, g->lo[a], g->hi[a]);
  const int32_t* n0 = &g->levels[0].nx;
  for (int l = 0; l < g->num_levels; ++l) {
    const mipnerf_b200_grid_level& lv = g->levels[l];
    if (!bricks && !lv.cells) return fail(MIPNERF_B200_EINVAL, "level %d: cells is NULL", l);
    if (bricks && lv.cells)
      return fail(MIPNERF_B200_EINVAL, "level %d: levels[%d].cells is set; the cells are read from bricks", l, l);
    if (bricks && !bricks->table[l]) return fail(MIPNERF_B200_EINVAL, "level %d: bricks->table[%d] is NULL", l, l);
    const int32_t n[3] = {lv.nx, lv.ny, lv.nz};
    for (int a = 0; a < 3; ++a)
      if (n[a] < 2 || (int64_t)(n[a] - 1) << l != (int64_t)n0[a] - 1)
        return fail(MIPNERF_B200_EINVAL, "level %d: %d x %d x %d points, need >= 2 per axis and (n_0 - 1) / 2^%d + 1",
                    l, lv.nx, lv.ny, lv.nz, l);
  }
  return MIPNERF_B200_OK;
}

// The uint8 rows of mipnerf_b200_grid_render_u8 and mipnerf_b200_grid_render_bricks (`sh` checked non-NULL by the
// caller): no levels[l].sh, finite scale / offset entries in use.
int check_sh_u8(const mipnerf_b200_grid* g, const mipnerf_b200_grid_sh_u8* sh) {
  const int nc = (g->degree + 1) * (g->degree + 1);
  for (int l = 0; l < g->num_levels; ++l) {
    if (g->levels[l].sh)
      return fail(MIPNERF_B200_EINVAL, "level %d: levels[%d].sh is set; the uint8 rows are read from sh->rows", l, l);
    for (int k = 0; k < nc; ++k)
      for (int ch = 0; ch < 3; ++ch)
        if (!std::isfinite(sh->scale[l][k][ch]) || !std::isfinite(sh->offset[l][k][ch]))
          return fail(MIPNERF_B200_EINVAL, "level %d coefficient %d channel %d: scale=%g offset=%g, need finite", l, k,
                      ch, sh->scale[l][k][ch], sh->offset[l][k][ch]);
  }
  return MIPNERF_B200_OK;
}

// The shared prologue of the entry points that march rays through a grid, in the order they refuse: grid, rays,
// viewdirs, the outputs (`out`: {rgb, distance, acc} of an entry point that renders, NULL for the others), the step,
// the bricks (`bricks`: the bricks argument of a _bricks entry point, NULL for the dense ones), then check_grid.
int check_march(const mipnerf_b200_grid* g, const mipnerf_b200_rays* rays, float* const* out, float step,
                const mipnerf_b200_grid_bricks* const* bricks) {
  int rc;
  if (!g) return fail(MIPNERF_B200_EINVAL, "grid is NULL");
  if ((rc = check_rays(rays))) return rc;
  if (rays->num_rays > 0 && !rays->viewdirs) return fail(MIPNERF_B200_EINVAL, "rays->viewdirs is NULL");
  if (out && rays->num_rays > 0 && (!out[0] || !out[1] || !out[2]))
    return fail(MIPNERF_B200_EINVAL, "rgb / distance / acc is NULL");
  if (!(step > 0.f) || !std::isfinite(step)) return fail(MIPNERF_B200_EINVAL, "step=%g: need a finite step > 0", step);
  if (bricks && !*bricks) return fail(MIPNERF_B200_EINVAL, "bricks is NULL");
  return check_grid(g, bricks ? *bricks : nullptr);
}

mipnerf_b200_rays offset_rays(const mipnerf_b200_rays& r, int64_t off, int64_t count) {
  mipnerf_b200_rays o = r;
  o.origins = r.origins + off * 3;
  o.directions = r.directions + off * 3;
  o.viewdirs = r.viewdirs ? r.viewdirs + off * 3 : nullptr;
  o.radii = r.radii + off;
  o.near = r.near + off;
  o.far = r.far + off;
  o.num_rays = count;
  return o;
}

// Scratch layout for one chunk of R rays on the fp32 path.
struct Fp32Scratch {
  float *enc, *h0, *h1, *venc, *c0, *c1, *raw_rgb, *raw_density, *t[2], *w[2];
  size_t bytes;
};

Fp32Scratch carve_fp32(const mipnerf_b200_config* c, const Dims& d, int64_t rays, void* base,
                       bool mlp_only = false) {
  Fp32Scratch s{};
  const size_t m = (size_t)rays * c->num_samples;
  Carver cv{base};
  s.h0 = cv.floats(m * c->net_width);
  s.h1 = cv.floats(m * c->net_width);
  s.c0 = cv.floats(m * c->net_width_condition);
  s.c1 = cv.floats(m * c->net_width_condition);
  if (!mlp_only) {
    s.enc = cv.floats(m * d.xyz_dim);
    s.venc = cv.floats((size_t)rays * d.view_dim);
    s.raw_rgb = cv.floats(m * 3);
    s.raw_density = cv.floats(m);
    for (int i = 0; i < 2; ++i) {
      s.t[i] = cv.floats((size_t)rays * (c->num_samples + 1));
      s.w[i] = cv.floats(m);
    }
  }
  s.bytes = cv.off;
  return s;
}

// The trunk on the fp32 path (models/mip_nerf.py:93-97): x [m, xyz_dim] -> *out (h0 or h1), [m, net_width].
int trunk_fp32(const mipnerf_b200_config* c, const Dims& d, const mipnerf_b200_weights* w, const float* x, int64_t m,
               float* h0, float* h1, const float** out_h, cudaStream_t st) {
  const float* cur = x;
  int cur_k = d.xyz_dim;
  bool concat = false;
  for (int i = 0; i < c->net_depth; ++i) {
    const mipnerf_b200_linear& l = w->linears[i];
    float* out = (i & 1) ? h1 : h0;
    CUDA_TRY(mipnerf::launch_linear_f32(cur, cur_k, cur_k, concat ? x : nullptr, d.xyz_dim,
                                        concat ? d.xyz_dim : 0, 1, l.weight, l.bias, out, c->net_width, m,
                                        c->net_width, 1, st));
    cur = out;
    cur_k = c->net_width;
    concat = (i % c->skip_index == 0 && i > 0);  // models/mip_nerf.py:96-97
  }
  *out_h = cur;
  return MIPNERF_B200_OK;
}

// MLP.forward on the fp32 path (models/mip_nerf.py:75-111).
int mlp_forward_fp32(const mipnerf_b200_config* c, const Dims& d, const mipnerf_b200_weights* w,
                     const float* x, const float* venc, int64_t rays, int n, const Fp32Scratch& s,
                     float* raw_rgb, float* raw_density, cudaStream_t st) {
  const int64_t m = rays * n;
  const float* cur;
  int rc;
  if ((rc = trunk_fp32(c, d, w, x, m, s.h0, s.h1, &cur, st))) return rc;
  const int cur_k = c->net_width;
  const mipnerf_b200_linear& dl = w->linears[c->net_depth];
  CUDA_TRY(mipnerf::launch_linear_f32(cur, cur_k, cur_k, nullptr, 0, 0, 1, dl.weight, dl.bias, raw_density,
                                      1, m, 1, 0, st));
  const float* feat = cur;
  int feat_k = cur_k;
  if (c->use_viewdirs) {
    const mipnerf_b200_linear& el = w->linears[c->net_depth + 1];
    float* bott = (cur == s.h0) ? s.h1 : s.h0;
    CUDA_TRY(mipnerf::launch_linear_f32(cur, cur_k, cur_k, nullptr, 0, 0, 1, el.weight, el.bias, bott,
                                        c->net_width, m, c->net_width, 0, st));
    feat = bott;
    feat_k = c->net_width;
    for (int j = 0; j < c->net_depth_condition; ++j) {  // check_config: at least one
      const mipnerf_b200_linear& vl = w->linears[c->net_depth + 2 + j];
      float* out = (j & 1) ? s.c1 : s.c0;
      CUDA_TRY(mipnerf::launch_linear_f32(feat, feat_k, feat_k, j == 0 ? venc : nullptr, d.view_dim,
                                          j == 0 ? d.view_dim : 0, n, vl.weight, vl.bias, out,
                                          c->net_width_condition, m, c->net_width_condition, 1, st));
      feat = out;
      feat_k = c->net_width_condition;
    }
  }
  const mipnerf_b200_linear& cl = w->linears[d.n_lin - 1];
  CUDA_TRY(mipnerf::launch_linear_f32(feat, feat_k, feat_k, nullptr, 0, 0, 1, cl.weight, cl.bias, raw_rgb, 3,
                                      m, 3, 0, st));
  return MIPNERF_B200_OK;
}

}  // namespace

extern "C" {

const char* mipnerf_b200_last_error(void) { return g_last_error.c_str(); }
int mipnerf_b200_abi_version(void) { return MIPNERF_B200_ABI_VERSION; }

size_t mipnerf_b200_workspace_bytes(const mipnerf_b200_config* cfg, int64_t num_rays, int precision) {
  Dims d;
  if (check_config(cfg, &d) != MIPNERF_B200_OK || num_rays < 0) return 0;
  if (precision == MIPNERF_B200_FP32)
    return carve_fp32(cfg, d, std::clamp<int64_t>(num_rays, 1, kChunkRaysFp32), nullptr).bytes;
  return mipnerf::tc_workspace_bytes(cfg, num_rays, precision);
}

size_t mipnerf_b200_packed_weights_bytes(const mipnerf_b200_config* cfg, int precision) {
  Dims d;
  if (check_config(cfg, &d) != MIPNERF_B200_OK) return 0;
  return mipnerf::tc_packed_bytes(cfg, precision);
}

int mipnerf_b200_pack_weights(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w, int precision,
                              void* packed_out, size_t packed_bytes, void* stream) {
  Dims d;
  int rc;
  if ((rc = check_config(cfg, &d))) return rc;
  if ((rc = check_weights(cfg, d, w))) return rc;
  if (!packed_out) return fail(MIPNERF_B200_EINVAL, "packed_out is NULL");
  const size_t need = mipnerf::tc_packed_bytes(cfg, precision);
  if (need == 0)
    return fail(MIPNERF_B200_EUNSUPPORTED, "no tensor-core kernel for this MLP shape / precision %d", precision);
  if (packed_bytes < need)
    return fail(MIPNERF_B200_EWORKSPACE, "packed buffer %zu < %zu bytes", packed_bytes, need);
  cudaError_t e = mipnerf::tc_pack_weights(cfg, w, precision, packed_out, (cudaStream_t)stream);
  if (e != cudaSuccess) return fail(MIPNERF_B200_ECUDA, "pack_weights: %s", cudaGetErrorString(e));
  return MIPNERF_B200_OK;
}

// randomized with density_noise > 0 (models/mip_nerf.py:232-233): the injected-noise entry points need the normals too
// (outs[l - first] is level l's output)
static int check_density_normals(const mipnerf_b200_config* cfg, int randomized, const mipnerf_b200_rng* rng,
                                 const mipnerf_b200_level_out* outs, int64_t num_rays, int first = 0) {
  if (!randomized || !(cfg->density_noise > 0.f) || rng || num_rays == 0) return MIPNERF_B200_OK;
  for (int l = first; l < cfg->num_levels; ++l)
    if (!outs[l - first].density_normal)
      return fail(MIPNERF_B200_EINVAL,
                  "randomized=1 with density_noise > 0 needs outs[%d].density_normal (injected noise) or the _rng "
                  "entry point (in-kernel Philox)", l - first);
  return MIPNERF_B200_OK;
}

// The level loop of mipnerf_b200_forward(_rng).  With `proposal` = {t_prev, w_prev} (mipnerf_b200_forward_proposed) it
// starts at level 1 with those in place of level 0's outputs, and outs[l - 1] is level l's output.
static int forward_impl(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w,
                        const mipnerf_b200_rays* rays, int randomized, const float* t_rand,
                        const float* u_jitter, const mipnerf_b200_rng* rng, int white_bkgd, int precision,
                        mipnerf_b200_level_out* outs, void* workspace, size_t workspace_bytes, void* stream,
                        const float* const* proposal = nullptr) {
  Dims d;
  int rc;
  if ((rc = check_config(cfg, &d))) return rc;
  const int first = proposal ? 1 : 0;
  if (proposal && cfg->num_levels < 2)
    return fail(MIPNERF_B200_EINVAL, "num_levels=%d: a forward from proposal weights needs >= 2 levels",
                cfg->num_levels);
  if ((rc = check_weights(cfg, d, w))) return rc;
  if ((rc = check_rays(rays))) return rc;
  if (!outs) return fail(MIPNERF_B200_EINVAL, "outs is NULL");
  if (proposal && rays->num_rays > 0 && (!proposal[0] || !proposal[1]))
    return fail(MIPNERF_B200_EINVAL, "t_prev / w_prev is NULL");
  if (cfg->use_viewdirs && rays->num_rays > 0 && !rays->viewdirs)
    return fail(MIPNERF_B200_EINVAL, "use_viewdirs but rays.viewdirs is NULL");
  if (randomized && !rng && ((!proposal && !t_rand) || (cfg->num_levels > 1 && !u_jitter)))
    return fail(MIPNERF_B200_EINVAL, proposal ? "randomized=1 needs u_jitter (injected noise) or the _rng entry point "
                                                "(in-kernel Philox)"
                                              : "randomized=1 needs t_rand and u_jitter (injected noise) or the _rng "
                                                "entry point (in-kernel Philox)");
  for (int l = first; l < cfg->num_levels; ++l)
    if (rays->num_rays > 0 && (!outs[l - first].comp_rgb || !outs[l - first].distance || !outs[l - first].acc))
      return fail(MIPNERF_B200_EINVAL, "outs[%d] misses comp_rgb/distance/acc", l - first);
  if ((rc = check_density_normals(cfg, randomized, rng, outs, rays->num_rays, first))) return rc;
  const size_t need = mipnerf_b200_workspace_bytes(cfg, rays->num_rays, precision);
  if (rays->num_rays > 0 && (!workspace || workspace_bytes < need))
    return fail(MIPNERF_B200_EWORKSPACE, "workspace %zu < %zu bytes", workspace_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  const int n = cfg->num_samples;
  const float rgb_scale = mipnerf::rgb_scale_of(cfg);

  if (precision != MIPNERF_B200_FP32) {
    if ((rc = check_tc(cfg, w, precision, "forward"))) return rc;
    cudaError_t e = mipnerf::tc_forward(cfg, w, rays, randomized, t_rand, u_jitter, rng, white_bkgd, precision,
                                        outs, workspace, workspace_bytes, st, nullptr, 0, 0, proposal);
    if (e != cudaSuccess) return fail(MIPNERF_B200_ECUDA, "tc_forward: %s", cudaGetErrorString(e));
    return MIPNERF_B200_OK;
  }

  for (int64_t off = 0; off < rays->num_rays; off += kChunkRaysFp32) {
    const int64_t cnt = (rays->num_rays - off) < kChunkRaysFp32 ? (rays->num_rays - off) : kChunkRaysFp32;
    const mipnerf_b200_rays rc_ = offset_rays(*rays, off, cnt);
    const Fp32Scratch s = carve_fp32(cfg, d, cnt, workspace);
    if (cfg->use_viewdirs)
      CUDA_TRY(mipnerf::launch_pos_enc(rc_.viewdirs, s.venc, cnt, 0, cfg->deg_view, 1, st));
    const float* t_prev = proposal ? proposal[0] + off * (n + 1) : nullptr;
    const float* w_prev = proposal ? proposal[1] + off * n : nullptr;
    for (int l = first; l < cfg->num_levels; ++l) {
      const mipnerf_b200_level_out& o = outs[l - first];
      float* t_cur = o.t_samples ? o.t_samples + off * (n + 1) : s.t[l & 1];
      float* w_cur = o.weights ? o.weights + off * n : s.w[l & 1];
      if (l == 0) {
        CUDA_TRY(mipnerf::launch_coarse_t(rc_.near, rc_.far, mipnerf::level_draws(randomized, t_rand, rng, off, 0, n + 1),
                                          t_cur, cnt, n, randomized, cfg->disparity, st));
      } else {
        CUDA_TRY(mipnerf::launch_resample(t_prev, w_prev, mipnerf::level_draws(randomized, u_jitter, rng, off, 1 + l, n + 1),
                                          t_cur, o.inds ? o.inds + off * (n + 1) : nullptr, cnt, n, n + 1,
                                          randomized, 1, cfg->resample_padding, st));
      }
      CUDA_TRY(mipnerf::launch_ipe_from_t(rc_.origins, rc_.directions, rc_.radii, t_cur, s.enc, cnt, n,
                                          cfg->min_deg_point, cfg->max_deg_point, cfg->disable_integration,
                                          st));
      if ((rc = mlp_forward_fp32(cfg, d, w, s.enc, cfg->use_viewdirs ? s.venc : nullptr, cnt, n, s, s.raw_rgb,
                                 s.raw_density, st)))
        return rc;
      CUDA_TRY(mipnerf::launch_add_density_noise(                                   // models/mip_nerf.py:232-233
          s.raw_density, mipnerf::density_noise_draws(cfg, randomized, o.density_normal, rng, off, l, n), cnt, n, st));
      CUDA_TRY(mipnerf::launch_composite(s.raw_rgb, s.raw_density, t_cur, rc_.directions,
                                         o.comp_rgb + off * 3, o.distance + off, o.acc + off,
                                         w_cur, cnt, n, white_bkgd, 1, cfg->density_bias, rgb_scale,
                                         cfg->rgb_padding, st));
      t_prev = t_cur;
      w_prev = w_cur;
    }
  }
  return MIPNERF_B200_OK;
}

int mipnerf_b200_forward(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w,
                         const mipnerf_b200_rays* rays, int randomized, const float* t_rand,
                         const float* u_jitter, int white_bkgd, int precision, mipnerf_b200_level_out* outs,
                         void* workspace, size_t workspace_bytes, void* stream) {
  return forward_impl(cfg, w, rays, randomized, t_rand, u_jitter, nullptr, white_bkgd, precision, outs, workspace,
                      workspace_bytes, stream);
}

int mipnerf_b200_forward_rng(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w,
                             const mipnerf_b200_rays* rays, const mipnerf_b200_rng* rng, int white_bkgd,
                             int precision, mipnerf_b200_level_out* outs, void* workspace,
                             size_t workspace_bytes, void* stream) {
  if (!rng) return fail(MIPNERF_B200_EINVAL, "rng is NULL");
  return forward_impl(cfg, w, rays, 1, nullptr, nullptr, rng, white_bkgd, precision, outs, workspace,
                      workspace_bytes, stream);
}

int mipnerf_b200_forward_proposed(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w,
                                  const mipnerf_b200_rays* rays, const float* t_prev, const float* w_prev,
                                  int randomized, const float* u_jitter, int white_bkgd, int precision,
                                  mipnerf_b200_level_out* outs, void* workspace, size_t workspace_bytes,
                                  void* stream) {
  const float* const proposal[2] = {t_prev, w_prev};
  return forward_impl(cfg, w, rays, randomized, nullptr, u_jitter, nullptr, white_bkgd, precision, outs, workspace,
                      workspace_bytes, stream, proposal);
}

int mipnerf_b200_forward_proposed_rng(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w,
                                      const mipnerf_b200_rays* rays, const float* t_prev, const float* w_prev,
                                      const mipnerf_b200_rng* rng, int white_bkgd, int precision,
                                      mipnerf_b200_level_out* outs, void* workspace, size_t workspace_bytes,
                                      void* stream) {
  if (!rng) return fail(MIPNERF_B200_EINVAL, "rng is NULL");
  const float* const proposal[2] = {t_prev, w_prev};
  return forward_impl(cfg, w, rays, 1, nullptr, nullptr, rng, white_bkgd, precision, outs, workspace,
                      workspace_bytes, stream, proposal);
}

int mipnerf_b200_philox_normal(const mipnerf_b200_rng* rng, int level, int64_t num_rays, int num_samples, float* out,
                               void* stream) {
  if (!rng || level < 0 || level >= 64 || num_rays < 0 || num_samples < 1 || (num_rays > 0 && !out))
    return fail(MIPNERF_B200_EINVAL, "bad argument");
  const mipnerf::Draws d = mipnerf::draws_philox(rng->seed, rng->offset, 0, mipnerf::kDensityNoiseStream + level, 1.f);
  CUDA_TRY(mipnerf::launch_philox_normal(d, out, num_rays, num_samples, (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

int mipnerf_b200_philox_uniform(const mipnerf_b200_rng* rng, int stream_id, int64_t num_rays, int ncols, float* out,
                                void* stream) {
  if (!rng || stream_id < 0 || num_rays < 0 || ncols < 1 || (num_rays > 0 && !out))
    return fail(MIPNERF_B200_EINVAL, "bad argument");
  const mipnerf::Draws d = mipnerf::level_draws(1, nullptr, rng, 0, stream_id, ncols);
  CUDA_TRY(mipnerf::launch_philox_uniform(d, out, num_rays, ncols, (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

// ---- training step -------------------------------------------------------------------------------
namespace {
constexpr int kMaxTrainDepth = 16;
struct TrainScratch {
  float *enc, *venc, *h[kMaxTrainDepth], *bott, *v, *raw_rgb, *raw_density;
  float *d_a, *d_b, *d_v, *d_raw_rgb, *d_raw_density, *part, *t[2], *w[2];
  float* vrow;      // tensor-core mode: per-ray view-direction bias [rays, net_width_condition]
  uint8_t* images;  // tensor-core mode: packed B operands (kTrainImages x kTrainImageBytes)
  size_t bytes;
};
constexpr int kTrainImages = 2 * kMaxTrainDepth + 8;
constexpr size_t kTrainImageBytes = 131072;  // 256 x 256 x 16 bit

// Per-layer scratch of m rows: a training chunk of `rays` rays, or (rays = 0) the fp32 query backward's points, one view
// encoding each.  The images come last: they are packed once per call into the first chunk's carve.
TrainScratch carve_train(const mipnerf_b200_config* c, const Dims& d, size_t m, int64_t rays, bool radiance, void* base) {
  TrainScratch s{};
  Carver cv{base};
  s.enc = cv.floats(m * d.xyz_dim);
  for (int i = 0; i < c->net_depth; ++i) s.h[i] = cv.floats(m * c->net_width);
  s.raw_density = cv.floats(m);
  s.d_a = cv.floats(m * c->net_width);
  s.d_b = cv.floats(m * c->net_width);
  s.d_raw_density = cv.floats(m);
  s.part = cv.floats(wgrad_part_floats(c, d));
  if (radiance) {
    s.venc = cv.floats((rays ? rays : m) * d.view_dim);
    s.bott = cv.floats(m * c->net_width);
    s.v = cv.floats(m * c->net_width_condition);
    s.raw_rgb = cv.floats(m * 3);
    s.d_v = cv.floats(m * c->net_width_condition);
    s.d_raw_rgb = cv.floats(m * 3);
  }
  if (rays) {
    for (int i = 0; i < 2; ++i) {
      s.t[i] = cv.floats((size_t)rays * (c->num_samples + 1));
      s.w[i] = cv.floats(m);
    }
    s.vrow = cv.floats((size_t)rays * c->net_width_condition);
    s.images = cv.bytes(kTrainImages * kTrainImageBytes);
  }
  s.bytes = cv.off;
  return s;
}

// The chunk-invariant head of the fused backward drivers' workspace: the wgrad partials, `image_slots` slots for the
// dgrad chain's B images and the level kernels' packed weights.  Carved first: the weights are packed once per call
// into the first chunk's carve and read by every chunk, so no buffer of a shorter last chunk may move onto them.
struct FusedHead {
  float* part;
  uint8_t *images, *packed;
};

FusedHead carve_fused_head(Carver& cv, const mipnerf_b200_config* c, const Dims& d, int precision, int image_slots) {
  FusedHead h;
  h.part = cv.floats(wgrad_part_floats(c, d));
  h.images = cv.bytes((size_t)image_slots * kTrainImageBytes);
  h.packed = cv.bytes(mipnerf::tc_packed_bytes(c, precision));
  return h;
}

// Operands of the tile-image backward chain for `rows` rows in whole 128-row tiles: the level kernel's dump (act
// [9][tiles][64 KB]: h_0..h_7, bottleneck; v [tiles][32 KB]: view-layer output) and the head's wgrad partials, set by
// the caller; the IPE features enc16 [tiles][32 KB], the fp32 view encoding (one row per view_div rows), d raw_rgb /
// d raw_density, the ReLU sign mask relu_bits [tiles * 128][32 B] and the gradient images.  bf16x3: each image, its lo.
struct TileChainOps {
  uint8_t *act, *v;
  float* part;
  uint8_t* enc16;
  float* venc;
  int view_div;
  float *d_raw_rgb, *d_raw_density;
  uint8_t *d_v, *d_a, *d_b, *relu_bits;
  int64_t rows, tiles;
};

// The chain's own operands for `rows` rows; without `radiance` (a density query) no view encoding, d raw_rgb or d_v.
TileChainOps carve_tile_chain(Carver& cv, const Dims& d, int precision, int64_t rows, int view_div, bool radiance) {
  TileChainOps o{};
  o.rows = rows;
  o.tiles = (rows + 127) / 128;
  o.view_div = view_div;
  const size_t x = mipnerf::is_x3(precision) ? 2 : 1, m = o.tiles * 128;  // tile images per operand: hi (, lo)
  if (radiance) {
    o.venc = cv.floats(m / view_div * d.view_dim);
    o.d_raw_rgb = cv.floats(m * 3);
    o.d_v = cv.bytes(x * o.tiles * 32768);
  }
  o.d_raw_density = cv.floats(m);
  o.enc16 = cv.bytes(x * o.tiles * 32768);
  o.relu_bits = cv.bytes(m * 32);
  o.d_a = cv.bytes(x * o.tiles * 65536);
  o.d_b = cv.bytes(x * o.tiles * 65536);
  return o;
}

// Scratch of the fused tensor-core training step (forward = the level kernels with the activation dump, backward on
// 16-bit tile images, train_t16.cu), one tile per ray.  Overlays the same workspace as TrainScratch.
struct FusedScratch {
  FusedHead head;
  // bf16x3: every tile image below is followed by its lo image of the same size (act: [2][9][rays][64 KB])
  uint8_t *act[2], *v[2];              // forward dump per level: [9][rays][64 KB], [rays][32 KB]
  float *raw_rgb[2], *raw_density[2], *t[2], *w[2];  // raw heads, fenceposts and weights per level
  TileChainOps chain;
  uint8_t* tcws;
  size_t tcws_bytes, bytes;
};

FusedScratch carve_fused(const mipnerf_b200_config* c, const Dims& d, int64_t rays, int precision, void* base) {
  FusedScratch s{};
  const size_t m = (size_t)rays * c->num_samples;
  Carver cv{base};
  const size_t x = precision == MIPNERF_B200_BF16X3 ? 2 : 1;  // tile images per operand: hi (, lo)
  // bf16x3: the image slots hold the lo images of the dgrad B operands as well
  s.head = carve_fused_head(cv, c, d, precision, kTrainImages);
  for (int l = 0; l < 2; ++l) {
    s.act[l] = cv.bytes(x * 9 * rays * 65536);
    s.v[l] = cv.bytes(x * rays * 32768);
    s.raw_rgb[l] = cv.floats(m * 3);
    s.raw_density[l] = cv.floats(m);
    s.t[l] = cv.floats((size_t)rays * (c->num_samples + 1));
    s.w[l] = cv.floats(m);
  }
  cv.floats(m * d.xyz_dim);  // unread; keeps the size mipnerf_b200_train_workspace_bytes_for has always returned
  s.chain = carve_tile_chain(cv, d, precision, m, c->num_samples, true);
  s.chain.part = s.head.part;
  s.tcws_bytes = mipnerf::tc_workspace_bytes(c, rays, precision);
  s.tcws = cv.bytes(s.tcws_bytes);
  s.bytes = cv.off;
  return s;
}

// The fused step needs the level kernels' architecture (8 x 256 trunk, ...) with one 128-row tile per ray (its
// activation dump is one tile per ray) and at most two levels; other shapes that train_tc_supported accepts, 256
// samples included, take the per-layer tensor-core path.
bool train_fused_supported(const mipnerf_b200_config* c, int precision) {
  return (precision == MIPNERF_B200_BF16 || precision == MIPNERF_B200_FP16 || precision == MIPNERF_B200_BF16X3) &&
         mipnerf::tc_supported(c, precision) &&
         c->num_samples == 128 &&
         mipnerf::tc_default_degrees(c) &&  // the backward's tile images carry the full 96 / 27 encodings
         c->num_levels <= 2 && c->net_depth == 8;
}

int check_train_config(const mipnerf_b200_config* c) {
  if (!c->use_viewdirs || c->net_depth_condition != 1)
    return fail(MIPNERF_B200_EUNSUPPORTED, "training: use_viewdirs=True with one view layer only");
  if (c->net_depth > kMaxTrainDepth)
    return fail(MIPNERF_B200_EUNSUPPORTED, "training: net_depth <= %d", kMaxTrainDepth);
  return MIPNERF_B200_OK;
}

inline bool takes_skip(const mipnerf_b200_config* c, int layer) {  // models/mip_nerf.py:40-42
  return layer > 1 && (layer - 1) % c->skip_index == 0;
}

// B operands of the training GEMMs, packed once per call (the weights change every optimiser step) into
// kTrainImageBytes slots at `base`; a null base only counts the slots.  bwd[i] = W_i[:, :256]^T for i = 1 .. depth + 1
// (depth / depth + 1: the bottleneck and the view layer), in bf16x3 with its lo image bwd_lo[i] kMaxTrainDepth + 2
// slots further on.  The per-layer path (`fwd`) also takes fwd[i] = W_i[:, :k_main] and skip[i] = W_i[:, 256:352]
// (fwd[depth] / fwd[depth + 1]: the bottleneck, the view layer's bottleneck columns).
struct LayerImages {
  const uint8_t *fwd[kMaxTrainDepth + 2], *skip[kMaxTrainDepth], *bwd[kMaxTrainDepth + 2], *bwd_lo[kMaxTrainDepth + 2];
  int slots;  // slots taken, lo images not counted
};

cudaError_t pack_layer_images(const mipnerf_b200_config* c, const Dims& d, const mipnerf_b200_weights* w, int precision,
                              bool fwd, uint8_t* base, LayerImages* im, cudaStream_t st) {
  const int depth = c->net_depth, W = c->net_width, Wc = c->net_width_condition;
  const int fmt = mipnerf::fmt_of(precision);
  const bool x3 = mipnerf::is_x3(precision);
  *im = LayerImages{};
  // columns [off, off + kk) of linear li as an nn x kk image (transposed: B[k][n] = W[n][k]) into the next slot
  auto pack = [&](int li, int off, int transposed, int nn, int kk, const uint8_t** out,
                  const uint8_t** out_lo = nullptr) {
    const size_t slot = im->slots++;
    if (!base) return cudaSuccess;
    const mipnerf_b200_linear& l = w->linears[li];
    uint8_t* dst = base + slot * kTrainImageBytes;
    *out = dst;
    if (out_lo) {
      uint8_t* lo = base + (slot + kMaxTrainDepth + 2) * kTrainImageBytes;
      *out_lo = lo;
      cudaError_t e = mipnerf::launch_pack_linear_image(l.weight, l.in_features, off, transposed, lo, nn, kk, fmt, st, 1);
      if (e != cudaSuccess) return e;
    }
    return mipnerf::launch_pack_linear_image(l.weight, l.in_features, off, transposed, dst, nn, kk, fmt, st);
  };
  auto bwd = [&](int li, int i, int kk) { return pack(li, 0, 1, W, kk, &im->bwd[i], x3 ? &im->bwd_lo[i] : nullptr); };
  cudaError_t e;
  for (int i = 0; i < depth; ++i) {
    if (fwd && (e = pack(i, 0, 0, W, i == 0 ? d.xyz_dim : W, &im->fwd[i]))) return e;
    if (fwd && takes_skip(c, i) && (e = pack(i, W, 0, W, d.xyz_dim, &im->skip[i]))) return e;
    if (i > 0 && (e = bwd(i, i, W))) return e;
  }
  if (fwd && (e = pack(depth + 1, 0, 0, W, W, &im->fwd[depth]))) return e;  // bottleneck
  if ((e = bwd(depth + 1, depth, W))) return e;
  if (fwd && (e = pack(depth + 2, 0, 0, Wc, W, &im->fwd[depth + 1]))) return e;  // view layer, bottleneck columns
  return bwd(depth + 2, depth + 1, Wc);
}

// Tensor-core GEMMs of the training step exist for the default widths only (linear_tc.cu), and the per-layer step's
// images must fit the kTrainImages slots carved from the workspace.
bool train_tc_supported(const mipnerf_b200_config* c, const Dims& d) {
  if (!(c->net_width == 256 && c->net_width_condition == 128 && d.xyz_dim == 96 && d.view_dim == 27 &&
        c->net_depth <= kMaxTrainDepth))
    return false;
  LayerImages im;
  pack_layer_images(c, d, nullptr, MIPNERF_B200_BF16, true, nullptr, &im, nullptr);
  return im.slots <= kTrainImages;
}

// The fused drivers' prologue, once per call (the weights change every optimiser step): the level kernels' image and
// the dgrad chain's transposed B operands (*im) packed into the head `h`; *wl: the weights with that packed image.
int pack_fused_weights(const mipnerf_b200_config* c, const Dims& d, const mipnerf_b200_weights* w, int precision,
                       const FusedHead& h, mipnerf_b200_weights* wl, LayerImages* im, cudaStream_t st) {
  *wl = *w;
  wl->packed = h.packed, wl->packed_precision = precision, wl->packed_bytes = mipnerf::tc_packed_bytes(c, precision);
  CUDA_TRY(mipnerf::tc_pack_weights(c, w, precision, h.packed, st));
  CUDA_TRY(pack_layer_images(c, d, w, precision, false, h.images, im, st));
  return MIPNERF_B200_OK;
}

// The gradient outputs of a backward pass: touched[i] (grads[i] already holds a sum to add to) starts at `accumulate`,
// the backward chains set it for every linear they reach, and every gradient still untouched after them (no rays or
// points, or the heads a density query does not reach) is written as exact zeros.
int zero_untouched(const Dims& d, const mipnerf_b200_weights* w, const mipnerf_b200_linear_grad* grads,
                   const bool* touched, cudaStream_t st) {
  for (int i = 0; i < d.n_lin; ++i)
    if (!touched[i]) {
      const mipnerf_b200_linear& l = w->linears[i];
      CUDA_TRY(cudaMemsetAsync(grads[i].weight_grad, 0, sizeof(float) * l.in_features * l.out_features, st));
      CUDA_TRY(cudaMemsetAsync(grads[i].bias_grad, 0, sizeof(float) * l.out_features, st));
    }
  return MIPNERF_B200_OK;
}

int check_grads(const Dims& d, const mipnerf_b200_linear_grad* grads, int num_grads) {
  if (num_grads != d.n_lin) return fail(MIPNERF_B200_EINVAL, "expected %d gradient pairs, got %d", d.n_lin, num_grads);
  for (int i = 0; i < d.n_lin; ++i)
    if (!grads[i].weight_grad || !grads[i].bias_grad) return fail(MIPNERF_B200_EINVAL, "grads[%d] has a NULL tensor", i);
  return MIPNERF_B200_OK;
}

// The precisions a backward pass from arbitrary cotangents takes: FP32 and BF16.  `what` names the entry point.
int check_cotangent_precision(int precision, const char* what) {
  if (precision == MIPNERF_B200_FP16)
    return fail(MIPNERF_B200_EUNSUPPORTED,
                "%s: FP16's fixed gradient scale is sized for the training loss and arbitrary cotangents can overflow "
                "or underflow it; use BF16 (fp32 range) or FP32", what);
  if (mipnerf::is_x3(precision))
    return fail(MIPNERF_B200_EUNSUPPORTED, "%s: the split-operand precisions are forward-only; use FP32 or BF16", what);
  return MIPNERF_B200_OK;
}

// The factor the training loss's gradient is emitted with.  fp16 gradients underflow: d loss / d activation is ~1e-7 ..
// 1e-4 per sample (the loss is a mean over the batch), below fp16's 6e-5 normal range.  The backward pass is linear in
// d loss / d raw, so render_backward emits it scaled by 2^10 (it is bounded by 2/3 per sample: no overflow), every
// 16-bit gradient operand carries that factor, and the fixed-order reduction of the wgrad partials takes it out again
// (without it, measured at depth 16, the per-layer step lost 62 % of layers.0's gradient against the fp32 step).  bf16
// has fp32's range: scale 1.
float grad_scale_of(int precision) { return precision == MIPNERF_B200_FP16 ? 1024.f : 1.f; }

// Where level l of the chunk [off, off + cnt) of a training step writes: its fenceposts and weights to the caller's
// outs[l] or the scratch t / w, its pixels to outs[l] or, with given fenceposts (whose recomputed pixels nobody reads),
// into the unused fencepost scratch t; inds and density_normal from the chunk's first ray.
mipnerf_b200_level_out chunk_level_out(const mipnerf_b200_level_out& o, int64_t off, int64_t cnt, int n, bool given_t,
                                       float* t, float* w) {
  mipnerf_b200_level_out r;
  r.comp_rgb = given_t ? t : o.comp_rgb + off * 3;
  r.distance = given_t ? t + 3 * cnt : o.distance + off;
  r.acc = given_t ? t + 4 * cnt : o.acc + off;
  r.weights = o.weights ? o.weights + off * n : w;
  r.t_samples = o.t_samples ? o.t_samples + off * (n + 1) : t;
  r.inds = o.inds ? o.inds + off * (n + 1) : nullptr;
  r.density_normal = o.density_normal ? o.density_normal + off * n : nullptr;
  return r;
}

// MLP.forward of m rows with every activation the backward needs kept in `s` (models/mip_nerf.py:75-111): the trunk
// s.h[] from s.enc and the density head into s.raw_density; unless `density_only`, the bottleneck s.bott, the view layer
// s.v (view encoding s.venc, or on the tensor cores its bias s.vrow, one row per `view_div` rows) and the colour head
// into s.raw_rgb.  tc: the 128- and 256-wide layers on the tensor cores (images `im`), the heads in fp32.
int mlp_forward_kept(const mipnerf_b200_config* c, const Dims& d, const mipnerf_b200_weights* w, bool tc, int precision,
                     const LayerImages& im, const TrainScratch& s, int64_t m, int view_div, bool density_only,
                     cudaStream_t st) {
  const int depth = c->net_depth, W = c->net_width, Wc = c->net_width_condition;
  for (int i = 0; i < depth; ++i) {
    const mipnerf_b200_linear& li = w->linears[i];
    const bool skip = takes_skip(c, i);
    const float* in = i == 0 ? s.enc : s.h[i - 1];
    const int k1 = i == 0 ? d.xyz_dim : W;
    if (!tc) {
      CUDA_TRY(mipnerf::launch_linear_f32(in, k1, k1, skip ? s.enc : nullptr, d.xyz_dim, skip ? d.xyz_dim : 0, 1,
                                          li.weight, li.bias, s.h[i], W, m, W, 1, st));
    } else if (!skip) {
      CUDA_TRY(mipnerf::launch_linear_tc(in, k1, im.fwd[i], s.h[i], W, m, W, k1, li.bias, nullptr, 1, nullptr, nullptr,
                                         nullptr, nullptr, 1, precision, st));
    } else {  // cat([h, enc]) as two K passes: the second adds the first's partial sums, the bias and the ReLU
      CUDA_TRY(mipnerf::launch_linear_tc(in, k1, im.fwd[i], s.h[i], W, m, W, k1, nullptr, nullptr, 1, nullptr, nullptr,
                                         nullptr, nullptr, 0, precision, st));
      CUDA_TRY(mipnerf::launch_linear_tc(s.enc, d.xyz_dim, im.skip[i], s.h[i], W, m, W, d.xyz_dim, li.bias, nullptr, 1,
                                         s.h[i], nullptr, nullptr, nullptr, 1, precision, st));
    }
  }
  const float* h_last = s.h[depth - 1];
  const mipnerf_b200_linear& dl = w->linears[depth];
  const mipnerf_b200_linear& el = w->linears[depth + 1];
  const mipnerf_b200_linear& vl = w->linears[depth + 2];
  const mipnerf_b200_linear& cl = w->linears[d.n_lin - 1];
  CUDA_TRY(mipnerf::launch_linear_f32(h_last, W, W, nullptr, 0, 0, 1, dl.weight, dl.bias, s.raw_density, 1, m, 1, 0, st));
  if (density_only) return MIPNERF_B200_OK;
  if (!tc) {
    CUDA_TRY(mipnerf::launch_linear_f32(h_last, W, W, nullptr, 0, 0, 1, el.weight, el.bias, s.bott, W, m, W, 0, st));
    CUDA_TRY(mipnerf::launch_linear_f32(s.bott, W, W, s.venc, d.view_dim, d.view_dim, view_div, vl.weight, vl.bias, s.v,
                                        Wc, m, Wc, 1, st));
  } else {
    CUDA_TRY(mipnerf::launch_linear_tc(h_last, W, im.fwd[depth], s.bott, W, m, W, W, el.bias, nullptr, 1, nullptr,
                                       nullptr, nullptr, nullptr, 0, precision, st));
    CUDA_TRY(mipnerf::launch_linear_tc(s.bott, W, im.fwd[depth + 1], s.v, Wc, m, Wc, W, nullptr, s.vrow, view_div,
                                       nullptr, nullptr, nullptr, nullptr, 1, precision, st));
  }
  CUDA_TRY(mipnerf::launch_linear_f32(s.v, Wc, Wc, nullptr, 0, 0, 1, cl.weight, cl.bias, s.raw_rgb, 3, m, 3, 0, st));
  return MIPNERF_B200_OK;
}

// The per-layer backward chain of m rows from d raw_rgb / d raw_density (s.d_raw_rgb, s.d_raw_density) through the
// colour head, view layer, bottleneck + density head and trunk into `grads`, on the activations mlp_forward_kept left in
// `s` (same `tc`, `view_div`, `density_only`).  With density_only it starts at the density head: d h_last is then the
// rank-1 term d_raw_density . W_density alone, which dgrad_f32 with an empty dY computes without a GEMM.  touched[i]:
// grads[i] already holds a sum to add to.  inv_gscale takes the fp16 step's gradient scale out of the wgrad sums.
int mlp_backward_chain(const mipnerf_b200_config* c, const Dims& d, const mipnerf_b200_weights* w, bool tc,
                       int precision, const LayerImages& im, const TrainScratch& s, int64_t m, int view_div,
                       bool density_only, const mipnerf_b200_linear_grad* grads, bool* touched, cudaStream_t st,
                       float inv_gscale = 1.f) {
  const int depth = c->net_depth, W = c->net_width, Wc = c->net_width_condition;
  // tensor-core mode: the wgrad partials of the 128- and 256-wide layers on the tensor cores as well (dy comes from
  // the 256-byte-aligned workspace carves, and an x2 always follows k1 = 256 columns); the two heads on fp32 FFMA
  auto wgrad = [&](int idx, const float* dy, const float* x1, int k1, const float* x2, int k2, int div) {
    const mipnerf_b200_linear& l = w->linears[idx];
    if (tc && mipnerf::wgrad_tc_shape_ok(l.out_features)) {  // tensor-core partials + same reduction
      int slices = 0;
      cudaError_t e2 = mipnerf::launch_wgrad_mn_partials({dy, l.out_features}, l.out_features, {x1, k1}, k1, {x2, k2},
                                                         k2, div, s.part, m, mipnerf::kWgradMaxSlices, precision,
                                                         &slices, st);
      if (e2 != cudaSuccess) return e2;
      e2 = mipnerf::launch_wgrad_reduce(s.part, slices, l.out_features, k1 + k2, grads[idx].weight_grad,
                                        grads[idx].bias_grad, touched[idx] ? 1 : 0, st, inv_gscale);
      touched[idx] = true;
      return e2;
    }
    cudaError_t e = mipnerf::launch_wgrad_f32(dy, l.out_features, x1, k1, k1, x2, k2, k2, div, s.part,
                                              grads[idx].weight_grad, grads[idx].bias_grad, touched[idx] ? 1 : 0,
                                              m, st, inv_gscale);
    touched[idx] = true;
    return e;
  };
  const float* h_last = s.h[depth - 1];
  const mipnerf_b200_linear& dl = w->linears[depth];
  const mipnerf_b200_linear& el = w->linears[depth + 1];
  const mipnerf_b200_linear& vl = w->linears[depth + 2];
  const mipnerf_b200_linear& cl = w->linears[d.n_lin - 1];
  if (density_only) {
    CUDA_TRY(wgrad(depth, s.d_raw_density, h_last, W, nullptr, 0, 1));
    CUDA_TRY(mipnerf::launch_dgrad_f32(nullptr, 0, el.weight, W, s.d_raw_density, dl.weight, h_last, s.d_b, m, W, st));
  } else {
    // colour head, view layer                                          (models/mip_nerf.py:106-110)
    CUDA_TRY(wgrad(d.n_lin - 1, s.d_raw_rgb, s.v, Wc, nullptr, 0, 1));
    CUDA_TRY(mipnerf::launch_color_dgrad(s.d_raw_rgb, cl.weight, s.v, s.d_v, m, Wc, st));
    CUDA_TRY(wgrad(depth + 2, s.d_v, s.bott, W, s.venc, d.view_dim, view_div));
    if (!tc)
      CUDA_TRY(mipnerf::launch_dgrad_f32(s.d_v, Wc, vl.weight, W + d.view_dim, nullptr, nullptr, nullptr, s.d_a, m, W,
                                         st));
    else
      CUDA_TRY(mipnerf::launch_linear_tc(s.d_v, Wc, im.bwd[depth + 1], s.d_a, W, m, W, Wc, nullptr, nullptr, 1, nullptr,
                                         nullptr, nullptr, nullptr, 0, precision, st));
    // bottleneck + density head share h_last                           (models/mip_nerf.py:98-101)
    CUDA_TRY(wgrad(depth + 1, s.d_a, h_last, W, nullptr, 0, 1));
    CUDA_TRY(wgrad(depth, s.d_raw_density, h_last, W, nullptr, 0, 1));
    if (!tc)
      CUDA_TRY(mipnerf::launch_dgrad_f32(s.d_a, W, el.weight, W, s.d_raw_density, dl.weight, h_last, s.d_b, m, W, st));
    else
      CUDA_TRY(mipnerf::launch_linear_tc(s.d_a, W, im.bwd[depth], s.d_b, W, m, W, W, nullptr, nullptr, 1, nullptr,
                                         s.d_raw_density, dl.weight, h_last, 0, precision, st));
  }
  // trunk                                                            (models/mip_nerf.py:93-97)
  float *cur = s.d_b, *other = s.d_a;
  for (int i = depth - 1; i >= 0; --i) {
    const bool skip = takes_skip(c, i);
    const float* in = i == 0 ? s.enc : s.h[i - 1];
    const int k1 = i == 0 ? d.xyz_dim : W;
    CUDA_TRY(wgrad(i, cur, in, k1, skip ? s.enc : nullptr, skip ? d.xyz_dim : 0, 1));
    if (i > 0) {
      if (!tc)
        CUDA_TRY(mipnerf::launch_dgrad_f32(cur, W, w->linears[i].weight, k1 + (skip ? d.xyz_dim : 0), nullptr, nullptr,
                                           s.h[i - 1], other, m, W, st));
      else
        CUDA_TRY(mipnerf::launch_linear_tc(cur, W, im.bwd[i], other, W, m, W, W, nullptr, nullptr, 1, nullptr, nullptr,
                                           nullptr, s.h[i - 1], 0, precision, st));
      float* tmp = cur;
      cur = other;
      other = tmp;
    }
  }
  return MIPNERF_B200_OK;
}

// Where the backward pass of a training driver starts: the loss of mipnerf_b200_loss, or cotangents of the rendered
// outputs (one entry per level).  Everything after the render backward only sees d raw_rgb / d raw_density.
struct GradSource {
  const mipnerf_b200_loss* loss;
  const mipnerf_b200_level_cotangent* cots;
};

// d raw_rgb / d raw_density of level l for the chunk [off, off + cnt) of a B-ray call.  `gscale` multiplies the loss
// gradient (the fp16 step's fixed scale, 1 otherwise).
cudaError_t launch_grad_source(const GradSource& g, const mipnerf_b200_config* c, int l, int64_t off, int64_t B,
                               int64_t cnt, const float* raw_rgb, const float* raw_dens, const float* t,
                               const float* dirs, int white_bkgd, float rgb_scale, float gscale, float* d_raw_rgb,
                               float* d_raw_dens, cudaStream_t st) {
  const int n = c->num_samples;
  if (g.cots) {
    const mipnerf_b200_level_cotangent& k = g.cots[l];
    const mipnerf::RenderCot cot{k.d_comp_rgb ? k.d_comp_rgb + off * 3 : nullptr,
                                 k.d_distance ? k.d_distance + off : nullptr, k.d_acc ? k.d_acc + off : nullptr,
                                 k.d_weights ? k.d_weights + off * n : nullptr};
    return mipnerf::launch_render_vjp(raw_rgb, raw_dens, t, dirs, cot, white_bkgd, c->density_bias, rgb_scale,
                                      c->rgb_padding, d_raw_rgb, d_raw_dens, cnt, n, st);
  }
  const mipnerf_b200_loss* loss = g.loss;
  return mipnerf::launch_render_backward(
      raw_rgb, raw_dens, t, dirs, loss->target_rgb + off * 3, loss->lossmult ? loss->lossmult + off : nullptr,
      loss->mask_sum, loss->level_mse_mult[l] * gscale, loss->level_dist_mult[l] * loss->dist_scale * gscale,
      white_bkgd, c->density_bias, rgb_scale, c->rgb_padding, d_raw_rgb, d_raw_dens,
      loss->per_ray_sqerr ? loss->per_ray_sqerr + (int64_t)l * B + off : nullptr,
      loss->per_ray_distloss ? loss->per_ray_distloss + (int64_t)l * B + off : nullptr, cnt, n, st);
}
}  // namespace

size_t mipnerf_b200_train_workspace_bytes_for(const mipnerf_b200_config* cfg, int64_t num_rays, int precision) {
  Dims d;
  if (check_config(cfg, &d) != MIPNERF_B200_OK || check_train_config(cfg) != MIPNERF_B200_OK || num_rays < 0)
    return 0;
  if (precision == MIPNERF_B200_BF16X3) {  // the fused step only, in chunks of kChunkRaysX3
    if (!train_fused_supported(cfg, precision)) return 0;
    return carve_fused(cfg, d, std::clamp<int64_t>(num_rays, 1, kChunkRaysX3), precision, nullptr).bytes;
  }
  if (precision != MIPNERF_B200_FP32 && precision != MIPNERF_B200_BF16 && precision != MIPNERF_B200_FP16) return 0;
  if (precision != MIPNERF_B200_FP32 && !train_tc_supported(cfg, d)) return 0;  // forward_backward refuses it
  const int64_t r = std::clamp<int64_t>(num_rays, 1, kChunkRaysFp32);
  size_t bytes = carve_train(cfg, d, r * cfg->num_samples, r, true, nullptr).bytes;
  if (train_fused_supported(cfg, precision))  // the fused tensor-core step overlays the same buffer
    bytes = std::max(bytes, carve_fused(cfg, d, r, precision, nullptr).bytes);
  return bytes;
}

// one size for every non-split precision (what callers allocated before the split step existed)
size_t mipnerf_b200_train_workspace_bytes(const mipnerf_b200_config* cfg, int64_t num_rays) {
  size_t bytes = 0;
  for (int precision : {MIPNERF_B200_FP32, MIPNERF_B200_BF16, MIPNERF_B200_FP16}) {
    const size_t b = mipnerf_b200_train_workspace_bytes_for(cfg, num_rays, precision);
    if (b > bytes) bytes = b;
  }
  return bytes;
}

// The per-level backward chain of the fused training step, on 16-bit tile images: colour head, view layer, bottleneck
// + density head, trunk, into `grads` (touched[i]: grads[i] already holds a sum to add to; inv_gscale takes the fp16
// step's gradient scale out again), on the images im.bwd (im.bwd_lo in bf16x3).  density_only (a density query): the
// chain starts at the density head; d h_7
// is then the rank-1 term d_raw_density . W_density, masked by h_7 > 0, which the bottleneck's dgrad computes on an
// all-zero d_a with the mask read from the h_7 tile (there is no bottleneck wgrad to leave its sign bits behind).
int tile_backward_chain(const mipnerf_b200_config* cfg, const Dims& d, const mipnerf_b200_weights* w, int precision,
                        const LayerImages& im, const TileChainOps& o, bool density_only, float inv_gscale,
                        const mipnerf_b200_linear_grad* grads, bool* touched, cudaStream_t st) {
  const int depth = cfg->net_depth, W = cfg->net_width, Wc = cfg->net_width_condition;
  const bool x3 = mipnerf::is_x3(precision);
  const int fmt = mipnerf::fmt_of(precision);
  const int64_t m = o.tiles * 128;
  const mipnerf_b200_linear& dl = w->linears[depth];
  const mipnerf_b200_linear& cl = w->linears[d.n_lin - 1];
  // the rows of a query's last tile past its last point (view_div 1) take no cotangent and a zero view encoding
  if (o.rows < m) {
    CUDA_TRY(cudaMemsetAsync(o.d_raw_density + o.rows, 0, (size_t)(m - o.rows) * 4, st));
    if (!density_only) {
      CUDA_TRY(cudaMemsetAsync(o.d_raw_rgb + o.rows * 3, 0, (size_t)(m - o.rows) * 12, st));
      CUDA_TRY(cudaMemsetAsync(o.venc + o.rows * d.view_dim, 0, (size_t)(m - o.rows) * d.view_dim * 4, st));
    }
  }
  // MIPNERF_B200_TRAIN_MASKBITS=0: the dgrad GEMMs read the ReLU mask from the activation tile images again (A/B)
  const char* bits_env = getenv("MIPNERF_B200_TRAIN_MASKBITS");
  const bool use_bits = !(bits_env && bits_env[0] == '0');
  auto wgrad = [&](int idx, mipnerf::T16 dy, mipnerf::T16 x1, int k1, const mipnerf::WgradOperand& x2, int k2, int div,
                   bool emit_mask) {
    const mipnerf_b200_linear& l = w->linears[idx];
    int slices = 0;
    cudaError_t e2 = mipnerf::launch_wgrad_mn_partials(dy, l.out_features, x1, k1, x2, k2, div, o.part, m,
                                                       mipnerf::kWgradMaxSlices, fmt, &slices, st,
                                                       emit_mask && use_bits ? o.relu_bits : nullptr);
    if (e2 != cudaSuccess) return e2;
    e2 = mipnerf::launch_wgrad_reduce(o.part, slices, l.out_features, k1 + k2, grads[idx].weight_grad,
                                      grads[idx].bias_grad, touched[idx] ? 1 : 0, st, inv_gscale);
    touched[idx] = true;
    return e2;
  };
  // y = [mask] (x . B^T + r1 r1w) on tile images
  // (act: the layer input whose ReLU masks the output, read as the sign bits the preceding wgrad left behind, or
  // null for no mask; image_mask: read it from the activation tile itself)
  auto dgrad = [&](mipnerf::T16 x, int slot, mipnerf::T16Out y, int nn, int kk, const float* r1, const float* r1w,
                   const uint8_t* act_in, bool image_mask = false) {
    const bool bits_ok = use_bits && !image_mask;
    const void* mask = act_in && !bits_ok ? act_in : nullptr;
    const void* bits = act_in && bits_ok ? o.relu_bits : nullptr;
    return mipnerf::launch_linear_t16(x, {im.bwd[slot], im.bwd_lo[slot]}, y, m, nn, kk, r1, r1w, mask, fmt, st, bits);
  };
  // h_0..h_7, 8 = bottleneck: the dump is one carve of 9 layers of tiles, in bf16x3 followed by their lo images
  auto h16 = [&](int i) { return mipnerf::tile_pair(o.act + (size_t)i * o.tiles * 65536, 9 * o.tiles, 256, x3); };
  const mipnerf::T16 enc16 = mipnerf::tile_pair(o.enc16, o.tiles, 128, x3);
  const mipnerf::T16 v = mipnerf::tile_pair(o.v, o.tiles, 128, x3);
  const mipnerf::T16Out d_v = mipnerf::tile_pair(o.d_v, o.tiles, 128, x3);
  const mipnerf::T16Out d_a = mipnerf::tile_pair(o.d_a, o.tiles, 256, x3);
  const mipnerf::T16Out d_b = mipnerf::tile_pair(o.d_b, o.tiles, 256, x3);
  if (density_only) {
    CUDA_TRY(mipnerf::launch_wgrad_small_n_t16(o.d_raw_density, 1, h16(depth - 1), W, o.part, grads[depth].weight_grad,
                                               grads[depth].bias_grad, touched[depth] ? 1 : 0, m, fmt, st, inv_gscale));
    touched[depth] = true;
    CUDA_TRY(cudaMemsetAsync(o.d_a, 0, (size_t)o.tiles * 65536 * (x3 ? 2 : 1), st));
    CUDA_TRY(dgrad(d_a, depth, d_b, W, W, o.d_raw_density, dl.weight, h16(depth - 1).hi, /*image_mask=*/true));
  } else {
    // colour head, view layer                                          (models/mip_nerf.py:106-110)
    CUDA_TRY(mipnerf::launch_wgrad_small_n_t16(o.d_raw_rgb, 3, v, Wc, o.part, grads[d.n_lin - 1].weight_grad,
                                               grads[d.n_lin - 1].bias_grad, touched[d.n_lin - 1] ? 1 : 0, m, fmt, st,
                                               inv_gscale));
    touched[d.n_lin - 1] = true;
    CUDA_TRY(mipnerf::launch_color_dgrad_t16(o.d_raw_rgb, cl.weight, o.v, d_v, m, Wc, fmt, st));
    CUDA_TRY(wgrad(depth + 2, d_v, h16(8), W, {o.venc, d.view_dim}, d.view_dim, o.view_div, false));
    CUDA_TRY(dgrad(d_v, depth + 1, d_a, W, Wc, nullptr, nullptr, nullptr));
    // bottleneck + density head share h_7                              (models/mip_nerf.py:98-101)
    CUDA_TRY(wgrad(depth + 1, d_a, h16(depth - 1), W, {}, 0, 1, /*emit_mask=*/true));  // sign mask of h_7
    CUDA_TRY(mipnerf::launch_wgrad_small_n_t16(o.d_raw_density, 1, h16(depth - 1), W, o.part, grads[depth].weight_grad,
                                               grads[depth].bias_grad, touched[depth] ? 1 : 0, m, fmt, st, inv_gscale));
    touched[depth] = true;
    CUDA_TRY(dgrad(d_a, depth, d_b, W, W, o.d_raw_density, dl.weight, h16(depth - 1).hi));
  }
  // trunk                                                            (models/mip_nerf.py:93-97)
  mipnerf::T16Out cur = d_b, other = d_a;
  for (int i = depth - 1; i >= 0; --i) {
    const bool skip = takes_skip(cfg, i);
    if (i == 0)
      CUDA_TRY(wgrad(0, cur, enc16, d.xyz_dim, {}, 0, 1, false));
    else
      CUDA_TRY(wgrad(i, cur, h16(i - 1), W, skip ? enc16 : mipnerf::T16{}, skip ? d.xyz_dim : 0, 1, true));
    if (i > 0) {  // the wgrad just streamed h_{i-1} and left its sign mask behind: 32 B per row instead of 512
      CUDA_TRY(dgrad(cur, i, other, W, W, nullptr, nullptr, h16(i - 1).hi));
      std::swap(cur, other);
    }
  }
  return MIPNERF_B200_OK;
}

static int forward_backward_fused(const mipnerf_b200_config* cfg, const Dims& d, const mipnerf_b200_weights* w,
                                  const mipnerf_b200_rays* rays, int randomized, const float* t_rand,
                                  const float* u_jitter, const mipnerf_b200_rng* rng, int white_bkgd, int precision,
                                  const GradSource& src, bool given_t, mipnerf_b200_level_out* outs,
                                  const mipnerf_b200_linear_grad* grads, bool* touched, void* workspace,
                                  cudaStream_t st) {
  const int n = cfg->num_samples;
  const float rgb_scale = mipnerf::rgb_scale_of(cfg);
  const int64_t B = rays->num_rays;
  // bf16x3: every operand of the backward is a pair of bf16 tile images, hi and lo (the 16-bit launchers' format
  // argument is then bf16, and the *_lo arguments select their split kernels)
  const bool x3 = mipnerf::is_x3(precision);
  const int fmt = mipnerf::fmt_of(precision);
  const int64_t chunk = x3 ? kChunkRaysX3 : kChunkRaysFp32;
  mipnerf_b200_weights wl;
  LayerImages im;
  int rc;
  if ((rc = pack_fused_weights(cfg, d, w, precision, carve_fused(cfg, d, std::min(B, chunk), precision, workspace).head,
                               &wl, &im, st)))
    return rc;
  const float gscale = grad_scale_of(precision), inv_gscale = 1.f / gscale;
  for (int64_t off = 0; off < B; off += chunk) {
    const int64_t cnt = (B - off) < chunk ? (B - off) : chunk;
    const mipnerf_b200_rays rc_ = offset_rays(*rays, off, cnt);
    const FusedScratch s = carve_fused(cfg, d, cnt, precision, workspace);
    TileChainOps ops = s.chain;
    CUDA_TRY(mipnerf::launch_pos_enc(rc_.viewdirs, ops.venc, cnt, 0, cfg->deg_view, 1, st));
    // ---- forward of all levels: two launches, everything the backward needs is left behind as tile images
    mipnerf_b200_level_out lo[2];
    mipnerf::TcTrainDump dump{};
    for (int l = 0; l < cfg->num_levels; ++l) {
      lo[l] = chunk_level_out(outs[l], off, cnt, n, given_t, s.t[l], s.w[l]);
      dump.act[l] = s.act[l], dump.v[l] = s.v[l], dump.raw_rgb[l] = s.raw_rgb[l], dump.raw_density[l] = s.raw_density[l];
    }
    CUDA_TRY(mipnerf::tc_forward(cfg, &wl, &rc_, randomized, t_rand ? t_rand + off * (n + 1) : nullptr,
                                 u_jitter ? u_jitter + off * (n + 1) : nullptr, rng, white_bkgd, precision, lo, s.tcws,
                                 s.tcws_bytes, st, &dump, off, given_t ? 1 : 0));
    for (int l = 0; l < cfg->num_levels; ++l) {
      const float* t_cur = lo[l].t_samples;
      // the IPE features again (operand of two wgrads; the level kernel keeps its own 16-bit copy on chip), written
      // straight into a tile image so that those wgrads stage them by bulk copy like every other operand
      CUDA_TRY(mipnerf::launch_ipe_t16(rc_.origins, rc_.directions, rc_.radii, t_cur,
                                       mipnerf::tile_pair(ops.enc16, cnt, 128, x3), cnt, n, cfg->disable_integration,
                                       fmt, st));
      CUDA_TRY(launch_grad_source(src, cfg, l, off, B, cnt, s.raw_rgb[l], s.raw_density[l], t_cur, rc_.directions,
                                  white_bkgd, rgb_scale, gscale, ops.d_raw_rgb, ops.d_raw_density, st));
      ops.act = s.act[l], ops.v = s.v[l];
      if ((rc = tile_backward_chain(cfg, d, w, precision, im, ops, false, inv_gscale, grads, touched, st))) return rc;
    }
  }
  return MIPNERF_B200_OK;
}

// The training drivers: forward with every activation the backward needs, then the backward pass from `src`.
// given_t: each level's fenceposts come from outs[l].t_samples (read-only) instead of being sampled / resampled, and
// the recomputed pixels are not returned (the backward pass of MipNerf.forward, mipnerf_b200_backward).
static int forward_backward_impl(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w,
                                 const mipnerf_b200_rays* rays, int randomized, const float* t_rand,
                                 const float* u_jitter, const mipnerf_b200_rng* rng, int white_bkgd, int precision,
                                 const GradSource& src, bool given_t, mipnerf_b200_level_out* outs,
                                 const mipnerf_b200_linear_grad* grads, int num_grads, int accumulate,
                                 void* workspace, size_t workspace_bytes, void* stream) {
  Dims d;
  int rc;
  if ((rc = check_config(cfg, &d))) return rc;
  if ((rc = check_train_config(cfg))) return rc;
  if ((rc = check_weights(cfg, d, w))) return rc;
  if ((rc = check_rays(rays))) return rc;
  const bool x3 = mipnerf::is_x3(precision);
  const bool tc = precision == MIPNERF_B200_BF16 || precision == MIPNERF_B200_FP16 || x3;
  if (x3 && (src.cots || !train_fused_supported(cfg, precision)))
    return fail(MIPNERF_B200_EUNSUPPORTED,
                "training: BF16X3 is the one split-operand training precision, for the fused training-loss step only "
                "(8x256 / 1x128 MLP, default encodings, 128 samples, at most two levels; no backward from cotangents); "
                "use FP32 (parity), BF16 or FP16");
  if (precision != MIPNERF_B200_FP32 && !tc) return fail(MIPNERF_B200_EINVAL, "precision %d", precision);
  if (tc && !train_tc_supported(cfg, d))
    return fail(MIPNERF_B200_EUNSUPPORTED,
                "tensor-core training GEMMs: 8x256 trunk / 128 view layer / 96-d IPE only; use MIPNERF_B200_FP32");
  if (!outs || !(src.loss || src.cots) || !grads) return fail(MIPNERF_B200_EINVAL, "outs / loss / grads is NULL");
  if (src.cots && (rc = check_cotangent_precision(precision, "backward from arbitrary cotangents"))) return rc;
  if ((rc = check_grads(d, grads, num_grads))) return rc;
  if (src.loss && (!src.loss->level_mse_mult || !src.loss->level_dist_mult))
    return fail(MIPNERF_B200_EINVAL, "loss multipliers are NULL");
  if (src.loss && rays->num_rays > 0 && (!src.loss->target_rgb || !src.loss->mask_sum || !rays->viewdirs))
    return fail(MIPNERF_B200_EINVAL, "target_rgb / mask_sum / viewdirs is NULL");
  if (rays->num_rays > 0 && !rays->viewdirs) return fail(MIPNERF_B200_EINVAL, "viewdirs is NULL");
  if (!given_t && randomized && !rng && (!t_rand || (cfg->num_levels > 1 && !u_jitter)))
    return fail(MIPNERF_B200_EINVAL,
                "randomized=1 needs t_rand and u_jitter (injected noise) or the _rng entry point (in-kernel Philox)");
  for (int l = 0; l < cfg->num_levels; ++l) {
    if (!given_t && rays->num_rays > 0 && (!outs[l].comp_rgb || !outs[l].distance || !outs[l].acc))
      return fail(MIPNERF_B200_EINVAL, "outs[%d] misses comp_rgb/distance/acc", l);
    if (given_t && rays->num_rays > 0 && !outs[l].t_samples)
      return fail(MIPNERF_B200_EINVAL, "t_samples[%d] is NULL", l);
  }
  if ((rc = check_density_normals(cfg, randomized, rng, outs, rays->num_rays))) return rc;
  const size_t need = x3 ? mipnerf_b200_train_workspace_bytes_for(cfg, rays->num_rays, precision)
                        : mipnerf_b200_train_workspace_bytes(cfg, rays->num_rays);
  if (rays->num_rays > 0 && (!workspace || workspace_bytes < need))
    return fail(MIPNERF_B200_EWORKSPACE, "workspace %zu < %zu bytes", workspace_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  const int n = cfg->num_samples, depth = cfg->net_depth;
  const float rgb_scale = mipnerf::rgb_scale_of(cfg);
  const int64_t B = rays->num_rays;
  const float gscale = grad_scale_of(precision);
  // with rays, the chains reach every linear (check_train_config: one view layer)
  bool touched[kMaxTrainDepth + 8];
  std::fill_n(touched, d.n_lin, accumulate != 0);
  if (tc && B > 0 && train_fused_supported(cfg, precision)) {
    if ((rc = forward_backward_fused(cfg, d, w, rays, randomized, t_rand, u_jitter, rng, white_bkgd, precision, src,
                                     given_t, outs, grads, touched, workspace, st)))
      return rc;
    return zero_untouched(d, w, grads, touched, st);
  }
  // ---- tensor-core mode: B operands of every forward / dgrad GEMM, packed once per call
  LayerImages im{};
  if (tc && B > 0) {
    const int64_t r = std::min(B, kChunkRaysFp32);
    CUDA_TRY(pack_layer_images(cfg, d, w, precision, true, carve_train(cfg, d, r * n, r, true, workspace).images, &im,
                               st));
  }

  for (int64_t off = 0; off < B; off += kChunkRaysFp32) {
    const int64_t cnt = (B - off) < kChunkRaysFp32 ? (B - off) : kChunkRaysFp32;
    const int64_t m = cnt * n;
    const mipnerf_b200_rays rc_ = offset_rays(*rays, off, cnt);
    const TrainScratch s = carve_train(cfg, d, m, cnt, true, workspace);
    CUDA_TRY(mipnerf::launch_pos_enc(rc_.viewdirs, s.venc, cnt, 0, cfg->deg_view, 1, st));
    if (tc) {
      const mipnerf_b200_linear& vl0 = w->linears[depth + 2];
      CUDA_TRY(mipnerf::launch_view_bias_from_enc(s.venc, vl0.weight, vl0.bias, s.vrow, cnt, st));
    }
    const float *t_prev = nullptr, *w_prev = nullptr;
    for (int l = 0; l < cfg->num_levels; ++l) {
      const mipnerf_b200_level_out lo = chunk_level_out(outs[l], off, cnt, n, given_t, s.t[l & 1], s.w[l & 1]);
      // ---- forward of this level, every activation kept (models/mip_nerf.py:203-240)
      if (given_t) {
        // the caller's fenceposts: nothing to sample
      } else if (l == 0) {
        CUDA_TRY(mipnerf::launch_coarse_t(rc_.near, rc_.far, mipnerf::level_draws(randomized, t_rand, rng, off, 0, n + 1),
                                          lo.t_samples, cnt, n, randomized, cfg->disparity, st));
      } else {
        CUDA_TRY(mipnerf::launch_resample(t_prev, w_prev, mipnerf::level_draws(randomized, u_jitter, rng, off, 1 + l, n + 1),
                                          lo.t_samples, lo.inds, cnt, n, n + 1, randomized, 1, cfg->resample_padding, st));
      }
      CUDA_TRY(mipnerf::launch_ipe_from_t(rc_.origins, rc_.directions, rc_.radii, lo.t_samples, s.enc, cnt, n,
                                          cfg->min_deg_point, cfg->max_deg_point, cfg->disable_integration, st));
      if ((rc = mlp_forward_kept(cfg, d, w, tc, precision, im, s, m, n, false, st))) return rc;
      // density noise (models/mip_nerf.py:232-233), in place: render_backward then takes softplus' at the noisy point
      CUDA_TRY(mipnerf::launch_add_density_noise(
          s.raw_density, mipnerf::density_noise_draws(cfg, randomized, outs[l].density_normal, rng, off, l, n), cnt, n, st));
      CUDA_TRY(mipnerf::launch_composite(s.raw_rgb, s.raw_density, lo.t_samples, rc_.directions, lo.comp_rgb,
                                         lo.distance, lo.acc, lo.weights, cnt, n, white_bkgd, 1, cfg->density_bias,
                                         rgb_scale, cfg->rgb_padding, st));

      // ---- backward of this level (its fenceposts are constants, so levels are independent here)
      CUDA_TRY(launch_grad_source(src, cfg, l, off, B, cnt, s.raw_rgb, s.raw_density, lo.t_samples, rc_.directions,
                                  white_bkgd, rgb_scale, gscale, s.d_raw_rgb, s.d_raw_density, st));
      if ((rc = mlp_backward_chain(cfg, d, w, tc, precision, im, s, m, n, false, grads, touched, st, 1.f / gscale)))
        return rc;
      t_prev = lo.t_samples;
      w_prev = lo.weights;
    }
  }
  return zero_untouched(d, w, grads, touched, st);
}

int mipnerf_b200_forward_backward(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w,
                                  const mipnerf_b200_rays* rays, int randomized, const float* t_rand,
                                  const float* u_jitter, int white_bkgd, int precision,
                                  const mipnerf_b200_loss* loss, mipnerf_b200_level_out* outs,
                                  const mipnerf_b200_linear_grad* grads, int num_grads, int accumulate,
                                  void* workspace, size_t workspace_bytes, void* stream) {
  return forward_backward_impl(cfg, w, rays, randomized, t_rand, u_jitter, nullptr, white_bkgd, precision,
                               GradSource{loss, nullptr}, false, outs, grads, num_grads, accumulate, workspace,
                               workspace_bytes, stream);
}

int mipnerf_b200_forward_backward_rng(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w,
                                      const mipnerf_b200_rays* rays, const mipnerf_b200_rng* rng, int white_bkgd,
                                      int precision, const mipnerf_b200_loss* loss, mipnerf_b200_level_out* outs,
                                      const mipnerf_b200_linear_grad* grads, int num_grads, int accumulate,
                                      void* workspace, size_t workspace_bytes, void* stream) {
  if (!rng) return fail(MIPNERF_B200_EINVAL, "rng is NULL");
  return forward_backward_impl(cfg, w, rays, 1, nullptr, nullptr, rng, white_bkgd, precision, GradSource{loss, nullptr},
                               false, outs, grads, num_grads, accumulate, workspace, workspace_bytes, stream);
}

int mipnerf_b200_backward(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w, const mipnerf_b200_rays* rays,
                          const float* const* t_samples, int randomized, const mipnerf_b200_rng* rng,
                          const float* const* density_normal, int white_bkgd, int precision,
                          const mipnerf_b200_level_cotangent* cots, const mipnerf_b200_linear_grad* grads,
                          int num_grads, int accumulate, void* workspace, size_t workspace_bytes, void* stream) {
  if (!cfg) return fail(MIPNERF_B200_EINVAL, "config is NULL");
  if (!t_samples || !cots) return fail(MIPNERF_B200_EINVAL, "t_samples / cots is NULL");
  if (cfg->num_levels < 1 || cfg->num_levels > 64) return fail(MIPNERF_B200_EINVAL, "num_levels=%d", cfg->num_levels);
  mipnerf_b200_level_out outs[64];
  for (int l = 0; l < cfg->num_levels; ++l) {
    outs[l] = mipnerf_b200_level_out{};
    outs[l].t_samples = const_cast<float*>(t_samples[l]);  // read only (given_t)
    outs[l].density_normal = density_normal ? density_normal[l] : nullptr;
  }
  if (rng)  // in-kernel normals: injected ones are ignored, as by the _rng forward
    for (int l = 0; l < cfg->num_levels; ++l) outs[l].density_normal = nullptr;
  return forward_backward_impl(cfg, w, rays, randomized, nullptr, nullptr, rng, white_bkgd, precision,
                               GradSource{nullptr, cots}, true, outs, grads, num_grads, accumulate, workspace,
                               workspace_bytes, stream);
}

int mipnerf_b200_linear_tc(const float* x, const float* weight, const float* bias, float* y, int64_t m, int n,
                           int k, int relu, int precision, void* scratch, size_t scratch_bytes, void* stream) {
  if (m < 0 || !mipnerf::linear_tc_shape_ok(n, k))
    return fail(MIPNERF_B200_EUNSUPPORTED, "linear_tc: n in {128,256}, k in {96,128,256} (got n=%d k=%d)", n, k);
  if (precision != MIPNERF_B200_BF16 && precision != MIPNERF_B200_FP16)
    return fail(MIPNERF_B200_EINVAL, "linear_tc: precision must be BF16 or FP16");
  if (m > 0 && (!x || !weight || !y)) return fail(MIPNERF_B200_EINVAL, "NULL tensor");
  const size_t need = mipnerf::linear_tc_image_bytes(n, k);
  if (!scratch || scratch_bytes < need) return fail(MIPNERF_B200_EWORKSPACE, "scratch %zu < %zu bytes", scratch_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  CUDA_TRY(mipnerf::launch_pack_linear_image(weight, k, 0, 0, scratch, n, k, precision, st));
  CUDA_TRY(mipnerf::launch_linear_tc(x, k, scratch, y, n, m, n, k, bias, nullptr, 1, nullptr, nullptr, nullptr, nullptr,
                                     relu, precision, st));
  return MIPNERF_B200_OK;
}

size_t mipnerf_b200_wgrad_tc_scratch_bytes(int n, int k) {
  if (n < 1 || k < 1) return 0;
  return sizeof(float) * (size_t)mipnerf::kWgradMaxSlices * n * (k + 1);
}

int mipnerf_b200_wgrad_tc(const float* dy, int n, const float* x1, int k1, const float* x2, int k2, int x2_row_div,
                          int64_t m, float* dw, float* db, int precision, void* scratch, size_t scratch_bytes,
                          void* stream) {
  if (m < 0 || k1 < 1 || k2 < 0 || !mipnerf::wgrad_tc_shape_ok(n))
    return fail(MIPNERF_B200_EUNSUPPORTED, "wgrad_tc: n in {128,256} (got n=%d)", n);
  if (k2 > 0 && k1 % 256 != 0)  // no k tile of the kernel may straddle x1 and x2 (launch_wgrad_mn_partials)
    return fail(MIPNERF_B200_EUNSUPPORTED, "wgrad_tc: with x2, k1 must be a multiple of 256 (got k1=%d)", k1);
  if (precision != MIPNERF_B200_BF16 && precision != MIPNERF_B200_FP16)
    return fail(MIPNERF_B200_EINVAL, "wgrad_tc: precision must be BF16 or FP16");
  if (!dw || !db || (m > 0 && (!dy || !x1 || (k2 > 0 && !x2)))) return fail(MIPNERF_B200_EINVAL, "NULL tensor");
  if (m > 0 && (reinterpret_cast<uintptr_t>(dy) & 15) != 0)  // dy rows are staged with float4 loads
    return fail(MIPNERF_B200_EINVAL, "wgrad_tc: dy must be 16-byte aligned");
  const size_t need = mipnerf_b200_wgrad_tc_scratch_bytes(n, k1 + k2);
  if (!scratch || scratch_bytes < need) return fail(MIPNERF_B200_EWORKSPACE, "scratch %zu < %zu bytes", scratch_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  int slices = 0;
  CUDA_TRY(mipnerf::launch_wgrad_mn_partials({dy, n}, n, {x1, k1}, k1, {k2 > 0 ? x2 : nullptr, k2}, k2, x2_row_div,
                                             static_cast<float*>(scratch), m, mipnerf::kWgradMaxSlices, precision,
                                             &slices, st));
  CUDA_TRY(mipnerf::launch_wgrad_reduce(static_cast<float*>(scratch), slices, n, k1 + k2, dw, db, 0, st));
  return MIPNERF_B200_OK;
}

// ---- the bf16x3 training step's GEMMs on their own (operands split into hi / lo tile images here) ----
namespace {
size_t t16_pair(int64_t m, int cols) { return align_up(2 * mipnerf::t16_image_bytes(m, cols)); }
}  // namespace

size_t mipnerf_b200_linear_x3_scratch_bytes(int64_t m, int n, int k) {
  if (m < 0 || !(n == 128 || n == 256) || !(k == 128 || k == 256)) return 0;
  return t16_pair(m, k) + t16_pair(m, n) + align_up(mipnerf::t16_image_bytes(m, n)) +
         align_up(2 * mipnerf::linear_tc_image_bytes(n, k));
}

int mipnerf_b200_linear_x3(const float* x, const float* weight, const float* r1, const float* r1w, const float* mask,
                           float* y, int64_t m, int n, int k, void* scratch, size_t scratch_bytes, void* stream) {
  const size_t need = mipnerf_b200_linear_x3_scratch_bytes(m, n, k);
  if (need == 0) return fail(MIPNERF_B200_EUNSUPPORTED, "linear_x3: n, k in {128,256} (got n=%d k=%d)", n, k);
  if (m > 0 && (!x || !weight || !y || (r1 && !r1w))) return fail(MIPNERF_B200_EINVAL, "NULL tensor");
  if (!scratch || scratch_bytes < need) return fail(MIPNERF_B200_EWORKSPACE, "scratch %zu < %zu bytes", scratch_bytes, need);
  if (m == 0) return MIPNERF_B200_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t tiles = (m + 127) / 128, mp = tiles * 128;  // the images are whole 128-row tiles (zero rows past m)
  uint8_t* base = static_cast<uint8_t*>(scratch);
  const mipnerf::T16Out xh = mipnerf::tile_pair(base, tiles, k, true);
  const mipnerf::T16Out yh = mipnerf::tile_pair(base + t16_pair(m, k), tiles, n, true);
  uint8_t* mk = yh.hi + t16_pair(m, n);
  uint8_t* img = mk + align_up(mipnerf::t16_image_bytes(m, n));
  const size_t ib = mipnerf::linear_tc_image_bytes(n, k);
  CUDA_TRY(mipnerf::launch_t16_pack(x, k, k, m, xh, MIPNERF_B200_BF16, st));
  if (mask) CUDA_TRY(mipnerf::launch_t16_pack(mask, n, n, m, mk, MIPNERF_B200_BF16, st));
  CUDA_TRY(mipnerf::launch_pack_linear_image(weight, k, 0, 0, img, n, k, MIPNERF_B200_BF16, st));
  CUDA_TRY(mipnerf::launch_pack_linear_image(weight, k, 0, 0, img + ib, n, k, MIPNERF_B200_BF16, st, 1));
  if (r1 && mp != m) return fail(MIPNERF_B200_EINVAL, "linear_x3: r1 needs m a multiple of 128");
  CUDA_TRY(mipnerf::launch_linear_t16(xh, {img, img + ib}, yh, mp, n, k, r1, r1w, mask ? mk : nullptr,
                                      MIPNERF_B200_BF16, st));
  CUDA_TRY(mipnerf::launch_t16_unpack(yh, n, y, n, m, MIPNERF_B200_BF16, st));
  return MIPNERF_B200_OK;
}

size_t mipnerf_b200_wgrad_x3_scratch_bytes(int64_t m, int n, int k1, int k2, int x2_row_div) {
  if (m < 0 || n < 1 || k1 < 1 || k2 < 0) return 0;
  return align_up(mipnerf_b200_wgrad_tc_scratch_bytes(n, k1 + k2)) + t16_pair(m, n) + t16_pair(m, k1) +
         (k2 > 0 && x2_row_div <= 1 ? t16_pair(m, k2) : 0);
}

int mipnerf_b200_wgrad_x3(const float* dy, int n, const float* x1, int k1, const float* x2, int k2, int x2_row_div,
                          int64_t m, float* dw, float* db, void* scratch, size_t scratch_bytes, void* stream) {
  if (m < 0 || k1 < 1 || k2 < 0 || !mipnerf::wgrad_tc_shape_ok(n))
    return fail(MIPNERF_B200_EUNSUPPORTED, "wgrad_x3: n in {128,256} (got n=%d)", n);
  if (k2 > 0 && k1 % 256 != 0)
    return fail(MIPNERF_B200_EUNSUPPORTED, "wgrad_x3: with x2, k1 must be a multiple of 256 (got k1=%d)", k1);
  if (!dw || !db || (m > 0 && (!dy || !x1 || (k2 > 0 && !x2)))) return fail(MIPNERF_B200_EINVAL, "NULL tensor");
  if (x2_row_div < 1) x2_row_div = 1;
  const size_t need = mipnerf_b200_wgrad_x3_scratch_bytes(m, n, k1, k2, x2_row_div);
  if (!scratch || scratch_bytes < need) return fail(MIPNERF_B200_EWORKSPACE, "scratch %zu < %zu bytes", scratch_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t tiles = (m + 127) / 128, mp = tiles * 128;  // zero rows past m add nothing
  uint8_t* base = static_cast<uint8_t*>(scratch);
  float* part = reinterpret_cast<float*>(base);
  const mipnerf::T16Out dyh =
      mipnerf::tile_pair(base + align_up(mipnerf_b200_wgrad_tc_scratch_bytes(n, k1 + k2)), tiles, n, true);
  const mipnerf::T16Out x1h = mipnerf::tile_pair(dyh.hi + t16_pair(m, n), tiles, k1, true);
  const mipnerf::T16Out x2h = mipnerf::tile_pair(x1h.hi + t16_pair(m, k1), tiles, k2, true);
  const bool x2_img = k2 > 0 && x2_row_div == 1;
  if (x2_row_div > 1 && mp != m) return fail(MIPNERF_B200_EINVAL, "wgrad_x3: x2_row_div > 1 needs m a multiple of 128");
  CUDA_TRY(mipnerf::launch_t16_pack(dy, n, n, m, dyh, MIPNERF_B200_BF16, st));
  CUDA_TRY(mipnerf::launch_t16_pack(x1, k1, k1, m, x1h, MIPNERF_B200_BF16, st));
  if (x2_img) CUDA_TRY(mipnerf::launch_t16_pack(x2, k2, k2, m, x2h, MIPNERF_B200_BF16, st));
  int slices = 0;
  if (mp > 0) {
    const mipnerf::WgradOperand x2op = x2_img ? mipnerf::WgradOperand(x2h) : mipnerf::WgradOperand(x2, k2);
    CUDA_TRY(mipnerf::launch_wgrad_mn_partials(dyh, n, x1h, k1, k2 > 0 ? x2op : mipnerf::WgradOperand(), k2,
                                               x2_row_div, part, mp, mipnerf::kWgradMaxSlices, MIPNERF_B200_BF16,
                                               &slices, st));
    CUDA_TRY(mipnerf::launch_wgrad_reduce(part, slices, n, k1 + k2, dw, db, 0, st));
  } else {
    CUDA_TRY(cudaMemsetAsync(dw, 0, sizeof(float) * n * (k1 + k2), st));
    CUDA_TRY(cudaMemsetAsync(db, 0, sizeof(float) * n, st));
  }
  return MIPNERF_B200_OK;
}

int mipnerf_b200_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n,
                           double lr, double beta1, double beta2, double eps, int64_t step, double grad_scale,
                           void* stream) {
  if (n < 0 || step < 1) return fail(MIPNERF_B200_EINVAL, "bad n / step");
  if (n > 0 && (!param || !grad || !exp_avg || !exp_avg_sq)) return fail(MIPNERF_B200_EINVAL, "NULL tensor");
  const double bc1 = 1.0 - pow(beta1, (double)step), bc2 = 1.0 - pow(beta2, (double)step);
  CUDA_TRY(mipnerf::launch_adam(param, grad, exp_avg, exp_avg_sq, n, (float)(1.0 - beta1), (float)beta2,
                                (float)(1.0 - beta2), (float)eps, (float)(lr / bc1), (float)sqrt(bc2), (float)grad_scale,
                                (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

int mipnerf_b200_adam_step_multi(int count, float* const* params, const float* const* grads, float* const* exp_avg,
                                 float* const* exp_avg_sq, const int64_t* sizes, double lr, double beta1, double beta2,
                                 double eps, int64_t step, double grad_scale, void* stream) {
  if (count < 0 || step < 1) return fail(MIPNERF_B200_EINVAL, "bad count / step");
  if (count > 0 && (!params || !grads || !exp_avg || !exp_avg_sq || !sizes)) return fail(MIPNERF_B200_EINVAL, "NULL array");
  for (int i = 0; i < count; ++i)  // every tensor before the first launch: a refusal leaves all of them untouched
    if (sizes[i] < 0 || (sizes[i] > 0 && (!params[i] || !grads[i] || !exp_avg[i] || !exp_avg_sq[i])))
      return fail(MIPNERF_B200_EINVAL, "tensor %d: NULL pointer or negative size", i);
  const double bc1 = 1.0 - pow(beta1, (double)step), bc2 = 1.0 - pow(beta2, (double)step);
  for (int base = 0; base < count; base += mipnerf::kAdamMaxTensors) {
    mipnerf::AdamMulti t{};
    t.count = (count - base) < mipnerf::kAdamMaxTensors ? (count - base) : mipnerf::kAdamMaxTensors;
    for (int k = 0; k < t.count; ++k) {
      const int i = base + k;
      t.p[k] = params[i], t.g[k] = grads[i], t.m[k] = exp_avg[i], t.v[k] = exp_avg_sq[i], t.n[k] = sizes[i];
      t.blocks[k] = (int)((sizes[i] + 255) / 256);
    }
    CUDA_TRY(mipnerf::launch_adam_multi(t, (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2), (float)eps,
                                        (float)(lr / bc1), (float)sqrt(bc2), (float)grad_scale, (cudaStream_t)stream));
  }
  return MIPNERF_B200_OK;
}

int mipnerf_b200_distloss(const float* weights, const float* samples, int64_t num_rays, int num_samples,
                          float* per_ray_loss, void* stream) {
  if (num_rays < 0 || num_samples < 1) return fail(MIPNERF_B200_EINVAL, "bad sizes");
  if (num_rays > 0 && (!weights || !samples || !per_ray_loss)) return fail(MIPNERF_B200_EINVAL, "NULL tensor");
  CUDA_TRY(mipnerf::launch_distloss(weights, samples, per_ray_loss, num_rays, num_samples, (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

int mipnerf_b200_distloss_backward(const float* weights, const float* samples, int64_t num_rays, int num_samples,
                                   const float* grad_out, float scale, float* d_weights, void* stream) {
  if (num_rays < 0 || num_samples < 1) return fail(MIPNERF_B200_EINVAL, "bad sizes");
  if (num_rays > 0 && (!weights || !samples || !d_weights)) return fail(MIPNERF_B200_EINVAL, "NULL tensor");
  CUDA_TRY(mipnerf::launch_distloss_backward(weights, samples, grad_out, scale, d_weights, num_rays, num_samples,
                                             (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

// The interlevel loss entry points' refusals, in order: num_rays, the NULL tensors (`out`: per_ray_loss or d_w_hat),
// then n and n_hat.
static int check_interlevel(const float* t, const float* w, int n, const float* t_hat, const float* w_hat, int n_hat,
                            int64_t num_rays, const float* out) {
  if (num_rays < 0) return fail(MIPNERF_B200_EINVAL, "num_rays=%lld: need >= 0", (long long)num_rays);
  if (num_rays > 0 && (!t || !w || !t_hat || !w_hat || !out)) return fail(MIPNERF_B200_EINVAL, "NULL tensor");
  if (n < 1 || n_hat < 1) return fail(MIPNERF_B200_EINVAL, "n=%d, n_hat=%d: need >= 1", n, n_hat);
  return MIPNERF_B200_OK;
}

int mipnerf_b200_interlevel_loss(const float* t, const float* w, int n, const float* t_hat, const float* w_hat,
                                 int n_hat, int64_t num_rays, float* per_ray_loss, void* stream) {
  int rc;
  if ((rc = check_interlevel(t, w, n, t_hat, w_hat, n_hat, num_rays, per_ray_loss))) return rc;
  CUDA_TRY(mipnerf::launch_interlevel_loss(t, w, n, t_hat, w_hat, n_hat, num_rays, per_ray_loss,
                                           (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

int mipnerf_b200_interlevel_loss_backward(const float* t, const float* w, int n, const float* t_hat,
                                          const float* w_hat, int n_hat, int64_t num_rays, const float* grad_out,
                                          float scale, float* d_w_hat, void* stream) {
  int rc;
  if ((rc = check_interlevel(t, w, n, t_hat, w_hat, n_hat, num_rays, d_w_hat))) return rc;
  CUDA_TRY(mipnerf::launch_interlevel_loss_backward(t, w, n, t_hat, w_hat, n_hat, num_rays, grad_out, scale, d_w_hat,
                                                    (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

size_t mipnerf_b200_image_metrics_scratch_bytes(int height, int width, int channels) {
  if (height < 1 || width < 1 || channels < 1) return 0;
  return mipnerf::image_metrics_scratch_bytes(height, width, channels);
}

int mipnerf_b200_image_metrics(const float* pred, const float* target, int height, int width, int channels,
                               void* scratch, size_t scratch_bytes, float* out, void* stream) {
  if (height < 1 || width < 1 || channels < 1) return fail(MIPNERF_B200_EINVAL, "bad image shape");
  if (!pred || !target || !out) return fail(MIPNERF_B200_EINVAL, "NULL tensor");
  const size_t need = mipnerf::image_metrics_scratch_bytes(height, width, channels);
  if (!scratch || scratch_bytes < need) return fail(MIPNERF_B200_EWORKSPACE, "scratch %zu < %zu bytes", scratch_bytes, need);
  CUDA_TRY(mipnerf::launch_image_metrics(pred, target, height, width, channels, 11, 1.5f, 1.0f, scratch, out,
                                         (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

int mipnerf_b200_generate_rays(const float* c2w_host, int height, int width, float focal, float near, float far,
                               int row0, int rows, float* origins, float* directions, float* viewdirs,
                               float* radii, float* near_out, float* far_out, void* stream) {
  if (!c2w_host || height < 2 || width < 1 || !(focal > 0.f) || row0 < 0 || rows < 0 || row0 + rows > height)
    return fail(MIPNERF_B200_EINVAL, "bad frame geometry");
  if (rows > 0 && (!origins || !directions || !viewdirs || !radii || !near_out || !far_out))
    return fail(MIPNERF_B200_EINVAL, "NULL output");
  CUDA_TRY(mipnerf::launch_generate_rays(c2w_host, height, width, focal, near, far, row0, rows, origins, directions,
                                         viewdirs, radii, near_out, far_out, (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

int mipnerf_b200_rays_from_pixels(const float* cam_table, const int64_t* offsets, const int32_t* widths,
                                  int num_images, const int64_t* pixel_ids, int64_t count, const float* atlas,
                                  float* origins, float* directions, float* viewdirs, float* radii,
                                  float* lossmult, float* near_out, float* far_out, float* rgb, void* stream) {
  if (num_images < 1 || count < 0) return fail(MIPNERF_B200_EINVAL, "bad sizes");
  if (!cam_table || !offsets || !widths) return fail(MIPNERF_B200_EINVAL, "NULL scene table");
  if (count > 0 && (!pixel_ids || !origins || !directions || !viewdirs || !radii || !lossmult || !near_out || !far_out))
    return fail(MIPNERF_B200_EINVAL, "NULL ray tensor");
  if (rgb && !atlas) return fail(MIPNERF_B200_EINVAL, "rgb requested without a pixel atlas");
  CUDA_TRY(mipnerf::launch_rays_from_pixels(cam_table, offsets, widths, num_images, pixel_ids, count, atlas, origins,
                                            directions, viewdirs, radii, lossmult, near_out, far_out, rgb,
                                            (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

int mipnerf_b200_sample_along_rays(const mipnerf_b200_rays* rays, int num_samples, int randomized,
                                   int disparity, const float* t_rand, float* t_samples, float* means,
                                   float* covs, void* stream) {
  int rc;
  if ((rc = check_rays(rays))) return rc;
  if (num_samples < 1 || !t_samples) return fail(MIPNERF_B200_EINVAL, "bad num_samples / t_samples");
  if (randomized && !t_rand) return fail(MIPNERF_B200_EINVAL, "randomized=1 needs t_rand");
  cudaStream_t st = (cudaStream_t)stream;
  CUDA_TRY(mipnerf::launch_coarse_t(rays->near, rays->far, mipnerf::draws_from_array(randomized ? t_rand : nullptr),
                                    t_samples, rays->num_rays, num_samples, randomized, disparity, st));
  if (means && covs)
    CUDA_TRY(mipnerf::launch_cast_rays(rays->origins, rays->directions, rays->radii, t_samples, means, covs,
                                       rays->num_rays, num_samples, st));
  return MIPNERF_B200_OK;
}

int mipnerf_b200_cast_rays(const mipnerf_b200_rays* rays, const float* t_samples, int num_samples,
                           float* means, float* covs, void* stream) {
  int rc;
  if ((rc = check_rays(rays))) return rc;
  if (num_samples < 1 || !t_samples || !means || !covs) return fail(MIPNERF_B200_EINVAL, "NULL argument");
  CUDA_TRY(mipnerf::launch_cast_rays(rays->origins, rays->directions, rays->radii, t_samples, means, covs,
                                     rays->num_rays, num_samples, (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

int mipnerf_b200_integrated_pos_enc(const float* means, const float* covs, int64_t num_points, int min_deg,
                                    int max_deg, float* out, void* stream) {
  // an empty degree range is an [M, 0] encoding, as in the reference: nothing to read or write
  if (num_points < 0 || max_deg < min_deg || min_deg < -60 || max_deg > 60 ||
      (num_points > 0 && max_deg > min_deg && (!means || !covs || !out)))
    return fail(MIPNERF_B200_EINVAL, "bad argument");
  CUDA_TRY(mipnerf::launch_ipe(means, covs, out, num_points, min_deg, max_deg, (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

int mipnerf_b200_pos_enc(const float* x, int64_t num_points, int min_deg, int max_deg, int append_identity,
                         float* out, void* stream) {
  const bool empty = max_deg == min_deg && !append_identity;  // an [M, 0] output: nothing to read or write
  if (num_points < 0 || max_deg < min_deg || min_deg < -60 || max_deg > 60 ||
      (num_points > 0 && !empty && (!x || !out)))
    return fail(MIPNERF_B200_EINVAL, "bad argument");
  CUDA_TRY(mipnerf::launch_pos_enc(x, out, num_points, min_deg, max_deg, append_identity, (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

int mipnerf_b200_mlp_forward(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w, const float* x,
                             const float* view_enc, int64_t num_rays, int samples_per_ray, int precision,
                             float* raw_rgb, float* raw_density, void* workspace, size_t workspace_bytes,
                             void* stream) {
  Dims d;
  int rc;
  mipnerf_b200_config c2;
  if (!cfg) return fail(MIPNERF_B200_EINVAL, "config is NULL");
  c2 = *cfg;
  c2.num_samples = 32;  // the MLP itself does not care; validate the rest
  if ((rc = check_config(&c2, &d))) return rc;
  if ((rc = check_weights(cfg, d, w))) return rc;
  if (num_rays < 0 || samples_per_ray < 1) return fail(MIPNERF_B200_EINVAL, "bad sizes");
  if (num_rays == 0) return MIPNERF_B200_OK;
  if (!x || !raw_rgb || !raw_density || (cfg->use_viewdirs && !view_enc))
    return fail(MIPNERF_B200_EINVAL, "NULL tensor");
  cudaStream_t st = (cudaStream_t)stream;
  c2.num_samples = samples_per_ray;
  if (precision != MIPNERF_B200_FP32) {
    if (!mipnerf::tc_mlp_supported(cfg, samples_per_ray, precision))
      return fail(MIPNERF_B200_EUNSUPPORTED, "tensor-core MLP: default 8x256 model, 128 samples/ray only");
    if ((rc = check_tc(&c2, w, precision, "MLP"))) return rc;
    if (!workspace || workspace_bytes < mipnerf::tc_mlp_workspace_bytes(num_rays))
      return fail(MIPNERF_B200_EWORKSPACE, "workspace %zu < %zu bytes", workspace_bytes,
                  mipnerf::tc_mlp_workspace_bytes(num_rays));
    cudaError_t e = mipnerf::tc_mlp_forward(cfg, w, x, view_enc, num_rays, precision, raw_rgb, raw_density, workspace,
                                            st);
    if (e != cudaSuccess) return fail(MIPNERF_B200_ECUDA, "tc_mlp_forward: %s", cudaGetErrorString(e));
    return MIPNERF_B200_OK;
  }
  const int64_t per = std::max<int64_t>(kChunkRaysFp32 * 128 / samples_per_ray, 1);
  const size_t need = mipnerf_b200_mlp_workspace_bytes(cfg, num_rays, samples_per_ray, precision);
  if (!workspace || workspace_bytes < need)
    return fail(MIPNERF_B200_EWORKSPACE, "workspace %zu < %zu bytes", workspace_bytes, need);
  for (int64_t off = 0; off < num_rays; off += per) {
    const int64_t cnt = (num_rays - off) < per ? (num_rays - off) : per;
    const Fp32Scratch s = carve_fp32(&c2, d, cnt, workspace, /*mlp_only=*/true);
    const int64_t row = off * samples_per_ray;
    if ((rc = mlp_forward_fp32(cfg, d, w, x + row * d.xyz_dim, view_enc ? view_enc + off * d.view_dim : nullptr,
                               cnt, samples_per_ray, s, raw_rgb + row * 3, raw_density + row, st)))
      return rc;
  }
  return MIPNERF_B200_OK;
}

size_t mipnerf_b200_mlp_workspace_bytes(const mipnerf_b200_config* cfg, int64_t num_rays, int samples_per_ray,
                                        int precision) {
  Dims d;
  if (!cfg || num_rays < 0 || samples_per_ray < 1) return 0;
  mipnerf_b200_config c2 = *cfg;
  c2.num_samples = 32;
  if (check_config(&c2, &d) != MIPNERF_B200_OK) return 0;
  if (precision != MIPNERF_B200_FP32) return mipnerf::tc_mlp_workspace_bytes(num_rays);
  c2.num_samples = samples_per_ray;
  const int64_t per = std::clamp<int64_t>(num_rays, 1, std::max<int64_t>(kChunkRaysFp32 * 128 / samples_per_ray, 1));
  return carve_fp32(&c2, d, per, nullptr, true).bytes;
}

int mipnerf_b200_volumetric_rendering(const float* rgb, const float* density, const float* t_samples,
                                      const float* dirs, int64_t num_rays, int num_samples, int white_bkgd,
                                      float* comp_rgb, float* distance, float* acc, float* weights,
                                      void* stream) {
  if (num_rays < 0 || num_samples < 1) return fail(MIPNERF_B200_EINVAL, "bad sizes");
  // the kernel reads each ray's rows with a compile-time stride: any other count would be read as a smaller one
  if (int rc = check_num_samples(num_samples)) return rc;
  if (num_rays == 0) return MIPNERF_B200_OK;
  if (!rgb || !density || !t_samples || !dirs || !comp_rgb || !distance || !acc)
    return fail(MIPNERF_B200_EINVAL, "NULL tensor");
  CUDA_TRY(mipnerf::launch_composite(rgb, density, t_samples, dirs, comp_rgb, distance, acc, weights, num_rays,
                                     num_samples, white_bkgd, 0, 0.f, 1.f, 0.f, (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

int mipnerf_b200_sorted_piecewise_constant_pdf(const float* bins, const float* weights, int64_t num_rays,
                                               int num_bins, int num_samples, int randomized,
                                               const float* u_jitter, float* samples, int64_t* inds,
                                               void* stream) {
  if (num_rays < 0 || num_bins < 1 || num_samples < 2) return fail(MIPNERF_B200_EINVAL, "bad sizes");
  if (num_bins % 32 != 0 || num_bins > kMaxResampleBins)
    return fail(MIPNERF_B200_EUNSUPPORTED, "num_bins=%d: need a multiple of 32, <= %d", num_bins, kMaxResampleBins);
  if (num_rays == 0) return MIPNERF_B200_OK;
  if (!bins || !weights || !samples || (randomized && !u_jitter)) return fail(MIPNERF_B200_EINVAL, "NULL tensor");
  CUDA_TRY(mipnerf::launch_resample(bins, weights, mipnerf::draws_from_array(randomized ? u_jitter : nullptr), samples,
                                    inds, num_rays, num_bins, num_samples, randomized, 0, 0.f, (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

int mipnerf_b200_resample_along_rays(const mipnerf_b200_rays* rays, const float* t_samples, const float* weights,
                                     int num_samples, int randomized, const float* u_jitter,
                                     float resample_padding, float* new_t_samples, float* means, float* covs,
                                     int64_t* inds, void* stream) {
  int rc;
  if ((rc = check_rays(rays))) return rc;
  if (num_samples < 32 || num_samples % 32 != 0 || num_samples > kMaxResampleBins)
    return fail(MIPNERF_B200_EUNSUPPORTED, "num_samples=%d: need a multiple of 32, <= %d", num_samples,
                kMaxResampleBins);
  if (rays->num_rays == 0) return MIPNERF_B200_OK;
  if (!t_samples || !weights || !new_t_samples || (randomized && !u_jitter))
    return fail(MIPNERF_B200_EINVAL, "NULL tensor");
  cudaStream_t st = (cudaStream_t)stream;
  CUDA_TRY(mipnerf::launch_resample(t_samples, weights, mipnerf::draws_from_array(randomized ? u_jitter : nullptr),
                                    new_t_samples, inds, rays->num_rays, num_samples, num_samples + 1, randomized, 1,
                                    resample_padding, st));
  if (means && covs)
    CUDA_TRY(mipnerf::launch_cast_rays(rays->origins, rays->directions, rays->radii, new_t_samples, means,
                                       covs, rays->num_rays, num_samples, st));
  return MIPNERF_B200_OK;
}

// ---- density queries and isosurface extraction ----------------------------------------------------
namespace {
// the fp32 density query runs as many points per chunk as the fp32 forward has samples per chunk
constexpr int64_t kChunkPointsFp32 = kChunkRaysFp32 * 128;

struct DensityScratch {
  float *zero_covs, *enc, *h0, *h1, *raw;
  size_t bytes;
};
DensityScratch carve_density(const mipnerf_b200_config* c, const Dims& d, int64_t m, void* base) {
  DensityScratch s{};
  Carver cv{base};
  s.zero_covs = cv.floats((size_t)m * 3);
  s.enc = cv.floats((size_t)m * d.xyz_dim);
  s.h0 = cv.floats((size_t)m * c->net_width);
  s.h1 = cv.floats((size_t)m * c->net_width);
  s.raw = cv.floats((size_t)m);
  s.bytes = cv.off;
  return s;
}

// The arguments every field query checks first: config, weights, point count, means and precision.
int check_query(const mipnerf_b200_config* c, Dims* d, const mipnerf_b200_weights* w, int64_t num_points,
                const float* means, int precision) {
  int rc;
  if ((rc = check_config(c, d))) return rc;
  if ((rc = check_weights(c, *d, w))) return rc;
  if (num_points < 0) return fail(MIPNERF_B200_EINVAL, "num_points=%lld", (long long)num_points);
  if (num_points > 0 && !means) return fail(MIPNERF_B200_EINVAL, "means is NULL");
  if (precision < MIPNERF_B200_FP32 || precision > MIPNERF_B200_BF16X3)
    return fail(MIPNERF_B200_EINVAL, "precision %d", precision);
  return MIPNERF_B200_OK;
}

// The IPE stage kernel on query points [off, off + m) into enc (models/mip.py:322-350): their covariances, or zero
// ones in zero_covs when covs is NULL or integration is disabled.
int query_ipe_fp32(const mipnerf_b200_config* c, const float* means, const float* covs, int64_t off, int64_t m,
                   float* zero_covs, float* enc, cudaStream_t st) {
  const float* cv = covs ? covs + off * 3 : nullptr;
  if (!cv || c->disable_integration) {
    CUDA_TRY(cudaMemsetAsync(zero_covs, 0, (size_t)m * 3 * sizeof(float), st));
    cv = zero_covs;
  }
  CUDA_TRY(mipnerf::launch_ipe(means + off * 3, cv, enc, m, c->min_deg_point, c->max_deg_point, st));
  return MIPNERF_B200_OK;
}

// The density of m points from their IPE features (models/mip_nerf.py:93-98, 237): the fp32 trunk in h0 / h1 (*h: its
// output), density_layer into raw and, unless density is NULL, the softplus into density.
int density_fp32(const mipnerf_b200_config* c, const Dims& d, const mipnerf_b200_weights* w, const float* enc,
                 int64_t m, float* h0, float* h1, const float** h, float* raw, float* density, cudaStream_t st) {
  int rc;
  if ((rc = trunk_fp32(c, d, w, enc, m, h0, h1, h, st))) return rc;
  const mipnerf_b200_linear& dl = w->linears[c->net_depth];
  CUDA_TRY(mipnerf::launch_linear_f32(*h, c->net_width, c->net_width, nullptr, 0, 0, 1, dl.weight, dl.bias, raw, 1, m,
                                      1, 0, st));
  if (density) CUDA_TRY(mipnerf::launch_density_activation(raw, density, m, c->density_bias, st));
  return MIPNERF_B200_OK;
}
}  // namespace

size_t mipnerf_b200_density_workspace_bytes(const mipnerf_b200_config* cfg, int64_t num_points, int precision) {
  Dims d;
  if (check_config(cfg, &d) != MIPNERF_B200_OK || num_points < 0 || precision != MIPNERF_B200_FP32) return 0;
  return carve_density(cfg, d, std::clamp<int64_t>(num_points, 1, kChunkPointsFp32), nullptr).bytes;
}

int mipnerf_b200_query_density(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w, const float* means,
                               const float* covs, int64_t num_points, int precision, float* raw_density,
                               float* density, void* workspace, size_t workspace_bytes, void* stream) {
  Dims d;
  int rc;
  if ((rc = check_query(cfg, &d, w, num_points, means, precision))) return rc;
  if (!raw_density && !density) return fail(MIPNERF_B200_EINVAL, "raw_density and density are both NULL");
  if (precision != MIPNERF_B200_FP32 && (rc = check_tc(cfg, w, precision, "density query"))) return rc;
  const size_t need = mipnerf_b200_density_workspace_bytes(cfg, num_points, precision);
  if (num_points > 0 && need > 0 && (!workspace || workspace_bytes < need))
    return fail(MIPNERF_B200_EWORKSPACE, "workspace %zu < %zu bytes", workspace_bytes, need);
  if (num_points == 0) return MIPNERF_B200_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (precision != MIPNERF_B200_FP32) {
    cudaError_t e = mipnerf::tc_query_density(cfg, w, means, covs, num_points, precision, raw_density, density, st);
    if (e != cudaSuccess) return fail(MIPNERF_B200_ECUDA, "tc_query_density: %s", cudaGetErrorString(e));
    return MIPNERF_B200_OK;
  }
  for (int64_t off = 0; off < num_points; off += kChunkPointsFp32) {
    const int64_t m = std::min(num_points - off, kChunkPointsFp32);
    const DensityScratch s = carve_density(cfg, d, m, workspace);
    const float* h;
    if ((rc = query_ipe_fp32(cfg, means, covs, off, m, s.zero_covs, s.enc, st))) return rc;
    if ((rc = density_fp32(cfg, d, w, s.enc, m, s.h0, s.h1, &h, raw_density ? raw_density + off : s.raw,
                           density ? density + off : nullptr, st)))
      return rc;
  }
  return MIPNERF_B200_OK;
}

namespace {
struct RadianceScratch {
  float *zero_covs, *enc, *venc, *raw_rgb, *raw_density;
  Fp32Scratch mlp;  // h0, h1, c0, c1 of mlp_forward_fp32
  size_t bytes;
};
RadianceScratch carve_radiance(const mipnerf_b200_config* c, const Dims& d, int64_t m, void* base) {
  RadianceScratch s{};
  Carver cv{base};
  s.zero_covs = cv.floats((size_t)m * 3);
  s.enc = cv.floats((size_t)m * d.xyz_dim);
  s.venc = cv.floats((size_t)m * d.view_dim);
  s.raw_rgb = cv.floats((size_t)m * 3);
  s.raw_density = cv.floats((size_t)m);
  s.mlp.h0 = cv.floats((size_t)m * c->net_width);
  s.mlp.h1 = cv.floats((size_t)m * c->net_width);
  s.mlp.c0 = cv.floats((size_t)m * c->net_width_condition);
  s.mlp.c1 = cv.floats((size_t)m * c->net_width_condition);
  s.bytes = cv.off;
  return s;
}
}  // namespace

size_t mipnerf_b200_radiance_workspace_bytes(const mipnerf_b200_config* cfg, int64_t num_points, int precision) {
  Dims d;
  if (check_config(cfg, &d) != MIPNERF_B200_OK || num_points < 0) return 0;
  if (precision != MIPNERF_B200_FP32)
    return mipnerf::tc_supported(cfg, precision) ? mipnerf::tc_radiance_workspace_bytes(num_points) : 0;
  return carve_radiance(cfg, d, std::clamp<int64_t>(num_points, 1, kChunkPointsFp32), nullptr).bytes;
}

int mipnerf_b200_query_radiance(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w, const float* means,
                                const float* covs, const float* viewdirs, int64_t num_points, int precision,
                                float* raw_rgb, float* raw_density, float* rgb, float* density, void* workspace,
                                size_t workspace_bytes, void* stream) {
  Dims d;
  int rc;
  if ((rc = check_query(cfg, &d, w, num_points, means, precision))) return rc;
  if (!raw_rgb && !raw_density && !rgb && !density) return fail(MIPNERF_B200_EINVAL, "every output is NULL");
  if (num_points > 0 && cfg->use_viewdirs && !viewdirs)
    return fail(MIPNERF_B200_EINVAL, "viewdirs is NULL with use_viewdirs");
  if (precision != MIPNERF_B200_FP32 && (rc = check_tc(cfg, w, precision, "radiance query"))) return rc;
  const size_t need = mipnerf_b200_radiance_workspace_bytes(cfg, num_points, precision);
  if (num_points > 0 && (need == 0 || !workspace || workspace_bytes < need))
    return fail(MIPNERF_B200_EWORKSPACE, "workspace %zu < %zu bytes", workspace_bytes, need);
  if (num_points == 0) return MIPNERF_B200_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (precision != MIPNERF_B200_FP32) {
    cudaError_t e = mipnerf::tc_query_radiance(cfg, w, means, covs, viewdirs, num_points, precision, raw_rgb,
                                               raw_density, rgb, density, workspace, workspace_bytes, st);
    if (e != cudaSuccess) return fail(MIPNERF_B200_ECUDA, "tc_query_radiance: %s", cudaGetErrorString(e));
    return MIPNERF_B200_OK;
  }
  // fp32: the IPE stage kernel, the view-direction encoding and the fp32 MLP with one sample per "ray" (each point its
  // own view encoding), then the activations (models/mip.py:322-363, models/mip_nerf.py:75-111, 236-237)
  const float rgb_scale = mipnerf::rgb_scale_of(cfg);
  for (int64_t off = 0; off < num_points; off += kChunkPointsFp32) {
    const int64_t m = std::min(num_points - off, kChunkPointsFp32);
    const RadianceScratch s = carve_radiance(cfg, d, m, workspace);
    if ((rc = query_ipe_fp32(cfg, means, covs, off, m, s.zero_covs, s.enc, st))) return rc;
    if (cfg->use_viewdirs) CUDA_TRY(mipnerf::launch_pos_enc(viewdirs + off * 3, s.venc, m, 0, cfg->deg_view, 1, st));
    float* rr = raw_rgb ? raw_rgb + off * 3 : s.raw_rgb;
    float* rd = raw_density ? raw_density + off : s.raw_density;
    if ((rc = mlp_forward_fp32(cfg, d, w, s.enc, cfg->use_viewdirs ? s.venc : nullptr, m, 1, s.mlp, rr, rd, st)))
      return rc;
    CUDA_TRY(mipnerf::launch_radiance_activation(rr, rd, rgb ? rgb + off * 3 : nullptr, density ? density + off : nullptr,
                                                 m, cfg->density_bias, rgb_scale, cfg->rgb_padding, st));
  }
  return MIPNERF_B200_OK;
}

namespace {
// Radiance under a shared direction set: per chunk of m points, the view layer's accumulators A [m rounded up to a
// 128-point tile][128] (W_view[:, :width] . bottleneck), and once per call the direction terms T [D][128]; fp32 adds
// the IPE, trunk and bottleneck activations, the raw densities and the zero bias / zero view row that let
// launch_linear_f32 compute A from the view layer's own weights.
struct RadianceDirsScratch {
  float *acc, *terms, *zero_covs, *enc, *h0, *h1, *raw, *zeros;
  size_t bytes;
};
RadianceDirsScratch carve_radiance_dirs(const mipnerf_b200_config* c, const Dims& d, int64_t m, int64_t num_dirs,
                                        int precision, void* base) {
  RadianceDirsScratch s{};
  Carver cv{base};
  s.acc = cv.floats((size_t)((m + 127) / 128 * 128) * c->net_width_condition);
  s.terms = cv.floats((size_t)num_dirs * c->net_width_condition);
  if (precision == MIPNERF_B200_FP32) {
    s.zero_covs = cv.floats((size_t)m * 3);
    s.enc = cv.floats((size_t)m * d.xyz_dim);
    s.h0 = cv.floats((size_t)m * c->net_width);
    s.h1 = cv.floats((size_t)m * c->net_width);
    s.raw = cv.floats((size_t)m);
    s.zeros = cv.floats((size_t)c->net_width_condition + d.view_dim);
  }
  s.bytes = cv.off;
  return s;
}
// the view layer splits into a per-point and a per-direction part only when it is the one layer before the colour head,
// 128 wide (the pair kernel's width)
bool radiance_dirs_supported(const mipnerf_b200_config* c, int precision) {
  if (precision != MIPNERF_B200_FP32) return mipnerf::tc_supported(c, precision);
  return c->use_viewdirs && c->net_depth_condition == 1 && c->net_width_condition == 128;
}
}  // namespace

size_t mipnerf_b200_radiance_dirs_workspace_bytes(const mipnerf_b200_config* cfg, int64_t num_points, int64_t num_dirs,
                                                  int precision) {
  Dims d;
  if (check_config(cfg, &d) != MIPNERF_B200_OK || num_points < 0 || num_dirs < 1 ||
      precision < MIPNERF_B200_FP32 || precision > MIPNERF_B200_BF16X3 || !radiance_dirs_supported(cfg, precision))
    return 0;
  return carve_radiance_dirs(cfg, d, std::clamp<int64_t>(num_points, 1, kChunkPointsFp32), num_dirs, precision, nullptr)
      .bytes;
}

int mipnerf_b200_query_radiance_dirs(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w, const float* means,
                                     const float* covs, int64_t num_points, const float* dirs, int64_t num_dirs,
                                     int precision, float* raw_rgb, float* rgb, float* raw_density, float* density,
                                     const float* table, int num_basis, int proj_raw, float* proj_out,
                                     void* workspace, size_t workspace_bytes, void* stream) {
  static_assert(kChunkPointsFp32 == mipnerf::kDensityChunkPoints, "one chunk size for every precision");
  Dims d;
  int rc;
  if ((rc = check_query(cfg, &d, w, num_points, means, precision))) return rc;
  if (num_dirs < 1) return fail(MIPNERF_B200_EINVAL, "num_dirs=%lld: need at least one direction", (long long)num_dirs);
  if (!raw_rgb && !rgb && !raw_density && !density && !proj_out) return fail(MIPNERF_B200_EINVAL, "every output is NULL");
  if (proj_out && !table) return fail(MIPNERF_B200_EINVAL, "proj_out without table");
  if (proj_out && (num_basis < 1 || num_basis > 16))
    return fail(MIPNERF_B200_EINVAL, "num_basis=%d: need 1..16 with proj_out", num_basis);
  if (!dirs) return fail(MIPNERF_B200_EINVAL, "dirs is NULL");
  if (!cfg->use_viewdirs)
    return fail(MIPNERF_B200_EUNSUPPORTED, "radiance under a direction set needs use_viewdirs (use query_radiance)");
  if (precision != MIPNERF_B200_FP32) {
    if ((rc = check_tc(cfg, w, precision, "radiance query"))) return rc;
  } else if (!radiance_dirs_supported(cfg, precision)) {
    return fail(MIPNERF_B200_EUNSUPPORTED, "radiance under a direction set: one 128-wide view layer only");
  }
  const size_t need = mipnerf_b200_radiance_dirs_workspace_bytes(cfg, num_points, num_dirs, precision);
  if (num_points > 0 && (need == 0 || !workspace || workspace_bytes < need))
    return fail(MIPNERF_B200_EWORKSPACE, "workspace %zu < %zu bytes", workspace_bytes, need);
  if (num_points == 0) return MIPNERF_B200_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const float rgb_scale = mipnerf::rgb_scale_of(cfg);
  const mipnerf_b200_linear& vl = w->linears[cfg->net_depth + 2];
  const mipnerf_b200_linear& cl = w->linears[d.n_lin - 1];
  const RadianceDirsScratch s0 =
      carve_radiance_dirs(cfg, d, std::min(num_points, kChunkPointsFp32), num_dirs, precision, workspace);
  // T: radiance mode's view-direction term of each direction (the tensor-core precisions), or the same sum over the
  // view layer's own weights (fp32)
  if (precision != MIPNERF_B200_FP32) {
    cudaError_t e = mipnerf::tc_view_terms(w, dirs, num_dirs, s0.terms, st);
    if (e != cudaSuccess) return fail(MIPNERF_B200_ECUDA, "tc_view_terms: %s", cudaGetErrorString(e));
  } else {
    CUDA_TRY(mipnerf::launch_view_terms(dirs, num_dirs, vl.weight + cfg->net_width, 1, cfg->net_width + d.view_dim,
                                        vl.bias, d.view_dim, cfg->deg_view, s0.terms, st));
    CUDA_TRY(cudaMemsetAsync(s0.zeros, 0, (size_t)(cfg->net_width_condition + d.view_dim) * sizeof(float), st));
  }
  for (int64_t off = 0; off < num_points; off += kChunkPointsFp32) {
    const int64_t m = std::min(num_points - off, kChunkPointsFp32);
    const RadianceDirsScratch& s = s0;  // every chunk reuses the first one's scratch, in stream order
    if (precision != MIPNERF_B200_FP32) {
      cudaError_t e = mipnerf::tc_query_view_acc(cfg, w, means + off * 3, covs ? covs + off * 3 : nullptr, m, precision,
                                                 s.acc, raw_density ? raw_density + off : nullptr,
                                                 density ? density + off : nullptr, st);
      if (e != cudaSuccess) return fail(MIPNERF_B200_ECUDA, "tc_query_view_acc: %s", cudaGetErrorString(e));
    } else {
      // the IPE stage kernel, the fp32 trunk, density_layer and extra_layer, then A = [bottleneck | 0] . W_view^T + 0:
      // the view layer's sum over its bottleneck columns (models/mip.py:322-350, models/mip_nerf.py:93-107)
      const float* h;
      if ((rc = query_ipe_fp32(cfg, means, covs, off, m, s.zero_covs, s.enc, st))) return rc;
      if ((rc = density_fp32(cfg, d, w, s.enc, m, s.h0, s.h1, &h, raw_density ? raw_density + off : s.raw,
                             density ? density + off : nullptr, st)))
        return rc;
      const mipnerf_b200_linear& el = w->linears[cfg->net_depth + 1];
      float* bott = h == s.h0 ? s.h1 : s.h0;
      CUDA_TRY(mipnerf::launch_linear_f32(h, cfg->net_width, cfg->net_width, nullptr, 0, 0, 1, el.weight, el.bias, bott,
                                          cfg->net_width, m, cfg->net_width, 0, st));
      CUDA_TRY(mipnerf::launch_linear_f32(bott, cfg->net_width, cfg->net_width, s.zeros + cfg->net_width_condition,
                                          d.view_dim, d.view_dim, (int)m, vl.weight, s.zeros, s.acc,
                                          cfg->net_width_condition, m, cfg->net_width_condition, 0, st));
    }
    CUDA_TRY(mipnerf::launch_radiance_pairs(
        s.acc, s.terms, cl.weight, cl.bias, m, num_dirs, rgb_scale, cfg->rgb_padding,
        raw_rgb ? raw_rgb + off * num_dirs * 3 : nullptr, rgb ? rgb + off * num_dirs * 3 : nullptr, table, num_basis,
        proj_raw, proj_out ? proj_out + off * num_basis * 3 : nullptr, st));
  }
  return MIPNERF_B200_OK;
}

namespace {
// Scratch of the bf16 query backward for one chunk of m points: the fused step's chain over whole tiles, its act / v
// the level kernel's query dump (h_0..h_7 and, radiance, the bottleneck; the view layer), and the raw heads.
struct QueryFusedScratch {
  FusedHead head;
  float* slots;  // radiance mode's view-direction terms, chunk-invariant too
  float *raw_rgb, *raw_density;
  TileChainOps chain;
  size_t slots_bytes, bytes;
};
QueryFusedScratch carve_query_fused(const mipnerf_b200_config* c, const Dims& d, int64_t m, bool radiance,
                                    void* base) {
  QueryFusedScratch s{};
  Carver cv{base};
  s.head = carve_fused_head(cv, c, d, MIPNERF_B200_BF16, kMaxTrainDepth + 2);
  s.slots_bytes = radiance ? mipnerf::tc_radiance_workspace_bytes(mipnerf::kDensityChunkPoints) : 0;
  s.slots = reinterpret_cast<float*>(cv.bytes(s.slots_bytes));
  s.chain = carve_tile_chain(cv, d, MIPNERF_B200_BF16, m, 1, radiance);
  s.chain.part = s.head.part;
  s.chain.act = cv.bytes((size_t)(radiance ? 9 : 8) * s.chain.tiles * 65536);
  s.raw_density = cv.floats((size_t)s.chain.tiles * 128);
  if (radiance) {
    s.chain.v = cv.bytes((size_t)s.chain.tiles * 32768);
    s.raw_rgb = cv.floats((size_t)s.chain.tiles * 128 * 3);
  }
  s.bytes = cv.off;
  return s;
}

// The configs the query backward takes: those of the training chain, and on the tensor cores (BF16) the default
// architecture and encodings (the tile images of the fused step's chain carry the full 96 / 27 encodings).
bool query_grad_supported(const mipnerf_b200_config* c, const Dims& d, int precision) {
  if (check_train_config(c) != MIPNERF_B200_OK) return false;
  if (precision == MIPNERF_B200_FP32) return true;
  return precision == MIPNERF_B200_BF16 && mipnerf::tc_supported(c, precision) && mipnerf::tc_default_degrees(c) &&
         c->net_depth == 8 && train_tc_supported(c, d);
}

// The cotangents of chunk [off, off + m) (radiance: all four; density: the density ones)
mipnerf::QueryCot chunk_cot(const mipnerf_b200_query_cotangent* cot, int64_t off, bool radiance) {
  return mipnerf::QueryCot{radiance && cot->d_raw_rgb ? cot->d_raw_rgb + off * 3 : nullptr,
                           cot->d_raw_density ? cot->d_raw_density + off : nullptr,
                           radiance && cot->d_rgb ? cot->d_rgb + off * 3 : nullptr,
                           cot->d_density ? cot->d_density + off : nullptr};
}

// fp32: the IPE stage kernel, pos_enc, the fp32 MLP with its activations kept and the per-layer chain
int query_backward_fp32(const mipnerf_b200_config* cfg, const Dims& d, const mipnerf_b200_weights* w,
                        const float* means, const float* covs, const float* viewdirs, int64_t num_points,
                        const mipnerf_b200_query_cotangent* cot, const mipnerf_b200_linear_grad* grads, bool* touched,
                        void* workspace, cudaStream_t st) {
  const bool radiance = viewdirs != nullptr;
  const float rgb_scale = mipnerf::rgb_scale_of(cfg);
  const LayerImages im{};
  int rc;
  for (int64_t off = 0; off < num_points; off += kChunkPointsFp32) {
    const int64_t m = std::min(num_points - off, kChunkPointsFp32);
    const TrainScratch s = carve_train(cfg, d, m, 0, radiance, workspace);
    float* zero_covs = Carver{workspace, s.bytes}.floats((size_t)m * 3);
    // the forward of the query (models/mip.py:322-363, models/mip_nerf.py:75-111), every activation kept
    if ((rc = query_ipe_fp32(cfg, means, covs, off, m, zero_covs, s.enc, st))) return rc;
    if (radiance) CUDA_TRY(mipnerf::launch_pos_enc(viewdirs + off * 3, s.venc, m, 0, cfg->deg_view, 1, st));
    if ((rc = mlp_forward_kept(cfg, d, w, false, MIPNERF_B200_FP32, im, s, m, 1, !radiance, st))) return rc;
    // the activations' VJP, then the training step's per-layer chain
    CUDA_TRY(mipnerf::launch_query_activation_vjp(s.raw_rgb, s.raw_density, chunk_cot(cot, off, radiance),
                                                  cfg->density_bias, rgb_scale, s.d_raw_rgb, s.d_raw_density, m, st));
    if ((rc = mlp_backward_chain(cfg, d, w, false, MIPNERF_B200_FP32, im, s, m, 1, !radiance, grads, touched, st)))
      return rc;
  }
  return MIPNERF_B200_OK;
}

// bf16: the query itself on the level kernel with the training dump (its outputs are the raw heads the VJP takes the
// activations' derivatives at), the IPE of the points as a tile image, then the fused training step's tile-image chain
int query_backward_bf16(const mipnerf_b200_config* cfg, const Dims& d, const mipnerf_b200_weights* w,
                        const float* means, const float* covs, const float* viewdirs, int64_t num_points,
                        const mipnerf_b200_query_cotangent* cot, const mipnerf_b200_linear_grad* grads, bool* touched,
                        void* workspace, cudaStream_t st) {
  const bool radiance = viewdirs != nullptr;
  const int prec = MIPNERF_B200_BF16;
  const float rgb_scale = mipnerf::rgb_scale_of(cfg);
  const int64_t chunk = mipnerf::kDensityChunkPoints;
  mipnerf_b200_weights wl;
  LayerImages im;
  int rc;
  if ((rc = pack_fused_weights(cfg, d, w, prec,
                               carve_query_fused(cfg, d, std::min(num_points, chunk), radiance, workspace).head, &wl,
                               &im, st)))
    return rc;
  for (int64_t off = 0; off < num_points; off += chunk) {
    const int64_t m = std::min(num_points - off, chunk);
    const QueryFusedScratch s = carve_query_fused(cfg, d, m, radiance, workspace);
    const TileChainOps& o = s.chain;
    const float* mp = means + off * 3;
    const float* cv = covs ? covs + off * 3 : nullptr;
    const mipnerf::TcQueryDump dump{o.act, o.v};
    cudaError_t e = radiance ? mipnerf::tc_query_radiance(cfg, &wl, mp, cv, viewdirs + off * 3, m, prec, s.raw_rgb,
                                                          s.raw_density, nullptr, nullptr, s.slots, s.slots_bytes, st,
                                                          &dump)
                             : mipnerf::tc_query_density(cfg, &wl, mp, cv, m, prec, s.raw_density, nullptr, st, &dump);
    if (e != cudaSuccess) return fail(MIPNERF_B200_ECUDA, "query backward, forward: %s", cudaGetErrorString(e));
    CUDA_TRY(mipnerf::launch_ipe_points_t16(mp, cv, o.enc16, m, cfg->disable_integration, prec, st));
    if (radiance) CUDA_TRY(mipnerf::launch_pos_enc(viewdirs + off * 3, o.venc, m, 0, cfg->deg_view, 1, st));
    CUDA_TRY(mipnerf::launch_query_activation_vjp(s.raw_rgb, s.raw_density, chunk_cot(cot, off, radiance),
                                                  cfg->density_bias, rgb_scale, o.d_raw_rgb, o.d_raw_density, m, st));
    if ((rc = tile_backward_chain(cfg, d, w, prec, im, o, !radiance, 1.f, grads, touched, st))) return rc;
  }
  return MIPNERF_B200_OK;
}
}  // namespace

size_t mipnerf_b200_query_backward_workspace_bytes(const mipnerf_b200_config* cfg, int64_t num_points, int radiance,
                                                   int precision) {
  Dims d;
  if (check_config(cfg, &d) != MIPNERF_B200_OK || num_points < 0 || !query_grad_supported(cfg, d, precision)) return 0;
  const int64_t m = std::clamp<int64_t>(num_points, 1, kChunkPointsFp32);
  if (precision == MIPNERF_B200_BF16) return carve_query_fused(cfg, d, m, radiance != 0, nullptr).bytes;
  return carve_train(cfg, d, m, 0, radiance != 0, nullptr).bytes + align_up((size_t)m * 3 * sizeof(float));
}

int mipnerf_b200_query_backward(const mipnerf_b200_config* cfg, const mipnerf_b200_weights* w, const float* means,
                                const float* covs, const float* viewdirs, int64_t num_points, int precision,
                                const mipnerf_b200_query_cotangent* cot, const mipnerf_b200_linear_grad* grads,
                                int num_grads, int accumulate, void* workspace, size_t workspace_bytes, void* stream) {
  Dims d;
  int rc;
  if ((rc = check_query(cfg, &d, w, num_points, means, precision))) return rc;
  if (!cot || !grads) return fail(MIPNERF_B200_EINVAL, "cot / grads is NULL");
  if ((rc = check_grads(d, grads, num_grads))) return rc;
  if ((rc = check_cotangent_precision(precision, "query backward"))) return rc;
  if ((rc = check_train_config(cfg))) return rc;
  if (!query_grad_supported(cfg, d, precision))
    return fail(MIPNERF_B200_EUNSUPPORTED,
                "query backward in BF16: the 8x256 / 1x128 MLP with max_deg_point=16, deg_view=4 only; use FP32");
  const bool radiance = viewdirs != nullptr;
  const size_t need = mipnerf_b200_query_backward_workspace_bytes(cfg, num_points, radiance, precision);
  if (num_points > 0 && (!workspace || workspace_bytes < need))
    return fail(MIPNERF_B200_EWORKSPACE, "workspace %zu < %zu bytes", workspace_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  bool touched[kMaxTrainDepth + 8];
  std::fill_n(touched, d.n_lin, accumulate != 0);
  if (num_points > 0) {
    auto* driver = precision == MIPNERF_B200_BF16 ? query_backward_bf16 : query_backward_fp32;
    if ((rc = driver(cfg, d, w, means, covs, viewdirs, num_points, cot, grads, touched, workspace, st))) return rc;
  }
  return zero_untouched(d, w, grads, touched, st);
}

size_t mipnerf_b200_isosurface_scratch_bytes(int nx, int ny, int nz) {
  if (nx < 2 || ny < 2 || nz < 2) return 0;
  return mipnerf::isosurface_scratch_bytes(nx, ny, nz);
}

int mipnerf_b200_isosurface_count(const float* grid, int nx, int ny, int nz, float iso, void* scratch,
                                  size_t scratch_bytes, int64_t* counts, void* stream) {
  if (nx < 2 || ny < 2 || nz < 2) return fail(MIPNERF_B200_EINVAL, "grid %d x %d x %d: need >= 2 per axis", nx, ny, nz);
  if (!grid || !counts) return fail(MIPNERF_B200_EINVAL, "grid / counts is NULL");
  const size_t need = mipnerf::isosurface_scratch_bytes(nx, ny, nz);
  if (!scratch || scratch_bytes < need) return fail(MIPNERF_B200_EWORKSPACE, "scratch %zu < %zu bytes", scratch_bytes, need);
  CUDA_TRY(mipnerf::launch_isosurface_count(grid, nx, ny, nz, iso, scratch, counts, (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

int mipnerf_b200_isosurface_emit(const float* grid, int nx, int ny, int nz, const float* lo_host, const float* hi_host,
                                 float iso, const void* scratch, float* verts, int32_t* faces, void* stream) {
  if (nx < 2 || ny < 2 || nz < 2) return fail(MIPNERF_B200_EINVAL, "grid %d x %d x %d: need >= 2 per axis", nx, ny, nz);
  if (!grid || !lo_host || !hi_host || !scratch) return fail(MIPNERF_B200_EINVAL, "grid / bounds / scratch is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  int64_t totals[2];
  CUDA_TRY(cudaMemcpyAsync(totals, mipnerf::isosurface_totals(scratch), sizeof(totals), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  if (totals[0] > INT32_MAX)
    return fail(MIPNERF_B200_EUNSUPPORTED, "%lld vertices: int32 face indices cannot address them",
                (long long)totals[0]);
  if ((totals[0] > 0 && !verts) || (totals[1] > 0 && !faces)) return fail(MIPNERF_B200_EINVAL, "verts / faces is NULL");
  if (totals[0] == 0) return MIPNERF_B200_OK;
  const int n[3] = {nx, ny, nz};
  float step[3];
  for (int a = 0; a < 3; ++a) step[a] = (hi_host[a] - lo_host[a]) / (float)(n[a] - 1);
  CUDA_TRY(mipnerf::launch_isosurface_emit(grid, nx, ny, nz, lo_host, step, iso, scratch, verts, faces, st));
  return MIPNERF_B200_OK;
}

int mipnerf_b200_isosurface_normals(const float* grid, int nx, int ny, int nz, const float* lo_host,
                                    const float* hi_host, float iso, const void* scratch, float* normals, void* stream) {
  if (nx < 2 || ny < 2 || nz < 2) return fail(MIPNERF_B200_EINVAL, "grid %d x %d x %d: need >= 2 per axis", nx, ny, nz);
  if (!grid || !lo_host || !hi_host || !scratch) return fail(MIPNERF_B200_EINVAL, "grid / bounds / scratch is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  int64_t totals[2];
  CUDA_TRY(cudaMemcpyAsync(totals, mipnerf::isosurface_totals(scratch), sizeof(totals), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  if (totals[0] > 0 && !normals) return fail(MIPNERF_B200_EINVAL, "normals is NULL");
  if (totals[0] == 0) return MIPNERF_B200_OK;
  const int n[3] = {nx, ny, nz};
  float step[3];
  for (int a = 0; a < 3; ++a) step[a] = (hi_host[a] - lo_host[a]) / (float)(n[a] - 1);
  CUDA_TRY(mipnerf::launch_isosurface_normals(grid, nx, ny, nz, step, iso, scratch, normals, st));
  return MIPNERF_B200_OK;
}

int mipnerf_b200_grid_render(const mipnerf_b200_grid* g, const mipnerf_b200_rays* rays, float step, int white_bkgd,
                             float* rgb, float* distance, float* acc, void* stream) {
  int rc;
  float* const out[3] = {rgb, distance, acc};
  if ((rc = check_march(g, rays, out, step, nullptr))) return rc;
  CUDA_TRY(mipnerf::launch_grid_render(*g, nullptr, nullptr, *rays, step, white_bkgd, rgb, distance, acc,
                                       mipnerf::kKernGridRender, (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

int mipnerf_b200_grid_render_u8(const mipnerf_b200_grid* g, const mipnerf_b200_grid_sh_u8* sh,
                                const mipnerf_b200_rays* rays, float step, int white_bkgd, float* rgb, float* distance,
                                float* acc, void* stream) {
  int rc;
  float* const out[3] = {rgb, distance, acc};
  if ((rc = check_march(g, rays, out, step, nullptr))) return rc;
  if (!sh) return fail(MIPNERF_B200_EINVAL, "sh is NULL");
  if ((rc = check_sh_u8(g, sh))) return rc;
  CUDA_TRY(mipnerf::launch_grid_render(*g, nullptr, sh, *rays, step, white_bkgd, rgb, distance, acc,
                                       mipnerf::kKernGridRenderU8, (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

int mipnerf_b200_grid_render_bricks(const mipnerf_b200_grid* g, const mipnerf_b200_grid_bricks* bricks,
                                    const mipnerf_b200_grid_sh_u8* sh_u8, const mipnerf_b200_rays* rays, float step,
                                    int white_bkgd, float* rgb, float* distance, float* acc, void* stream) {
  int rc;
  float* const out[3] = {rgb, distance, acc};
  if ((rc = check_march(g, rays, out, step, &bricks))) return rc;
  if (sh_u8 && (rc = check_sh_u8(g, sh_u8))) return rc;
  CUDA_TRY(mipnerf::launch_grid_render(*g, bricks, sh_u8, *rays, step, white_bkgd, rgb, distance, acc,
                                       mipnerf::kKernGridRenderBricks, (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

int mipnerf_b200_grid_render_backward(const mipnerf_b200_grid* g, const mipnerf_b200_rays* rays, float step,
                                      int white_bkgd, const float* d_rgb, const float* d_distance, const float* d_acc,
                                      const mipnerf_b200_grid_grads* grads, void* stream) {
  int rc;
  if ((rc = check_march(g, rays, nullptr, step, nullptr))) return rc;
  if (!grads) return fail(MIPNERF_B200_EINVAL, "grads is NULL");
  for (int l = 0; l < g->num_levels; ++l)
    if (g->levels[l].sh && (!grads->density[l] || !grads->sh[l]))
      return fail(MIPNERF_B200_EINVAL, "level %d has kept points: grads->density[%d] / grads->sh[%d] is NULL", l, l, l);
  CUDA_TRY(mipnerf::launch_grid_render_backward(*g, *rays, step, white_bkgd, d_rgb, d_distance, d_acc, *grads,
                                                (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

int mipnerf_b200_grid_visibility(const mipnerf_b200_grid* g, const mipnerf_b200_rays* rays, float step,
                                 float* const* max_weight, void* stream) {
  int rc;
  if ((rc = check_march(g, rays, nullptr, step, nullptr))) return rc;
  if (!max_weight) return fail(MIPNERF_B200_EINVAL, "max_weight is NULL");
  for (int l = 0; l < g->num_levels; ++l)
    if (g->levels[l].sh && !max_weight[l])
      return fail(MIPNERF_B200_EINVAL, "level %d has kept points: max_weight[%d] is NULL", l, l);
  CUDA_TRY(mipnerf::launch_grid_visibility(*g, nullptr, *rays, step, max_weight, mipnerf::kKernGridVisibility,
                                           (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

int mipnerf_b200_grid_visibility_bricks(const mipnerf_b200_grid* g, const mipnerf_b200_grid_bricks* bricks,
                                        const mipnerf_b200_rays* rays, float step, float* const* max_weight,
                                        void* stream) {
  int rc;
  if ((rc = check_march(g, rays, nullptr, step, &bricks))) return rc;
  if (!max_weight) return fail(MIPNERF_B200_EINVAL, "max_weight is NULL");
  // a level may have kept points wherever it stores a brick: its rows need not be baked yet, so levels[l].sh cannot
  // tell
  for (int l = 0; l < g->num_levels; ++l)
    if (bricks->pool[l] && !max_weight[l])
      return fail(MIPNERF_B200_EINVAL, "level %d stores bricks: max_weight[%d] is NULL", l, l);
  CUDA_TRY(mipnerf::launch_grid_visibility(*g, bricks, *rays, step, max_weight, mipnerf::kKernGridVisibilityBricks,
                                           (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

int mipnerf_b200_grid_proposal(const mipnerf_b200_grid* g, const mipnerf_b200_grid_bricks* bricks,
                               const mipnerf_b200_rays* rays, const float* t_samples, int num_samples, float* weights,
                               void* stream) {
  int rc;
  if (!g) return fail(MIPNERF_B200_EINVAL, "grid is NULL");
  if ((rc = check_rays(rays))) return rc;
  if (rays->num_rays > 0 && (!t_samples || !weights)) return fail(MIPNERF_B200_EINVAL, "t_samples / weights is NULL");
  if (num_samples < 1 || num_samples > 256)
    return fail(MIPNERF_B200_EINVAL, "num_samples=%d: need 1..256", num_samples);
  if ((rc = check_grid(g, bricks))) return rc;
  CUDA_TRY(mipnerf::launch_grid_proposal(*g, bricks, *rays, t_samples, num_samples, weights, (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

int mipnerf_b200_grid_proposal_backward(const mipnerf_b200_grid* g, const mipnerf_b200_rays* rays,
                                        const float* t_samples, int num_samples, const float* d_weights,
                                        const mipnerf_b200_grid_grads* grads, void* stream) {
  int rc;
  if (!g) return fail(MIPNERF_B200_EINVAL, "grid is NULL");
  if ((rc = check_rays(rays))) return rc;
  if (rays->num_rays > 0 && (!t_samples || !d_weights || !grads))
    return fail(MIPNERF_B200_EINVAL, "t_samples / d_weights / grads is NULL");
  if (num_samples < 1 || num_samples > 256)
    return fail(MIPNERF_B200_EINVAL, "num_samples=%d: need 1..256", num_samples);
  if ((rc = check_grid(g))) return rc;
  if (rays->num_rays == 0) return MIPNERF_B200_OK;
  for (int l = 0; l < g->num_levels; ++l)
    if (g->levels[l].sh && !grads->density[l])
      return fail(MIPNERF_B200_EINVAL, "level %d has kept points: grads->density[%d] is NULL", l, l);
  CUDA_TRY(mipnerf::launch_grid_proposal_backward(*g, *rays, t_samples, num_samples, d_weights, *grads,
                                                  (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

int mipnerf_b200_grid_tv(const mipnerf_b200_grid* g, const int64_t* const* points, const int64_t* num_points,
                         float eps, float* const* tv_density, float* const* tv_sh, const float* weights,
                         const mipnerf_b200_grid_grads* grads, void* stream) {
  int rc;
  if (!g) return fail(MIPNERF_B200_EINVAL, "grid is NULL");
  if ((rc = check_grid(g))) return rc;
  if (!(eps > 0.f) || !std::isfinite(eps)) return fail(MIPNERF_B200_EINVAL, "eps=%g: need a finite eps > 0", eps);
  if (!points || !num_points) return fail(MIPNERF_B200_EINVAL, "points / num_points is NULL");
  if (grads && !weights) return fail(MIPNERF_B200_EINVAL, "grads is set: weights is NULL");
  for (int l = 0; l < g->num_levels; ++l) {
    const mipnerf_b200_grid_level& lv = g->levels[l];
    const int64_t m = num_points[l], n = (int64_t)lv.nx * lv.ny * lv.nz;
    if (m < 0 || m > n)
      return fail(MIPNERF_B200_EINVAL, "level %d: num_points=%lld, need 0..%lld (the lattice's points)", l,
                  (long long)m, (long long)n);
    if (m > 0 && (!lv.sh || !points[l]))
      return fail(MIPNERF_B200_EINVAL, "level %d has %lld kept points: levels[%d].sh / points[%d] is NULL", l,
                  (long long)m, l, l);
  }
  CUDA_TRY(mipnerf::launch_grid_tv(*g, points, num_points, eps, tv_density, tv_sh, weights, grads,
                                   (cudaStream_t)stream));
  return MIPNERF_B200_OK;
}

}  // extern "C"
