// kernels.h — internal (C++) launcher prototypes shared by the translation units of
// libmipnerf_b200.so.  The public surface is include/mipnerf_b200.h.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <type_traits>

#include "draws.h"

struct mipnerf_b200_grid;  // include/mipnerf_b200.h
struct mipnerf_b200_grid_bricks;
struct mipnerf_b200_grid_grads;
struct mipnerf_b200_grid_sh_u8;
struct mipnerf_b200_rays;

namespace mipnerf {

// ---- ray_kernels.cu ----
cudaError_t launch_distloss(const float* weights, const float* t, float* out, int64_t num_rays, int n,
                            cudaStream_t st);
// d_w[r,i] = grad_out * scale * ((2/3) (t_{i+1} - t_i) w_i + 2 S_i),  S_i = sum_j w_j |m_i - m_j|  (grad_out NULL = 1)
cudaError_t launch_distloss_backward(const float* weights, const float* t, const float* grad_out, float scale,
                                     float* d_w, int64_t num_rays, int n, cudaStream_t st);
// mip-NeRF 360's interlevel loss per ray (include/mipnerf_b200.h) and its gradient in w_hat, written (grad_out NULL = 1)
cudaError_t launch_interlevel_loss(const float* t, const float* w, int n, const float* t_hat, const float* w_hat,
                                   int m, int64_t num_rays, float* out, cudaStream_t st);
cudaError_t launch_interlevel_loss_backward(const float* t, const float* w, int n, const float* t_hat,
                                            const float* w_hat, int m, int64_t num_rays, const float* grad_out,
                                            float scale, float* d_w_hat, cudaStream_t st);
cudaError_t launch_generate_rays(const float* c2w_host, int height, int width, float focal, float near_v,
                                 float far_v, int row0, int rows, float* origins, float* directions,
                                 float* viewdirs, float* radii, float* near_o, float* far_o, cudaStream_t st);
cudaError_t launch_rays_from_pixels(const float* cam_table, const int64_t* offsets, const int32_t* widths,
                                    int num_images, const int64_t* pixel_ids, int64_t count, const float* atlas,
                                    float* origins, float* directions, float* viewdirs, float* radii,
                                    float* lossmult, float* near_o, float* far_o, float* rgb, cudaStream_t st);
cudaError_t launch_coarse_t(const float* near, const float* far, const Draws& t_rand, float* t_out,
                            int64_t num_rays, int n, int randomized, int disparity, cudaStream_t st);
cudaError_t launch_philox_uniform(const Draws& d, float* out, int64_t num_rays, int ncols, cudaStream_t st);
cudaError_t launch_philox_normal(const Draws& d, float* out, int64_t num_rays, int ncols, cudaStream_t st);
// raw_density [num_rays, ncols] += d.scale * normal (models/mip_nerf.py:232-233); no-op when `d` is inactive
cudaError_t launch_add_density_noise(float* raw_density, const Draws& d, int64_t num_rays, int ncols, cudaStream_t st);
cudaError_t launch_cast_rays(const float* origins, const float* directions, const float* radii,
                             const float* t, float* means, float* covs, int64_t num_rays, int n,
                             cudaStream_t st);
cudaError_t launch_ipe(const float* means, const float* covs, float* out, int64_t num_points,
                       int min_deg, int max_deg, cudaStream_t st);
cudaError_t launch_ipe_from_t(const float* origins, const float* directions, const float* radii,
                              const float* t, float* out, int64_t num_rays, int n, int min_deg,
                              int max_deg, int disable_integration, cudaStream_t st);
cudaError_t launch_pos_enc(const float* x, float* out, int64_t num_points, int min_deg, int max_deg,
                           int append_identity, cudaStream_t st);
cudaError_t launch_composite(const float* rgb, const float* dens, const float* t, const float* dirs,
                             float* comp_rgb, float* distance, float* acc, float* weights,
                             int64_t num_rays, int n, int white_bkgd, int activate,
                             float density_bias, float rgb_scale, float rgb_padding, cudaStream_t st);
cudaError_t launch_resample(const float* bins, const float* weights, const Draws& jitter, float* out,
                            int64_t* inds, int64_t num_rays, int nb, int ns, int randomized, int blur,
                            float padding, cudaStream_t st);
// density[i] = softplus(raw[i] + density_bias)  (models/mip_nerf.py:237)
cudaError_t launch_density_activation(const float* raw, float* density, int64_t n, float density_bias, cudaStream_t st);
// rgb[i,c] = rgb_activation(raw_rgb[i,c]), density[i] = softplus(raw_density[i] + density_bias) (models/mip_nerf.py:
// 236-237); either output may be null
cudaError_t launch_radiance_activation(const float* raw_rgb, const float* raw_density, float* rgb, float* density,
                                       int64_t n, float density_bias, float rgb_scale, float rgb_padding,
                                       cudaStream_t st);

// ---- isosurface.cu (marching tetrahedra; grid [nz, ny, nx], x fastest) ----
size_t isosurface_scratch_bytes(int nx, int ny, int nz);
// the device int64 [2] (vertices, faces) that launch_isosurface_count leaves at the start of the scratch
const int64_t* isosurface_totals(const void* scratch);
cudaError_t launch_isosurface_count(const float* grid, int nx, int ny, int nz, float iso, void* scratch,
                                    int64_t* counts, cudaStream_t st);
// lo / step: HOST float[3] (lattice point idx at lo + idx * step per axis)
cudaError_t launch_isosurface_emit(const float* grid, int nx, int ny, int nz, const float* lo, const float* step,
                                   float iso, const void* scratch, float* verts, int32_t* faces, cudaStream_t st);
// after launch_isosurface_emit on the same scratch: the unit normal of every vertex (step: HOST float[3])
cudaError_t launch_isosurface_normals(const float* grid, int nx, int ny, int nz, const float* step, float iso,
                                      const void* scratch, float* normals, cudaStream_t st);

// ---- grid_render.cu (ray marching through a baked grid; arguments checked by the caller; id: a KernelId) ----
cudaError_t launch_grid_render(const mipnerf_b200_grid& grid, const mipnerf_b200_grid_bricks* bricks,
                               const mipnerf_b200_grid_sh_u8* sh, const mipnerf_b200_rays& rays, float step,
                               int white_bkgd, float* rgb, float* distance, float* acc, int id, cudaStream_t st);
cudaError_t launch_grid_render_backward(const mipnerf_b200_grid& grid, const mipnerf_b200_rays& rays, float step,
                                        int white_bkgd, const float* d_rgb, const float* d_distance,
                                        const float* d_acc, const mipnerf_b200_grid_grads& grads, cudaStream_t st);
cudaError_t launch_grid_visibility(const mipnerf_b200_grid& grid, const mipnerf_b200_grid_bricks* bricks,
                                   const mipnerf_b200_rays& rays, float step, float* const* max_weight, int id,
                                   cudaStream_t st);
// bricks NULL: the dense cells
cudaError_t launch_grid_proposal(const mipnerf_b200_grid& grid, const mipnerf_b200_grid_bricks* bricks,
                                 const mipnerf_b200_rays& rays, const float* t_samples, int num_samples,
                                 float* weights, cudaStream_t st);
// dense fp32 cells; adds into grads.density only
cudaError_t launch_grid_proposal_backward(const mipnerf_b200_grid& grid, const mipnerf_b200_rays& rays,
                                          const float* t_samples, int num_samples, const float* d_weights,
                                          const mipnerf_b200_grid_grads& grads, cudaStream_t st);
template <class F>  // f(std::integral_constant<int, NC>{}), NC = (degree + 1)^2 for degree 0..3: the grid kernels' NC
void with_sh_coeffs(int degree, F&& f) {
  if (degree == 0) return f(std::integral_constant<int, 1>{});
  if (degree == 1) return f(std::integral_constant<int, 4>{});
  if (degree == 2) return f(std::integral_constant<int, 9>{});
  f(std::integral_constant<int, 16>{});
}

// ---- grid_tv.cu (total-variation prior of a baked grid; arguments checked by the caller) ----
cudaError_t launch_grid_tv(const mipnerf_b200_grid& grid, const int64_t* const* points, const int64_t* num_points,
                           float eps, float* const* tv_density, float* const* tv_sh, const float* weights,
                           const mipnerf_b200_grid_grads* grads, cudaStream_t st);

// ---- metrics.cu ----
size_t image_metrics_scratch_bytes(int height, int width, int channels);
cudaError_t launch_image_metrics(const float* pred, const float* target, int height, int width, int channels,
                                 int window, float sigma, float max_val, void* scratch, float* out, cudaStream_t st);

// ---- linear_f32.cu ----
// Y[M,N] = act( [X1 | X2[row / x2_row_div]] @ W[N, K1+K2]^T + bias ),  fp32 FFMA.
cudaError_t launch_linear_f32(const float* x1, int ld1, int k1, const float* x2, int ld2, int k2,
                              int x2_row_div, const float* w, const float* bias, float* y, int ldy,
                              int64_t m, int n, int relu, cudaStream_t st);

// ---- train_kernels.cu (fp32 training step: backward + Adam) ----
constexpr int kWgradMaxSlices = 160;
int wgrad_num_slices(int64_t m, int tiles, int sms);
cudaError_t launch_render_backward(const float* raw_rgb, const float* raw_dens, const float* t, const float* dirs,
                                   const float* target, const float* lossmult, const float* mask_sum,
                                   float mse_mult, float dist_mult, int white_bkgd, float density_bias,
                                   float rgb_scale, float rgb_padding, float* d_raw_rgb, float* d_raw_dens,
                                   float* sqerr_out, float* dist_out, int64_t num_rays, int n, cudaStream_t st);
// cotangents of one level's rendered outputs (each [B,3] / [B] / [B] / [B,N], NULL = zero), for launch_render_vjp
struct RenderCot {
  const float *d_comp_rgb, *d_distance, *d_acc, *d_weights;
};
// d raw_rgb / d raw_density of  sum <cot, (comp_rgb, distance, acc, weights)>  (render_backward_kernel's recompute)
cudaError_t launch_render_vjp(const float* raw_rgb, const float* raw_dens, const float* t, const float* dirs,
                              const RenderCot& cot, int white_bkgd, float density_bias, float rgb_scale,
                              float rgb_padding, float* d_raw_rgb, float* d_raw_dens, int64_t num_rays, int n,
                              cudaStream_t st);
// cotangents of a field query's outputs (raw heads [P,3] / [P] and activated rgb / density), NULL = zero
struct QueryCot {
  const float *d_raw_rgb, *d_raw_density, *d_rgb, *d_density;
};
// d raw_rgb / d raw_density of  <cot, (raw_rgb, raw_density, rgb, density)>  of m points; d_raw_rgb null: density only
cudaError_t launch_query_activation_vjp(const float* raw_rgb, const float* raw_dens, const QueryCot& cot,
                                        float density_bias, float rgb_scale, float* d_raw_rgb, float* d_raw_dens,
                                        int64_t m, cudaStream_t st);
cudaError_t launch_color_dgrad(const float* d_rgb, const float* wc, const float* v, float* d_v, int64_t m,
                               int k_dim, cudaStream_t st);
// dX[m,k] = (act[m,k] > 0 or act == NULL) * (dY[m,:n_dim] @ W[:n_dim, :k_dim] (row stride ldw) + r1[m] * r1w[k])
cudaError_t launch_dgrad_f32(const float* dy, int n_dim, const float* w, int ldw, const float* r1,
                             const float* r1w, const float* act, float* dx, int64_t m, int k_dim,
                             cudaStream_t st);
// dW[n_dim, k1+k2] (+)= dY^T @ [X1 | X2[row / x2_row_div]],  db[n_dim] (+)= colsum(dY); `part` holds
// up to kWgradMaxSlices * n_dim * (k1+k2+1) floats of per-slice partial sums.  `scale` multiplies the sums before
// they are stored / added (1 / the fp16 step's gradient scale).
cudaError_t launch_wgrad_f32(const float* dy, int n_dim, const float* x1, int ld1, int k1, const float* x2,
                             int ld2, int k2, int x2_row_div, float* part, float* dw, float* db,
                             int accumulate, int64_t m, cudaStream_t st, float scale = 1.f);
// c1 = fl32(1 - beta1), c2 = fl32(1 - beta2), each rounded once from double (torch's Adam weights)
cudaError_t launch_adam(float* p, const float* g, float* m, float* v, int64_t n, float c1, float beta2, float c2,
                        float eps, float step_size, float bc2_sqrt, float grad_scale, cudaStream_t st);
constexpr int kAdamMaxTensors = 32;
struct AdamMulti {  // passed by value in the kernel parameters
  float* p[kAdamMaxTensors];
  const float* g[kAdamMaxTensors];
  float* m[kAdamMaxTensors];
  float* v[kAdamMaxTensors];
  int64_t n[kAdamMaxTensors];
  int blocks[kAdamMaxTensors];  // ceil(n / 256)
  int count;
};
cudaError_t launch_adam_multi(const AdamMulti& t, float c1, float beta2, float c2, float eps, float step_size,
                              float bc2_sqrt, float grad_scale, cudaStream_t st);

// A 16-bit tile image (train_t16.cu's layout below) and, in bf16x3, its lo image of the same shape; lo null: a plain
// 16-bit image.  Byte is const uint8_t for an operand (T16) and uint8_t for an output (T16Out), which converts to T16.
template <typename Byte>
struct TileImage {
  Byte* hi = nullptr;
  Byte* lo = nullptr;
  TileImage(Byte* hi = nullptr, Byte* lo = nullptr) : hi(hi), lo(lo) {}
  template <typename B>
  TileImage(const TileImage<B>& o) : hi(o.hi), lo(o.lo) {}
};
using T16 = TileImage<const uint8_t>;
using T16Out = TileImage<uint8_t>;
// The pair of a carve of `tiles` tiles of `cols` columns at hi, laid out as hi, then lo `tiles` tiles further on
// (split false: the plain image at hi).
template <typename Byte>
TileImage<Byte> tile_pair(Byte* hi, int64_t tiles, int cols, bool split) {
  return {hi, split ? hi + (size_t)tiles * ((cols + 63) / 64) * 16384 : nullptr};
}

// ---- linear_tc.cu (wgmma linear layer for the training step's forward / dgrad GEMMs) ----
size_t linear_tc_image_bytes(int n, int k);
bool linear_tc_shape_ok(int n, int k);
// B image of  W[:, off:off+k]  (transposed == 0, n rows)  or of  W[off:off+k, :n]^T  (transposed == 1)
// lo != 0: the low halves fl16(w - fl16(w)) of the split precisions (the level kernel's lo stage image convention)
cudaError_t launch_pack_linear_image(const float* w, int ldw, int off, int transposed, void* image, int n, int k,
                                     int precision, cudaStream_t st, int lo = 0);
// Y = [mask>0] * relu?( X[M,:k] . B^T + bias[col] + row_bias[row/row_div][col] + prev[row][col] + r1[row]*r1w[col] )
cudaError_t launch_linear_tc(const float* x, int ldx, const void* image, float* y, int ldy, int64_t m, int n, int k,
                             const float* bias, const float* row_bias, int row_div, const float* prev,
                             const float* r1, const float* r1w, const float* mask, int relu, int precision,
                             cudaStream_t st);

bool wgrad_tc_shape_ok(int n_dim);
// One operand of launch_wgrad_mn_partials: an fp32 row-major matrix with leading dimension ld, or a tile image (pair)
// whose rows are its k columns.  The default operand is absent.
struct WgradOperand {
  const float* f32 = nullptr;
  int ld = 0;
  T16 image;
  WgradOperand() = default;
  WgradOperand(const float* p, int ld) : f32(p), ld(ld) {}
  template <typename Byte>
  WgradOperand(TileImage<Byte> image) : image(image) {}
  bool is_image() const { return image.hi != nullptr; }
  bool absent() const { return !f32 && !is_image(); }
};
// Wgrad partials only; the caller runs the fixed-order reduction (launch_wgrad_reduce) afterwards with the slice count
// returned in *slices_out.  dy (an fp32 dy: ld == n_dim, 16-byte aligned) and x1 are required, x2 (k2 columns) may be
// absent.  Tile-image operands need m a multiple of 128, and x2 as an image x2_row_div == 1.  No k tile may straddle
// x1 and x2: k2 > 0 needs k1 % 256 == 0.  bf16x3: dy and x1 are pairs, and so is x2 if it is an image.
cudaError_t launch_wgrad_mn_partials(const WgradOperand& dy, int n_dim, const WgradOperand& x1, int k1,
                                     const WgradOperand& x2, int k2, int x2_row_div, float* part, int64_t m,
                                     int max_slices, int precision, int* slices_out, cudaStream_t st,
                                     void* mask_out = nullptr);
// fixed-order reduction of [slices, n_dim, k_dim + 1] partials into dW / db (train_kernels.cu)
cudaError_t launch_wgrad_reduce(const float* part, int slices, int n_dim, int k_dim, float* dw, float* db,
                                int accumulate, cudaStream_t st, float scale = 1.f);

// ---- train_t16.cu (backward pass on 16-bit tile images: [tile = 128 rows][64-column slab][128 rows x 128 B, SW128]) ----
// The split (bf16x3) backward carries every operand as two such images, hi = fl16(x) and lo = fl16(x - hi): the
// TileImage pairs below (lo null: the 16-bit path; lo given: bf16x3, and precision must be bf16).
size_t t16_image_bytes(int64_t rows, int cols);
cudaError_t launch_t16_pack(const float* src, int ld, int cols, int64_t m, T16Out image, int precision,
                            cudaStream_t st);
cudaError_t launch_ipe_t16(const float* origins, const float* directions, const float* radii, const float* t,
                           T16Out image, int64_t num_rays, int n, int disable_integration, int precision,
                           cudaStream_t st);
// the IPE of query points [num_points, 3] (covs null: zero) as a tile image, whole tiles (rows past num_points: the IPE
// of a zero Gaussian), with the query modes' ipe_pair<false>
cudaError_t launch_ipe_points_t16(const float* means, const float* covs, void* image, int64_t num_points,
                                  int disable_integration, int precision, cudaStream_t st);
// a pair: dst = hi + lo
cudaError_t launch_t16_unpack(T16 image, int cols, float* dst, int ld, int64_t m, int precision, cudaStream_t st);
// y = [mask > 0] * (x . B^T + r1 * r1w), B the weight image (launch_pack_linear_image).  mask: a tile image like y
// (zero where mask <= 0), or mask_bits: [m][32 B] sign bits of a 256-column image (wgrad_mn_kernel's by-product); at
// most one of them.  bf16x3 (x.lo given): x, the weight image and y are pairs.
cudaError_t launch_linear_t16(T16 x, T16 image, T16Out y, int64_t m, int n, int k, const float* r1, const float* r1w,
                              const void* mask, int precision, cudaStream_t st, const void* mask_bits = nullptr);
cudaError_t launch_color_dgrad_t16(const float* d_rgb, const float* wc, const void* v, T16Out d_v, int64_t m, int k_dim,
                                   int precision, cudaStream_t st);
cudaError_t launch_wgrad_small_n_t16(const float* dy, int n_dim, T16 x, int k_dim, float* part, float* dw, float* db,
                                     int accumulate, int64_t m, int precision, cudaStream_t st, float scale = 1.f);

// ---- mlp_tc.cu ----
// out[ray][n] = b[n] + W[n, in_main : in_main + view_dim] . venc[ray]   (view-direction part of the view layer)
cudaError_t launch_view_bias_from_enc(const float* venc, const float* w, const float* b, float* out,
                                      int64_t num_rays, cudaStream_t st);
// terms[d][n] = bias[n] + sum_{k < nk} w[k sk + n sn] enc_k(dirs[d])  (fmaf, k in order; enc: pos_enc of num_deg
// degrees with append_identity, nk <= 27), n < 128
cudaError_t launch_view_terms(const float* dirs, int64_t num_dirs, const float* w, int64_t sk, int64_t sn,
                              const float* bias, int nk, int num_deg, float* terms, cudaStream_t st);
// Per (point p, direction d): raw = W_color . max(acc[p] + terms[d], 0) + b_color (128 wide, the level kernel's order),
// rgb = its activation, into raw_rgb / rgb [P][D][3] (either may be null); proj (may be null) [P][num_basis][3] =
// sum over d in order of table[d][k] (raw if proj_raw else rgb), num_basis 1..16.
cudaError_t launch_radiance_pairs(const float* acc, const float* terms, const float* w_color, const float* b_color,
                                  int64_t num_points, int64_t num_dirs, float rgb_scale, float rgb_padding,
                                  float* raw_rgb, float* rgb, const float* table, int num_basis, int proj_raw,
                                  float* proj, cudaStream_t st);

}  // namespace mipnerf
