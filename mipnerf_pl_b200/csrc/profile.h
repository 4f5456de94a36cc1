// profile.h — per-kernel launch counters and optional CUDA-event timing inside the library.
// bench.py uses it for `gpu_launches` and for the dominant kernel's live launch duration
// (`roofline.achieved`); with timing disabled the only cost is one counter increment per launch.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace mipnerf {

enum KernelId : int {
  kKernCoarseT = 0,
  kKernCastRays,
  kKernIpe,
  kKernPosEnc,
  kKernLinearF32,
  kKernComposite,
  kKernResample,
  kKernPackWeights,
  kKernMlpLevelTc,   // fused wgmma level kernel (IPE + MLP + compositing)
  kKernMlpTc,        // wgmma MLP on explicit features
  kKernRayGen,       // on-device pinhole ray generation
  kKernDistloss,
  kKernRayPrologue,  // view-direction bias + coarse fenceposts in front of the fused level kernels
  kKernRenderBackward,
  kKernDgrad,
  kKernWgrad,
  kKernAdam,
  kKernLinearTc,     // stand-alone wgmma linear layer (training forward / dgrad)
  kKernWgradTc,      // wgmma wgrad partials
  kKernImageMetrics, // PSNR + SSIM of a rendered frame
  kKernDensityTc,    // density-only mode of the wgmma level kernel (IPE + trunk + density head)
  kKernIsosurface,   // marching-tetrahedra isosurface extraction (count / scan / emit)
  kKernRadianceTc,   // radiance mode of the wgmma level kernel (IPE + per-point view term + the whole MLP)
  kKernRadianceDirsTc,  // view-accumulator mode of the wgmma level kernel (IPE + the MLP up to the view layer's GEMM)
  kKernRadiancePairs,   // per-(point, direction) view layer + colour head (+ projection) of a shared direction set
  kKernInterlevelLoss,  // mip-NeRF 360's interlevel loss of proposal weights, and its gradient
  kKernGridProposalBackward,  // gradient of a baked grid's proposal weights with respect to its densities
  kKernGridProposal,   // proposal weights of a baked grid at a forward's level-0 intervals
  kKernGridTv,         // total-variation terms and gradient of a baked grid's kept points
  kKernGridVisibilityBricks,  // grid_visibility on a baked grid whose cells are 8^3-point bricks
  kKernGridRenderBricks,  // ray marching through a baked grid whose cells are 8^3-point bricks
  kKernGridRenderBackward,  // gradient of the baked-grid ray marcher with respect to the densities and SH rows
  kKernGridRenderU8,    // ray marching through a baked grid whose SH rows are uint8, dequantized in the kernel
  kKernGridVisibility,  // largest blending weight per kept baked-grid point over a batch of rays
  kKernGridRender,      // ray marching through a baked density + SH grid
  kKernCount
};

const char* kernel_name(int id);

// RAII bracket around one kernel launch on `st`.
struct LaunchScope {
  LaunchScope(int id, cudaStream_t st);
  ~LaunchScope();
  int id_;
  cudaStream_t st_;
  int slot_;
};

}  // namespace mipnerf
