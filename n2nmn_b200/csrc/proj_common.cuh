// Work description shared by the two implementations of the conv_image contraction
// (wgmma TF32: proj_wgmma.cuh; fp32 CUDA cores: proj_simt.cuh).
//
// The contraction  m[r, :] = X[r, :] · W_img + b_img  runs over the flattened (image, pixel) row
// axis r = b*HW + p of the feature grid (models_clevr/nmn3_modules.py:101 through
// util/empty_safe_conv.py:8-32). It depends on the image only, never on the node, so it is done
// once per (image, weight set) and its consumers are folded into the epilogue:
//   PS_FIND : every Find / Filter node of the image reduces the row on the fly
//               att[p] = Σ_c m[p,c]·(τ∘w2)[c] · rsqrt(max(Σ_c m[p,c]²·τ²[c], 1e-12)) + b2
//             (l2_normalize + conv_eltwise, nmn3_modules.py:107-108) — m never reaches HBM;
//   others  : rows of images that host a consumer (FindSameProperty's conv_image map, or one of
//             the fc_att maps, see ProjSetId) are stored to `mbuf` (bias included) for the node
//             kernel.
#pragma once
#include "common.cuh"

namespace n2nmn {

struct ProjParams {
  const ProjWork* work;   // 128-row tiles (common.cuh)
  int num_tiles;
  int total_rows;   // rows of ONE segment: N*HW
  int num_seg;      // segments covered by this launch
  int seg_images;   // N: images per segment (global image g = seg*N + b)
  int n_tiles;      // Mp / 256
  int k_blocks;     // ceil(Dk / 32)
  int HW, M, Mp, Dk, feat_pitch;
  const float* feat_seg[kMaxSeg];   // [N*HW, feat_pitch] per segment (CUDA-core path only)
  const float* bias[NUM_PROJ_SETS];      // [Mp], zero padded
  const float* w_orig[NUM_PROJ_SETS];    // [Dk][M] (CUDA-core path only)
  // fused consumers of PS_FIND: CSR over the images of all segments
  const int32_t* img_ptr;     // [N+1]
  const int32_t* node_text;   // text row of each CSR entry
  const int32_t* node_out;    // arena slot of each CSR entry
  const float* tauw;          // [text rows][Mp]: τ∘w2 and τ² from the text kernel
  const float* tau2;
  const float* elt_b;         // conv_eltwise bias of FindModule, [1]
  float* arena;               // [slots][HW]
  // stored sets
  const int32_t* mslot;       // [NUM_PROJ_SETS][num_images] -> slot in mbuf or -1
  int num_images;             // num_seg * N
  float* mbuf;                // [slots][HW][Mp]
};

}  // namespace n2nmn
