// How the 2-D models (ResNetSE, Res2Net, ERes2Net, CAM++) plan their convolutions over image grids, in one place (image_plan.cu).  The plan
// itself (PlanStep, PlanModel and the executor) is shared with ECAPA-TDNN: plan.h.
//
// Layout: every activation is split-bf16 planes over rows (b, h+1, w+1) of a [B, H+2, W+2] grid whose border rows are zero and
// are never written (freq = H, time = W, channels last).  With that layout
//   * a 3x3 conv (padding 1) is the gather-GEMM with 9 taps at row offsets dh*(W+2)+dw -- the zero border IS the padding; a 32 ->
//     32 channel one runs on the weight-stationary patch kernel (conv3x3.cu) instead, unless PPV_CONV3X3=0;
//   * a strided conv is computed on the input grid and only the rows on the stride lattice are stored, straight into the output
//     grid (epilogue row remap: the strided 3x3 convs cost 4x their FLOPs in exchange for no strided-gather TMA path);
//   * BatchNorm(eval) directly after a conv is folded into the conv's weights and bias at finalize (ArenaBuilder::fold_conv);
//   * a 1x1 conv over a 32-column window may run on the CUDA cores (pointwise.cu), unless PPV_POINTWISE=0.
#pragma once
#include <vector>

#include "common.h"
#include "plan.h"

namespace ppv {

// levels[0] = the stem grid H x W; each next level halves H, and W too if `halve_w` (a stride-2 conv's output grid)
void image_pyramid(ImageGeo* levels, int n, int H, int W, bool halve_w);
// Planes epilogue of a conv over grid `gin` whose outputs on the (stride_h, stride_w) lattice are stored into `out` on grid `gout`
Epilogue image_epilogue(const Planes& out, const ImageGeo& gin, const ImageGeo& gout, int stride_h, int stride_w);
// the nine K-sources of a 3x3 conv over columns [col0, col0 + ncols) of `p` on grid `g`, taps in (dh, dw) order
void image_taps(std::vector<GemmSource>* v, const Planes& p, int col0, int ncols, const ImageGeo& g);

// The head ResNetSE and Res2Net share (resnet_se.py:133-139, res2net.py:161-167): the last grid flattened to [B, T', cat] ->
// AttentiveStatisticsPooling(cat, 128) with the global context (pooling.py:86-125) -> bn2 -> Linear -> bn3.  The attention TDNN's
// weight splits into the part over x (att1) and the part over [mean; std] (fold: a per-utterance bias); bn3 folds into fc.
struct AspHead {
    GemmWeights fold, att1, att2, fc;
    float *att1_bn_scale = nullptr, *att1_bn_shift = nullptr, *bn2_scale = nullptr, *bn2_shift = nullptr;
    int cat = 0, att = 128, embd = 0;
};
// the workspace buffers the head writes: flat [B T', cat] is its input
struct AspHeadBuffers {
    Planes flat, gstat, pooled, attp;
    float *fold_out = nullptr, *pooled_raw = nullptr, *emb_out = nullptr;
};
// Reads "pooling.*", "bn2.norm.*", "linear.*" and "bn3.norm.*" (the reference's names) into the arena.
bool prepare_asp_head(ArenaBuilder& ab, AspHead* h, int cat, int att, int embd);

}  // namespace ppv
