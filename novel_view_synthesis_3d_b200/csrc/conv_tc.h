// conv_tc.h -- wgmma/TMA implicit-GEMM convolution (bf16 in, fp32 accumulate in registers) + bf16 weight shadows.
#pragma once
#include "kernels.h"

// One conv/dense leaf of the flat fp32 parameter buffer and where its bf16 shadows live in the workspace.
struct WeightPrepEntry {
  long long src;      // element offset of the kernel in the flat fp32 params ([seg][tap][Ci][segw])
  long long dstT;     // byte offset in the workspace of the forward shadow  [Co][tap][Ci]   (-1: none)
  long long dstC;     // byte offset of the data-gradient shadow (plain bf16 cast)            (-1: none)
  long long prefix;   // first global element index of this entry
  long long tprefix;  // first 64x64 tile index of this entry (filled in by launch_weight_prep)
  int Ci, Co, taps, nseg;
};
#define XU_PREP_MAX 160
struct WeightPrepTable {
  int n;
  long long total;
  WeightPrepEntry e[XU_PREP_MAX];
};
void launch_weight_prep(const WeightPrepTable& tab, const float* params, void* ws, cudaStream_t s);

// mode 0: forward conv (N,H,W,Ci)->(N,H,W,Co);  mode 1: its data gradient.  true if the tensor-core kernel takes it.
bool conv_tc_supported(int dtype, int mode, int N, int H, int W, int Ci, int Co, int ks, int stride, int nseg);
// true if the forward epilogue can also emit the GroupNorm input statistics of its output (ConvArgs::cstats)
bool conv_tc_stats_supported(int mode, int N, int Ho, int Wo);
// `a` as for launch_conv_simt (a.w is ignored); wshadow = the bf16 shadow for a.mode (see WeightPrepEntry).
void launch_conv_tc(const ConvArgs& a, const void* wshadow, cudaStream_t s);

// weight gradient on the tensor cores (+ bias gradient); everything else stays on launch_wgrad_simt
bool wgrad_tc_supported(int dtype, int N, int H, int W, int Ci, int Co, int ks, int stride, int nseg);
void launch_wgrad_tc(const WgradArgs& a, cudaStream_t s);
