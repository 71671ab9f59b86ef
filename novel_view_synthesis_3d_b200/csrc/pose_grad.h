// pose_grad.h -- the gradient of the loss w.r.t. the camera rays and the cameras (pose_grad.cu).
#pragma once
#include <cuda_runtime.h>

// The cameras of one forward and where their ray gradient goes.
struct PoseGradArgs {
  const float* R1; const float* t1; const float* R2; const float* t2; const float* K;   // (B,3,3) / (B,3)
  const float* kinv;        // (B,3,3) fp32 K^-1 the forward used (generated rays)
  const float* rays;        // (B,2,S,S,6) explicit rays, or nullptr (generated from the cameras)
  const float* cond_mask;   // (B)
  float* d_rays;            // (B,2,S,S,6) out
  int B, S, E, convention;
};
// One pose-embedding convolution: 3x3, 144 -> E, stride s, SAME padding lo (top / left), output So x So.
struct PoseLevel {
  const void* dy;      // its output gradient (2B, So, So, E), activation dtype
  const float* w;      // fp32 kernel [tap][144][E]
  float alpha;         // scale of dy
  int So, s, lo;
};
struct PoseLevels {
  PoseLevel l[8];
  int n;
};

// wgmma kernel of one level (bf16): reads the forward's bf16 weight shadow [E][tap][144]; accumulate = add into d_rays.
bool pose_grad_tc_supported(int So, int E);
void launch_pose_grad_tc(const PoseGradArgs& a, const PoseLevel& L, const void* wshadow, int accumulate, cudaStream_t s);
// SIMT kernel over several levels (fp32, or bf16 with the weights rounded to bf16 as the shadows are).
void launch_pose_grad_simt(int dtype, const PoseGradArgs& a, const PoseLevels& lv, int accumulate, cudaStream_t s);
// generated rays: d_rays -> dR1, dt1, dR2, dt2, dK (each may be nullptr)
void launch_camera_grad(const PoseGradArgs& a, float* dR1, float* dt1, float* dR2, float* dt2, float* dK, cudaStream_t s);
