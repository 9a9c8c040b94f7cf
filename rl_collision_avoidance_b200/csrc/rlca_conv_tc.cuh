// rlca_conv_tc.cuh — internal interface of the wgmma conv tower (rlca_conv_tc.cu).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

int rlca_conv_tc_init();
size_t rlca_conv_tc_image_floats();
// builds the pre-swizzled tf32 hi/lo operand image of both towers' conv weights (index 0 actor, 1 critic)
void rlca_conv_tc_prep(const float *const cv1w[2], const float *const cv1b[2], const float *const cv2w[2],
                       const float *const cv2b[2], float *img, cudaStream_t s);
// F = [2][nb][4096] relu(conv2(relu(conv1(obs)))) in flatten order c*128+q; Fs (optional) = [tower][hi,lo][nb][4096]
int rlca_conv_tc_forward(const float *obs, const float *img, float *F, float *Fs, int nb, int num_sms, cudaStream_t s);

// ---- backward: part = [2 towers][slots][3616] per-CTA partial gradients (cv2w | cv2b | cv1w | cv1b), summed by
// conv_part_reduce_kernel; dF = d(relu(conv2)) unmasked, Fmask = the forward features (mask = Fmask > 0)
size_t rlca_conv_tc_bwd_image_floats();
int rlca_conv_tc_bwd_slots(int nb, int num_sms);
void rlca_conv_tc_bwd_prep(const float *const cv1w[2], const float *const cv1b[2], const float *const cv2w[2],
                           const float *const cv2b[2], float *img, cudaStream_t s);
int rlca_conv_tc_backward(const float *obs, const float *img, const float *dF, const float *Fmask, float *part, int nb,
                          int num_sms, cudaStream_t s);
