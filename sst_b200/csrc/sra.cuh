// internal declarations shared by the SRA translation units
#pragma once
#include <cuda_fp16.h>
#include "common.cuh"

void sstb_gemm_rows(cudaStream_t st, const float* A, int lda, const float* W, const float* bias, const float* res, int ldr,
                    float* out, int ldo, int M_cap, const int32_t* M_dev, int N, int K, int act, const float* pos_tab,
                    const int32_t* pos_code, int posL, int pos_maxw, int pos_ndim, int pos_ncols);
void sstb_gemm_rows_ex(cudaStream_t st, const float* A, int lda, const float* W, int ldw, const float* bias, const float* res,
                       int ldr, const long long* res_index, float* out, int ldo, int M_cap, const int32_t* M_dev, int N, int K,
                       int act, const float* pos_tab, const int32_t* pos_code, int posL, int pos_maxw, int pos_ndim, int pos_ncols);
// fp32-tolerance row GEMM on the tensor core (csrc/spconv.cu, split-fp16 operands): out = act(A . W^T + bias) + res.  Returns
// SSTB_ERR_UNSUPPORTED (nothing launched) when the shape does not fit (K, N multiples of 64) - callers then use sstb_gemm_rows.
// Each row of A and each output channel of W is lifted by a power of two to the top of fp16's range before it is split into an
// fp16 pair (as in sstb200_spconv_forward), so the result is homogeneous in the scale of either operand: an element within 2^-16
// of its row's (channel's) largest |value| keeps 22 significant bits, a smaller one an absolute error of 2^-38 of that largest,
// at any magnitude fp32 holds.  Unscaled, the pair loses bits for every |x| below about 2^-3 - which is where nn.Linear's default
// init (|w| <= 1 / sqrt(K)) and xavier's (|w| <= sqrt(6 / (K + N))) put the weights of an encoder layer, and where small
// activation rows lie.
int sstb_gemm_rows_x3(sstb200_ctx* c, const float* A, int lda, const float* W, const float* bias, const float* res, int ldr, float* out,
                      int ldo, int M_cap, const int32_t* M_dev, int N, int K, int act);
void sstb_add_norm_act(cudaStream_t st, const float* a, const float* b, const float* gamma, const float* beta,
                       const float* bn_mean, const float* bn_var, float eps, float* out, int n_cap, const int32_t* n_dev, int d, int act);
void sstb_add_norm(cudaStream_t st, const float* a, const float* b, const float* gamma, const float* beta,
                   const float* bn_mean, const float* bn_var, float eps, float* out, int n_cap, const int32_t* n_dev, int d);
int sstb_win_attn_fp32(sstb200_ctx* c, const float* qkv, int d, int nhead, int n_cap, const int32_t* n_dev,
                       const int32_t* win_offsets, const int32_t* tok_perm, const int32_t* tok_win, const float* tau,
                       int tau_n, float tau_min, float* out);
int sstb_sra_layer_fp32(sstb200_ctx* c, const sstb200_sra_layer* L, const sstb200_sra_plan* P, const float* x, float* y,
                        int n_cap, const int32_t* n_dev);
int sstb_sra_layer_bf16(sstb200_ctx* c, const sstb200_sra_layer* L, const sstb200_sra_plan* P, const float* x, float* y,
                        int n_cap, const int32_t* n_dev);

#define SSTB_MAX_STACK 64   // encoder layers per stack call (kernel-parameter arrays of per-layer pointers)
// Fused post-attention chain (csrc/sra_chain2.cu).  next / next_plan / next_qkv: fuse the NEXT layer's q|k|v projection into the
// chain.  bn_fold: the layer's folded eval-mode BatchNorm (sstb_sra_bn_fold), required when the layer uses BatchNorm.
int sstb_sra_chain2(sstb200_ctx* c, const sstb200_sra_layer* L, const __half* att, const float* x, float* y, int n_cap,
                    const int32_t* n_dev, const sstb200_sra_layer* next = nullptr, const sstb200_sra_plan* next_plan = nullptr,
                    void* next_qkv = nullptr, const float* bn_fold = nullptr);
// layer_cfg use_bn (eval-mode BatchNorm instead of LayerNorm): out[l][4][128] = {scale1, shift1, scale2, shift2} per layer;
// rows of LayerNorm layers are left untouched.  bn_fold of sstb_sra_chain2 = that layer's 512 floats.
int sstb_sra_bn_fold(sstb200_ctx* c, const sstb200_sra_layer* layers, int num_layers, float* out);
int sstb_sra_stack_bf16(sstb200_ctx* c, const sstb200_sra_layer* layers, int num_layers, const sstb200_sra_plan* plans /*[2]*/,
                        const float* x, float* y, float* scratch, int n_cap, const int32_t* n_dev);

void sstb_sir_segmax_finalize(cudaStream_t st, const uint32_t* ord, int G, int C, float* out, int ldo, int col0);
