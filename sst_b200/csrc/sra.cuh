// internal declarations of the SRA encoder layer, shared by its translation units (sra_*.cu)
#pragma once
#include <cuda_fp16.h>
#include "common.cuh"

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
