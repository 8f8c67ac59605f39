// misc.h — prototypes of the misc.cuh kernels that car_train.cu launches.  They are defined once, in car_api.cu (through misc.cuh),
// and misc.cuh includes this file: a signature that changes on one side only leaves car_train.cu's call without a definition.
#pragma once
#include "common.cuh"

__global__ void rope_kv_write_kernel(const bf16* __restrict__ qkv, const float* __restrict__ rope, bf16* __restrict__ q,
                                     bf16* __restrict__ kc, bf16* __restrict__ vc, int rows, int Tq, int d, int H, int S);
__global__ void swiglu_kernel(const bf16* __restrict__ g, const bf16* __restrict__ u, bf16* __restrict__ out, long long n);
