// b200sd_internal.h — declarations shared between the .cu translation units of libb200sd.so.
#pragma once
#include <cuda_runtime.h>
#include "../../../include/b200sd.h"

namespace b200sd {

int gemm_tc(const void* A, long long lda, const void* Wt, void* D, long long ldd, int M, int N, int K, int block_n,
            const b200sd_epilogue* epi, int is_bf16, int max_ctas, cudaStream_t stream);

int conv_tc(const void* X, long long pitch_c, int NB, int Hin, int Win, int C, const void* Wt, int ksize, int stride,
            int pad, int pad_end, void* D, long long ldd, int Cout, int block_n, const b200sd_epilogue* epi,
            int is_bf16, int max_ctas, cudaStream_t stream);

int attention_tc(const void* Q, long long ldq, const void* K, long long ldk, const void* V, long long ldv, void* O,
                 long long ldo, int B, int heads, int Sq, int Skv, const int* kv_len, int d, int d_pad, float scale,
                 int v_ones_col, int is_bf16, cudaStream_t stream);

}  // namespace b200sd
