// api.cu — extern "C" entry points for the tensor-core ops (declared in include/b200sd.h).
#include "b200sd_internal.h"

extern "C" int b200sd_linear(const void* A, long long lda, const void* Wt, void* D, long long ldd, int M, int N, int K,
                             int block_n, const b200sd_epilogue* epi, int dtype, int max_ctas, void* stream) {
  return b200sd::gemm_tc(A, lda, Wt, D, ldd, M, N, K, block_n, epi, dtype == B200SD_BF16 ? 1 : 0, max_ctas,
                         static_cast<cudaStream_t>(stream));
}

extern "C" int b200sd_conv2d(const void* X, long long pitch_c, int NB, int Hin, int Win, int C, const void* Wt,
                             int ksize, int stride, int pad, int pad_end, void* D, long long ldd, int Cout,
                             int block_n, const b200sd_epilogue* epi, int dtype, int max_ctas, void* stream) {
  return b200sd::conv_tc(X, pitch_c, NB, Hin, Win, C, Wt, ksize, stride, pad, pad_end, D, ldd, Cout, block_n, epi,
                         dtype == B200SD_BF16 ? 1 : 0, max_ctas, static_cast<cudaStream_t>(stream));
}

extern "C" int b200sd_conv2d_scaled(const void* X, long long pitch_c, int NB, int Hin, int Win, int C, const void* Wt,
                                    int ksize, int stride, int pad, int pad_end, void* D, long long ldd, int Cout,
                                    int block_n, const b200sd_epilogue* epi, float res_scale, int dtype, int max_ctas,
                                    void* stream) {
  return b200sd::conv_tc(X, pitch_c, NB, Hin, Win, C, Wt, ksize, stride, pad, pad_end, D, ldd, Cout, block_n, epi,
                         dtype == B200SD_BF16 ? 1 : 0, max_ctas, static_cast<cudaStream_t>(stream), true, res_scale);
}

extern "C" int b200sd_attention(const void* Q, long long ldq, const void* K, long long ldk, const void* V,
                                long long ldv, void* O, long long ldo, int B, int heads, int Sq, int Skv, int d,
                                int d_pad, float scale, int v_ones_col, int dtype, void* stream) {
  return b200sd::attention_tc(Q, ldq, K, ldk, V, ldv, O, ldo, B, heads, Sq, Skv, nullptr, d, d_pad, scale, v_ones_col,
                              dtype == B200SD_BF16 ? 1 : 0, static_cast<cudaStream_t>(stream));
}

extern "C" int b200sd_attention_varlen(const void* Q, long long ldq, const void* K, long long ldk, const void* V,
                                       long long ldv, void* O, long long ldo, int B, int heads, int Sq, int Skv,
                                       const int* kv_len, int d, int d_pad, float scale, int v_ones_col, int dtype,
                                       void* stream) {
  if (!kv_len) return B200SD_ERR_INVALID;
  return b200sd::attention_tc(Q, ldq, K, ldk, V, ldv, O, ldo, B, heads, Sq, Skv, kv_len, d, d_pad, scale, v_ones_col,
                              dtype == B200SD_BF16 ? 1 : 0, static_cast<cudaStream_t>(stream));
}
