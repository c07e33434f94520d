// C entry points to the fused FFN kernel for tools/ffn_bench.py.  The tool compiles this file (which includes tc_gemm.cu,
// so the kernel is built from the library's own source with the library's flags) twice into bench_out/: as is, and with
// -DB200ST_MLP_TIMELINE for the per-warpgroup stamps; both are linked against the library's other objects.
#include "../neurst_b200/csrc/tc_gemm.cu"

using namespace b200st;

static DropoutSpec bits_spec(float p, const void* bits) {
  DropoutSpec s = no_dropout();
  if (p > 0.f) { s.p = p; s.scale = 1.f / (1.f - p); s.bits = static_cast<const uint8_t*>(bits); }
  return s;
}

extern "C" {

int ffnb_fwd(const void* X, int dtype, int M, int d, int ffn, const void* W1, const float* b1, const void* W2, const float* b2,
             float p_ffn, const void* bits_ffn, float p_post, const void* bits_post, void* F1, float* x_out, void* stream,
             int* tickets) {
  return fused_mlp_fwd(X, dtype, M, d, ffn, W1, b1, W2, b2, bits_spec(p_ffn, bits_ffn), bits_spec(p_post, bits_post), F1, x_out,
                       static_cast<cudaStream_t>(stream), tickets);
}

int ffnb_bwd(const void* dY, int dtype, int M, int d, int ffn, const void* W1, const void* W2, const void* F1, float scale,
             void* dF1, float* dH, void* stream, int* tickets) {
  return fused_mlp_bwd(dY, dtype, M, d, ffn, W1, W2, F1, scale, dF1, dH, static_cast<cudaStream_t>(stream), tickets);
}

// CTAs of the launch fused_mlp_fwd / fused_mlp_bwd makes at this shape (the timeline buffer's first dimension)
int ffnb_grid(int M, int ffn) {
  int splits = 1;
  if (mlp_splits(ceil_div(M, BM), ffn / 128, &splits)) return -1;
  return ceil_div(M, BM) * splits;
}

// 0 when the library was built with the timeline, 1 when not
int ffnb_set_timeline(unsigned long long* buf) {
#ifdef B200ST_MLP_TIMELINE
  return cudaMemcpyToSymbol(g_mlp_timeline, &buf, sizeof(buf)) == cudaSuccess ? 0 : 2;
#else
  (void)buf;
  return 1;
#endif
}

}  // extern "C"
