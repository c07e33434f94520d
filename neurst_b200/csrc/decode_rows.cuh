// The decoder step on more than 8 rows (decode_rows.cu): 16-bit shadow weights only, projections on wgmma.
#pragma once
#include "model.cuh"

namespace b200st {

constexpr int kDecodeMaxRows = 256;        // B200ST_DECODE_MAX_ROWS

int64_t rows_scratch_floats(const Config& c, int B);
// x [B, d] sits at scratch offset 0 (written by the embedding kernel before rows_step), logits [B, V] at this offset
int64_t rows_logits_offset(const Config& c, int B);
// Checks what the wide step needs beyond check_state (shadow, dims, shared memory); nothing is launched.
int rows_check(const Model& m, const Buffers& buf, const DecodeState& st, int beam);
// Dynamic shared memory of the wide step's self- and cross-attention kernels, and the call that sets both kernels' limits.
// A caller of rows_check sets them once, to the largest need of the models it steps: the limit belongs to the kernel, so
// setting it model after model could lower it below an earlier model's need.
size_t rows_self_smem(const Config& c, int max_len);
size_t rows_cross_smem(const Config& c, int Tm, int beam);
int rows_raise_smem(size_t self_bytes, size_t cross_bytes);
// Every decoder layer and the tied logits of one step on st.B rows; anc / beam as step_launch in decode.cu.
int rows_step(const Model& m, const Buffers& buf, const DecodeState& st, const int32_t* time_dev, float* logits, const int* anc,
              int beam, cudaStream_t s);
// greedy_pick_kernel's selection rules with one block per row; the last block to finish publishes time / all_finished
int rows_greedy_pick(const float* logits, int64_t* ids, int32_t* finished, int32_t* length, float* logprob, int64_t* out,
                     int32_t* time, int32_t* all_finished, uint32_t* ticket, int B, int V, int eos, int unk, int min_len,
                     int max_steps, cudaStream_t s);

}  // namespace b200st
