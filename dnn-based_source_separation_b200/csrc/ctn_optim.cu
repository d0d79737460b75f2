// Training-step remainder (SURVEY.md 8f-3): global-norm gradient clipping + Adam over the FLAT gradient bucket the native
// backward writes (ctn_b200/models/_train.py), as two streaming kernels instead of the ~350 tiny launches of
// torch.nn.utils.clip_grad_norm_ + torch.optim.Adam.  Reference: egs/wsj0-mix/common/src/driver.py:149-157
// (optimizer.zero_grad / clip_grad_norm_(max_norm) / optimizer.step), torch.optim.Adam semantics (no amsgrad):
//   g <- g * min(1, max_norm / (||g||_2 + 1e-6));  [g += wd * p];  m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;
//   p -= lr / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps)
// The step counter t and the learning rate live in DEVICE memory so that the whole training step can be replayed from a CUDA
// graph (and the LR halved by the scheduler, egs/wsj0-mix/conv-tasnet/src/adhoc_driver.py:25-39, without re-capture).
#include "ctn_internal.h"

namespace {

// chunk table entry: tensor index and element offset inside the tensor; one block per chunk of CHUNK elements
constexpr int CHUNK = 2048;

// Sum of squares over the chunks of the table, i.e. over exactly the tensors k_clip_adam updates: a frozen tensor or padding that
// shares the bucket stays out of the norm, as its .grad stays out of torch.nn.utils.clip_grad_norm_.  One block per chunk, its
// CHUNK / 256 loads per thread issued together; scalar loads, because the tensors' offsets are arbitrary; squares exact in double.
__global__ void __launch_bounds__(256) k_sumsq(const int2* __restrict__ chunks, const long long* __restrict__ flat_off,
                                               const int* __restrict__ numel, const float* __restrict__ g, double* __restrict__ out) {
  __shared__ double red[64];
  const int2 ch = chunks[blockIdx.x];
  const float* gt = g + flat_off[ch.x] + ch.y;
  const int len = numel[ch.x] - ch.y < CHUNK ? numel[ch.x] - ch.y : CHUNK;
  float v[CHUNK / 256];
#pragma unroll
  for (int k = 0; k < CHUNK / 256; ++k) {
    const int e = threadIdx.x + 256 * k;
    v[k] = e < len ? gt[e] : 0.f;
  }
  double s = 0.0, dummy = 0.0;
#pragma unroll
  for (int k = 0; k < CHUNK / 256; ++k) s += (double)v[k] * v[k];
  block_sum2_d(s, dummy, red);
  if (threadIdx.x == 0) atomicAdd(out, s);
}

__global__ void __launch_bounds__(256) k_clip_adam(const int2* __restrict__ chunks, float* const* __restrict__ params,
                                                   const long long* __restrict__ flat_off, const int* __restrict__ numel,
                                                   const float* __restrict__ flat_grad, float* __restrict__ exp_avg,
                                                   float* __restrict__ exp_avg_sq, const double* __restrict__ sumsq,
                                                   const float* __restrict__ lr_p, const long long* __restrict__ step_p, float beta1,
                                                   float beta2, float eps, float wd, float max_norm, float* __restrict__ norm_out) {
  const int2 ch = chunks[blockIdx.x];
  const int ti = ch.x, e0 = ch.y;
  const int n = numel[ti];
  const long long fo = flat_off[ti];
  float* __restrict__ p = params[ti];
  const float total_norm = (float)sqrt(*sumsq);
  float clip = 1.f;
  if (max_norm > 0.f) {
    clip = max_norm / (total_norm + 1e-6f);  // torch.nn.utils.clip_grad_norm_
    clip = clip < 1.f ? clip : 1.f;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0 && norm_out) *norm_out = total_norm;
  const long long t = *step_p + 1;  // this step's index (the counter itself is advanced by k_step_advance afterwards)
  const float lr = *lr_p;
  const float bc1 = 1.f - powf(beta1, (float)t), bc2 = 1.f - powf(beta2, (float)t);
  const float step_size = lr / bc1, bc2_sqrt = sqrtf(bc2);
  const int end = e0 + CHUNK < n ? e0 + CHUNK : n;
  for (int e = e0 + threadIdx.x; e < end; e += blockDim.x) {
    float g = flat_grad[fo + e] * clip;
    const float w = p[e];
    if (wd != 0.f) g = fmaf(wd, w, g);
    const float m = exp_avg[fo + e] + (1.f - beta1) * (g - exp_avg[fo + e]);  // lerp, as torch's single-tensor Adam
    const float v = beta2 * exp_avg_sq[fo + e] + (1.f - beta2) * g * g;
    exp_avg[fo + e] = m;
    exp_avg_sq[fo + e] = v;
    const float denom = sqrtf(v) / bc2_sqrt + eps;
    p[e] = w - step_size * (m / denom);
  }
}
__global__ void k_step_advance(long long* step_p) { *step_p += 1; }

}  // namespace

extern "C" int ctn_clip_adam_chunks(const int* numel, int n_tensors, int* chunk_tensor, int* chunk_offset, int capacity) {
  if (!numel || n_tensors <= 0) return CTN_EINVAL;
  int c = 0;
  for (int i = 0; i < n_tensors; ++i)
    for (int e = 0; e < numel[i]; e += CHUNK) {
      if (chunk_tensor && c < capacity) { chunk_tensor[c] = i; chunk_offset[c] = e; }
      ++c;
    }
  return c;  // number of chunks (call with null outputs to size the table)
}

extern "C" int ctn_clip_adam_step(const int32_t* chunk_table, int n_chunks, float* const* params, const long long* flat_off,
                                  const int32_t* numel, int n_tensors, const float* flat_grad, size_t flat_numel, float* exp_avg,
                                  float* exp_avg_sq, double* sumsq_scratch, const float* lr, long long* step, float beta1, float beta2,
                                  float eps, float weight_decay, float max_norm, float* norm_out, ctn_stream_t stream) {
  LaunchScope scope(flat_grad);
  if (!chunk_table || n_chunks <= 0 || !params || !flat_off || !numel || n_tensors <= 0 || !flat_grad || !exp_avg || !exp_avg_sq ||
      !sumsq_scratch || !lr || !step)
    return CTN_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(sumsq_scratch, 0, sizeof(double), st);
  if (e != cudaSuccess) return (int)e;
  const int2* chunks = reinterpret_cast<const int2*>(chunk_table);
  k_sumsq<<<n_chunks, 256, 0, st>>>(chunks, flat_off, numel, flat_grad, sumsq_scratch);
  CTN_COUNT_LAUNCH();
  k_clip_adam<<<n_chunks, 256, 0, st>>>(chunks, params, flat_off, numel, flat_grad, exp_avg, exp_avg_sq,
                                        sumsq_scratch, lr, step, beta1, beta2, eps, weight_decay, max_norm, norm_out);
  CTN_COUNT_LAUNCH();
  k_step_advance<<<1, 1, 0, st>>>(step);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}
