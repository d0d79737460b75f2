// Causal Conv-TasNet (cLN instead of gLN, all-left padding of the depthwise conv): forward pipeline in the reference's
// operation order (src/models/tdcn.py:107-147,177-196 with causal=True; src/modules/norm.py:42-95).
//
// cLN's statistics at frame t cover all channels and ALL frames <= t, so they are only known after a scan over time of
// the complete tensor: the stack cannot defer / fold the normalisation the way the gLN path does.  Each block is therefore
//   h = PReLU(W1 x + b1)  [contraction, fused bias+PReLU epilogue]   -> cLN1 (step sums -> scan -> apply, in place)
//   u = PReLU(dwconv_causal(h) + bd)                                  -> cLN2
//   r = [Wo; Ws] u  [contraction]   ;   x += r[:Bc] + bo ; skip += r[Bc:] + bs
// The contractions are the same wgmma / FFMA kernels as everywhere else; their operands are materialised tensors without
// operand scales, so the f16x3 mode runs them on tf32 pieces (ctn_pw).  The rest are streaming kernels (HBM-bound).
// Note: the reference's own cLN cannot run on CUDA (its frame counter is built on the CPU, norm.py:83), so this path has
// no GPU baseline in the reference at all.
#include <string.h>
#include "ctn_internal.h"

namespace {

struct CausalWs {
  double* cln;   // [B][frames<=pitch][2]
  double* dummy; // [B][2] sink for the unused gLN statistics of the EPI_H epilogue
  float* wimg;
  float* Wcat;   // (Bc+Sc, H)
  float* r;      // (B, Bc+Sc, pitch)
};

void carve(Carver& cv, const ctn_config_t* c, int B, int pitch, CausalWs* ws) {
  // images of pw1, [out; skip] and (with an encoder) the head
  const int Bc = c->bottleneck, H = c->hidden;
  const int shapes[][2] = {{H, Bc}, {Bc + c->skip, H}, {Bc, c->n_basis}};
  ws->cln = cv.take<double>((size_t)B * pitch * 2);
  ws->dummy = cv.take<double>((size_t)B * 2);
  ws->wimg = cv.take<float>(ctn_pw_wimg_max_bytes(shapes, c->n_basis > 0 ? 3 : 2, c->math) / sizeof(float));
  ws->Wcat = cv.take<float>((size_t)(c->bottleneck + c->skip) * c->hidden);
  ws->r = cv.take<float>((size_t)B * pitch * (c->bottleneck + c->skip));
}

// u[c][t] = PReLU( sum_k wd[c][k] * h[c][t + k*d - pad_left] + bd[c] ), h = 0 outside [0, frames)   (tdcn.py:123-132,181-184)
__global__ void __launch_bounds__(256) k_dw_plain(const float* __restrict__ h, float* __restrict__ u, const float* __restrict__ wd,
                                                  const float* __restrict__ bd, const float* __restrict__ slope, int C, int frames,
                                                  int pitch, int P, int dil, int pad_left) {
  const int b = blockIdx.y;
  const float a = slope[0];
  for (int c = blockIdx.x; c < C; c += gridDim.x) {
    const float* hr = h + ((size_t)b * C + c) * pitch;
    float* ur = u + ((size_t)b * C + c) * pitch;
    const float bc = bd[c];
    for (int t = threadIdx.x; t < pitch; t += 256) {
      float v = 0.f;
      if (t < frames) {
        float acc = bc;
        for (int k = 0; k < P; ++k) {
          const int tt = t + k * dil - pad_left;
          if (tt >= 0 && tt < frames) acc = fmaf(wd[c * P + k], hr[tt], acc);
        }
        v = prelu_f(acc, a);
      }
      ur[t] = v;
    }
  }
}

// rows of r (B, Mt, pitch): m < Bc (has_out): xout = xin + r + bo[m] ; else skip (+)= r + bs[j]      (tdcn.py:144-145, :39)
// xin == xout updates the residual stream in place.  A thread owns 4 consecutive frames (128-bit loads / stores).
__global__ void __launch_bounds__(256) k_res_skip(const float* __restrict__ r, int Mt, const float* xin, float* xout,
                                                  float* __restrict__ skip, const float* __restrict__ bo,
                                                  const float* __restrict__ bs, int Bc, int Sc, int has_out, int skip_init,
                                                  int frames, int pitch) {
  const int b = blockIdx.y;
  for (int m = blockIdx.x; m < Mt; m += gridDim.x) {
    const float* rr = r + ((size_t)b * Mt + m) * pitch;
    const bool is_x = has_out && m < Bc;
    const int j = m - (has_out ? Bc : 0);
    const float* src = is_x ? xin + ((size_t)b * Bc + m) * pitch : skip + ((size_t)b * Sc + j) * pitch;
    float* dst = is_x ? xout + ((size_t)b * Bc + m) * pitch : skip + ((size_t)b * Sc + j) * pitch;
    const float bb = is_x ? bo[m] : bs[j];
    const bool fresh = !is_x && skip_init;
    for (int t = threadIdx.x * 4; t < pitch; t += 1024) {
      float4 v = zero4();
      if (t < frames) {
        const float4 q = ld4(rr + t);
        const float4 base = fresh ? zero4() : ld4(src + t);
        v = mask4(make_float4(base.x + q.x + bb, base.y + q.y + bb, base.z + q.z + bb, base.w + q.w + bb), t, frames);
      }
      st4(dst + t, v);
    }
  }
}

// y[b][c][t] += bias[c] (valid columns only)
__global__ void __launch_bounds__(256) k_bias_rows(float* __restrict__ y, const float* __restrict__ bias, int C, int frames, int pitch) {
  const int b = blockIdx.y;
  for (int c = blockIdx.x; c < C; c += gridDim.x) {
    float* r = y + ((size_t)b * C + c) * pitch;
    const float bc = bias[c];
    for (int t = threadIdx.x; t < pitch; t += 256) r[t] = t < frames ? r[t] + bc : 0.f;
  }
}

}  // namespace

size_t ctn_causal_ws_bytes(const ctn_config_t* c, int B, int pitch) {
  Carver cv(nullptr);
  CausalWs ws;
  carve(cv, c, B, pitch, &ws);
  return cv.off + 256;
}

int ctn_causal_head(const ctn_config_t* c, const ctn_params_t* p, const float* w, float* tmp, float* x0, int B, int frames,
                    int pitch, void* cws, cudaStream_t st) {
  Carver cv(cws);
  CausalWs ws;
  carve(cv, c, B, pitch, &ws);
  const int N = c->n_basis, Bc = c->bottleneck;
  // cLN0 (conv_tasnet.py:333-334,370) then the bottleneck 1x1 (:335,371)
  CTN_TRY(ctn_cln_pitch_fwd(w, p->norm0_g, p->norm0_b, tmp, B, N, frames, pitch, c->eps, ws.cln, st));
  PwArgs a;
  memset(&a, 0, sizeof(a));
  a.A = tmp; a.W = p->bn_w; a.D = x0; a.B = B; a.M = Bc; a.K = N; a.frames = frames; a.pitch = pitch;
  { StageTimer tm(CTN_ST_HEAD, st); CTN_TRY(ctn_pw(a, PRO_NONE, EPI_RAW, c->math, ws.wimg, st)); }
  k_bias_rows<<<grid_cb(Bc, B), 256, 0, st>>>(x0, p->bn_b, Bc, frames, pitch);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

int ctn_causal_tcn(const ctn_config_t* c, const ctn_block_params_t* blocks, float* x, float* skip, float* h, float* u, int B,
                   int frames, int pitch, void* cws, cudaStream_t st) {
  Carver cv(cws);
  CausalWs ws;
  carve(cv, c, B, pitch, &ws);
  const int R = c->num_blocks, X = c->num_layers, Bc = c->bottleneck, H = c->hidden, Sc = c->skip, P = c->sep_kernel;
  for (int i = 0; i < R * X; ++i) {
    const ctn_block_params_t& q = blocks[i];
    const bool has_out = q.out_w != nullptr;
    if (!has_out && i != R * X - 1) return CTN_EINVAL;
    const int dil = 1 << (i % X);
    const int pad_left = (P - 1) * dil;  // causal: all of the padding on the left (tdcn.py:125-127)
    // h = PReLU(W1 x + b1)
    PwArgs a;
    memset(&a, 0, sizeof(a));
    a.A = x; a.W = q.bottleneck_w; a.D = h; a.B = B; a.M = H; a.K = Bc; a.frames = frames; a.pitch = pitch;
    a.bias = q.bottleneck_b; a.slope = q.prelu1; a.stats_out = ws.dummy;
    { StageTimer tm(CTN_ST_PW1, st); CTN_TRY(ctn_pw(a, PRO_NONE, EPI_H, c->math, ws.wimg, st)); }
    {
      StageTimer tm(CTN_ST_DW, st);
      CTN_TRY(ctn_cln_pitch_fwd(h, q.norm1_g, q.norm1_b, h, B, H, frames, pitch, c->eps_tcn, ws.cln, st));
      CTN_TRY(ctn_dw_plain_fwd(h, u, q.dw_w, q.dw_b, q.prelu2, B, H, frames, pitch, P, dil, pad_left, st));
      CTN_TRY(ctn_cln_pitch_fwd(u, q.norm2_g, q.norm2_b, u, B, H, frames, pitch, c->eps_tcn, ws.cln, st));
    }
    const int Mt = has_out ? Bc + Sc : Sc;
    CTN_TRY(ctn_block_wcat(q, Bc, Sc, H, ws.Wcat, st));
    memset(&a, 0, sizeof(a));
    a.A = u; a.W = ws.Wcat; a.D = ws.r; a.B = B; a.M = Mt; a.K = H; a.frames = frames; a.pitch = pitch;
    { StageTimer tm(CTN_ST_PW2, st); CTN_TRY(ctn_pw(a, PRO_NONE, EPI_RAW, c->math, ws.wimg, st)); }
    { StageTimer tm(CTN_ST_FIN, st);
      CTN_TRY(ctn_res_skip_fwd(ws.r, Mt, x, x, skip, q.out_b, q.skip_b, Bc, Sc, has_out ? 1 : 0, i == 0 ? 1 : 0, B, frames, pitch, st)); }
  }
  return CTN_OK;
}

// The per-frame kernels above, shared with the online (chunk-by-chunk) pipeline of ctn_online.cu and the un-fused training
// forward of ctn_train.cu: same kernels, same launch shape.
int ctn_res_skip_fwd(const float* r, int Mt, const float* xin, float* xout, float* skip, const float* bo, const float* bs, int Bc, int Sc,
                     int has_out, int skip_init, int B, int frames, int pitch, cudaStream_t st) {
  k_res_skip<<<grid_cb(Mt, B), 256, 0, st>>>(r, Mt, xin, xout, skip, bo, bs, Bc, Sc, has_out, skip_init, frames, pitch);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

int ctn_block_wcat(const ctn_block_params_t& q, int Bc, int Sc, int H, float* wcat, cudaStream_t st) {
  const bool has_out = q.out_w != nullptr;
  cudaError_t e = cudaSuccess;
  if (has_out) e = cudaMemcpyAsync(wcat, q.out_w, sizeof(float) * (size_t)Bc * H, cudaMemcpyDeviceToDevice, st);
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(wcat + (has_out ? (size_t)Bc * H : 0), q.skip_w, sizeof(float) * (size_t)Sc * H, cudaMemcpyDeviceToDevice, st);
  return e == cudaSuccess ? CTN_OK : (int)e;
}

int ctn_dw_plain_fwd(const float* h, float* u, const float* wd, const float* bd, const float* slope, int B, int C, int frames, int pitch,
                     int P, int dil, int pad_left, cudaStream_t st) {
  k_dw_plain<<<grid_cb(C, B), 256, 0, st>>>(h, u, wd, bd, slope, C, frames, pitch, P, dil, pad_left);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}

int ctn_bias_rows_fwd(float* y, const float* bias, int C, int B, int frames, int pitch, cudaStream_t st) {
  k_bias_rows<<<grid_cb(C, B), 256, 0, st>>>(y, bias, C, frames, pitch);
  CTN_COUNT_LAUNCH();
  CTN_RETURN_IF_CUDA_ERR();
  return CTN_OK;
}
