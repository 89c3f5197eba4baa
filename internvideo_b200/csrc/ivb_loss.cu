// ivb_loss.cu — decoder heads' normalisation + alignment losses, contrastive loss, pixel targets,
// and the flat AdamW step: HBM-bound kernels with warp-shuffle row reductions.
//
//   LayerNorm -> L2-normalise   Linear_Decoder / MLP_Decoder.forward  internvideo2_pretrain.py:355-365,393-403
//   (2 - 2 sum_c out*tgt).mean() engines/engine_for_pretraining.py:131-136
//   video-text contrastive       InternVideo2/multi_modality/models/criterions.py:15-55,65-103,200-216
//   pixel-reconstruction target  InternVideo1/Pretrain/VideoMAE/engine_for_pretraining.py:66-98 + MSE :43,106
#include <math.h>

#define IVB_COLRED_FLOATS (4L << 20)
#include "ivb_colred.cuh"
#include "ivb_internal.h"
#include "ivb_ptx.cuh"

namespace ivb {

__device__ __forceinline__ void ld8_bf16(const __nv_bfloat16* p, float v[8]) {
  uint4 u = *reinterpret_cast<const uint4*>(p);
  float2 f0 = unpack_bf16(u.x), f1 = unpack_bf16(u.y), f2 = unpack_bf16(u.z), f3 = unpack_bf16(u.w);
  v[0] = f0.x; v[1] = f0.y; v[2] = f1.x; v[3] = f1.y; v[4] = f2.x; v[5] = f2.y; v[6] = f3.x; v[7] = f3.y;
}
__device__ __forceinline__ void ld8_f32(const float* p, float v[8]) {
  float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void st8_bf16(__nv_bfloat16* p, const float v[8]) {
  uint4 w;
  w.x = pack_bf16(v[0], v[1]); w.y = pack_bf16(v[2], v[3]);
  w.z = pack_bf16(v[4], v[5]); w.w = pack_bf16(v[6], v[7]);
  *reinterpret_cast<uint4*>(p) = w;
}
template <bool F32>
__device__ __forceinline__ void ld8(const void* p, long off, float v[8]) {
  if (F32) ld8_f32(reinterpret_cast<const float*>(p) + off, v);
  else ld8_bf16(reinterpret_cast<const __nv_bfloat16*>(p) + off, v);
}

// ---------------------------------------------------------------- LayerNorm + L2 normalise
// out = y / ||y||,  y = LN(z) * w + b.   stats[row] = {mean, rstd, 1/||y||}.
// If tgt != nullptr also accumulates loss_sum += sum_rows (2 - 2 <out, tgt>)  (engine :131-136).
template <bool TGT_F32>
__global__ void __launch_bounds__(256)
ln_l2_fwd_kernel(const __nv_bfloat16* __restrict__ z, long ldz, const __nv_bfloat16* __restrict__ w,
                 const __nv_bfloat16* __restrict__ bsh, float eps, int M, int C,
                 __nv_bfloat16* __restrict__ out, long ldo, float* __restrict__ stats,
                 const void* __restrict__ tgt, long ldt, float* __restrict__ loss_sum) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const float invC = 1.f / C;
  float loss_acc = 0.f;
  for (long row = static_cast<long>(blockIdx.x) * wpb + (threadIdx.x >> 5); row < M;
       row += static_cast<long>(gridDim.x) * wpb) {
    const __nv_bfloat16* zr = z + row * ldz;
    float s = 0.f;
    for (int c = lane * 8; c < C; c += 256) { float v[8]; ld8_bf16(zr + c, v);
#pragma unroll
      for (int k = 0; k < 8; ++k) s += v[k]; }
    const float mean = warp_sum(s) * invC;
    float ss = 0.f;
    for (int c = lane * 8; c < C; c += 256) { float v[8]; ld8_bf16(zr + c, v);
#pragma unroll
      for (int k = 0; k < 8; ++k) { const float d = v[k] - mean; ss += d * d; } }
    const float rstd = rsqrtf(warp_sum(ss) * invC + eps);
    float n2 = 0.f, dot = 0.f;
    for (int c = lane * 8; c < C; c += 256) {
      float v[8], wv[8], bv[8];
      ld8_bf16(zr + c, v); ld8_bf16(w + c, wv); ld8_bf16(bsh + c, bv);
      float t[8];
      if (tgt) ld8<TGT_F32>(tgt, row * ldt + c, t);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float y = (v[k] - mean) * rstd * wv[k] + bv[k];
        n2 += y * y;
        if (tgt) dot += y * t[k];
      }
    }
    n2 = warp_sum(n2);
    const float inv_n = rsqrtf(n2);
    if (tgt) { dot = warp_sum(dot); if (lane == 0) loss_acc += 2.f - 2.f * dot * inv_n; }
    if (out) {
      for (int c = lane * 8; c < C; c += 256) {
        float v[8], wv[8], bv[8], o[8];
        ld8_bf16(zr + c, v); ld8_bf16(w + c, wv); ld8_bf16(bsh + c, bv);
#pragma unroll
        for (int k = 0; k < 8; ++k) o[k] = ((v[k] - mean) * rstd * wv[k] + bv[k]) * inv_n;
        st8_bf16(out + row * ldo + c, o);
      }
    }
    if (lane == 0 && stats) { stats[row * 3 + 0] = mean; stats[row * 3 + 1] = rstd; stats[row * 3 + 2] = inv_n; }
  }
  if (tgt && loss_sum) {
    __shared__ float red[8];
    if (lane == 0) red[threadIdx.x >> 5] = loss_acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f;
      for (int k = 0; k < wpb; ++k) t += red[k];
      atomicAdd(loss_sum, t);
    }
  }
}

// d_out = gscale * dout_tensor  (dout_tensor is the upstream gradient, or the TARGET itself when the
// loss is (2-2<out,tgt>).mean(): then gscale = -2 * g / rows).  Computes dz (bf16), dw, db (fp32, accumulated in a fixed order).
// dynamic smem: float acc[2][warps][C]
template <bool DO_F32>
__global__ void __launch_bounds__(256)
ln_l2_bwd_kernel(const __nv_bfloat16* __restrict__ z, long ldz, const __nv_bfloat16* __restrict__ w,
                 const __nv_bfloat16* __restrict__ bsh, const float* __restrict__ stats, int M, int C,
                 const void* __restrict__ dout, long lddo, float gscale_host,
                 const float* __restrict__ gscale_dev, __nv_bfloat16* __restrict__ dz, long lddz,
                 float* __restrict__ dw, float* __restrict__ db) {
  extern __shared__ float acc_smem[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int wpb = blockDim.x >> 5;
  const float invC = 1.f / C;
  const float gs = gscale_host * (gscale_dev ? *gscale_dev : 1.f);
  const bool want = dw != nullptr;
  float* accw = acc_smem + static_cast<long>(warp) * C;
  float* accb = acc_smem + static_cast<long>(wpb + warp) * C;
  if (want) for (int i = lane; i < C; i += 32) { accw[i] = 0.f; accb[i] = 0.f; }
  __syncwarp();
  for (long row = static_cast<long>(blockIdx.x) * wpb + warp; row < M; row += static_cast<long>(gridDim.x) * wpb) {
    const __nv_bfloat16* zr = z + row * ldz;
    const float mean = stats[row * 3], rstd = stats[row * 3 + 1], inv_n = stats[row * 3 + 2];
    // pass 1: a = <do, out> (out = y*inv_n)
    float a = 0.f;
    for (int c = lane * 8; c < C; c += 256) {
      float v[8], wv[8], bv[8], g[8];
      ld8_bf16(zr + c, v); ld8_bf16(w + c, wv); ld8_bf16(bsh + c, bv); ld8<DO_F32>(dout, row * lddo + c, g);
#pragma unroll
      for (int k = 0; k < 8; ++k) a += g[k] * gs * ((v[k] - mean) * rstd * wv[k] + bv[k]) * inv_n;
    }
    a = warp_sum(a);
    // dy = inv_n * (do - out * a);  LN backward: g = dy*w ; dx = rstd*(g - mean(g) - xhat*mean(g*xhat))
    float s1 = 0.f, s2 = 0.f;
    for (int c = lane * 8; c < C; c += 256) {
      float v[8], wv[8], bv[8], g[8];
      ld8_bf16(zr + c, v); ld8_bf16(w + c, wv); ld8_bf16(bsh + c, bv); ld8<DO_F32>(dout, row * lddo + c, g);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float xh = (v[k] - mean) * rstd;
        const float o = (xh * wv[k] + bv[k]) * inv_n;
        const float dy = inv_n * (g[k] * gs - o * a);
        s1 += dy * wv[k];
        s2 += dy * wv[k] * xh;
      }
    }
    s1 = warp_sum(s1) * invC; s2 = warp_sum(s2) * invC;
    for (int c = lane * 8; c < C; c += 256) {
      float v[8], wv[8], bv[8], g[8], o8[8];
      ld8_bf16(zr + c, v); ld8_bf16(w + c, wv); ld8_bf16(bsh + c, bv); ld8<DO_F32>(dout, row * lddo + c, g);
      float dyv[8], xhv[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float xh = (v[k] - mean) * rstd;
        const float o = (xh * wv[k] + bv[k]) * inv_n;
        const float dy = inv_n * (g[k] * gs - o * a);
        dyv[k] = dy; xhv[k] = xh;
        o8[k] = rstd * (dy * wv[k] - s1 - xh * s2);
      }
      st8_bf16(dz + row * lddz + c, o8);
      if (want) {
        float4* aw = reinterpret_cast<float4*>(accw + c);
        float4* ab = reinterpret_cast<float4*>(accb + c);
        float4 w0 = aw[0], w1 = aw[1], b0 = ab[0], b1 = ab[1];
        w0.x += dyv[0] * xhv[0]; w0.y += dyv[1] * xhv[1]; w0.z += dyv[2] * xhv[2]; w0.w += dyv[3] * xhv[3];
        w1.x += dyv[4] * xhv[4]; w1.y += dyv[5] * xhv[5]; w1.z += dyv[6] * xhv[6]; w1.w += dyv[7] * xhv[7];
        b0.x += dyv[0]; b0.y += dyv[1]; b0.z += dyv[2]; b0.w += dyv[3];
        b1.x += dyv[4]; b1.y += dyv[5]; b1.z += dyv[6]; b1.w += dyv[7];
        aw[0] = w0; aw[1] = w1; ab[0] = b0; ab[1] = b1;
      }
    }
  }
  if (want) {
    __syncthreads();
    for (int i = threadIdx.x; i < C; i += blockDim.x) {
      float sw = 0.f, sb = 0.f;
      for (int k = 0; k < wpb; ++k) { sw += acc_smem[static_cast<long>(k) * C + i]; sb += acc_smem[static_cast<long>(wpb + k) * C + i]; }
      colred_put(0, gridDim.x, blockIdx.x, C, i, sw);
      if (db) colred_put(1, gridDim.x, blockIdx.x, C, i, sb);
    }
  }
}

// ---------------------------------------------------------------- flat AdamW (fp32 master, bf16 model copy)
template <bool G_F32>
__global__ void adamw_kernel(float* __restrict__ master, float* __restrict__ m, float* __restrict__ v,
                             const void* __restrict__ grad, __nv_bfloat16* __restrict__ param_bf16,
                             long n, float lr, float beta1, float beta2, float eps, float wd,
                             float bc1, float bc2, float grad_scale_host,
                             const float* __restrict__ grad_scale_dev, const float* __restrict__ dyn) {
  const long i = (static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4;
  if (i >= n) return;
  if (dyn != nullptr) {  // device-resident {lr, step}: keeps a captured CUDA graph valid across steps
    lr = dyn[0];
    bc1 = 1.f - powf(beta1, dyn[1]);
    bc2 = 1.f - powf(beta2, dyn[1]);
  }
  const float gs_dev = grad_scale_dev ? *grad_scale_dev : 1.f;
  // a device scale that is not a positive finite number marks a bad step (NaN/Inf global gradient norm:
  // engine.step(check_finite) — engine_for_pretraining.py:151-161 aborts there): leave every state untouched
  if (!(gs_dev > 0.f) || gs_dev > 3.0e38f) return;
  const float grad_scale = grad_scale_host * gs_dev;
  float g[4], p[4], mm[4], vv[4];
  const int cnt = (n - i) >= 4 ? 4 : static_cast<int>(n - i);
  // 16-byte vector path when the 4-element group is whole and every base pointer is 16 B aligned
  const bool vec = cnt == 4 &&
                   ((reinterpret_cast<uintptr_t>(master) | reinterpret_cast<uintptr_t>(m) |
                     reinterpret_cast<uintptr_t>(v)) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(grad) & (G_F32 ? 15 : 7)) == 0 &&
                   (reinterpret_cast<uintptr_t>(param_bf16) & 7) == 0;
  if (vec) {
    const float4 p4 = *reinterpret_cast<const float4*>(master + i);
    const float4 m4 = *reinterpret_cast<const float4*>(m + i);
    const float4 v4 = *reinterpret_cast<const float4*>(v + i);
    p[0] = p4.x; p[1] = p4.y; p[2] = p4.z; p[3] = p4.w;
    mm[0] = m4.x; mm[1] = m4.y; mm[2] = m4.z; mm[3] = m4.w;
    vv[0] = v4.x; vv[1] = v4.y; vv[2] = v4.z; vv[3] = v4.w;
    if (G_F32) {
      const float4 g4 = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(grad) + i);
      g[0] = g4.x; g[1] = g4.y; g[2] = g4.z; g[3] = g4.w;
    } else {
      const uint2 gb = *reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(grad) + i);
      const float2 a = unpack_bf16(gb.x), b = unpack_bf16(gb.y);
      g[0] = a.x; g[1] = a.y; g[2] = b.x; g[3] = b.y;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) g[k] *= grad_scale;
  } else {
    for (int k = 0; k < cnt; ++k) {
      g[k] = (G_F32 ? reinterpret_cast<const float*>(grad)[i + k]
                    : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(grad)[i + k])) * grad_scale;
      p[k] = master[i + k]; mm[k] = m[i + k]; vv[k] = v[i + k];
    }
  }
  const float inv_bc1 = 1.f / bc1, inv_bc2 = 1.f / bc2, decay = 1.f - lr * wd;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (k < cnt) {
      p[k] *= decay;
      mm[k] = beta1 * mm[k] + (1.f - beta1) * g[k];
      vv[k] = beta2 * vv[k] + (1.f - beta2) * g[k] * g[k];
      p[k] -= lr * (mm[k] * inv_bc1) / (sqrtf(vv[k] * inv_bc2) + eps);
    }
  }
  if (vec) {
    *reinterpret_cast<float4*>(master + i) = make_float4(p[0], p[1], p[2], p[3]);
    *reinterpret_cast<float4*>(m + i) = make_float4(mm[0], mm[1], mm[2], mm[3]);
    *reinterpret_cast<float4*>(v + i) = make_float4(vv[0], vv[1], vv[2], vv[3]);
    uint2 pb;
    pb.x = pack_bf16(p[0], p[1]); pb.y = pack_bf16(p[2], p[3]);
    *reinterpret_cast<uint2*>(param_bf16 + i) = pb;
  } else {
    for (int k = 0; k < cnt; ++k) {
      master[i + k] = p[k]; m[i + k] = mm[k]; v[i + k] = vv[k];
      param_bf16[i + k] = __float2bfloat16(p[k]);
    }
  }
}

// ---------------------------------------------------------------- contrastive loss (video-text)
// cosv2t [G,G] fp32 = vn @ tn^T (wgmma GEMM).  S = cos / temp.  idx int64 [G].
// row pass: lse_r[i], tsum_r[i] = sum_j tg[i,j] S[i,j] ; col pass: lse_c[i], tsum_c[i] = sum_j tg[i,j] S[j,i]
// loss = 1/(2G) sum_i [(lse_r[i] - tsum_r[i]) + (lse_c[i] - tsum_c[i])]          (criterions.py:93-102)
__global__ void __launch_bounds__(256)
vtc_stats_kernel(const float* __restrict__ cosm, const long long* __restrict__ idx, int G, float inv_temp,
                 const float* __restrict__ temp_dev,
                 float* __restrict__ lse_r, float* __restrict__ lse_c, float* __restrict__ loss) {
  // a device-resident temperature (the learnable `temp` parameter) overrides the host value: no D2H
  // sync per step and a captured CUDA graph follows the parameter as it trains
  if (temp_dev != nullptr) inv_temp = 1.f / *temp_dev;
  // blocks [0, G): row i ; blocks [G, 2G): column i
  const int which = blockIdx.x / G;
  const int i = blockIdx.x % G;
  const long long my = idx[i];
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < G; j += blockDim.x) {
    const float s = (which == 0 ? cosm[static_cast<long>(i) * G + j] : cosm[static_cast<long>(j) * G + i]) * inv_temp;
    mx = fmaxf(mx, s);
  }
  __shared__ float red[8];
  __shared__ float bc;
  mx = warp_max(mx);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x == 0) { float t = red[0]; for (int k = 1; k < 8; ++k) t = fmaxf(t, red[k]); bc = t; }
  __syncthreads();
  mx = bc;
  float se = 0.f, ts = 0.f, cnt = 0.f;
  for (int j = threadIdx.x; j < G; j += blockDim.x) {
    const float s = (which == 0 ? cosm[static_cast<long>(i) * G + j] : cosm[static_cast<long>(j) * G + i]) * inv_temp;
    se += __expf(s - mx);
    if (idx[j] == my) { ts += s; cnt += 1.f; }
  }
  __shared__ float r2[3][8];
  se = warp_sum(se); ts = warp_sum(ts); cnt = warp_sum(cnt);
  if ((threadIdx.x & 31) == 0) { r2[0][threadIdx.x >> 5] = se; r2[1][threadIdx.x >> 5] = ts; r2[2][threadIdx.x >> 5] = cnt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b2 = 0.f, c = 0.f;
    for (int k = 0; k < 8; ++k) { a += r2[0][k]; b2 += r2[1][k]; c += r2[2][k]; }
    const float lse = mx + __logf(a);
    (which == 0 ? lse_r : lse_c)[i] = lse;
    atomicAdd(loss, (lse - b2 / c) * (0.5f / G));
  }
}

// dS[a,b] = gs/(2G) * [ exp(S-lse_r[a]) + exp(S-lse_c[b]) - 2*tg[a,b] ] ; written as bf16 d(cos) = dS/temp
// and dtemp accumulated: dtemp += sum dS * (-S/temp).
__global__ void __launch_bounds__(256)
vtc_grad_kernel(const float* __restrict__ cosm, const long long* __restrict__ idx, int G, float inv_temp,
                const float* __restrict__ temp_dev,
                const float* __restrict__ lse_r, const float* __restrict__ lse_c, float gscale_host,
                const float* __restrict__ gscale_dev, __nv_bfloat16* __restrict__ dcos, float* __restrict__ dtemp) {
  if (temp_dev != nullptr) inv_temp = 1.f / *temp_dev;
  const int a = blockIdx.x;
  const float gs = gscale_host * (gscale_dev ? *gscale_dev : 1.f) * (0.5f / G);
  const long long my = idx[a];
  float cnt = 0.f;
  for (int j = threadIdx.x; j < G; j += blockDim.x) cnt += (idx[j] == my) ? 1.f : 0.f;
  __shared__ float red[8];
  __shared__ float bc;
  cnt = warp_sum(cnt);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) { float t = 0.f; for (int k = 0; k < 8; ++k) t += red[k]; bc = t; }
  __syncthreads();
  const float inv_cnt = 1.f / bc;
  const float la = lse_r[a];
  float dt = 0.f;
  for (int b = threadIdx.x; b < G; b += blockDim.x) {
    const float s = cosm[static_cast<long>(a) * G + b] * inv_temp;
    const float tg = (idx[b] == my) ? inv_cnt : 0.f;
    const float ds = gs * (__expf(s - la) + __expf(s - lse_c[b]) - 2.f * tg);
    dcos[static_cast<long>(a) * G + b] = __float2bfloat16(ds * inv_temp);
    dt += ds * (-s * inv_temp);
  }
  dt = warp_sum(dt);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = dt;
  __syncthreads();
  if (threadIdx.x == 0 && dtemp) { float t = 0.f; for (int k = 0; k < 8; ++k) t += red[k]; atomicAdd(dtemp, t); }
}

// F.normalize(x, dim=-1) rows (eps 1e-12): out bf16, inv_norm saved.   x fp32 or bf16.
template <bool XF32>
__global__ void l2norm_rows_kernel(const void* __restrict__ x, long ldx, int M, int C,
                                   __nv_bfloat16* __restrict__ out, long ldo, float* __restrict__ inv_norm) {
  const long row = static_cast<long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  float ss = 0.f;
  for (int c = lane * 8; c < C; c += 256) { float v[8]; ld8<XF32>(x, row * ldx + c, v);
#pragma unroll
    for (int k = 0; k < 8; ++k) ss += v[k] * v[k]; }
  ss = warp_sum(ss);
  const float inv = 1.f / fmaxf(sqrtf(ss), 1e-12f);
  for (int c = lane * 8; c < C; c += 256) { float v[8], o[8]; ld8<XF32>(x, row * ldx + c, v);
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = v[k] * inv;
    st8_bf16(out + row * ldo + c, o); }
  if (lane == 0 && inv_norm) inv_norm[row] = inv;
}
// backward of F.normalize: dx = inv * (dy - xn * <dy, xn>)   (dy fp32, xn bf16) -> dx fp32
__global__ void l2norm_rows_bwd_kernel(const float* __restrict__ dy, long lddy, const __nv_bfloat16* __restrict__ xn,
                                       long ldxn, const float* __restrict__ inv_norm, int M, int C,
                                       float* __restrict__ dx, long lddx) {
  const long row = static_cast<long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  float dot = 0.f;
  for (int c = lane * 8; c < C; c += 256) { float g[8], v[8]; ld8_f32(dy + row * lddy + c, g); ld8_bf16(xn + row * ldxn + c, v);
#pragma unroll
    for (int k = 0; k < 8; ++k) dot += g[k] * v[k]; }
  dot = warp_sum(dot);
  const float inv = inv_norm[row];
  for (int c = lane * 8; c < C; c += 256) { float g[8], v[8]; ld8_f32(dy + row * lddy + c, g); ld8_bf16(xn + row * ldxn + c, v);
    float* o = dx + row * lddx + c;
    *reinterpret_cast<float4*>(o) = make_float4(inv * (g[0] - v[0] * dot), inv * (g[1] - v[1] * dot), inv * (g[2] - v[2] * dot), inv * (g[3] - v[3] * dot));
    *reinterpret_cast<float4*>(o + 4) = make_float4(inv * (g[4] - v[4] * dot), inv * (g[5] - v[5] * dot), inv * (g[6] - v[6] * dot), inv * (g[7] - v[7] * dot)); }
}

// ---------------------------------------------------------------- IV1 pixel targets + MSE
// One CTA (C warps) per masked patch: warp c normalises channel c over the tub*P*P pixels
// (mean / unbiased variance, +1e-6 on the std), labels layout 'b n (p c)'.
__global__ void pixel_target_kernel(const __nv_bfloat16* __restrict__ video, const int* __restrict__ midx,
                                    int n_mask, int B, int C, int T, int H, int W, int tub, int P,
                                    int normalize, const float* __restrict__ mean3, const float* __restrict__ std3,
                                    float* __restrict__ labels) {
  const int row = blockIdx.x;            // b * n_mask + m
  const int b = row / n_mask;
  const int c = threadIdx.x >> 5;        // channel
  const int lane = threadIdx.x & 31;
  if (c >= C) return;
  const int tok = midx[row];
  const int gw = W / P, gh = H / P;
  const int f = tok / (gh * gw), py = (tok / gw) % gh, px = tok % gw;
  const int npix = tub * P * P;
  const float mu_c = mean3[c], sd_c = std3[c];
  float s = 0.f;
  for (int i = lane; i < npix; i += 32) {
    const int dx = i % P, dy = (i / P) % P, dt = i / (P * P);
    const long src = (((static_cast<long>(b) * C + c) * T + (f * tub + dt)) * H + (py * P + dy)) * W + (px * P + dx);
    s += __bfloat162float(video[src]) * sd_c + mu_c;
  }
  const float mean = warp_sum(s) / npix;
  float ss = 0.f;
  for (int i = lane; i < npix; i += 32) {
    const int dx = i % P, dy = (i / P) % P, dt = i / (P * P);
    const long src = (((static_cast<long>(b) * C + c) * T + (f * tub + dt)) * H + (py * P + dy)) * W + (px * P + dx);
    const float d = __bfloat162float(video[src]) * sd_c + mu_c - mean;
    ss += d * d;
  }
  const float var = warp_sum(ss) / (npix - 1);
  const float inv = 1.f / (sqrtf(var) + 1e-6f);
  float* out = labels + static_cast<long>(row) * npix * C;
  for (int i = lane; i < npix; i += 32) {
    const int dx = i % P, dy = (i / P) % P, dt = i / (P * P);
    const long src = (((static_cast<long>(b) * C + c) * T + (f * tub + dt)) * H + (py * P + dy)) * W + (px * P + dx);
    const float u = __bfloat162float(video[src]) * sd_c + mu_c;
    out[static_cast<long>(i) * C + c] = normalize ? (u - mean) * inv : u;
  }
}

__device__ __forceinline__ void unpack8q(const uint4& u, float v[8]) {
  float2 f0 = unpack_bf16(u.x), f1 = unpack_bf16(u.y), f2 = unpack_bf16(u.z), f3 = unpack_bf16(u.w);
  v[0] = f0.x; v[1] = f0.y; v[2] = f1.x; v[3] = f1.y; v[4] = f2.x; v[5] = f2.y; v[6] = f3.x; v[7] = f3.y;
}

// Register-resident backward (C <= 256*NCH, bf16 upstream gradient / target): z and dout rows read once, all loads
// in flight together, the three sweeps run over registers (210 us vs 247 us for the streaming kernel at C = 3200;
// the same treatment of the FORWARD was slower — see ivb_ln_l2_fwd — and is not kept).
// dynamic smem: float acc[2][warps][C]
template <int NCH>
__global__ void __launch_bounds__(128, 2)
ln_l2_bwd_reg_kernel(const __nv_bfloat16* __restrict__ z, long ldz, const __nv_bfloat16* __restrict__ w,
                     const __nv_bfloat16* __restrict__ bsh, const float* __restrict__ stats, int M, int C,
                     const __nv_bfloat16* __restrict__ dout, long lddo, float gscale_host,
                     const float* __restrict__ gscale_dev, __nv_bfloat16* __restrict__ dz, long lddz,
                     float* __restrict__ dw, float* __restrict__ db) {
  extern __shared__ float acc_smem[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int wpb = blockDim.x >> 5;
  const int nch = C >> 3;
  const float invC = 1.f / C;
  const float gs = gscale_host * (gscale_dev ? *gscale_dev : 1.f);
  const bool want = dw != nullptr;
  float* accw = acc_smem + static_cast<long>(warp) * C;
  float* accb = acc_smem + static_cast<long>(wpb + warp) * C;
  if (want) for (int i = lane; i < C; i += 32) { accw[i] = 0.f; accb[i] = 0.f; }
  __syncwarp();
  for (long row = static_cast<long>(blockIdx.x) * wpb + warp; row < M; row += static_cast<long>(gridDim.x) * wpb) {
    uint4 zq[NCH], gq[NCH];
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c = lane + 32 * i;
      if (c < nch) {
        zq[i] = *reinterpret_cast<const uint4*>(z + row * ldz + c * 8);
        gq[i] = *reinterpret_cast<const uint4*>(dout + row * lddo + c * 8);
      }
    }
    const float mean = stats[row * 3], rstd = stats[row * 3 + 1], inv_n = stats[row * 3 + 2];
    float a = 0.f;     // <do, out>, out = y * inv_n
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c = lane + 32 * i;
      if (c < nch) {
        float v[8], wv[8], bv[8], g[8];
        unpack8q(zq[i], v); unpack8q(gq[i], g); ld8_bf16(w + c * 8, wv); ld8_bf16(bsh + c * 8, bv);
#pragma unroll
        for (int k = 0; k < 8; ++k) a += g[k] * gs * ((v[k] - mean) * rstd * wv[k] + bv[k]) * inv_n;
      }
    }
    a = warp_sum(a);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c = lane + 32 * i;
      if (c < nch) {
        float v[8], wv[8], bv[8], g[8];
        unpack8q(zq[i], v); unpack8q(gq[i], g); ld8_bf16(w + c * 8, wv); ld8_bf16(bsh + c * 8, bv);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float xh = (v[k] - mean) * rstd;
          const float o = (xh * wv[k] + bv[k]) * inv_n;
          const float dy = inv_n * (g[k] * gs - o * a);
          s1 += dy * wv[k];
          s2 += dy * wv[k] * xh;
        }
      }
    }
    s1 = warp_sum(s1) * invC; s2 = warp_sum(s2) * invC;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int c = lane + 32 * i;
      if (c < nch) {
        float v[8], wv[8], bv[8], g[8], o8[8], dyv[8], xhv[8];
        unpack8q(zq[i], v); unpack8q(gq[i], g); ld8_bf16(w + c * 8, wv); ld8_bf16(bsh + c * 8, bv);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float xh = (v[k] - mean) * rstd;
          const float o = (xh * wv[k] + bv[k]) * inv_n;
          const float dy = inv_n * (g[k] * gs - o * a);
          dyv[k] = dy; xhv[k] = xh;
          o8[k] = rstd * (dy * wv[k] - s1 - xh * s2);
        }
        st8_bf16(dz + row * lddz + c * 8, o8);
        if (want) {
          float4* aw = reinterpret_cast<float4*>(accw + c * 8);
          float4* ab = reinterpret_cast<float4*>(accb + c * 8);
          float4 w0 = aw[0], w1 = aw[1], b0 = ab[0], b1 = ab[1];
          w0.x += dyv[0] * xhv[0]; w0.y += dyv[1] * xhv[1]; w0.z += dyv[2] * xhv[2]; w0.w += dyv[3] * xhv[3];
          w1.x += dyv[4] * xhv[4]; w1.y += dyv[5] * xhv[5]; w1.z += dyv[6] * xhv[6]; w1.w += dyv[7] * xhv[7];
          b0.x += dyv[0]; b0.y += dyv[1]; b0.z += dyv[2]; b0.w += dyv[3];
          b1.x += dyv[4]; b1.y += dyv[5]; b1.z += dyv[6]; b1.w += dyv[7];
          aw[0] = w0; aw[1] = w1; ab[0] = b0; ab[1] = b1;
        }
      }
    }
  }
  if (want) {
    __syncthreads();
    for (int i = threadIdx.x; i < C; i += blockDim.x) {
      float sw = 0.f, sb = 0.f;
      for (int k = 0; k < wpb; ++k) { sw += acc_smem[static_cast<long>(k) * C + i]; sb += acc_smem[static_cast<long>(wpb + k) * C + i]; }
      colred_put(0, gridDim.x, blockIdx.x, C, i, sw);
      if (db) colred_put(1, gridDim.x, blockIdx.x, C, i, sb);
    }
  }
}

// loss_sum += sum (pred - label)^2 ; dpred(bf16) = gscale * 2 (pred - label) (optional)
__global__ void __launch_bounds__(256)
mse_kernel(const __nv_bfloat16* __restrict__ pred, const float* __restrict__ label, long n,
           float* __restrict__ loss_sum, float gscale_host, const float* __restrict__ gscale_dev,
           __nv_bfloat16* __restrict__ dpred) {
  const float gs = gscale_host * (gscale_dev ? *gscale_dev : 1.f);
  float acc = 0.f;
  for (long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const float d = __bfloat162float(pred[i]) - label[i];
    acc += d * d;
    if (dpred) dpred[i] = __float2bfloat16(2.f * gs * d);
  }
  __shared__ float red[8];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0 && loss_sum) { float t = 0.f; for (int k = 0; k < 8; ++k) t += red[k]; atomicAdd(loss_sum, t); }
}

}  // namespace ivb

using namespace ivb;

extern "C" int ivb_ln_l2_fwd(const void* z, long ldz, const void* weight, const void* bias, float eps,
                             int M, int C, void* out, long ldo, float* stats, const void* target,
                             int target_is_f32, long ldt, float* loss_sum, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0) return 0;
  if ((C & 7) || (ldz & 7)) return set_error("ivb_ln_l2_fwd: C/ld must be multiples of 8");
  long blocks = (M + 7) / 8;
  const long cap = static_cast<long>(num_sms()) * 8;
  if (blocks > cap) blocks = cap;
  auto zz = reinterpret_cast<const __nv_bfloat16*>(z);
  auto ww = reinterpret_cast<const __nv_bfloat16*>(weight);
  auto bb = reinterpret_cast<const __nv_bfloat16*>(bias);
  auto oo = reinterpret_cast<__nv_bfloat16*>(out);
  if (target_is_f32) ln_l2_fwd_kernel<true><<<(int)blocks, 256, 0, stream>>>(zz, ldz, ww, bb, eps, M, C, oo, ldo, stats, target, ldt, loss_sum);
  else ln_l2_fwd_kernel<false><<<(int)blocks, 256, 0, stream>>>(zz, ldz, ww, bb, eps, M, C, oo, ldo, stats, target, ldt, loss_sum);
  count_launch();
  return check_launch("ln_l2_fwd_kernel");
}

template <bool DO_F32>
static int launch_ln_l2_bwd(const void* z, long ldz, const void* weight, const void* bias,
                            const float* stats, int M, int C, const void* dout, long lddo, float gh,
                            const float* gd, void* dz, long lddz, float* dw, float* db, cudaStream_t stream) {
  auto kern = ln_l2_bwd_kernel<DO_F32>;
  int wpb = 8;
  size_t smem = dw ? static_cast<size_t>(2) * wpb * C * sizeof(float) : 0;
  while (smem > 200 * 1024 && wpb > 1) { wpb /= 2; smem /= 2; }
  if (smem > 48 * 1024) {
    static bool set[64] = {};
    if (first_use_on_device(set)) {
      cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
      if (e != cudaSuccess) return set_error_cuda("cudaFuncSetAttribute(ln_l2_bwd)", e);
    }
  }
  long blocks = (M + wpb * 2 - 1) / (wpb * 2);
  const long cap = static_cast<long>(num_sms()) * (smem > 96 * 1024 ? 2 : 4);
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  if (colred_check(2, blocks, C, "ln_l2_bwd: gradient scratch too small")) return 1;
  kern<<<(int)blocks, wpb * 32, smem, stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(z), ldz, reinterpret_cast<const __nv_bfloat16*>(weight),
      reinterpret_cast<const __nv_bfloat16*>(bias), stats, M, C, dout, lddo, gh, gd,
      reinterpret_cast<__nv_bfloat16*>(dz), lddz, dw, db);
  count_launch();
  if (int rc = check_launch("ln_l2_bwd_kernel")) return rc;
  return dw ? colred_finish(2, (int)blocks, C, dw, db, nullptr, stream) : 0;
}

template <int NCH>
static int launch_ln_l2_bwd_reg(const void* z, long ldz, const void* weight, const void* bias,
                                const float* stats, int M, int C, const void* dout, long lddo, float gh,
                                const float* gd, void* dz, long lddz, float* dw, float* db, cudaStream_t stream) {
  auto kern = ln_l2_bwd_reg_kernel<NCH>;
  const int wpb = 4;
  const size_t smem = dw ? static_cast<size_t>(2) * wpb * C * sizeof(float) : 0;   // <= 104 KB at C = 3200: 2 CTAs/SM
  if (smem > 48 * 1024) {
    static bool set[64] = {};
    if (first_use_on_device(set)) {
      cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 110 * 1024);
      if (e != cudaSuccess) return set_error_cuda("cudaFuncSetAttribute(ln_l2_bwd_reg)", e);
    }
  }
  long blocks = (M + wpb * 2 - 1) / (wpb * 2);
  const long cap = static_cast<long>(num_sms()) * 2;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  if (colred_check(2, blocks, C, "ln_l2_bwd: gradient scratch too small")) return 1;
  kern<<<(int)blocks, wpb * 32, smem, stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(z), ldz, reinterpret_cast<const __nv_bfloat16*>(weight),
      reinterpret_cast<const __nv_bfloat16*>(bias), stats, M, C, reinterpret_cast<const __nv_bfloat16*>(dout), lddo,
      gh, gd, reinterpret_cast<__nv_bfloat16*>(dz), lddz, dw, db);
  count_launch();
  if (int rc = check_launch("ln_l2_bwd_reg_kernel")) return rc;
  return dw ? colred_finish(2, (int)blocks, C, dw, db, nullptr, stream) : 0;
}

extern "C" int ivb_ln_l2_bwd(const void* z, long ldz, const void* weight, const void* bias,
                             const float* stats, int M, int C, const void* dout, int dout_is_f32,
                             long lddo, float gscale_host, const float* gscale_dev, void* dz, long lddz,
                             float* dweight, float* dbias, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0) return 0;
  if ((C & 7) || (ldz & 7) || (lddz & 7) || (lddo & 7)) return set_error("ivb_ln_l2_bwd: C/ld must be multiples of 8");
  if (!dout_is_f32 && C <= 256 * 13) {
    const int nchunks = (C + 255) / 256;
    if (nchunks <= 3) return launch_ln_l2_bwd_reg<3>(z, ldz, weight, bias, stats, M, C, dout, lddo, gscale_host, gscale_dev, dz, lddz, dweight, dbias, stream);
    if (nchunks <= 6) return launch_ln_l2_bwd_reg<6>(z, ldz, weight, bias, stats, M, C, dout, lddo, gscale_host, gscale_dev, dz, lddz, dweight, dbias, stream);
    return launch_ln_l2_bwd_reg<13>(z, ldz, weight, bias, stats, M, C, dout, lddo, gscale_host, gscale_dev, dz, lddz, dweight, dbias, stream);
  }
  if (dout_is_f32) return launch_ln_l2_bwd<true>(z, ldz, weight, bias, stats, M, C, dout, lddo, gscale_host, gscale_dev, dz, lddz, dweight, dbias, stream);
  return launch_ln_l2_bwd<false>(z, ldz, weight, bias, stats, M, C, dout, lddo, gscale_host, gscale_dev, dz, lddz, dweight, dbias, stream);
}

extern "C" int ivb_adamw_step(float* master, float* exp_avg, float* exp_avg_sq, const void* grad,
                              int grad_is_f32, void* param_bf16, long n, float lr, float beta1,
                              float beta2, float eps, float weight_decay, int step, float grad_scale,
                              const float* grad_scale_dev, const float* dyn_lr_step, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (n <= 0) return 0;
  const float bc1 = 1.f - powf(beta1, static_cast<float>(step));
  const float bc2 = 1.f - powf(beta2, static_cast<float>(step));
  const int threads = 256;
  const long blocks = (n + threads * 4 - 1) / (threads * 4);
  if (grad_is_f32)
    adamw_kernel<true><<<(unsigned)blocks, threads, 0, stream>>>(master, exp_avg, exp_avg_sq, grad, reinterpret_cast<__nv_bfloat16*>(param_bf16), n, lr, beta1, beta2, eps, weight_decay, bc1, bc2, grad_scale, grad_scale_dev, dyn_lr_step);
  else
    adamw_kernel<false><<<(unsigned)blocks, threads, 0, stream>>>(master, exp_avg, exp_avg_sq, grad, reinterpret_cast<__nv_bfloat16*>(param_bf16), n, lr, beta1, beta2, eps, weight_decay, bc1, bc2, grad_scale, grad_scale_dev, dyn_lr_step);
  count_launch();
  return check_launch("adamw_kernel");
}

extern "C" int ivb_vtc_loss_fwd(const float* cos_v2t, const long long* idx, int G, float temp,
                                const float* temp_dev, float* lse_row, float* lse_col, float* loss,
                                void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (G <= 0) return 0;
  if (temp_dev == nullptr && !(temp > 0.f)) return set_error("ivb_vtc_loss_fwd: temp must be > 0");
  vtc_stats_kernel<<<2 * G, 256, 0, stream>>>(cos_v2t, idx, G, 1.f / temp, temp_dev, lse_row, lse_col, loss);
  count_launch();
  return check_launch("vtc_stats_kernel");
}

extern "C" int ivb_vtc_loss_bwd(const float* cos_v2t, const long long* idx, int G, float temp,
                                const float* temp_dev,
                                const float* lse_row, const float* lse_col, float gscale_host,
                                const float* gscale_dev, void* dcos_bf16, float* dtemp, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (G <= 0) return 0;
  vtc_grad_kernel<<<G, 256, 0, stream>>>(cos_v2t, idx, G, 1.f / temp, temp_dev, lse_row, lse_col, gscale_host,
                                         gscale_dev, reinterpret_cast<__nv_bfloat16*>(dcos_bf16), dtemp);
  count_launch();
  return check_launch("vtc_grad_kernel");
}

extern "C" int ivb_l2norm_rows_fwd(const void* x, int x_is_f32, long ldx, int M, int C, void* out,
                                   long ldo, float* inv_norm, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0) return 0;
  if ((C & 7) || (ldx & 7) || (ldo & 7)) return set_error("ivb_l2norm_rows_fwd: C/ld must be multiples of 8");
  const int wpb = 8;
  const unsigned grid = (M + wpb - 1) / wpb;
  if (x_is_f32) l2norm_rows_kernel<true><<<grid, wpb * 32, 0, stream>>>(x, ldx, M, C, reinterpret_cast<__nv_bfloat16*>(out), ldo, inv_norm);
  else l2norm_rows_kernel<false><<<grid, wpb * 32, 0, stream>>>(x, ldx, M, C, reinterpret_cast<__nv_bfloat16*>(out), ldo, inv_norm);
  count_launch();
  return check_launch("l2norm_rows_kernel");
}

extern "C" int ivb_l2norm_rows_bwd(const float* dy, long lddy, const void* xn, long ldxn,
                                   const float* inv_norm, int M, int C, float* dx, long lddx,
                                   void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0) return 0;
  if ((C & 7) || (lddy & 7) || (ldxn & 7) || (lddx & 7)) return set_error("ivb_l2norm_rows_bwd: C/ld must be multiples of 8");
  const int wpb = 8;
  l2norm_rows_bwd_kernel<<<(M + wpb - 1) / wpb, wpb * 32, 0, stream>>>(dy, lddy, reinterpret_cast<const __nv_bfloat16*>(xn), ldxn, inv_norm, M, C, dx, lddx);
  count_launch();
  return check_launch("l2norm_rows_bwd_kernel");
}

extern "C" int ivb_pixel_targets(const void* video, const int* masked_idx, int n_mask, int B, int C,
                                 int T, int H, int W, int tubelet, int patch, int normalize,
                                 const float* mean3, const float* std3, float* labels, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (B <= 0 || n_mask <= 0) return 0;
  if (C > 8) return set_error("ivb_pixel_targets: at most 8 channels");
  pixel_target_kernel<<<B * n_mask, C * 32, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(video), masked_idx, n_mask, B, C, T, H, W, tubelet, patch, normalize, mean3, std3, labels);
  count_launch();
  return check_launch("pixel_target_kernel");
}

extern "C" int ivb_mse_loss(const void* pred_bf16, const float* label, long n, float* loss_sum,
                            float gscale_host, const float* gscale_dev, void* dpred_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (n <= 0) return 0;
  long blocks = (n + 255) / 256;
  const long cap = static_cast<long>(num_sms()) * 8;
  if (blocks > cap) blocks = cap;
  mse_kernel<<<(unsigned)blocks, 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(pred_bf16), label, n, loss_sum, gscale_host, gscale_dev, reinterpret_cast<__nv_bfloat16*>(dpred_bf16));
  count_launch();
  return check_launch("mse_kernel");
}

// ---------------------------------------------------------------- single-query attention pooling
// AttentionPoolingBlock / CrossAttention with ONE query per clip (internvideo2_pretrain.py:61-76, 107-114):
//   s_j = scale * <q_h, k_{j,h}> ; p = softmax_j(s) ; o_h = sum_j p_j v_{j,h}.   One CTA per (head, clip).
namespace ivb {

__device__ __forceinline__ float block_reduce_128(float v, float* red, bool is_max) {
  v = is_max ? warp_max(v) : warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = red[0];
  for (int k = 1; k < 4; ++k) r = is_max ? fmaxf(r, red[k]) : r + red[k];
  return r;
}

__global__ void __launch_bounds__(128)
pool_attn_fwd_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k, long ldk,
                     const __nv_bfloat16* __restrict__ v, long ldv, int n, int H, int d, float scale,
                     __nv_bfloat16* __restrict__ out, float* __restrict__ probs) {
  extern __shared__ float sm[];          // [d] q_h | [n] scores/probs | [4] red
  float* sq = sm;
  float* sp = sm + d;
  float* red = sp + n;
  const int h = blockIdx.x, b = blockIdx.y, D = H * d;
  for (int i = threadIdx.x; i < d; i += blockDim.x) sq[i] = __bfloat162float(q[static_cast<long>(b) * D + h * d + i]) * scale;
  __syncthreads();
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const __nv_bfloat16* kr = k + (static_cast<long>(b) * n + j) * ldk + h * d;
    float s = 0.f;
    for (int c = 0; c < d; c += 8) {
      float kv[8];
      ld8_bf16(kr + c, kv);
#pragma unroll
      for (int t = 0; t < 8; ++t) s += kv[t] * sq[c + t];
    }
    sp[j] = s;
    mx = fmaxf(mx, s);
  }
  mx = block_reduce_128(mx, red, true);
  float se = 0.f;
  for (int j = threadIdx.x; j < n; j += blockDim.x) { const float e = __expf(sp[j] - mx); sp[j] = e; se += e; }
  se = block_reduce_128(se, red, false);
  const float inv = 1.f / se;
  __syncthreads();
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const float pj = sp[j] * inv;
    sp[j] = pj;
    probs[(static_cast<long>(b) * H + h) * n + j] = pj;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    float o = 0.f;
    const __nv_bfloat16* vc = v + static_cast<long>(b) * n * ldv + h * d + c;
    for (int j = 0; j < n; ++j) o += sp[j] * __bfloat162float(vc[static_cast<long>(j) * ldv]);
    out[static_cast<long>(b) * D + h * d + c] = __float2bfloat16(o);
  }
}

__global__ void __launch_bounds__(128)
pool_attn_bwd_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k, long ldk,
                     const __nv_bfloat16* __restrict__ v, long ldv, const float* __restrict__ probs,
                     const __nv_bfloat16* __restrict__ dout, int n, int H, int d, float scale,
                     __nv_bfloat16* __restrict__ dq, __nv_bfloat16* __restrict__ dk, long lddk,
                     __nv_bfloat16* __restrict__ dv, long lddv) {
  extern __shared__ float sm[];          // [d] q_h*scale | [d] do_h | [n] ds | [4] red
  float* sq = sm;
  float* sdo = sm + d;
  float* sds = sdo + d;
  float* red = sds + n;
  const int h = blockIdx.x, b = blockIdx.y, D = H * d;
  for (int i = threadIdx.x; i < d; i += blockDim.x) {
    sq[i] = __bfloat162float(q[static_cast<long>(b) * D + h * d + i]) * scale;
    sdo[i] = __bfloat162float(dout[static_cast<long>(b) * D + h * d + i]);
  }
  __syncthreads();
  const float* pr = probs + (static_cast<long>(b) * H + h) * n;
  float acc = 0.f;
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const __nv_bfloat16* vr = v + (static_cast<long>(b) * n + j) * ldv + h * d;
    float dp = 0.f;
    for (int c = 0; c < d; c += 8) {
      float vv[8];
      ld8_bf16(vr + c, vv);
#pragma unroll
      for (int t = 0; t < 8; ++t) dp += vv[t] * sdo[c + t];
    }
    sds[j] = dp;
    acc += pr[j] * dp;
  }
  acc = block_reduce_128(acc, red, false);
  __syncthreads();
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const float pj = pr[j];
    const float ds = pj * (sds[j] - acc);
    sds[j] = ds;
    __nv_bfloat16* dkr = dk + (static_cast<long>(b) * n + j) * lddk + h * d;
    __nv_bfloat16* dvr = dv + (static_cast<long>(b) * n + j) * lddv + h * d;
    for (int c = 0; c < d; c += 8) {
      float a[8], bb[8];
#pragma unroll
      for (int t = 0; t < 8; ++t) { a[t] = ds * sq[c + t]; bb[t] = pj * sdo[c + t]; }
      st8_bf16(dkr + c, a);
      st8_bf16(dvr + c, bb);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    float g = 0.f;
    const __nv_bfloat16* kc = k + static_cast<long>(b) * n * ldk + h * d + c;
    for (int j = 0; j < n; ++j) g += sds[j] * __bfloat162float(kc[static_cast<long>(j) * ldk]);
    dq[static_cast<long>(b) * D + h * d + c] = __float2bfloat16(g * scale);
  }
}

}  // namespace ivb

extern "C" int ivb_pool_attn_fwd(const void* q, const void* k, long ldk, const void* v, long ldv, int B,
                                 int n, int H, int d, float scale, void* out, float* probs, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (B <= 0) return 0;
  if ((d & 7) || (ldk & 7) || (ldv & 7)) return set_error("ivb_pool_attn_fwd: d/ld must be multiples of 8");
  const size_t smem = (static_cast<size_t>(d) + n + 8) * sizeof(float);
  if (smem > 48 * 1024) return set_error("ivb_pool_attn_fwd: sequence too long for the single-query kernel");
  pool_attn_fwd_kernel<<<dim3(H, B), 128, smem, stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(q), reinterpret_cast<const __nv_bfloat16*>(k), ldk,
      reinterpret_cast<const __nv_bfloat16*>(v), ldv, n, H, d, scale, reinterpret_cast<__nv_bfloat16*>(out), probs);
  count_launch();
  return check_launch("pool_attn_fwd_kernel");
}

extern "C" int ivb_pool_attn_bwd(const void* q, const void* k, long ldk, const void* v, long ldv,
                                 const float* probs, const void* dout, int B, int n, int H, int d,
                                 float scale, void* dq, void* dk, long lddk, void* dv, long lddv,
                                 void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (B <= 0) return 0;
  if ((d & 7) || (ldk & 7) || (ldv & 7) || (lddk & 7) || (lddv & 7)) return set_error("ivb_pool_attn_bwd: d/ld must be multiples of 8");
  const size_t smem = (2 * static_cast<size_t>(d) + n + 8) * sizeof(float);
  if (smem > 48 * 1024) return set_error("ivb_pool_attn_bwd: sequence too long for the single-query kernel");
  pool_attn_bwd_kernel<<<dim3(H, B), 128, smem, stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(q), reinterpret_cast<const __nv_bfloat16*>(k), ldk,
      reinterpret_cast<const __nv_bfloat16*>(v), ldv, probs, reinterpret_cast<const __nv_bfloat16*>(dout), n, H, d,
      scale, reinterpret_cast<__nv_bfloat16*>(dq), reinterpret_cast<__nv_bfloat16*>(dk), lddk,
      reinterpret_cast<__nv_bfloat16*>(dv), lddv);
  count_launch();
  return check_launch("pool_attn_bwd_kernel");
}
