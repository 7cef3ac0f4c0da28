// Test-only entry points: one run_linear call on either GEMM path (the SIMT fp32 kernel or the wgmma split-fp16 kernel) in
// any of its modes, one 3x3 convolution layer on either path (k_conv3x3 or k_conv_ps), the wgmma kernel's column-segment /
// rotary epilogue, and one batched launch of the split-fp16 flash attention kernel.
#include <stdlib.h>

#include <vector>

#include "common.cuh"
#include "conv_ps.cuh"
#include "linear.cuh"

// fp32 -> fp16 hi plane and UNSCALED lo plane (the operand format of the attention kernel)
static __global__ void k_split_unscaled_f32(const float* __restrict__ x, size_t n, __half* __restrict__ hi, __half* __restrict__ lo) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) tc::split_h_unscaled(x[i], hi[i], lo[i]);
}

// One fp32 operand on the device: the host values, and their hi / lo * 2^11 planes (the producing epilogues' format)
struct DbgOperand {
  DevBuf f, h, l;
};
static int dbg_upload_split(b2_context* ctx, cudaStream_t st, const float* host, size_t n, DbgOperand& o) {
  if (n == 0) return B2_OK;
  B2_CUDA(ctx, o.f.ensure(n * 4));
  B2_CUDA(ctx, o.h.ensure(n * 2));
  B2_CUDA(ctx, o.l.ensure(n * 2));
  B2_CUDA(ctx, cudaMemcpyAsync(o.f.p, host, n * 4, cudaMemcpyHostToDevice, st));
  B2_LAUNCH(ctx, k_split_f32, (unsigned)((n + 255) / 256), 256, 0, st, o.f.as<float>(), n, o.h.as<__half>(), o.l.as<__half>());
  B2_CHECK_LAUNCH(ctx);
  return B2_OK;
}
extern "C" int b2_debug_linear_host(b2_context* ctx, const b2_linear_launch* L, const b2_linear_problem* P, int np) {
  if (!ctx || !L || !P || np <= 0 || (L->path != 0 && L->path != 1) || L->k1 < 0 || L->k2 < 0) return B2_ERR_ARG;
  const bool tc = L->path == 1, hm = L->head_major != 0;
  if (!P[0].b || P[0].ldb < L->k1 + L->k2) return b2_fail(ctx, B2_ERR_ARG, "b2_debug_linear_host: problem 0 needs a B operand");
  // the kernel takes the residual's and the planes' leading dimensions once per launch: every problem must agree
  int maxn = 0, ldr = -1, ldch = -1;
  for (int i = 0; i < np; ++i) {
    const b2_linear_problem& p = P[i];
    if (p.m < 0 || p.n < 0) return b2_fail(ctx, B2_ERR_ARG, "b2_debug_linear_host: negative m or n");
    if (p.m == 0 || p.n == 0) continue;
    maxn = p.n > maxn ? p.n : maxn;
    if (!p.a1 || p.lda1 < L->k1 || (L->k2 && (!p.a2 || p.lda2 < L->k2)) || (L->per_problem_b && (!p.b || p.ldb < L->k1 + L->k2)))
      return b2_fail(ctx, B2_ERR_ARG, "b2_debug_linear_host: a missing operand or a leading dimension below its K");
    if (!p.c && !p.c_hi) return b2_fail(ctx, B2_ERR_ARG, "b2_debug_linear_host: a problem without an output");
    if (!p.c_hi != !p.c_lo) return b2_fail(ctx, B2_ERR_ARG, "b2_debug_linear_host: planes come in pairs (c_hi and c_lo)");
    if (!tc && (p.c_hi || !p.c)) return b2_fail(ctx, B2_ERR_ARG, "b2_debug_linear_host: the SIMT path writes an fp32 output only");
    if (p.c && !hm && p.ldc < p.n) return b2_fail(ctx, B2_ERR_ARG, "b2_debug_linear_host: ldc below n");
    if (L->resid_in_place && (!p.c || p.resid || hm))
      return b2_fail(ctx, B2_ERR_ARG, "b2_debug_linear_host: an in-place residual needs a row-major fp32 output and no resid");
    const int r = L->resid_in_place ? p.ldc : (p.resid ? p.ldr : -1);
    if (r >= 0 && ((ldr >= 0 && r != ldr) || r < p.n)) return b2_fail(ctx, B2_ERR_ARG, "b2_debug_linear_host: residual pitches differ or are below n");
    if (r >= 0) ldr = r;
    if (p.c_hi && !hm) {
      if ((ldch >= 0 && p.ldch != ldch) || p.ldch < p.n) return b2_fail(ctx, B2_ERR_ARG, "b2_debug_linear_host: plane pitches differ or are below n");
      ldch = p.ldch;
    }
  }
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  struct Bufs {
    DbgOperand a1, a2, b;
    DevBuf r, c, ch, cl;
  };
  std::vector<Bufs> d(np);
  DevBuf dBias, dErr;
  B2_CUDA(ctx, dErr.ensure(16));
  B2_CUDA(ctx, cudaMemsetAsync(dErr.p, 0, 16, st));
  if (L->bias && maxn) {
    B2_CUDA(ctx, dBias.ensure((size_t)maxn * 4));
    B2_CUDA(ctx, cudaMemcpyAsync(dBias.p, L->bias, (size_t)maxn * 4, cudaMemcpyHostToDevice, st));
  }
  int rc;
  if (!L->per_problem_b && (rc = dbg_upload_split(ctx, st, P[0].b, (size_t)maxn * P[0].ldb, d[0].b))) return rc;
  std::vector<LinArgs> la(np);
  for (int i = 0; i < np; ++i) {
    const b2_linear_problem& p = P[i];
    Bufs& q = d[i];
    LinArgs& a = la[i];
    // run_linear reads K and the epilogue of the launch from problem 0, which may be an empty one
    a.K1 = L->k1, a.K2 = L->k2, a.bias = L->bias ? dBias.as<float>() : nullptr, a.scale = L->scale;
    a.ldr = ldr > 0 ? ldr : 0, a.ldch = ldch > 0 ? ldch : 0;
    a.head_major = L->head_major, a.relu = L->relu, a.gelu = L->gelu, a.lo_unscaled = L->lo_unscaled, a.M = p.m, a.N = p.n;
    if (!L->per_problem_b) a.w = d[0].b.f.as<float>(), a.ldb = P[0].ldb;  // the weight of the launch, its planes through TcWeights
    if (p.m == 0 || p.n == 0) continue;  // run_linear skips the problem
    const size_t m = (size_t)p.m, hm_elems = (size_t)cdiv(p.n, 64) * m * 64;
    if ((rc = dbg_upload_split(ctx, st, p.a1, m * p.lda1, q.a1))) return rc;
    if (L->k2 && (rc = dbg_upload_split(ctx, st, p.a2, m * p.lda2, q.a2))) return rc;
    if (L->per_problem_b && (rc = dbg_upload_split(ctx, st, p.b, (size_t)p.n * p.ldb, q.b))) return rc;
    if (p.resid && (rc = dbg_upload(ctx, st, p.resid, m * p.ldr * 4, 0, q.r))) return rc;
    if (p.c && (rc = dbg_upload(ctx, st, p.c, (hm ? hm_elems : m * p.ldc) * 4, (size_t)GW_M * (hm ? 64 : p.ldc) * 4, q.c))) return rc;
    if (p.c_hi) {
      const size_t e = hm ? hm_elems : m * p.ldch, g = (size_t)GW_M * (hm ? 64 : p.ldch) * 2;
      if ((rc = dbg_upload(ctx, st, p.c_hi, e * 2, g, q.ch)) || (rc = dbg_upload(ctx, st, p.c_lo, e * 2, g, q.cl))) return rc;
    }
    a.a1f = q.a1.f.as<float>(), a.a1p = {q.a1.h.as<__half>(), q.a1.l.as<__half>()}, a.lda1 = p.lda1;
    if (L->k2) a.a2f = q.a2.f.as<float>(), a.a2p = {q.a2.h.as<__half>(), q.a2.l.as<__half>()}, a.lda2 = p.lda2;
    if (L->per_problem_b) a.bf = q.b.f.as<float>(), a.bp = {q.b.h.as<__half>(), q.b.l.as<__half>()}, a.ldb = p.ldb;
    a.resid = L->resid_in_place ? q.c.as<float>() : (p.resid ? q.r.as<float>() : nullptr);
    a.cf = p.c ? q.c.as<float>() : nullptr, a.ldc = p.ldc, a.tc_want_f32 = p.c != nullptr;
    a.cp = {q.ch.as<__half>(), q.cl.as<__half>()};
  }
  if (tc) B2_CUDA(ctx, cudaFuncSetAttribute(k_gemm_ws, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GW_SMEM));
  TcWeights tw{d[0].b.f.as<float>(), d[0].b.h.as<__half>(), d[0].b.l.as<__half>(), dErr.as<int>(), tc};
  tw.sm_count = ctx->sm_count;
  if ((rc = run_linear(ctx, st, tw, la.data(), np))) return rc;
  bool guard_ok = true;
  for (int i = 0; i < np; ++i) {
    const b2_linear_problem& p = P[i];
    const Bufs& q = d[i];
    if (p.m == 0 || p.n == 0) continue;
    const size_t m = (size_t)p.m, e = hm ? (size_t)cdiv(p.n, 64) * m * 64 : 0;
    if (p.c && (rc = dbg_download(ctx, st, p.c, (hm ? e : m * p.ldc) * 4, (size_t)GW_M * (hm ? 64 : p.ldc) * 4, q.c, guard_ok))) return rc;
    if (p.c_hi) {
      const size_t eh = hm ? e : m * p.ldch, g = (size_t)GW_M * (hm ? 64 : p.ldch) * 2;
      if ((rc = dbg_download(ctx, st, p.c_hi, eh * 2, g, q.ch, guard_ok)) || (rc = dbg_download(ctx, st, p.c_lo, eh * 2, g, q.cl, guard_ok))) return rc;
    }
  }
  if (!guard_ok) return b2_fail(ctx, B2_ERR_STATE, "b2_debug_linear_host: the kernel wrote past row m of an output");
  int err = 0;
  B2_CUDA(ctx, cudaMemcpyAsync(&err, dErr.p, 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  if (err) return b2_fail(ctx, B2_ERR_STATE, "wgmma pipeline timed out on an mbarrier (kernel bug)");
  return B2_OK;
}

extern "C" int b2_debug_conv_host(b2_context* ctx, const b2_conv_layer* L) {
  if (!ctx || !L) return B2_ERR_ARG;
  const b2_conv_layer& c = *L;
  const int H = c.height, W = c.width, Cin = c.cin, Cout = c.cout;
  const bool tc = c.path == 1, pool = c.pool != 0;
  if (c.path != 0 && c.path != 1) return b2_fail(ctx, B2_ERR_ARG, "b2_debug_conv_host: path must be 0 (SIMT) or 1 (wgmma)");
  if (!c.in || !c.weight || !c.bias) return b2_fail(ctx, B2_ERR_ARG, "b2_debug_conv_host: missing input, weight or bias");
  if (!c.out && !c.out_hi) return b2_fail(ctx, B2_ERR_ARG, "b2_debug_conv_host: no output");
  if (!c.out_hi != !c.out_lo) return b2_fail(ctx, B2_ERR_ARG, "b2_debug_conv_host: planes come in pairs (out_hi and out_lo)");
  if (H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0) return b2_fail(ctx, B2_ERR_ARG, "b2_debug_conv_host: a size below 1");
  if (pool && (H < 2 || W < 2)) return b2_fail(ctx, B2_ERR_ARG, "b2_debug_conv_host: the pooled output would be empty");
  // k_conv3x3 has ReLU built in, pads by 1, loads Cin in steps of CK channels and writes 64-channel blocks of fp32
  if (!tc && (!c.relu || c.dilation != 1 || Cin % CK || Cout % 64 || c.out_hi || c.ctas))
    return b2_fail(ctx, B2_ERR_ARG, "b2_debug_conv_host: the SIMT path needs ReLU, dilation 1, Cin a multiple of 8, Cout of 64, an fp32 "
                                    "output only and its own grid");
  const int OH = pool ? H / 2 : H, OW = pool ? W / 2 : W;
  const size_t nin = (size_t)H * W * Cin, nout = (size_t)OH * OW * Cout, nw = (size_t)Cout * 9 * Cin;
  const size_t guard = ((size_t)CP_TH * OW + CP_TW) * Cout;  // elements: a tile's rows below the output and a tile's width past them
  // weights OIHW -> [co][tap * Cin + ci] for the implicit GEMM (conv_ps_repack's order), [tap][ci][co] for the SIMT kernel
  std::vector<float> wk(nw);
  for (int o = 0; o < Cout; ++o)
    for (int i = 0; i < Cin; ++i)
      for (int tp = 0; tp < 9; ++tp) {
        const float v = c.weight[((size_t)o * Cin + i) * 9 + tp];
        if (tc) wk[(size_t)o * 9 * Cin + (size_t)tp * Cin + i] = v;
        else wk[((size_t)tp * Cin + i) * Cout + o] = v;
      }
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  DbgOperand x, w;
  DevBuf xp, b, of, op, err;
  int rc;
  B2_CUDA(ctx, err.ensure(16));
  B2_CUDA(ctx, cudaMemsetAsync(err.p, 0, 16, st));
  B2_CUDA(ctx, b.ensure((size_t)Cout * 4));
  B2_CUDA(ctx, cudaMemcpyAsync(b.p, c.bias, (size_t)Cout * 4, cudaMemcpyHostToDevice, st));
  if (tc) {
    if ((rc = dbg_upload_split(ctx, st, wk.data(), nw, w))) return rc;
    // the input's planes in one buffer, lo after hi, as conv_ps_run reads them
    B2_CUDA(ctx, x.f.ensure(nin * 4));
    B2_CUDA(ctx, xp.ensure(nin * 2 * 2));
    B2_CUDA(ctx, cudaMemcpyAsync(x.f.p, c.in, nin * 4, cudaMemcpyHostToDevice, st));
    B2_LAUNCH(ctx, k_split_f32, (unsigned)((nin + 255) / 256), 256, 0, st, x.f.as<float>(), nin, xp.as<__half>(), xp.as<__half>() + nin);
    B2_CHECK_LAUNCH(ctx);
  } else {
    if ((rc = dbg_upload(ctx, st, c.in, nin * 4, 0, x.f)) || (rc = dbg_upload(ctx, st, wk.data(), nw * 4, 0, w.f))) return rc;
  }
  if (c.out && (rc = dbg_upload(ctx, st, c.out, nout * 4, guard * 4, of))) return rc;
  if (c.out_hi) {  // one buffer, lo after hi (conv_ps_run's layout), then the guard
    B2_CUDA(ctx, op.ensure((2 * nout + guard) * 2));
    B2_CUDA(ctx, cudaMemcpyAsync(op.p, c.out_hi, nout * 2, cudaMemcpyHostToDevice, st));
    B2_CUDA(ctx, cudaMemcpyAsync(op.as<__half>() + nout, c.out_lo, nout * 2, cudaMemcpyHostToDevice, st));
    B2_CUDA(ctx, cudaMemsetAsync(op.as<__half>() + 2 * nout, 0xFF, guard * 2, st));
  }
  if (tc) {
    B2_CUDA(ctx, cudaFuncSetAttribute(k_conv_ps<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CP_SMEM));
    B2_CUDA(ctx, cudaFuncSetAttribute(k_conv_ps<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CpGeom<2>::SMEM));
    rc = conv_ps_run(ctx, st, xp.as<__half>(), H, W, Cin, Cout, pool, c.relu != 0, c.dilation, w.h.as<__half>(), w.l.as<__half>(), b.as<float>(),
                     c.out_hi ? op.as<__half>() : nullptr, c.out ? of.as<float>() : nullptr, err.as<int>(), "debug", c.ctas);
  } else {
    rc = conv3x3_simt_run(ctx, st, x.f.as<float>(), w.f.as<float>(), b.as<float>(), of.as<float>(), H, W, Cin, Cout, pool);
  }
  if (rc) return rc;
  bool guard_ok = true;
  if (c.out && (rc = dbg_download(ctx, st, c.out, nout * 4, guard * 4, of, guard_ok))) return rc;
  if (c.out_hi) {
    std::vector<unsigned char> g(guard * 2);
    B2_CUDA(ctx, cudaMemcpyAsync(c.out_hi, op.p, nout * 2, cudaMemcpyDeviceToHost, st));
    B2_CUDA(ctx, cudaMemcpyAsync(c.out_lo, op.as<__half>() + nout, nout * 2, cudaMemcpyDeviceToHost, st));
    B2_CUDA(ctx, cudaMemcpyAsync(g.data(), op.as<__half>() + 2 * nout, guard * 2, cudaMemcpyDeviceToHost, st));
    B2_CUDA(ctx, cudaStreamSynchronize(st));
    for (unsigned char v : g) guard_ok = guard_ok && v == 0xFF;
  }
  if (!guard_ok) return b2_fail(ctx, B2_ERR_STATE, "b2_debug_conv_host: the kernel wrote past the end of an output");
  int e = 0;
  B2_CUDA(ctx, cudaMemcpyAsync(&e, err.p, 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  if (e) return b2_fail(ctx, B2_ERR_STATE, "wgmma pipeline timed out on an mbarrier (kernel bug)");
  return B2_OK;
}

extern "C" int b2_debug_gemm_segments_host(b2_context* ctx, const float* A, const float* B, const float* bias, int M, int K, int nseg,
                                           int rot_mask, const float* cs, const float* sn, int separate, uint16_t* out_hi, uint16_t* out_lo) {
  if (!ctx || !A || !B || !bias || !out_hi || !out_lo || M <= 0 || K <= 0 || (K % 64) || nseg < 1 || nseg > GW_SEGS ||
      (rot_mask && (!cs || !sn || separate)))
    return B2_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  const int N = 256 * nseg;
  const size_t ep = (size_t)M * 256;  // halves of one segment's plane
  DevBuf dA, dB, dBias, dCs, dSn, dErr, dAh, dAl, dBh, dBl, dH, dL;
  B2_CUDA(ctx, dA.ensure((size_t)M * K * 4));
  B2_CUDA(ctx, dB.ensure((size_t)N * K * 4));
  B2_CUDA(ctx, dBias.ensure((size_t)N * 4));
  B2_CUDA(ctx, dCs.ensure((size_t)M * 32 * 4));
  B2_CUDA(ctx, dSn.ensure((size_t)M * 32 * 4));
  B2_CUDA(ctx, dErr.ensure(16));
  B2_CUDA(ctx, dAh.ensure((size_t)M * K * 2));
  B2_CUDA(ctx, dAl.ensure((size_t)M * K * 2));
  B2_CUDA(ctx, dBh.ensure((size_t)N * K * 2));
  B2_CUDA(ctx, dBl.ensure((size_t)N * K * 2));
  B2_CUDA(ctx, dH.ensure(nseg * ep * 2));
  B2_CUDA(ctx, dL.ensure(nseg * ep * 2));
  B2_CUDA(ctx, cudaMemcpyAsync(dA.p, A, (size_t)M * K * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(dB.p, B, (size_t)N * K * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(dBias.p, bias, (size_t)N * 4, cudaMemcpyHostToDevice, st));
  if (rot_mask) {
    B2_CUDA(ctx, cudaMemcpyAsync(dCs.p, cs, (size_t)M * 32 * 4, cudaMemcpyHostToDevice, st));
    B2_CUDA(ctx, cudaMemcpyAsync(dSn.p, sn, (size_t)M * 32 * 4, cudaMemcpyHostToDevice, st));
  }
  B2_CUDA(ctx, cudaMemsetAsync(dErr.p, 0, 16, st));
  B2_LAUNCH(ctx, k_split_f32, (unsigned)(((size_t)M * K + 255) / 256), 256, 0, st, dA.as<float>(), (size_t)M * K, dAh.as<__half>(), dAl.as<__half>());
  B2_LAUNCH(ctx, k_split_f32, (unsigned)(((size_t)N * K + 255) / 256), 256, 0, st, dB.as<float>(), (size_t)N * K, dBh.as<__half>(), dBl.as<__half>());
  B2_CUDA(ctx, cudaFuncSetAttribute(k_gemm_ws, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GW_SMEM));
  TcWeights tw{nullptr, nullptr, nullptr, dErr.as<int>(), true};
  tw.sm_count = ctx->sm_count;
  __half *H = dH.as<__half>(), *L = dL.as<__half>(), *Bh = dBh.as<__half>(), *Bl = dBl.as<__half>();
  LinArgs a;
  a.a1p = {dAh.as<__half>(), dAl.as<__half>()}, a.lda1 = K, a.K1 = K, a.ldb = K, a.M = M, a.head_major = 1, a.lo_unscaled = 1;
  for (int s = 0; s < (separate ? nseg : 1); ++s) {
    if (separate) {  // segment s as a linear of its own: its 256 rows of B and of the bias
      a.bp = {Bh + (size_t)s * 256 * K, Bl + (size_t)s * 256 * K}, a.bias = dBias.as<float>() + s * 256, a.N = 256;
      a.cp = {H + s * ep, L + s * ep};
    } else {
      a.bp = {Bh, Bl}, a.bias = dBias.as<float>(), a.N = N, a.seg_n = 256;
      for (int j = 0; j < nseg; ++j) a.seg_p[j] = {H + j * ep, L + j * ep};
      a.rot_mask = rot_mask, a.cs = dCs.as<float>(), a.sn = dSn.as<float>();
    }
    const int rc = run_linear(ctx, st, tw, &a, 1);
    if (rc != B2_OK) return rc;
  }
  int err = 0;
  B2_CUDA(ctx, cudaMemcpyAsync(out_hi, H, nseg * ep * 2, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(out_lo, L, nseg * ep * 2, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(&err, dErr.p, 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  if (err) return b2_fail(ctx, B2_ERR_STATE, "wgmma pipeline timed out on an mbarrier (kernel bug)");
  return B2_OK;
}

extern "C" int b2_debug_attention_host(b2_context* ctx, int np, const int* nq, const int* nk, int heads, float scale, int single,
                                       const float* q, const float* k, const float* v, float* o) {
  if (!ctx || !nq || !nk || !q || !k || !v || !o || np <= 0 || np > AP_MAXP || heads <= 0) return B2_ERR_ARG;
  size_t eq = 0, ek = 0;  // elements of q (and o), of k (and v)
  for (int z = 0; z < np; ++z) {
    if (nq[z] <= 0 || nk[z] <= 0) return B2_ERR_ARG;
    eq += (size_t)nq[z] * heads * 64, ek += (size_t)nk[z] * heads * 64;
  }
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  const size_t n = eq + 2 * ek;  // q, k, v back to back
  DevBuf dIn, dPl, dO, dErr, part, ml, cnt;
  B2_CUDA(ctx, dIn.ensure(n * 4));
  B2_CUDA(ctx, dPl.ensure(n * 2 * 2));
  B2_CUDA(ctx, dO.ensure(eq * 2 * 2));
  B2_CUDA(ctx, dErr.ensure(16));
  float* in = dIn.as<float>();
  B2_CUDA(ctx, cudaMemcpyAsync(in, q, eq * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(in + eq, k, ek * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(in + eq + ek, v, ek * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemsetAsync(dErr.p, 0, 16, st));
  __half *hi = dPl.as<__half>(), *lo = hi + n, *oh = dO.as<__half>(), *ol = oh + eq;
  B2_LAUNCH(ctx, k_split_unscaled_f32, (unsigned)((n + 255) / 256), 256, 0, st, in, n, hi, lo);
  B2_CUDA(ctx, cudaFuncSetAttribute(k_flash_ps<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AS_SMEM));
  B2_CUDA(ctx, cudaFuncSetAttribute(k_flash_ps<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AS_SMEM));
  FlashPlanes fp[AP_MAXP];
  size_t qo = 0, ko = eq;
  for (int z = 0; z < np; ++z) {
    const size_t vo = ko + ek;
    fp[z] = {{hi + qo, lo + qo}, {hi + ko, lo + ko}, {hi + vo, lo + vo}, {oh + qo, ol + qo}, nq[z], nk[z], heads, 64 * heads};
    qo += (size_t)nq[z] * heads * 64, ko += (size_t)nk[z] * heads * 64;
  }
  TcWeights tw{nullptr, nullptr, nullptr, dErr.as<int>(), true};
  tw.attn_part = &part, tw.attn_ml = &ml, tw.attn_cnt = &cnt, tw.sm_count = ctx->sm_count;
  const int rc = run_flash_planes(ctx, st, tw, fp, np, scale, single != 0);
  if (rc != B2_OK) return rc;
  std::vector<__half> ho(2 * eq);
  int err = 0;
  B2_CUDA(ctx, cudaMemcpyAsync(ho.data(), oh, eq * 2 * 2, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(&err, dErr.p, 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  // o = hi + lo * 2^-11 (the SINGLE variant writes lo = 0)
  for (size_t i = 0; i < eq; ++i) o[i] = __half2float(ho[i]) + __half2float(ho[eq + i]) * tc::LO_INV;
  if (err) return b2_fail(ctx, B2_ERR_STATE, "wgmma attention timed out on an mbarrier (kernel bug)");
  return B2_OK;
}
