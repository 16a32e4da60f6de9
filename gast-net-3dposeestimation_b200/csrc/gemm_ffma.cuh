// FP32 (FFMA) tile GEMM with the fused epilogues of the GAST-Net lifting path.
//
//   out[rows of a frame tile, N] = epilogue( [A_seg0 | A_seg1 | A_seg2][rows, K] . W[N, K]^T )
//
// Rows are (frame, joint) positions in channels-last layout; a CTA owns `fpt` whole frames
// (fpt*J <= 128 rows) so that the joint-mixing epilogues (SemCH neighbour mix, global
// attention) never leave the tile.  A segments are gathered with a per-frame remap, which is
// how the dilated / strided temporal convolutions (gast_net.py:145-148,222-224), the
// residual slices (:170,:243) and the channel concatenations (:28, local_attention.py:142)
// are expressed without materialising anything.
//
// This is the exact-fp32 core: used for shapes the tensor-core core does not take (K % 32 != 0,
// tiny widths) and as the on-GPU cross-check of the tensor-core path.
#pragma once
#include "gast_common.cuh"

namespace gast {

constexpr int FF_BM = 128;
constexpr int FF_BN = 128;
constexpr int FF_BK = 16;
constexpr int FF_THREADS = 256;
constexpr int FF_LDS = FF_BM + 4;  // smem leading dim (floats), keeps float4 alignment

enum { EPI_PLAIN = 0, EPI_SEMCH = 1, EPI_GLOBAL = 2 };

// dynamic smem (floats): main loop tiles, reused by the epilogues
//   main loop : 2 * BK * LDS (A) + 2 * BK * LDS (B)
//   EPI_SEMCH : H1 staging 128 x 64
//   EPI_GLOBAL: G staging 128 x 128, attention fpt*heads*J*J, ab 128 x 8
__host__ __device__ inline size_t ffma_smem_bytes(int epi, int J, int fpt, int hpt) {
  size_t main_f = 4 * FF_BK * FF_LDS;
  size_t f = main_f;
  if (epi == EPI_SEMCH) f = (main_f > 128 * 64) ? main_f : 128 * 64;
  if (epi == EPI_GLOBAL) {
    size_t g = 128 * 128 + (size_t)fpt * hpt * J * J + 128 * 2 * 4;
    f = (main_f > g) ? main_f : g;
  }
  return f * sizeof(float) + 3 * 128 * sizeof(long long);
}

// The epilogues run on 256 threads: the whole block of the FFMA core, the two consumer warpgroups of the
// tensor-core core (whose producer warpgroup has left by then), so they synchronise on named barrier 1 over 256.
__device__ __forceinline__ void epi_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// Fused epilogues shared by both GEMM cores.  `acc` holds the 128 x 128 tile product in the FFMA thread layout:
// thread tid (of 256) owns rows {ty*4+i, 64+ty*4+i} (i<4) and cols {tx*4+j, 64+tx*4+j} (j<4), ty = tid/16,
// tx = tid%16.  `smem` is free scratch of at least ffma_smem_bytes() - 3*128*8 bytes; callers synchronise before.
// The tile is frames f0 .. f0 + nf - 1 (vrows rows) x columns n0 .. n0 + 127, column tile `ctile` (n0 = 128 ctile).
template <int EPI>
__device__ __forceinline__ void gemm_epilogue(const GemmP& p, const float (&acc)[8][8], float* smem, int tid,
                                              int f0, int nf, int vrows, int n0, int ctile) {
  const int J = p.J;
  const int ty = tid >> 4, tx = tid & 15;
  if (EPI == EPI_PLAIN) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      int r = (i < 4) ? (ty * 4 + i) : (64 + ty * 4 + i - 4);
      if (r >= vrows) continue;
      int fr = r / J, j = r - fr * J;
      long long orow = ((long long)(f0 + fr) * J + j);
      const float* resrow = nullptr;
      if (p.res) {
        long long fin = map_frame(p.res_map, f0 + fr);
        resrow = p.res + (fin * J + j) * (long long)p.res_ld;
      }
#pragma unroll
      for (int g = 0; g < 2; ++g) {
        int n = n0 + g * 64 + tx * 4;
        if (n >= p.N) continue;
        float v[4] = {acc[i][g * 4 + 0], acc[i][g * 4 + 1], acc[i][g * 4 + 2], acc[i][g * 4 + 3]};
        if (p.bias) {
          float4 bb = ldg4(p.bias + n);
          v[0] += bb.x; v[1] += bb.y; v[2] += bb.z; v[3] += bb.w;
        }
        if (p.relu) {
#pragma unroll
          for (int q = 0; q < 4; ++q) v[q] = fmaxf(v[q], 0.f);
        }
        if (resrow) {
          float4 rr = ldg4(resrow + n);
          v[0] += rr.x; v[1] += rr.y; v[2] += rr.z; v[3] += rr.w;
        }
        *reinterpret_cast<float4*>(p.out + orow * p.ld_out + n) = make_float4(v[0], v[1], v[2], v[3]);
      }
    }
  } else if (EPI == EPI_SEMCH) {
    // tile = 64 channels of one mask: cols [0,64) = X.W0 (self), cols [64,128) = X.W1 (neighbours)
    float* Hs = smem;  // [128][64]
    // the caller synchronised after its main loop: smem is free
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      int r = (i < 4) ? (ty * 4 + i) : (64 + ty * 4 + i - 4);
      *reinterpret_cast<float4*>(Hs + r * 64 + tx * 4) =
          make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]);
    }
    epi_sync();
    const int mask = ctile / p.tiles_per_mask;
    const int c0 = (ctile - mask * p.tiles_per_mask) * 64 + tx * 4;
    if (c0 < p.C) {
      const NbrTable& nb = p.nbr[mask];
      const float* coef = p.coef[mask];
      float4 sh = make_float4(0.f, 0.f, 0.f, 0.f);
      if (p.shift) sh = ldg4(p.shift + mask * p.C + c0);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        int r = (i < 4) ? (ty * 4 + i) : (64 + ty * 4 + i - 4);
        if (r >= vrows) continue;
        int fr = r / J, ji = r - fr * J;
        float v0 = sh.x, v1 = sh.y, v2 = sh.z, v3 = sh.w;
        for (int z = nb.row_ptr[ji]; z < nb.row_ptr[ji + 1]; ++z) {
          int jj = nb.col[z];
          float4 cf = ldg4(coef + (long long)z * p.C + c0);
          float4 hv;
          if (jj == ji) hv = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
          else hv = *reinterpret_cast<const float4*>(Hs + (fr * J + jj) * 64 + tx * 4);
          v0 = fmaf(cf.x, hv.x, v0); v1 = fmaf(cf.y, hv.y, v1);
          v2 = fmaf(cf.z, hv.z, v2); v3 = fmaf(cf.w, hv.w, v3);
        }
        if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); v2 = fmaxf(v2, 0.f); v3 = fmaxf(v3, 0.f); }
        long long orow = ((long long)(f0 + fr) * J + ji);
        *reinterpret_cast<float4*>(p.out + orow * p.ld_out + mask * p.C + c0) = make_float4(v0, v1, v2, v3);
      }
    }
  } else {  // EPI_GLOBAL
    // tile = 128 stacked g channels; stage G(+bias) then y[i,:] = sum_j att_h[i,j] G[j,:]
    float* Gs = smem;                                  // [128][128]
    const int H2 = 2 * p.heads;
    const int h_first = n0 / p.Cg;
    int h_last = (min(n0 + FF_BN, p.N) - 1) / p.Cg;
    const int hpt = h_last - h_first + 1;
    float* att = Gs + 128 * 128;                       // [nf][hpt][J][J]
    float* abs_ = att + p.fpt * hpt * J * J;           // [128][H2]
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      int r = (i < 4) ? (ty * 4 + i) : (64 + ty * 4 + i - 4);
#pragma unroll
      for (int g = 0; g < 2; ++g) {
        int nl = g * 64 + tx * 4;
        int n = n0 + nl;
        float4 bb = make_float4(0.f, 0.f, 0.f, 0.f);
        if (p.bg && n < p.N) bb = ldg4(p.bg + n);
        *reinterpret_cast<float4*>(Gs + r * 128 + nl) =
            make_float4(acc[i][g * 4 + 0] + bb.x, acc[i][g * 4 + 1] + bb.y,
                        acc[i][g * 4 + 2] + bb.z, acc[i][g * 4 + 3] + bb.w);
      }
    }
    for (int i = tid; i < vrows * H2; i += FF_THREADS) {
      int r = i / H2, q = i - r * H2;
      abs_[r * H2 + q] = p.ab[((long long)f0 * J + r) * H2 + q];
    }
    epi_sync();
    // attention rows: softmax_j(LeakyReLU_0.2(a_i + b_j)) + C_k[i,j]   (global_attention.py:72-76)
    for (int i = tid; i < nf * hpt * J; i += FF_THREADS) {
      int ji = i % J;
      int t = i / J;
      int hh = t % hpt, fr = t / hpt;
      int h = h_first + hh;
      float a = abs_[(fr * J + ji) * H2 + 2 * h];
      float mx = -3.4e38f;
      float* row = att + ((fr * hpt + hh) * J + ji) * J;
      for (int j = 0; j < J; ++j) {
        float s = a + abs_[(fr * J + j) * H2 + 2 * h + 1];
        s = (s >= 0.f) ? s : 0.2f * s;
        row[j] = s;
        mx = fmaxf(mx, s);
      }
      float sum = 0.f;
      for (int j = 0; j < J; ++j) { float e = expf(row[j] - mx); row[j] = e; sum += e; }
      float inv = 1.f / sum;
      const float* ck = p.ck + ((long long)h * J + ji) * J;
      for (int j = 0; j < J; ++j) row[j] = row[j] * inv + ck[j];
    }
    epi_sync();
    const bool vec = (p.Cg % 4) == 0;
    for (int i = tid; i < vrows * 32; i += FF_THREADS) {
      int r = i >> 5, nl = (i & 31) * 4;
      int n = n0 + nl;
      if (n >= p.N) continue;
      int fr = r / J, ji = r - fr * J;
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (vec) {
        int hh = n / p.Cg - h_first;
        const float* arow = att + ((fr * hpt + hh) * J + ji) * J;
        for (int j = 0; j < J; ++j) {
          float w = arow[j];
          float4 g = *reinterpret_cast<const float4*>(Gs + (fr * J + j) * 128 + nl);
          v[0] = fmaf(w, g.x, v[0]); v[1] = fmaf(w, g.y, v[1]);
          v[2] = fmaf(w, g.z, v[2]); v[3] = fmaf(w, g.w, v[3]);
        }
      } else {
        for (int q = 0; q < 4; ++q) {
          if (n + q >= p.N) break;
          int hh = (n + q) / p.Cg - h_first;
          const float* arow = att + ((fr * hpt + hh) * J + ji) * J;
          float s = 0.f;
          for (int j = 0; j < J; ++j) s = fmaf(arow[j], Gs[(fr * J + j) * 128 + nl + q], s);
          v[q] = s;
        }
      }
      long long orow = ((long long)(f0 + fr) * J + ji);
      *reinterpret_cast<float4*>(p.out + orow * p.ld_out + n) = make_float4(v[0], v[1], v[2], v[3]);
    }
  }
}

template <int EPI>
__global__ void __launch_bounds__(FF_THREADS, 2)
gemm_ffma_kernel(const __grid_constant__ GemmP p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  long long* rowbase = reinterpret_cast<long long*>(smem_raw);          // [3][128]
  float* smem = reinterpret_cast<float*>(smem_raw + 3 * 128 * sizeof(long long));
  float* As = smem;                          // [2][BK][LDS]
  float* Bs = smem + 2 * FF_BK * FF_LDS;     // [2][BK][LDS]

  const int tid = threadIdx.x;
  const int J = p.J;
  const int f0 = blockIdx.x * p.fpt;
  const int nf = min(p.fpt, p.F - f0);
  const int vrows = nf * J;                  // valid rows in this tile
  const int n0 = blockIdx.y * FF_BN;

  // per-row gather offsets of every A segment
  for (int i = tid; i < p.nseg * 128; i += FF_THREADS) {
    int s = i >> 7, r = i & 127;
    long long off = -1;
    if (r < vrows) {
      int fr = r / J, j = r - fr * J;
      long long fin = map_frame(p.seg[s].map, f0 + fr);
      off = (fin * J + j) * (long long)p.seg[s].ld;
    }
    rowbase[s * 128 + r] = off;
  }
  __syncthreads();

  // loader mapping: 512 float4 per operand chunk, 2 per thread
  const int l_row0 = tid >> 2;        // 0..63 (second: +64)
  const int l_kq = tid & 3;           // which float4 of the 16-wide chunk

  // compute mapping
  const int ty = tid >> 4, tx = tid & 15;

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  float4 ra[2], rb[2];

  int seg = 0, k0 = 0, kcol = 0;      // current chunk: segment, offset in segment, column base in W
  int nchunks = 0;
  for (int s = 0; s < p.nseg; ++s) nchunks += (p.seg[s].K + FF_BK - 1) / FF_BK;

  auto load_chunk = [&](int s, int kk, int kc) {
    const float* base = p.seg[s].base;
    const int Ks = p.seg[s].K;
    const int Kc = p.seg[s].Kc;
    const long long tstride = p.seg[s].tap_stride;
    const int k = kk + l_kq * 4;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      int r = l_row0 + h * 64;
      long long off = rowbase[s * 128 + r];
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (off >= 0 && k < Ks) {
        int tap = k / Kc;
        v = ldg4(base + off + tap * tstride + (k - tap * Kc));
      }
      ra[h] = v;
      int n = n0 + r;
      float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
      if (n < p.N && k < Ks) w = ldg4(p.W + (long long)n * p.ldw + kc + k);
      rb[h] = w;
    }
  };
  auto store_chunk = [&](int buf) {
    float* a = As + buf * FF_BK * FF_LDS;
    float* b = Bs + buf * FF_BK * FF_LDS;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      int r = l_row0 + h * 64;
      int kb = l_kq * 4;
      a[(kb + 0) * FF_LDS + r] = ra[h].x; a[(kb + 1) * FF_LDS + r] = ra[h].y;
      a[(kb + 2) * FF_LDS + r] = ra[h].z; a[(kb + 3) * FF_LDS + r] = ra[h].w;
      b[(kb + 0) * FF_LDS + r] = rb[h].x; b[(kb + 1) * FF_LDS + r] = rb[h].y;
      b[(kb + 2) * FF_LDS + r] = rb[h].z; b[(kb + 3) * FF_LDS + r] = rb[h].w;
    }
  };
  auto advance = [&]() {
    k0 += FF_BK;
    if (k0 >= p.seg[seg].K) { kcol += p.seg[seg].K; k0 = 0; ++seg; }
  };

  load_chunk(seg, k0, kcol);
  store_chunk(0);
  advance();
  __syncthreads();

  for (int c = 0; c < nchunks; ++c) {
    const int buf = c & 1;
    const bool more = (c + 1 < nchunks);
    if (more) load_chunk(seg, k0, kcol);
    const float* a = As + buf * FF_BK * FF_LDS;
    const float* b = Bs + buf * FF_BK * FF_LDS;
#pragma unroll
    for (int k = 0; k < FF_BK; ++k) {
      float4 a0 = *reinterpret_cast<const float4*>(a + k * FF_LDS + ty * 4);
      float4 a1 = *reinterpret_cast<const float4*>(a + k * FF_LDS + 64 + ty * 4);
      float4 b0 = *reinterpret_cast<const float4*>(b + k * FF_LDS + tx * 4);
      float4 b1 = *reinterpret_cast<const float4*>(b + k * FF_LDS + 64 + tx * 4);
      float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (more) {
      store_chunk(buf ^ 1);
      advance();
    }
    __syncthreads();
  }

  gemm_epilogue<EPI>(p, acc, smem, tid, f0, nf, vrows, n0, blockIdx.y);
}

}  // namespace gast
