// lion_b200 -- kernels of the fused network path.
//
// Data layout in HBM (all fp32):
//   PF  "packed features"  [B][G][R][4]   G = ceil(C/4) channel groups, R rows (points, or
//                                         centre x neighbour pairs); one float4 = 4 channels of
//                                         one row.  A latent x[B,N,4] *is* a PF with G=1.
//   C4  coordinates        [B][N] float4  (x, y, z, 0)
//   VG  voxel grid         [B][G][P][4]   P = (r+2)^3 zero-haloed positions,
//                                         pos(x,y,z) = ((x+1)*(r+2) + (y+1))*(r+2) + (z+1)
// Channel groups are the unit of concatenation (cat along C = adjacent groups) and every
// global access is a coalesced float4 along rows.  The zero halo turns a 3x3x3 convolution
// into 27 constant row offsets (implicit GEMM without im2col or bounds checks), which is what
// the wgmma kernel (conv_tc.cu) exploits with shifted shared-memory operand descriptors.
#pragma once
#include <cuda_fp16.h>
#include "common.cuh"
#include "point_core.cuh"
#include "model.cuh"

namespace lion {

__device__ __forceinline__ float4 f4_max(float4 a, float4 b) {
  return make_float4(fmaxf(a.x, b.x), fmaxf(a.y, b.y), fmaxf(a.z, b.z), fmaxf(a.w, b.w));
}
__device__ __forceinline__ float4 f4_scale(float4 a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }
__device__ __forceinline__ float4 f4_add(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ float4 f4_fma(float4 a, float s, float4 c) {
  return make_float4(fmaf(a.x, s, c.x), fmaf(a.y, s, c.y), fmaf(a.z, s, c.z), fmaf(a.w, s, c.w));
}

// ------------------------------------------------------------------------------------
// latent x[B][N][D] (D<=4 floats per point... here D==4) -> C4 coordinates
// ------------------------------------------------------------------------------------
__global__ void k_make_coords(const float4* __restrict__ x, float4* __restrict__ c4, int total) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  float4 v = x[i];
  v.w = 0.0f;
  c4[i] = v;
}

// ------------------------------------------------------------------------------------
// voxelisation prep, once per distinct (coords, r) of a forward (4 instead of 14 per step).
// One CTA per shape: statistics -> normalised coords -> voxel ids -> an in-shared-memory
// bitonic sort of (voxel id, point id) keys, which yields for every occupied voxel the list of
// its points in ascending point order.  The scatter-mean that follows is then a plain store
// per voxel: no atomics, no count grid, and -- unlike the reference's float atomicAdd
// (voxelization/vox.cu:66-68) -- bit-reproducible from run to run.
// ------------------------------------------------------------------------------------
constexpr int VOXP_THREADS = 1024;
constexpr int VOXP_MAXN = 4096;

__global__ void __launch_bounds__(VOXP_THREADS)
k_vox_prep(const float4* __restrict__ c4, float4* __restrict__ nc, int* __restrict__ s_order, int* __restrict__ s_ppos,
           int* __restrict__ s_len, unsigned char* __restrict__ occ, int occ_stride, int N, int r,
           int* __restrict__ s_cidx /*[B][N] or null*/, int* __restrict__ nocc /*[B]*/, int* __restrict__ vgrid /*[B][(r+2)^3], pre-set to -1*/) {
  int b = blockIdx.x;
  const float4* c = c4 + (size_t)b * N;
  __shared__ float s_stat[4];
  __shared__ unsigned s_key[VOXP_MAXN];
  // mean (torch-CUDA summation order: bit-exact voxel indices, point_core.cuh) and max centred norm
  vox_stats_block<VOXP_THREADS / 32>([&](int k, float& x, float& y, float& z) { float4 v = c[k]; x = v.x; y = v.y; z = v.z; }, N,
                                     3 * (int)gridDim.x, 3LL * b, s_stat);
  float mx = s_stat[0], my = s_stat[1], mz = s_stat[2], nrm = s_stat[3];
  int n2 = 1;
  while (n2 < N) n2 <<= 1;
  int bits = 0;
  while ((1 << bits) < n2) ++bits;                 // point-id bits
  for (int k = threadIdx.x; k < n2; k += blockDim.x) {
    unsigned key = 0xffffffffu;
    if (k < N) {
      float4 p = c[k];
      float v[3];
      vox_normalize(__fsub_rn(p.x, mx), __fsub_rn(p.y, my), __fsub_rn(p.z, mz), nrm, r, 1, 0.0f, v);
      int xi = (int)rintf(v[0]), yi = (int)rintf(v[1]), zi = (int)rintf(v[2]);   // half-to-even, like torch.round
      nc[(size_t)b * N + k] = make_float4(v[0], v[1], v[2], 0.0f);
      key = ((unsigned)(xi * r * r + yi * r + zi) << bits) | (unsigned)k;
    }
    s_key[k] = key;
  }
  __syncthreads();
  for (int kk = 2; kk <= n2; kk <<= 1) {
    for (int j = kk >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n2; i += blockDim.x) {
        int ixj = i ^ j;
        if (ixj > i) {
          unsigned a = s_key[i], bb = s_key[ixj];
          bool up = (i & kk) == 0;
          if ((a > bb) == up) { s_key[i] = bb; s_key[ixj] = a; }
        }
      }
      __syncthreads();
    }
  }
  int rp = r + 2;
  unsigned mask = (1u << bits) - 1u;
  // occupied voxels in ascending voxel order get compact ids 0..n_occ-1 (the rank of their leading slot): the sparse
  // first convolution (k_sparse_conv_gather) works on the compact list instead of the 94 %-empty grid
  __shared__ int s_wsum[VOXP_THREADS / 32];
  __shared__ int s_base;
  if (threadIdx.x == 0) s_base = 0;
  __syncthreads();
  for (int s0 = 0; s0 < N; s0 += blockDim.x) {           // uniform trip count: barriers inside
    const int s = s0 + threadIdx.x;
    unsigned key = 0;
    int vox = -1;
    bool lead = false;
    if (s < N) {
      key = s_key[s];
      vox = (int)(key >> bits);
      lead = (s == 0) || ((int)(s_key[s - 1] >> bits) != vox);
    }
    const unsigned bal = __ballot_sync(0xffffffffu, lead);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (lane == 0) s_wsum[wid] = __popc(bal);
    __syncthreads();
    int before = s_base + __popc(bal & ((1u << lane) - 1u));
    for (int w = 0; w < wid; ++w) before += s_wsum[w];
    int total = 0;
    for (int w = 0; w < VOXP_THREADS / 32; ++w) total += s_wsum[w];
    __syncthreads();
    if (threadIdx.x == 0) s_base += total;
    if (s < N) {
      int len = 0, pp = -1;
      if (lead) {
        len = 1;
        while (s + len < N && (int)(s_key[s + len] >> bits) == vox) ++len;
        int xi = vox / (r * r), yi = (vox / r) % r, zi = vox % r;
        pp = ((xi + 1) * rp + (yi + 1)) * rp + (zi + 1);
        occ[(size_t)b * occ_stride + (pp >> 6)] = 1;       // 64-row occupancy flags (pre-zeroed) for the sparse-input conv
        if (vgrid) vgrid[(size_t)b * rp * rp * rp + pp] = before;
      }
      s_order[(size_t)b * N + s] = (int)(key & mask);
      s_ppos[(size_t)b * N + s] = pp;
      s_len[(size_t)b * N + s] = len;
      if (s_cidx) s_cidx[(size_t)b * N + s] = lead ? before : -1;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0 && nocc) nocc[b] = s_base;
}

// scatter-mean into the COMPACT voxel list: row cidx of xc[B][G][N] = mean feature of occupied voxel cidx (same
// summation order as k_scatter); rows n_occ..N-1 are zeroed.
__global__ void k_scatter_compact(const float4* __restrict__ feat, const int* __restrict__ s_order, const int* __restrict__ s_cidx,
                                  const int* __restrict__ s_len, const int* __restrict__ nocc, float4* __restrict__ xc, int G, int N) {
  int b = blockIdx.z, g = blockIdx.y;
  int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= N) return;
  float4* dst = xc + ((size_t)b * G + g) * N;
  if (s >= nocc[b]) dst[s] = make_float4(0.f, 0.f, 0.f, 0.f);
  int ci = s_cidx[(size_t)b * N + s];
  if (ci < 0) return;
  int len = s_len[(size_t)b * N + s];
  float inv = 1.0f / (float)len;
  const float4* f = feat + ((size_t)b * G + g) * N;
  const int* ord = s_order + (size_t)b * N + s;
  float4 acc = f4_scale(f[ord[0]], inv);
  for (int k = 1; k < len; ++k) acc = f4_add(acc, f4_scale(f[ord[k]], inv));
  dst[ci] = acc;
}

// Sparse first convolution of a PVConv, second half.  y[b][v][t][c] = W[t]^T x[v] for every occupied voxel v and tap t
// (one dense GEMM over the compact list, k_ygemm in sparse_conv.cu); here every interior output voxel p sums,
// in ascending tap order, the rows y[vgrid[p + off(t)]][t] of its occupied neighbours -- each y row is read exactly
// once -- adds the bias, stores the raw convolution output and accumulates the GroupNorm statistics.  Deterministic.
// A voxel none of whose 27 neighbours is occupied ("inactive": 67-84 % of the voxels of the prior's latent points at r = 32)
// holds exactly the bias: bit j of mask[b][w] is set when voxel 32 w + j is active, and only active voxels are stored
// unless store_all (k_act_grid substitutes the bias for the rest; probes read the whole grid).  The GroupNorm sums
// still cover every voxel.
//   one warp = 32 consecutive interior voxels; accumulators [32][C] in shared memory; C <= 64 (2 channels per lane)
//   grid = (ceil(r^3 / (32 * warps)), B), block = 32 * warps, dynamic smem = warps * (32 * (C + 2) floats + SPG_LIST int2)
constexpr int SPG_LIST = 256;      // contribution-list entries per warp (packed: v << 10 | tap << 5 | voxel-in-warp)
constexpr int SPG_BATCH = 16;      // y rows in flight per warp
// consume a warp's contribution list: SPG_BATCH independent 4*C-byte row reads in flight, then the adds in list order.
// NOT inlined: the tap loop below is fully unrolled and an inlined copy per tap made a 12 600-instruction kernel whose
// fetch stalls dominated (ncu: 25 % of the samples on no-instruction / EXIT).
template <int C>
__device__ __noinline__ void spg_flush(float* __restrict__ acc, const unsigned* __restrict__ list, int n,
                                       const float* __restrict__ yb, int ldy, int lane) {
  constexpr int CPL = C / 32, PITCH = C + 2;
  __syncwarp();
  for (int i0 = 0; i0 < n; i0 += SPG_BATCH) {
    float2 val[SPG_BATCH];
    int jj[SPG_BATCH];
#pragma unroll
    for (int k = 0; k < SPG_BATCH; ++k) {
      jj[k] = -1;
      if (i0 + k < n) {
        const unsigned e = list[i0 + k];
        const float* src = yb + (size_t)(e >> 10) * ldy + ((e >> 5) & 31) * C + lane * CPL;
        if (CPL == 2) val[k] = __ldg(reinterpret_cast<const float2*>(src));
        else val[k] = make_float2(__ldg(src), 0.0f);
        jj[k] = (int)(e & 31);
      }
    }
#pragma unroll
    for (int k = 0; k < SPG_BATCH; ++k) {
      if (jj[k] >= 0) {
        float* a = acc + jj[k] * PITCH + lane * CPL;
        a[0] += val[k].x;
        if (CPL == 2) a[1] += val[k].y;
      }
    }
  }
  __syncwarp();
}

template <int C>
__global__ void __launch_bounds__(128)
k_sparse_conv_gather(const float* __restrict__ y, int ldy, const int* __restrict__ vgrid, const float* __restrict__ bias,
                     float4* __restrict__ out, double* __restrict__ ssum, double* __restrict__ ssq, int stat_stride,
                     int r, int Nrows, unsigned* __restrict__ mask, bool store_all) {
  static_assert(C == 32 || C == 64, "two (or one) channels per lane");
  constexpr int CPL = C / 32;                     // channels per lane
  constexpr int PITCH = C + 2;
  extern __shared__ float s_acc[];
  __shared__ float s_red[2][4][C];
  const int b = blockIdx.y, lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int rp = r + 2, P = rp * rp * rp, V = r * r * r;
  const int q = (blockIdx.x * nw + wid) * 32 + lane;          // interior voxel (x, y, z) flattened
  const bool live = q < V;
  int p = 0;
  if (live) { int z = q % r, yy = (q / r) % r, x = q / (r * r); p = ((x + 1) * rp + (yy + 1)) * rp + (z + 1); }
  float* acc = s_acc + (size_t)wid * 32 * PITCH;
  // the 27 neighbour ids of this lane's voxel: independent loads, all in flight together (a rolled tap loop serialised
  // 27 L2 round trips per warp)
  const int* vg = vgrid + (size_t)b * P;
  int nb[27];
#pragma unroll
  for (int t = 0; t < 27; ++t) {
    const int off = ((t / 9) - 1) * rp * rp + (((t / 3) % 3) - 1) * rp + ((t % 3) - 1);
    nb[t] = live ? __ldg(vg + p + off) : -1;
  }
  // accumulators start at the bias
  {
    float bv[CPL];
#pragma unroll
    for (int k = 0; k < CPL; ++k) bv[k] = bias ? bias[lane * CPL + k] : 0.0f;
    for (int j = 0; j < 32; ++j)
#pragma unroll
      for (int k = 0; k < CPL; ++k) acc[j * PITCH + lane * CPL + k] = bv[k];
  }
  const float* yb = y + (size_t)b * Nrows * ldy;
  // contributions (occupied neighbour v of lane j's voxel, tap t) are listed in shared memory in (t, j) order and then
  // consumed in that order: the accumulation order per output voxel is ascending t whatever the batching
  unsigned* list = reinterpret_cast<unsigned*>(s_acc + (size_t)nw * 32 * PITCH) + wid * SPG_LIST;
  int n = 0;
  bool any = false;                               // this lane's voxel has an occupied neighbour
#pragma unroll
  for (int t = 0; t < 27; ++t) {
    const int v = nb[t];
    const unsigned m = __ballot_sync(0xffffffffu, v >= 0);
    any |= v >= 0;
    if (n + 32 > SPG_LIST) { spg_flush<C>(acc, list, n, yb, ldy, lane); n = 0; }
    if (v >= 0) list[n + __popc(m & ((1u << lane) - 1u))] = ((unsigned)v << 10) | ((unsigned)t << 5) | (unsigned)lane;
    n += __popc(m);
  }
  spg_flush<C>(acc, list, n, yb, ldy, lane);
  const int word = (int)blockIdx.x * nw + wid;
  const unsigned active = __ballot_sync(0xffffffffu, any);
  if (lane == 0 && word * 32 < V) mask[(size_t)b * ((V + 31) / 32) + word] = active;
  // store (PF/VG layout: consecutive lanes = consecutive z) and statistics
  if (live && (store_all || any)) {
#pragma unroll
    for (int g = 0; g < C / 4; ++g) {
      const float* a = acc + lane * PITCH + g * 4;
      out[((size_t)b * (C / 4) + g) * P + p] = make_float4(a[0], a[1], a[2], a[3]);
    }
  }
  float cs[2][CPL], cq[2][CPL];
#pragma unroll
  for (int k = 0; k < CPL; ++k) { cs[0][k] = cs[1][k] = 0.0f; cq[0][k] = cq[1][k] = 0.0f; }
  // (signed: with the unsigned blockIdx.x the difference wraps for the warps past V, and min() then counts 32 rows)
  const int nlive = max(0, min(32, V - word * 32));
  for (int j = 0; j < nlive; j += 2) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (j + h < nlive) {
#pragma unroll
        for (int k = 0; k < CPL; ++k) { const float a = acc[(j + h) * PITCH + lane * CPL + k]; cs[h][k] += a; cq[h][k] = fmaf(a, a, cq[h][k]); }
      }
    }
  }
#pragma unroll
  for (int k = 0; k < CPL; ++k) { s_red[0][wid][lane * CPL + k] = cs[0][k] + cs[1][k]; s_red[1][wid][lane * CPL + k] = cq[0][k] + cq[1][k]; }
  __syncthreads();
  if (threadIdx.x < C) {
    float a = 0.0f, qq = 0.0f;
    for (int w = 0; w < nw; ++w) { a += s_red[0][w][threadIdx.x]; qq += s_red[1][w][threadIdx.x]; }
    atomicAdd(ssum + (size_t)b * stat_stride + threadIdx.x, (double)a);
    atomicAdd(ssq + (size_t)b * stat_stride + threadIdx.x, (double)qq);
  }
}

// Class-valued 64-row blocks of the second 3x3x3 convolution of a PVConv whose first one ran sparse.  Its input (k_act_grid
// with the gather's activity mask) holds one value per (shape, channel) at every inactive interior voxel, so an output
// voxel none of whose 27 neighbours is active depends on its border class only (conv_tc.cu: Params::cls_flag).  Block
// k of shape b -- rows p_begin + 64 k .. + 63 of the row tiles' span [p_begin, p_end) = [rp^2, (rp-1) rp^2) -- is
// flagged (flags[b][k] = 1) when no interior row of it lies within one voxel of an active one; the nblk blocks cover the
// row tiles, those past p_end hold no interior row and are flagged.  One warp per block, two rows per lane.  Also
// writes the all-clear activity mask of the 3x3x3 grid that computes the class values (zmask[b], one word) and adds
// the flagged blocks to *count.
__global__ void __launch_bounds__(256) k_conv2_flags(const unsigned* __restrict__ mask, int r, int nblk,
                                                     unsigned char* __restrict__ flags, int stride,
                                                     unsigned* __restrict__ zmask, unsigned long long* __restrict__ count) {
  __shared__ int s_n;
  const int b = blockIdx.y, lane = threadIdx.x & 31, k = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int rp = r + 2, p_end = (rp - 1) * rp * rp;
  const unsigned* mb = mask + (size_t)b * ((r * r * r + 31) / 32);
  if (threadIdx.x == 0) s_n = 0;
  if (blockIdx.x == 0 && threadIdx.x == 0) zmask[b] = 0u;
  __syncthreads();
  bool hit = false;
  if (k < nblk) {
    for (int h = 0; h < 2; ++h) {
      const int p = rp * rp + 64 * k + 32 * h + lane;
      const int x = p / (rp * rp), y = (p / rp) % rp, z = p % rp;
      if (p >= p_end || y < 1 || y > r || z < 1 || z > r) continue;
      for (int dx = -1; dx <= 1; ++dx)
        for (int dy = -1; dy <= 1; ++dy)
          for (int dz = -1; dz <= 1; ++dz) {
            const int xx = x + dx, yy = y + dy, zz = z + dz;
            if (xx < 1 || xx > r || yy < 1 || yy > r || zz < 1 || zz > r) continue;
            const int q = ((xx - 1) * r + (yy - 1)) * r + (zz - 1);
            hit |= ((__ldg(mb + (q >> 5)) >> (q & 31)) & 1u) != 0;
          }
    }
  }
  const bool flag = !__any_sync(0xffffffffu, hit);
  if (k < nblk && lane == 0) {
    flags[(size_t)b * stride + k] = flag ? 1 : 0;
    if (flag) atomicAdd(&s_n, 1);
  }
  __syncthreads();
  if (threadIdx.x == 0 && s_n) atomicAdd(count, (unsigned long long)s_n);
}

// scatter-mean of PF rows into a (pre-zeroed) VG: one thread per (occupied voxel, channel group)
// sums its points in ascending point order, each term scaled by 1/count first as the
// reference does (vox.cu:65-68), and stores once.
__global__ void k_scatter(const float4* __restrict__ feat, const int* __restrict__ s_order, const int* __restrict__ s_ppos,
                          const int* __restrict__ s_len, float4* __restrict__ grid, int G, int N, int P) {
  int b = blockIdx.z, g = blockIdx.y;
  int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= N) return;
  int pp = s_ppos[(size_t)b * N + s];
  if (pp < 0) return;
  int len = s_len[(size_t)b * N + s];
  float inv = 1.0f / (float)len;
  const float4* f = feat + ((size_t)b * G + g) * N;
  const int* ord = s_order + (size_t)b * N + s;
  float4 acc = f4_scale(f[ord[0]], inv);
  for (int k = 1; k < len; ++k) acc = f4_add(acc, f4_scale(f[ord[k]], inv));
  grid[((size_t)b * G + g) * P + pp] = acc;
}

// ------------------------------------------------------------------------------------
// SIMT reference convolution (3x3x3 over a VG, or 1x1 over a PF with ntaps == 1).
// Correctness scaffold and small-shape fallback; the tensor-core kernel (conv_tc.cu) has the
// same contract:
//   out[b][co/4][p] = bias + sum_taps sum_ci W[tap][ci][co] * in[b][ci/4][p + off[tap]]
//   for the interior rows p of [p_begin, p_end);  ssum/ssq[b][co] += sum / sum of squares over them.
//   Rows whose (y,z) lie in the halo are not part of the result: this kernel writes them as zeros, the
//   tensor-core kernel leaves them unwritten, so readers of a 3x3x3 output (k_act_grid, k_devox_fuse,
//   k_vg_to_cm) read interior rows only.
// ------------------------------------------------------------------------------------
// ConvGeom: model.cuh

template <int COT>
__global__ void __launch_bounds__(128)
k_conv_simt(const float4* __restrict__ in, const float* __restrict__ Wt, const float* __restrict__ bias,
            float4* __restrict__ out, double* __restrict__ ssum, double* __restrict__ ssq,
            int Gin, int cin_pad, int cout_pad, int Gout_store, ConvGeom geo) {
  extern __shared__ float s_w[];   // [ntaps][4][COT]
  int b = blockIdx.z;
  int co0 = blockIdx.y * COT;
  int p = geo.p_begin + blockIdx.x * 128 + threadIdx.x;
  bool inrange = p < geo.p_end;
  bool valid = inrange;
  if (geo.rp > 0 && inrange) {
    int z = p % geo.rp, y = (p / geo.rp) % geo.rp;
    valid = (z >= 1 && z <= geo.rp - 2 && y >= 1 && y <= geo.rp - 2);
  }
  float acc[COT];
#pragma unroll
  for (int o = 0; o < COT; ++o) acc[o] = 0.0f;
  const float4* inb = in + (size_t)b * Gin * geo.rows;
  for (int g = 0; g < Gin; ++g) {
    __syncthreads();
    for (int i = threadIdx.x; i < geo.ntaps * 4 * COT; i += 128) {
      int o = i % COT, j = (i / COT) % 4, t = i / (4 * COT);
      s_w[i] = Wt[((size_t)t * cin_pad + g * 4 + j) * cout_pad + co0 + o];
    }
    __syncthreads();
    if (valid) {
      const float4* ig = inb + (size_t)g * geo.rows + p;
      for (int t = 0; t < geo.ntaps; ++t) {
        float4 v = __ldg(ig + geo.off[t]);
        const float* w = s_w + t * 4 * COT;
#pragma unroll
        for (int o = 0; o < COT; ++o) {
          acc[o] = fmaf(v.x, w[o], acc[o]);
          acc[o] = fmaf(v.y, w[COT + o], acc[o]);
          acc[o] = fmaf(v.z, w[2 * COT + o], acc[o]);
          acc[o] = fmaf(v.w, w[3 * COT + o], acc[o]);
        }
      }
    }
  }
#pragma unroll
  for (int o = 0; o < COT; ++o) acc[o] = valid ? acc[o] + (bias ? bias[co0 + o] : 0.0f) : 0.0f;
  if (inrange) {
#pragma unroll
    for (int q = 0; q < COT / 4; ++q) {
      int g = co0 / 4 + q;
      if (g < Gout_store)
        out[((size_t)b * Gout_store + g) * geo.rows + p] = make_float4(acc[4 * q], acc[4 * q + 1], acc[4 * q + 2], acc[4 * q + 3]);
    }
  }
  if (ssum) {
    int lane = threadIdx.x & 31;
#pragma unroll
    for (int o = 0; o < COT; ++o) {
      float s = warp_sum(acc[o]);
      float q = warp_sum(acc[o] * acc[o]);
      if (lane == 0) {
        atomicAdd(ssum + (size_t)b * cout_pad + co0 + o, (double)s);
        atomicAdd(ssq + (size_t)b * cout_pad + co0 + o, (double)q);
      }
    }
  }
}

// ------------------------------------------------------------------------------------
// AdaGN folding: GroupNorm(8, C, eps 1e-5, affine) followed by *factor + bias
// (models/adagn.py:45-65) collapses to y = scale[b][c] * x + shift[b][c] once the (b, group)
// statistics are known; SE3d (models/pvcnn2_ada.py:27-41) needs only the per-channel mean of
// y, which is affine in the per-channel mean of x, so its gate folds in as well.
//   grid = B, block = C (<= 512; C multiple of 8)
// ------------------------------------------------------------------------------------
struct PrepJob {
  const double* ssum; const double* ssq; int stat_stride;
  const float* gamma; const float* beta;
  const float* style_fb /*[B][2C] for this layer*/; int fb_stride;
  const float* se_w1 /*[C/8][C] or null*/; const float* se_w2 /*[C][C/8]*/;
  float* scale; float* shift; int C; double count;
};
// grid = (B, number of jobs <= 2), block = the larger C; dynamic smem = (C + C/8) floats of the largest SE job.
// Two layers whose statistics are complete at the same point of the stream (a PVConv's first convolution and its
// point branch) are folded by ONE launch: each tiny launch costs 4-5 us on the step's critical path.
__global__ void k_affine_prep(PrepJob j0, PrepJob j1) {
  extern __shared__ float s_f[];   // [C] se input, [C/8] hidden
  __shared__ double s_gs[8], s_gq[8];
  const PrepJob& J = blockIdx.y == 0 ? j0 : j1;
  const int C = J.C;
  int b = blockIdx.x, c = threadIdx.x;
  const bool on = c < C;
  int cpg = C / 8;
  if (c < 8) { s_gs[c] = 0; s_gq[c] = 0; }
  __syncthreads();
  double s = 0.0, q = 0.0;
  if (on) {
    s = J.ssum[(size_t)b * J.stat_stride + c]; q = J.ssq[(size_t)b * J.stat_stride + c];
    atomicAdd(&s_gs[c / cpg], s);
    atomicAdd(&s_gq[c / cpg], q);
  }
  __syncthreads();
  float sc = 0.f, sh = 0.f;
  if (on) {
    double n = J.count * cpg;
    double mean = s_gs[c / cpg] / n;
    double var = s_gq[c / cpg] / n - mean * mean;
    if (var < 0) var = 0;
    float rstd = (float)(1.0 / sqrt(var + 1e-5));
    float f = J.style_fb[(size_t)b * J.fb_stride + c], bb = J.style_fb[(size_t)b * J.fb_stride + C + c];
    float ga = J.gamma[c], be = J.beta[c];
    sc = rstd * ga * f;
    sh = (be - (float)mean * rstd * ga) * f + bb;
  }
  if (J.se_w1) {                                   // block-uniform
    int H = C / 8;
    float* s_h = s_f + C;
    if (on) s_f[c] = sc * (float)(s / J.count) + sh;     // mean over voxels of the AdaGN output
    __syncthreads();
    // squeeze: one warp per hidden unit, lanes stride the C inputs (coalesced, C / 32 independent loads per lane) -- a
    // thread per hidden unit walked 128 weights serially, ~5 us of the 12 us these launches took at C = 128
    if ((blockDim.x & 31) == 0) {
      for (int o = (int)(threadIdx.x >> 5); o < H; o += (int)(blockDim.x >> 5)) {
        float a = 0.0f;
        for (int k = (int)(threadIdx.x & 31); k < C; k += 32) a = fmaf(J.se_w1[o * C + k], s_f[k], a);
        a = warp_sum(a);
        if ((threadIdx.x & 31) == 0) s_h[o] = fmaxf(a, 0.0f);
      }
    } else if (c < H) {      // channel counts that are not a multiple of the warp size (none in the shipped configs)
      float a = 0.0f;
      for (int k = 0; k < C; ++k) a = fmaf(J.se_w1[c * C + k], s_f[k], a);
      s_h[c] = fmaxf(a, 0.0f);
    }
    __syncthreads();
    if (on) {
      float a = 0.0f;
      for (int k = 0; k < H; ++k) a = fmaf(J.se_w2[c * H + k], s_h[k], a);
      float gate = 1.0f / (1.0f + expf(-a));
      sc *= gate;
      sh *= gate;
    }
  }
  if (on) {
    J.scale[(size_t)b * C + c] = sc;
    J.shift[(size_t)b * C + c] = sh;
  }
}

// all AdaGN style Linears of a network in one launch: out[b][off_l + o] = W_l[o] . style[b] + bias_l[o]
__global__ void k_style_linear(const StyleLayer* __restrict__ layers, const float* __restrict__ style, int S,
                               float* __restrict__ out, int out_stride) {
  extern __shared__ float s_style[];
  StyleLayer L = layers[blockIdx.x];
  int b = blockIdx.y;
  for (int i = threadIdx.x; i < S; i += blockDim.x) s_style[i] = style[(size_t)b * S + i];
  __syncthreads();
  int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if (!L.w) {     // plain GroupNorm (non-Ada blocks): factor = 1, bias = 0
    for (int o = threadIdx.x; o < L.n_out; o += blockDim.x) out[(size_t)b * out_stride + L.out_off + o] = o < L.n_out / 2 ? 1.0f : 0.0f;
    return;
  }
  for (int o = wid; o < L.n_out; o += nw) {
    float a = 0.0f;
    for (int k = lane; k < S; k += 32) a = fmaf(L.w[(size_t)o * S + k], s_style[k], a);
    a = warp_sum(a);
    if (lane == 0) out[(size_t)b * out_stride + L.out_off + o] = a + L.b[o];
  }
}

// max over the rows of a PF: out[b][c] = max_i in[b][c/4][i].c%4   (PointNetPlusEncoder: features.max(-1), shapelatent_modules.py:46)
__global__ void k_max_rows(const float4* __restrict__ in, float* __restrict__ out, int G, int R) {
  int b = blockIdx.y, g = blockIdx.x;
  const float4* src = in + ((size_t)b * G + g) * R;
  float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
  for (int i = threadIdx.x; i < R; i += blockDim.x) m = f4_max(m, src[i]);
  m.x = warp_max(m.x); m.y = warp_max(m.y); m.z = warp_max(m.z); m.w = warp_max(m.w);
  __shared__ float4 s_m[8];
  int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) s_m[wid] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) m = f4_max(m, s_m[w]);
    *reinterpret_cast<float4*>(out + ((size_t)b * G + g) * 4) = m;
  }
}
// [B][N][3] -> PF / C4 [B][N] float4 (x, y, z, 0): networks whose points carry no extra feature channel
__global__ void k_pad3(const float* __restrict__ x, float4* __restrict__ o, int total) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < total) o[i] = make_float4(x[3 * (size_t)i], x[3 * (size_t)i + 1], x[3 * (size_t)i + 2], 0.0f);
}
// PF with G groups -> point-major [B][R][C]
__global__ void k_pf_to_pm(const float4* __restrict__ src, float* __restrict__ dst, int G, int C, int R) {
  int b = blockIdx.z, g = blockIdx.y;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R) return;
  float4 v = src[((size_t)b * G + g) * R + i];
  float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    int c = g * 4 + j;
    if (c < C) dst[((size_t)b * R + i) * C + c] = vv[j];
  }
}

// generic small dense layer on [B][K] rows: out = act(W x + b); act 0 none, 1 leaky(0.1)
__global__ void k_small_linear(const float* __restrict__ W, const float* __restrict__ bias, const float* __restrict__ x,
                               int x_stride, float* __restrict__ out, int out_stride, int K, int O, int act) {
  extern __shared__ float s_x[];
  int b = blockIdx.x;
  for (int i = threadIdx.x; i < K; i += blockDim.x) s_x[i] = x[(size_t)b * x_stride + i];
  __syncthreads();
  int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int o = wid; o < O; o += nw) {
    float a = 0.0f;
    for (int k = lane; k < K; k += 32) a = fmaf(W[(size_t)o * K + k], s_x[k], a);
    a = warp_sum(a);
    if (lane == 0) {
      a += bias ? bias[o] : 0.0f;
      if (act == 1) a = a > 0.0f ? a : 0.1f * a;
      out[(size_t)b * out_stride + o] = a;
    }
  }
}

// sinusoidal timestep embedding (models/latent_points_ada.py:101-115); freqs computed on the
// host in float64 and rounded to fp32 exactly like the reference
__global__ void k_time_sinusoid(const float* __restrict__ t, const float* __restrict__ freqs, float* __restrict__ out,
                                int half, float scale) {
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < half; i += blockDim.x) {     // any time_dim, whatever the block size
    float e = __fmul_rn(__fmul_rn(t[b], scale), freqs[i]);
    out[(size_t)b * 2 * half + i] = sinf(e);
    out[(size_t)b * 2 * half + half + i] = cosf(e);
  }
}

// ------------------------------------------------------------------------------------
// elementwise passes
// ------------------------------------------------------------------------------------
// Where a consumer gets the folded AdaGN affine of its (b, 4-channel group): either the arrays
// k_affine_prep wrote (scale != null; the SE-gated case), or -- saving that launch on the critical
// path -- straight from the GroupNorm statistics the producing convolution accumulated: the block
// computes its four (scale, shift) pairs once (same formulas as k_affine_prep, group sums in channel
// order) and shares them through shared memory.  Must be called by ALL threads of the block.
struct AffSrc {
  const float* scale; const float* shift;
  const double* ssum; const double* ssq; int stat_stride;
  const float* gamma; const float* beta; const float* fb; int fb_stride;
  double count;
};
__device__ __forceinline__ void aff_block_load(const AffSrc& a, int b, int g, int C, float4& s, float4& t) {
  if (a.scale) {
    s = *reinterpret_cast<const float4*>(a.scale + (size_t)b * C + g * 4);
    t = *reinterpret_cast<const float4*>(a.shift + (size_t)b * C + g * 4);
    return;
  }
  __shared__ float s_aff[8];
  if (threadIdx.x < 4) {
    const int c = g * 4 + threadIdx.x, cpg = C / 8, c0 = (c / cpg) * cpg;
    const double* ps = a.ssum + (size_t)b * a.stat_stride + c0;
    const double* pq = a.ssq + (size_t)b * a.stat_stride + c0;
    double gs = 0.0, gq = 0.0;
    for (int k = 0; k < cpg; ++k) { gs += ps[k]; gq += pq[k]; }
    const double n = a.count * cpg;
    const double mean = gs / n;
    double var = gq / n - mean * mean;
    if (var < 0) var = 0;
    const float rstd = (float)(1.0 / sqrt(var + 1e-5));
    const float f = a.fb[(size_t)b * a.fb_stride + c], bb = a.fb[(size_t)b * a.fb_stride + C + c];
    const float ga = a.gamma[c], be = a.beta[c];
    s_aff[threadIdx.x] = rstd * ga * f;
    s_aff[4 + threadIdx.x] = (be - (float)mean * rstd * ga) * f + bb;
  }
  __syncthreads();
  s = make_float4(s_aff[0], s_aff[1], s_aff[2], s_aff[3]);
  t = make_float4(s_aff[4], s_aff[5], s_aff[6], s_aff[7]);
}

// VG: y = swish(scale*x + shift) on interior voxels, 0 on every halo position (incl. x planes).
// ACT_U positions per thread, loads issued before any use: a 16-byte access per thread leaves too
// few bytes in flight per SM to cover HBM latency (4.3 TB/s measured with one access per thread).
constexpr int ACT_U = 4;
// 8 floats -> one 16-byte row of 8 halves, each rounded to nearest even
__device__ __forceinline__ float4 h8_pack(float4 a, float4 b) {
  union { __half2 h[4]; float4 f; } u;
  u.h[0] = __floats2half2_rn(a.x, a.y); u.h[1] = __floats2half2_rn(a.z, a.w);
  u.h[2] = __floats2half2_rn(b.x, b.y); u.h[3] = __floats2half2_rn(b.z, b.w);
  return u.f;
}

// The output form F16 (the input of the FP16 second convolution): block (x, y, b) covers channels 8y .. 8y + 7, i.e. fp32
// groups 2y and 2y + 1 of `in` (G of them), applies the same affine and Swish in fp32 and stores one row of 8 halves
// (rounded to nearest even) per position into out [B][G/2][P][8].  Otherwise block (x, y, b) covers group y and stores
// the TF32-rounded float4 into out [B][G][P][4].  Halo positions are exactly 0 in both forms.
// Blocks with blockIdx.x >= nb_act do k_unscatter's job instead (us_ppos != null): they restore the all-zero
// invariant of the persistent scatter grid that the first convolution has finished reading by now (one launch less
// per PVConv on the critical path); block (x, y, z) zeroes its 256 points in groups y, y + gridDim.y, ... < us_G.
// mask (the sparse first convolution's activity bits, k_sparse_conv_gather; null = read every interior position): an
// interior position whose bit is clear is neither read nor recomputed -- its input is exactly bias (null = 0), and the
// block computes that position's output once, with the same expression.
template <bool F16>
__global__ void k_act_grid(const float4* __restrict__ in, float4* __restrict__ out, AffSrc aff, int G, int C, int rp, int P,
                           int nb_act, const int* __restrict__ us_ppos, float4* __restrict__ us_grid, int us_G, int us_N,
                           const unsigned* __restrict__ mask, const float* __restrict__ bias) {
  constexpr int NG = F16 ? 2 : 1;                       // fp32 input groups per output row
  int b = blockIdx.z, g = blockIdx.y;
  if ((int)blockIdx.x >= nb_act) {
    int sidx = ((int)blockIdx.x - nb_act) * blockDim.x + threadIdx.x;
    if (sidx >= us_N) return;
    int pp = us_ppos[(size_t)b * us_N + sidx];
    if (pp >= 0)
      for (int gg = g; gg < us_G; gg += gridDim.y) us_grid[((size_t)b * us_G + gg) * P + pp] = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  float4 s[NG], t[NG];
#pragma unroll
  for (int k = 0; k < NG; ++k) {
    if (k) __syncthreads();                              // (aff_block_load's shared slots are reused)
    aff_block_load(aff, b, NG * g + k, C, s[k], t[k]);
  }
  const float4* src = in + ((size_t)b * G + NG * g) * P;
  float4* dst = out + ((size_t)b * (G / NG) + g) * P;
  const int p0 = blockIdx.x * (blockDim.x * ACT_U) + threadIdx.x;
  const int r = rp - 2;
  const unsigned* mb = mask ? mask + (size_t)b * ((r * r * r + 31) / 32) : nullptr;
  float4 cst = make_float4(0.f, 0.f, 0.f, 0.f);          // the output of an inactive position
  if (mask) {
    float4 bv[NG];
#pragma unroll
    for (int k = 0; k < NG; ++k) {
      const int c0 = (NG * g + k) * 4;
      bv[k] = bias ? make_float4(bias[c0], bias[c0 + 1], bias[c0 + 2], bias[c0 + 3]) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if constexpr (F16) cst = h8_pack(f4_swish(f4_affine(bv[0], s[0], t[0])), f4_swish(f4_affine(bv[1], s[1], t[1])));
    else cst = f4_tf32(f4_swish(f4_affine(bv[0], s[0], t[0])));
  }
  float4 v[ACT_U][NG];
  bool interior[ACT_U], active[ACT_U];
  // p -> (x, y, z) by multiply-high with m = ceil(2^32 / rp) (exact while p * rp < 2^32): the four positions of a thread
  // cost one integer division instead of sixteen -- at 1 float4 per clock per SM this pass is instruction-bound, not
  // HBM-bound, once the index arithmetic and an IEEE division per Swish are in the loop
  const unsigned rp_m = 0xffffffffu / (unsigned)rp + 1u;
#pragma unroll
  for (int u = 0; u < ACT_U; ++u) {
    int p = p0 + u * blockDim.x;
    const int q = (int)__umulhi((unsigned)p, rp_m), x = (int)__umulhi((unsigned)q, rp_m);
    const int z = p - q * rp, y = q - x * rp;
    interior[u] = p < P && z >= 1 && z <= rp - 2 && y >= 1 && y <= rp - 2 && x >= 1 && x <= rp - 2;
    active[u] = interior[u];
    if (mb && interior[u]) {
      const int qi = ((x - 1) * r + (y - 1)) * r + (z - 1);      // interior voxel index, as the gather numbers it
      active[u] = (__ldg(mb + (qi >> 5)) >> (qi & 31)) & 1u;
    }
#pragma unroll
    for (int k = 0; k < NG; ++k) {
      v[u][k] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (active[u]) v[u][k] = __ldcs(src + (size_t)k * P + p);     // read once: streaming
    }
  }
#pragma unroll
  for (int u = 0; u < ACT_U; ++u) {
    int p = p0 + u * blockDim.x;
    if (p < P) {
      float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
      if (active[u]) {                                   // sole consumer: the second 3x3x3 convolution
        if constexpr (F16) o = h8_pack(f4_swish(f4_affine(v[u][0], s[0], t[0])), f4_swish(f4_affine(v[u][1], s[1], t[1])));
        else o = f4_tf32(f4_swish(f4_affine(v[u][0], s[0], t[0])));
      } else if (interior[u]) {
        o = cst;
      }
      dst[p] = o;
    }
  }
}

// PF: y = swish(scale*x + shift); written at group offset g_off of a destination with Gd groups.
// POOL > 1: max over POOL consecutive rows (neighbours of one centre) after the activation.
template <int POOL>
__global__ void k_act_rows(const float4* __restrict__ in, float4* __restrict__ out, AffSrc aff, int G, int C, int R_out, int Gd,
                           int g_off, int flags) {
  int b = blockIdx.z, g = blockIdx.y;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  float4 s, t;
  aff_block_load(aff, b, g, C, s, t);
  if (i >= R_out) return;
  const float4* src = in + ((size_t)b * G + g) * (size_t)R_out * POOL + (size_t)i * POOL;
  float4 r = f4_affine(src[0], s, t);
  if (!(flags & 2)) r = f4_swish(r);
#pragma unroll 4
  for (int k = 1; k < POOL; ++k) r = f4_max(r, f4_swish(f4_affine(src[k], s, t)));
  if (flags & 1) r = f4_tf32(r);
  out[((size_t)b * Gd + g_off + g) * R_out + i] = r;
}

// PF -> PF with max over 32 consecutive rows (the neighbours of one centre) after the activation:
// one warp per output row, lane k reads neighbour k (one coalesced 512-byte access per warp instead
// of 32 strided ones per thread), butterfly max.  The result is the same set maximum as
// k_act_rows<32>, bit for bit.
__global__ void k_act_rows_pool32(const float4* __restrict__ in, float4* __restrict__ out, AffSrc aff, int G, int C, int R_out,
                                  int Gd, int g_off) {
  int b = blockIdx.z, g = blockIdx.y;
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  float4 s, t;
  aff_block_load(aff, b, g, C, s, t);
  const float4* src = in + ((size_t)b * G + g) * (size_t)R_out * 32;
  constexpr int ROWS = 4;                                  // rows per warp, loads issued together
  const int i0 = (blockIdx.x * wpb + (threadIdx.x >> 5)) * ROWS;
  float4 v[ROWS];
#pragma unroll
  for (int u = 0; u < ROWS; ++u) {
    v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (i0 + u < R_out) v[u] = __ldcs(src + (size_t)(i0 + u) * 32 + lane);
  }
#pragma unroll
  for (int u = 0; u < ROWS; ++u) {
    if (i0 + u < R_out) {                                  // warp-uniform
      float4 r = f4_swish(f4_affine(v[u], s, t));
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        r.x = fmaxf(r.x, __shfl_xor_sync(0xffffffffu, r.x, o));
        r.y = fmaxf(r.y, __shfl_xor_sync(0xffffffffu, r.y, o));
        r.z = fmaxf(r.z, __shfl_xor_sync(0xffffffffu, r.z, o));
        r.w = fmaxf(r.w, __shfl_xor_sync(0xffffffffu, r.w, o));
      }
      if (lane == 0) out[((size_t)b * Gd + g_off + g) * R_out + i0 + u] = r;
    }
  }
}

// pooled SharedMLP tail: mm[b][g][centre] = (min4, max4) over the centre's 32 neighbours of the raw convolution output
// (written by the convolution's epilogue).  y = swish(scale*x + shift) is monotonic-then-quasi-convex in x, so its
// maximum over the neighbours is attained at one of the two extremes: the same set maximum as k_act_rows_pool32.
__global__ void k_act_pool_minmax(const float4* __restrict__ mm, float4* __restrict__ out, AffSrc aff, int G, int C, int R_out,
                                  int Gd, int g_off) {
  int b = blockIdx.z, g = blockIdx.y;
  float4 s, t;
  aff_block_load(aff, b, g, C, s, t);
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R_out) return;
  const float4* src = mm + (((size_t)b * G + g) * R_out + i) * 2;
  float4 lo = f4_swish(f4_affine(src[0], s, t)), hi = f4_swish(f4_affine(src[1], s, t));
  out[((size_t)b * Gd + g_off + g) * R_out + i] = make_float4(fmaxf(lo.x, hi.x), fmaxf(lo.y, hi.y), fmaxf(lo.z, hi.z), fmaxf(lo.w, hi.w));
}

// per-channel sum / sum of squares over the rows of a PF (stand-alone AdaGN / SE3d entry points;
// on the fused path these statistics come out of the convolution epilogue instead)
__global__ void k_row_stats(const float4* __restrict__ in, double* __restrict__ ssum, double* __restrict__ ssq, int G, int R,
                            int stat_stride) {
  int b = blockIdx.z, g = blockIdx.y;
  float s[4] = {0, 0, 0, 0}, q[4] = {0, 0, 0, 0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < R; i += gridDim.x * blockDim.x) {
    float4 v = in[((size_t)b * G + g) * R + i];
    s[0] += v.x; s[1] += v.y; s[2] += v.z; s[3] += v.w;
    q[0] += v.x * v.x; q[1] += v.y * v.y; q[2] += v.z * v.z; q[3] += v.w * v.w;
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float a = warp_sum(s[j]), c = warp_sum(q[j]);
    if ((threadIdx.x & 31) == 0) {
      atomicAdd(ssum + (size_t)b * stat_stride + g * 4 + j, (double)a);
      atomicAdd(ssq + (size_t)b * stat_stride + g * 4 + j, (double)c);
    }
  }
}

// SE3d gate from channel means (models/pvcnn2_ada.py:27-41): gate[b][c] = sigmoid(W2 relu(W1 mean)); grid = B, block = C
__global__ void k_se_gate(const double* __restrict__ ssum, int stat_stride, const float* __restrict__ w1, const float* __restrict__ w2,
                          float* __restrict__ gate, int C, double count) {
  extern __shared__ float s_f[];
  int b = blockIdx.x, c = threadIdx.x, H = C / 8;
  float* s_h = s_f + C;
  s_f[c] = (float)(ssum[(size_t)b * stat_stride + c] / count);
  __syncthreads();
  if (c < H) {
    float a = 0.0f;
    for (int k = 0; k < C; ++k) a = fmaf(w1[c * C + k], s_f[k], a);
    s_h[c] = fmaxf(a, 0.0f);
  }
  __syncthreads();
  float a = 0.0f;
  for (int k = 0; k < H; ++k) a = fmaf(w2[c * H + k], s_h[k], a);
  gate[(size_t)b * C + c] = 1.0f / (1.0f + expf(-a));
}
// y = x * gate[b][c] on channel-major data [B][C][V];  also plain swish when gate == nullptr
__global__ void k_scale_or_swish(const float* __restrict__ x, const float* __restrict__ gate, float* __restrict__ y, size_t V, size_t total) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  float v = x[i];
  y[i] = gate ? v * gate[i / V] : swishf(v);
}

// copy groups of a PF into another PF at a group offset (channel concatenation)
__global__ void k_copy_groups(const float4* __restrict__ src, float4* __restrict__ dst, int Gs, int Gd, int g_off, int R) {
  int b = blockIdx.z, g = blockIdx.y;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R) return;
  dst[((size_t)b * Gd + g_off + g) * R + i] = src[((size_t)b * Gs + g) * R + i];
}

// broadcast a per-shape vector v[b][4*Gv] over all rows (the time embedding "expand")
__global__ void k_fill_groups(const float* __restrict__ v, int v_stride, float4* __restrict__ dst, int Gd, int g_off, int R) {
  int b = blockIdx.z, g = blockIdx.y;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R) return;
  dst[((size_t)b * Gd + g_off + g) * R + i] = *reinterpret_cast<const float4*>(v + (size_t)b * v_stride + g * 4);
}

// ------------------------------------------------------------------------------------
// trilinear devoxelisation fused with: AdaGN-2 + SE affine of the raw second conv output,
// + the point branch swish(AdaGN(conv1x1)) (PVConv.forward, models/pvcnn2_ada.py:267-277)
// ------------------------------------------------------------------------------------
__global__ void k_devox_fuse(const float4* __restrict__ raw, const float4* __restrict__ nc, const float* __restrict__ scale,
                             const float* __restrict__ shift, const float4* __restrict__ rawp, AffSrc aff_p,
                             float4* __restrict__ out, int G, int C, int N, int r, int P, int Gd, int g_off) {
  int b = blockIdx.z, g = blockIdx.y;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  float4 sp = make_float4(0.f, 0.f, 0.f, 0.f), tp = sp;
  if (rawp) aff_block_load(aff_p, b, g, C, sp, tp);
  if (i >= N) return;
  float4 c = nc[(size_t)b * N + i];
  int rp = r + 2;
  float xl = floorf(c.x), yl = floorf(c.y), zl = floorf(c.z);
  float x1 = c.x - xl, y1 = c.y - yl, z1 = c.z - zl;
  float x0 = 1.0f - x1, y0 = 1.0f - y1, z0 = 1.0f - z1;
  float w[8] = {x0 * y0 * z0, x0 * y0 * z1, x0 * y1 * z0, x0 * y1 * z1, x1 * y0 * z0, x1 * y0 * z1, x1 * y1 * z0, x1 * y1 * z1};
  int hx = (x1 > 0.0f) ? rp * rp : 0, hy = (y1 > 0.0f) ? rp : 0, hz = (z1 > 0.0f) ? 1 : 0;
  int i0 = (((int)xl + 1) * rp + ((int)yl + 1)) * rp + ((int)zl + 1);
  int idx[8] = {i0, i0 + hz, i0 + hy, i0 + hy + hz, i0 + hx, i0 + hx + hz, i0 + hx + hy, i0 + hx + hy + hz};
  float4 s = *reinterpret_cast<const float4*>(scale + (size_t)b * C + g * 4);
  float4 t = *reinterpret_cast<const float4*>(shift + (size_t)b * C + g * 4);
  const float4* rg = raw + ((size_t)b * G + g) * P;
  float4 acc = f4_scale(f4_affine(__ldg(rg + idx[0]), s, t), w[0]);
#pragma unroll
  for (int k = 1; k < 8; ++k) acc = f4_fma(f4_affine(__ldg(rg + idx[k]), s, t), w[k], acc);
  if (rawp) acc = f4_add(acc, f4_swish(f4_affine(rawp[((size_t)b * G + g) * N + i], sp, tp)));
  out[((size_t)b * Gd + g_off + g) * N + i] = acc;
}

// ------------------------------------------------------------------------------------
// set abstraction: FPS (+ centre coordinates), ball query, grouped input assembly
// ------------------------------------------------------------------------------------
template <int A, int C, bool FULL>
__global__ void __launch_bounds__(FPS_THREADS)
k_fps_c4(const float4* __restrict__ c4, int* __restrict__ idx, float4* __restrict__ centers, int N, int M, int VT) {
  extern __shared__ float s_fps[];
  int b = blockIdx.x;
  const float4* c = c4 + (size_t)b * N;
  int* io = idx + (size_t)b * M;
  float4* co = centers + (size_t)b * M;
  fps_block_emit<A, C, FULL>([&](int k, float& x, float& y, float& z) { float4 v = c[k]; x = v.x; y = v.y; z = v.z; },
                             [&](int j, int k, float x, float y, float z) { io[j] = k; co[j] = make_float4(x, y, z, 0.0f); },
                             N, M, VT, s_fps);
}

__global__ void k_ball_query_c4(const float4* __restrict__ centers, const float4* __restrict__ points, int* __restrict__ out,
                                int N, int M, float r2, int K) {
  int b = blockIdx.y;
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (warp >= M) return;
  float4 ce = centers[(size_t)b * M + warp];
  const float4* pt = points + (size_t)b * N;
  ball_query_warp([&](int k, float& x, float& y, float& z) { float4 v = __ldg(pt + k); x = v.x; y = v.y; z = v.z; },
                  ce.x, ce.y, ce.z, r2, N, K, out + ((size_t)b * M + warp) * K);
}

// grouped SA input: group 0 = neighbour xyz - centre xyz (BallQuery.forward, pvcnn2_ada.py:104-113),
// groups 1..Gf = neighbour features.  rows = M*U pairs.
__global__ void k_group_gather(const float4* __restrict__ feat, const float4* __restrict__ points,
                               const float4* __restrict__ centers, const int* __restrict__ nidx, float4* __restrict__ out,
                               int Gf, int N, int M, int U) {
  int b = blockIdx.z, g = blockIdx.y;    // g == 0: coordinates; g >= 1: features group g-1
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int MU = M * U;
  if (i >= MU) return;
  int k = nidx[(size_t)b * MU + i];
  float4 v;
  if (g == 0) {
    float4 p = points[(size_t)b * N + k], c = centers[(size_t)b * M + i / U];
    v = make_float4(p.x - c.x, p.y - c.y, p.z - c.z, 0.0f);
  } else {
    v = feat[((size_t)b * Gf + (g - 1)) * N + k];
  }
  out[((size_t)b * (Gf + 1) + g) * MU + i] = v;
}

// ------------------------------------------------------------------------------------
// feature propagation: 3-NN search + interpolation into a destination PF at a group offset
// ------------------------------------------------------------------------------------
__global__ void k_three_nn_c4(const float4* __restrict__ points, const float4* __restrict__ centers, int* __restrict__ idx,
                              float* __restrict__ wgt, int N, int M) {
  int b = blockIdx.y;
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  extern __shared__ float4 s_c4[];
  const float4* ce = centers + (size_t)b * M;
  float4 u = make_float4(0, 0, 0, 0);
  if (j < N) u = points[(size_t)b * N + j];
  ThreeNN st;
  st.init();
  const int TILE = 1024;
  for (int k0 = 0; k0 < M; k0 += TILE) {
    int n = min(TILE, M - k0);
    __syncthreads();
    for (int t = threadIdx.x; t < n; t += blockDim.x) s_c4[t] = ce[k0 + t];
    __syncthreads();
    for (int k = 0; k < n; ++k) {
      float4 c = s_c4[k];
      st.push(sqdist_ref(u.x - c.x, u.y - c.y, u.z - c.z), k0 + k);
    }
  }
  if (j >= N) return;
  float w0, w1, w2;
  st.weights(w0, w1, w2);
  size_t o = ((size_t)b * N + j) * 3;
  idx[o] = st.i0; idx[o + 1] = st.i1; idx[o + 2] = st.i2;
  wgt[o] = w0; wgt[o + 1] = w1; wgt[o + 2] = w2;
}

__global__ void k_interp_rows(const float4* __restrict__ cf, const int* __restrict__ idx, const float* __restrict__ wgt,
                              float4* __restrict__ dst, int Gs, int M, int N, int Gd, int g_off) {
  int b = blockIdx.z, g = blockIdx.y;
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  size_t o = ((size_t)b * N + j) * 3;
  const float4* f = cf + ((size_t)b * Gs + g) * M;
  float4 a = f4_scale(f[idx[o]], wgt[o]);                      // f[i1]*w1 + f[i2]*w2 + f[i3]*w3
  a = f4_fma(f[idx[o + 1]], wgt[o + 1], a);
  a = f4_fma(f[idx[o + 2]], wgt[o + 2], a);
  dst[((size_t)b * Gd + g_off + g) * N + j] = a;
}

// ------------------------------------------------------------------------------------
// linear attention (models/pvcnn2_ada.py:54-71).  qkv PF has 3*H*32 channels ordered
// (qkv, head, c).  ctx[b][h][d][e] = sum_n softmax_n(k[d])[n] * v[e][n];  out[e][n] = sum_d ctx[d][e] q[d][n]
// ------------------------------------------------------------------------------------
// Split over N (online softmax): block (h, b, c) handles the 128 points of chunk c and leaves an UNNORMALISED partial
// context plus its per-channel running max / sum; k_attn_apply merges the S = ceil(N/128) partials in its prologue.
// (Round 1 used one block per (b, head) looping over all N: 128 blocks, 57 us at N = 1024 -- latency-bound.)
//   part[b][h][c] = { ctx_c[32][32], max_c[32], sum_c[32] }   (ATTN_PART floats)
constexpr int ATTN_CHUNK = 128;
constexpr int ATTN_PART = 1024 + 64;
__global__ void __launch_bounds__(256)
k_attn_ctx(const float4* __restrict__ qkv, float* __restrict__ part, int H, int N) {
  const int h = blockIdx.x, b = blockIdx.y, c = blockIdx.z, S = gridDim.z;
  const int Gq = 3 * H * 8;                       // groups in qkv
  const int n0 = c * ATTN_CHUNK, nn = min(ATTN_CHUNK, N - n0);
  const float4* kb = qkv + ((size_t)b * Gq + (H + h) * 8) * N + n0;       // k: 8 groups x N
  const float4* vb = qkv + ((size_t)b * Gq + (2 * H + h) * 8) * N + n0;   // v
  __shared__ float s_k[32][ATTN_CHUNK + 1], s_v[32][ATTN_CHUNK + 1];
  const int tid = threadIdx.x;
  for (int i = tid; i < 8 * ATTN_CHUNK; i += 256) {
    const int g = i / ATTN_CHUNK, n = i % ATTN_CHUNK;
    float4 kv = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY), vv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (n < nn) { kv = kb[(size_t)g * N + n]; vv = vb[(size_t)g * N + n]; }
    s_k[g * 4 + 0][n] = kv.x; s_k[g * 4 + 1][n] = kv.y; s_k[g * 4 + 2][n] = kv.z; s_k[g * 4 + 3][n] = kv.w;
    s_v[g * 4 + 0][n] = vv.x; s_v[g * 4 + 1][n] = vv.y; s_v[g * 4 + 2][n] = vv.z; s_v[g * 4 + 3][n] = vv.w;
  }
  __syncthreads();
  // channel d = tid / 8: eight threads share its 128 entries
  const int d = tid >> 3, sub = tid & 7;
  float m = -INFINITY;
  for (int n = sub; n < ATTN_CHUNK; n += 8) m = fmaxf(m, s_k[d][n]);
  m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
  m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
  m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 4));
  float sum = 0.0f;
  for (int n = sub; n < ATTN_CHUNK; n += 8) {
    const float e = (n < nn) ? expf(s_k[d][n] - m) : 0.0f;
    s_k[d][n] = e;
    sum += e;
  }
  sum += __shfl_xor_sync(0xffffffffu, sum, 1);
  sum += __shfl_xor_sync(0xffffffffu, sum, 2);
  sum += __shfl_xor_sync(0xffffffffu, sum, 4);
  __syncthreads();
  const int e0 = sub * 4;
  float acc[4] = {0, 0, 0, 0};
  for (int n = 0; n < ATTN_CHUNK; ++n) {
    const float kk = s_k[d][n];
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j] = fmaf(kk, s_v[e0 + j][n], acc[j]);
  }
  float* o = part + (((size_t)b * H + h) * S + c) * ATTN_PART;
#pragma unroll
  for (int j = 0; j < 4; ++j) o[d * 32 + e0 + j] = acc[j];
  if (sub == 0) { o[1024 + d] = m; o[1024 + 32 + d] = sum; }
}

__global__ void __launch_bounds__(128)
k_attn_apply(const float4* __restrict__ qkv, const float* __restrict__ part, float4* __restrict__ out, int H, int N, int S) {
  int h = blockIdx.y, b = blockIdx.z;
  __shared__ float s_ctx[32 * 32];
  __shared__ float s_w[32][33];          // [chunk (<= 32)][d]: exp(max_c - max) / denominator
  const float* pb = part + ((size_t)b * H + h) * S * ATTN_PART;
  if (threadIdx.x < 32) {
    const int d = threadIdx.x;
    float M = -INFINITY;
    for (int c = 0; c < S; ++c) M = fmaxf(M, pb[(size_t)c * ATTN_PART + 1024 + d]);
    float den = 0.0f;
    for (int c = 0; c < S; ++c) den += expf(pb[(size_t)c * ATTN_PART + 1024 + d] - M) * pb[(size_t)c * ATTN_PART + 1024 + 32 + d];
    const float inv = 1.0f / den;
    for (int c = 0; c < S; ++c) s_w[c][d] = expf(pb[(size_t)c * ATTN_PART + 1024 + d] - M) * inv;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 1024; i += 128) {
    const int d = i >> 5;
    float a = 0.0f;
    for (int c = 0; c < S; ++c) a = fmaf(s_w[c][d], pb[(size_t)c * ATTN_PART + i], a);
    s_ctx[i] = a;
  }
  __syncthreads();
  int n = blockIdx.x * 128 + threadIdx.x;
  if (n >= N) return;
  int Gq = 3 * H * 8;
  const float4* qb = qkv + ((size_t)b * Gq + h * 8) * N;
  float acc[32];
#pragma unroll
  for (int e = 0; e < 32; ++e) acc[e] = 0.0f;
#pragma unroll
  for (int g = 0; g < 8; ++g) {
    float4 q = qb[(size_t)g * N + n];
    float qq[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float* c = s_ctx + (g * 4 + j) * 32;
#pragma unroll
      for (int e = 0; e < 32; ++e) acc[e] = fmaf(c[e], qq[j], acc[e]);
    }
  }
  float4* ob = out + ((size_t)b * (H * 8) + h * 8) * N;
#pragma unroll
  for (int g = 0; g < 8; ++g) ob[(size_t)g * N + n] = make_float4(acc[4 * g], acc[4 * g + 1], acc[4 * g + 2], acc[4 * g + 3]);
}

// ------------------------------------------------------------------------------------
// layout conversion at the module-level C ABI: [B][C][R] channel-major <-> PF
// ------------------------------------------------------------------------------------
__global__ void k_cm_to_pf(const float* __restrict__ src, float4* __restrict__ dst, int C, int G, int R) {
  int b = blockIdx.z, g = blockIdx.y;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R) return;
  float v[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    int c = g * 4 + j;
    v[j] = c < C ? src[((size_t)b * C + c) * R + i] : 0.0f;
  }
  dst[((size_t)b * G + g) * R + i] = make_float4(v[0], v[1], v[2], v[3]);
}
__global__ void k_pf_to_cm(const float4* __restrict__ src, float* __restrict__ dst, int C, int G, int R) {
  int b = blockIdx.z, g = blockIdx.y;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R) return;
  float4 v = src[((size_t)b * G + g) * R + i];
  float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    int c = g * 4 + j;
    if (c < C) dst[((size_t)b * C + c) * R + i] = vv[j];
  }
}
// dense voxel tensor [B][C][r^3] (flat index x*r^2 + y*r + z) <-> zero-haloed VG [B][G][(r+2)^3][4];
// the halo rows of the VG must already be zero.  tf32 != 0: round to TF32 (rna) for the tensor cores.
__global__ void k_cm_to_vg(const float* __restrict__ src, float4* __restrict__ dst, int C, int G, int r, int tf32) {
  int b = blockIdx.z, g = blockIdx.y;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int V = r * r * r, rp = r + 2;
  if (i >= V) return;
  int x = i / (r * r), y = (i / r) % r, z = i % r;
  size_t prow = ((size_t)(x + 1) * rp + (y + 1)) * rp + (z + 1);
  float v[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    int c = g * 4 + j;
    v[j] = c < C ? src[((size_t)b * C + c) * V + i] : 0.0f;
  }
  float4 o = make_float4(v[0], v[1], v[2], v[3]);
  if (tf32) o = f4_tf32(o);
  dst[((size_t)b * G + g) * ((size_t)rp * rp * rp) + prow] = o;
}
// the FP16 form of k_cm_to_vg: dst [B][G8][(r+2)^3] rows of 8 halves (channels 8 g8 .. 8 g8 + 7, rounded to nearest even)
__global__ void k_cm_to_vg_h8(const float* __restrict__ src, float4* __restrict__ dst, int C, int G8, int r) {
  int b = blockIdx.z, g = blockIdx.y;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int V = r * r * r, rp = r + 2;
  if (i >= V) return;
  int x = i / (r * r), y = (i / r) % r, z = i % r;
  size_t prow = ((size_t)(x + 1) * rp + (y + 1)) * rp + (z + 1);
  float v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    int c = g * 8 + j;
    v[j] = c < C ? src[((size_t)b * C + c) * V + i] : 0.0f;
  }
  dst[((size_t)b * G8 + g) * ((size_t)rp * rp * rp) + prow] = h8_pack(make_float4(v[0], v[1], v[2], v[3]), make_float4(v[4], v[5], v[6], v[7]));
}
// rows of 8 halves [B][G8][R] -> channel-major fp32 [B][C][R] (exact)
__global__ void k_h8_to_cm(const float4* __restrict__ src, float* __restrict__ dst, int C, int G8, int R) {
  int b = blockIdx.z, g = blockIdx.y;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R) return;
  union { float4 f; __half h[8]; } u;
  u.f = src[((size_t)b * G8 + g) * R + i];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    int c = g * 8 + j;
    if (c < C) dst[((size_t)b * C + c) * R + i] = __half2float(u.h[j]);
  }
}
__global__ void k_vg_to_cm(const float4* __restrict__ src, float* __restrict__ dst, int C, int G, int r) {
  int b = blockIdx.z, g = blockIdx.y;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int V = r * r * r, rp = r + 2;
  if (i >= V) return;
  int x = i / (r * r), y = (i / r) % r, z = i % r;
  size_t prow = ((size_t)(x + 1) * rp + (y + 1)) * rp + (z + 1);
  float4 v = src[((size_t)b * G + g) * ((size_t)rp * rp * rp) + prow];
  float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    int c = g * 4 + j;
    if (c < C) dst[((size_t)b * C + c) * V + i] = vv[j];
  }
}
__global__ void k_cm_to_c4(const float* __restrict__ src, float4* __restrict__ dst, int N) {
  int b = blockIdx.y;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const float* s = src + (size_t)b * 3 * N;
  dst[(size_t)b * N + i] = make_float4(s[i], s[i + N], s[i + 2 * N], 0.0f);
}
__global__ void k_c4_to_cm(const float4* __restrict__ src, float* __restrict__ dst, int N) {
  int b = blockIdx.y;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  float4 v = src[(size_t)b * N + i];
  float* d = dst + (size_t)b * 3 * N;
  d[i] = v.x; d[i + N] = v.y; d[i + 2 * N] = v.z;
}

}  // namespace lion
