// Streaming sm_90a kernels of the calibration E-step: every kernel makes one pass over planar
// coherencies / visibilities in HBM with 128-bit coalesced loads (a warp = one station p against
// 32 consecutive stations q, 512 contiguous bytes per polarisation product per timeslot).
//
//   k_predict_full   : V = sum_k J_kp C_k J_kq^H over all clusters, residual / cost
//                      (replaces predict_threadfn_withgain_full, lmfit.c:611-688, plus
//                       cost_func / robust_cost_func, robust_lbfgs.c:674-726)
//   k_grad_full      : LBFGS gradient over all clusters from a stored residual
//                      (replaces cpu_calc_deriv(_robust), robust_lbfgs.c:424-560,155-316, which
//                       loop per PARAMETER over all rows; here one pass over rows)
//   k_cluster_pass   : per-cluster E-step pass of the LM solver: model of one cluster, residual,
//                      cost and J^T e in a single sweep (replaces predict_threadfn_withgain(0),
//                      lmfit.c:64-124,233-296 + the J^T e dgemv of clmfit.c:315)
//   k_coh_gram       : per-baseline time sums conj(C) (x) C from which J^T J is assembled without
//                      ever forming the dense Jacobian (jacobian_threadfn, lmfit.c:392-474 +
//                      dgemm, clmfit.c:307)
#include "internal.cuh"
#include "tma.cuh"

// ------------------------------------------------------------------------------------------------
// layout conversion (API layout <-> planar device layout)
// ------------------------------------------------------------------------------------------------
// src: rows [r0, r0+nr) of the API coherency array, [row][M][4] complex; dst planar [M][4][R]
// block (32 clusters, 8 rows): 64 B contiguous reads per thread (2 KB per warp), 128 B row-runs out
#define XP_ROWS 8
__global__ void k_coh_to_planar(const double2 *__restrict__ src, double2 *__restrict__ dst,
                                long long r0, int nr, int M, long long R) {
  __shared__ double2 tile[4][XP_ROWS][33];
  const int kx = blockIdx.x * 32 + threadIdx.x;
  const int ry = blockIdx.y * XP_ROWS + threadIdx.y;
  if (kx < M && ry < nr) {
    const double2 *s = src + ((long long)ry * M + kx) * 4;
#pragma unroll
    for (int c = 0; c < 4; c++) tile[c][threadIdx.y][threadIdx.x] = s[c];
  }
  __syncthreads();
  const int tid = threadIdx.y * 32 + threadIdx.x;
  const int rr = tid % XP_ROWS, kk = tid / XP_ROWS;
  const int k = blockIdx.x * 32 + kk;
  const int r = blockIdx.y * XP_ROWS + rr;
  if (k < M && r < nr) {
#pragma unroll
    for (int c = 0; c < 4; c++) dst[((long long)k * 4 + c) * R + r0 + r] = tile[c][rr][kk];
  }
}

// planar [M][4][R] -> API layout rows [r0, r0+nr)
__global__ void k_coh_from_planar(const double2 *__restrict__ src, double2 *__restrict__ dst,
                                  long long r0, int nr, int M, long long R) {
  __shared__ double2 tile[4][XP_ROWS][33];
  const int tid = threadIdx.y * 32 + threadIdx.x;
  const int rr = tid % XP_ROWS, kk = tid / XP_ROWS;
  const int k = blockIdx.x * 32 + kk;
  const int r = blockIdx.y * XP_ROWS + rr;
  if (k < M && r < nr) {
#pragma unroll
    for (int c = 0; c < 4; c++) tile[c][rr][kk] = src[((long long)k * 4 + c) * R + r0 + r];
  }
  __syncthreads();
  const int kx = blockIdx.x * 32 + threadIdx.x;
  const int ry = blockIdx.y * XP_ROWS + threadIdx.y;
  if (kx < M && ry < nr) {
    double2 *d = dst + ((long long)ry * M + kx) * 4;
#pragma unroll
    for (int c = 0; c < 4; c++) d[c] = tile[c][threadIdx.y][threadIdx.x];
  }
}

// API visibilities [row][4] complex <-> planar [4][R]
__global__ void k_vis_to_planar(const double2 *__restrict__ src, double2 *__restrict__ dst,
                                long long R) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // over 4*R, c fastest in src
  if (i < 4 * R) {
    long long r = i >> 2;
    int c = (int)(i & 3);
    dst[(long long)c * R + r] = src[i];
  }
}
__global__ void k_vis_from_planar(const double2 *__restrict__ src, double2 *__restrict__ dst,
                                  long long R) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 4 * R) {
    long long r = i >> 2;
    int c = (int)(i & 3);
    dst[i] = src[(long long)c * R + r];
  }
}

// ------------------------------------------------------------------------------------------------
// deterministic grid reduction: per-CTA partial, the last CTA to arrive sums them in index order
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void grid_reduce_sum(double v, double *partials, double *out,
                                                unsigned int *counter) {
  __shared__ double wsum[32];
  __shared__ bool is_last;
  v = warp_sum(v);
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) wsum[w] = v;
  __syncthreads();
  unsigned int nblocks = gridDim.x * gridDim.y * gridDim.z;
  unsigned int bid = blockIdx.x + gridDim.x * (blockIdx.y + gridDim.y * blockIdx.z);
  if (threadIdx.x == 0) {
    double s = 0.0;
    int nw = (blockDim.x + 31) >> 5;
    for (int i = 0; i < nw; i++) s += wsum[i];
    partials[bid] = s;
    __threadfence();
    unsigned int t = atomicAdd(counter, 1u);
    is_last = (t == nblocks - 1);
  }
  __syncthreads();
  if (is_last) {
    // fixed-order tree: thread i sums partials i, i+T, ...; then block tree
    double s = 0.0;
    for (unsigned int i = threadIdx.x; i < nblocks; i += blockDim.x)
      s += ((volatile double *)partials)[i];
    s = warp_sum(s);
    __syncthreads();
    if (lane == 0) wsum[w] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
      double tot = 0.0;
      int nw = (blockDim.x + 31) >> 5;
      for (int i = 0; i < nw; i++) tot += wsum[i];
      *out = tot;
      *counter = 0;  // re-arm for the next launch
    }
  }
}

// ------------------------------------------------------------------------------------------------
// full predict over all clusters
// ------------------------------------------------------------------------------------------------

template <int TB>
__global__ void __launch_bounds__(TILE_THREADS)
k_predict_full(PredictArgs a) {
  const TileDesc td = a.tiles[blockIdx.x];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int p = td.pb * TILE_P + w;
  const int q = td.qb * TILE_Q + lane;
  const bool valid = (q > p) && (q < a.N);
  const int t0 = blockIdx.y * TB;
  double cost = 0.0;
  if (valid) {
    const long long b = baseline_index(p, q, a.N);
    double2 acc[TB][4];
    bool fl[TB];
    long long row[TB];
#pragma unroll
    for (int i = 0; i < TB; i++) {
      int t = t0 + i;
      row[i] = (long long)(t < a.tilesz ? t : a.tilesz - 1) * a.Nbase + b;
      fl[i] = (t < a.tilesz) ? (a.flag[row[i]] != 0) : true;
#pragma unroll
      for (int c = 0; c < 4; c++) acc[i][c] = make_double2(0.0, 0.0);
    }
    for (int k = 0; k < a.M; k++) {
      const ClusterDesc cd = a.clus[k];
      const double2 *ck = a.coh + (long long)k * 4 * a.R;
      double2 Jp[4], Jq[4];
      int cur = -1;
#pragma unroll
      for (int i = 0; i < TB; i++) {
        double2 C[4];
#pragma unroll
        for (int c = 0; c < 4; c++) C[c] = ld_stream(ck + (long long)c * a.R + row[i]);
        int px = row_chunk(row[i], a.R, cd.nchunk);
        if (px != cur) {
          const double *pblk = a.pp + a.chunk_poff[cd.chunk0 + px];
          load_jones(pblk, p, Jp);
          load_jones(pblk, q, Jq);
          cur = px;
        }
        double2 T1[4];
        mat_ab(Jp, C, T1);
        mat_abh_acc(T1, Jq, acc[i]);
      }
    }
#pragma unroll
    for (int i = 0; i < TB; i++) {
      if (t0 + i < a.tilesz) {
#pragma unroll
        for (int c = 0; c < 4; c++) {
          double2 m = fl[i] ? make_double2(0.0, 0.0) : acc[i][c];
          double2 xv = make_double2(0.0, 0.0);
          if (a.out_mode == 1 || a.cost_mode) xv = ld_stream(a.x + (long long)c * a.R + row[i]);
          double2 e = csub(xv, m);
          if (a.out_mode == 1) st_stream(a.out + (long long)c * a.R + row[i], e);
          if (a.out_mode == 2) st_stream(a.out + (long long)c * a.R + row[i], m);
          if (a.cost_mode == 1) {
            cost = fma(e.x, e.x, cost);
            cost = fma(e.y, e.y, cost);
          } else if (a.cost_mode == 2) {
            cost += log(1.0 + e.x * e.x * a.inv_nu);
            cost += log(1.0 + e.y * e.y * a.inv_nu);
          }
        }
      }
    }
  }
  if (a.cost_mode) grid_reduce_sum(cost, a.partials, a.cost, a.counter);
}

// ------------------------------------------------------------------------------------------------
// shared epilogue: reduce per-thread station gradients of a tile and add them to g (8 doubles per
// station).  Gp belongs to station p (shared by the whole warp), Gq to station q (one per lane,
// shared by the 8 warps of the CTA).  warp-shuffle reduction for p, smem transpose for q.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tile_reduce_station_grad(const double2 *Gp, const double2 *Gq,
                                                          double *gblk, int p, int q, int N,
                                                          bool pvalid, double (*sq)[8][TILE_Q],
                                                          double scale) {
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // station p: butterfly over the 32 lanes
  double vp[8];
#pragma unroll
  for (int c = 0; c < 4; c++) {
    vp[2 * c] = warp_sum(Gp[c].x);
    vp[2 * c + 1] = warp_sum(Gp[c].y);
  }
  if (pvalid && lane < 8) {
    double v = vp[0];
#pragma unroll
    for (int c = 1; c < 8; c++) v = (lane == c) ? vp[c] : v;
    atomicAdd(gblk + 8 * (long long)p + lane, scale * v);
  }
  // station q: [warp][component][lane] in smem, warp c sums component c over the 8 warps
#pragma unroll
  for (int c = 0; c < 4; c++) {
    sq[w][2 * c][lane] = Gq[c].x;
    sq[w][2 * c + 1][lane] = Gq[c].y;
  }
  __syncthreads();
  {
    double s = 0.0;
#pragma unroll
    for (int ww = 0; ww < TILE_P; ww++) s += sq[ww][w][lane];
    if (q < N && s != 0.0) atomicAdd(gblk + 8 * (long long)q + w, scale * s);
  }
  __syncthreads();
}

// contraction of the time-summed outer product W[i][j][l][m] = sum_t R_ij conj(C_lm) with the Jones
// matrices:   Gp = R Jq C^H -> Gp_il = sum_{j,m} Jq_jm W[i,j,l,m]
//             Gq = R^H Jp C -> Gq_jm = sum_{i,l} Jp_il conj(W[i,j,l,m])
// (the 8 reals of Gp/Gq are d(cost)/d(Re,Im of J_p,il / J_q,jm) up to the factor 2, see
//  DESIGN.md "closed-form gradient"; cf. the per-parameter E_col products of lmfit.c:436-466)
__device__ __forceinline__ void contract_W(const double2 *W, const double2 *Jp, const double2 *Jq,
                                           double2 *Gp, double2 *Gq) {
#pragma unroll
  for (int i = 0; i < 2; i++)
#pragma unroll
    for (int l = 0; l < 2; l++) {
      double2 s = make_double2(0.0, 0.0);
#pragma unroll
      for (int j = 0; j < 2; j++)
#pragma unroll
        for (int m = 0; m < 2; m++) cfma(s, Jq[2 * j + m], W[((i * 2 + j) * 2 + l) * 2 + m]);
      Gp[2 * i + l] = cadd(Gp[2 * i + l], s);
    }
#pragma unroll
  for (int j = 0; j < 2; j++)
#pragma unroll
    for (int m = 0; m < 2; m++) {
      double2 s = make_double2(0.0, 0.0);
#pragma unroll
      for (int i = 0; i < 2; i++)
#pragma unroll
        for (int l = 0; l < 2; l++) cfmac(s, Jp[2 * i + l], W[((i * 2 + j) * 2 + l) * 2 + m]);
      Gq[2 * j + m] = cadd(Gq[2 * j + m], s);
    }
}

// W += R (x) conj(C)
__device__ __forceinline__ void accum_W(double2 *W, const double2 *Rm, const double2 *C) {
#pragma unroll
  for (int ij = 0; ij < 4; ij++)
#pragma unroll
    for (int lm = 0; lm < 4; lm++) cfmac(W[ij * 4 + lm], Rm[ij], C[lm]);
}

// ------------------------------------------------------------------------------------------------
// LBFGS gradient over all clusters
// ------------------------------------------------------------------------------------------------

template <int TB>
__global__ void __launch_bounds__(TILE_THREADS)
k_grad_full(GradArgs a) {
  __shared__ double sq[TILE_P][8][TILE_Q];
  const TileDesc td = a.tiles[blockIdx.x];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int p = td.pb * TILE_P + w;
  const int q = td.qb * TILE_Q + lane;
  const bool valid = (q > p) && (q < a.N);
  const int t0 = blockIdx.y * TB;
  const long long b = valid ? baseline_index(p, q, a.N) : 0;
  double2 Rm[TB][4];
  long long row[TB];
  bool use[TB];
#pragma unroll
  for (int i = 0; i < TB; i++) {
    int t = t0 + i;
    row[i] = (long long)(t < a.tilesz ? t : a.tilesz - 1) * a.Nbase + b;
    use[i] = valid && (t < a.tilesz) && (a.flag[row[i]] == 0);
#pragma unroll
    for (int c = 0; c < 4; c++) {
      double2 e = make_double2(0.0, 0.0);
      if (use[i]) {
        e = ld_stream(a.res + (long long)c * a.R + row[i]);
        if (a.robust) {
          e.x = e.x / (a.nu + e.x * e.x);
          e.y = e.y / (a.nu + e.y * e.y);
        }
      }
      Rm[i][c] = e;
    }
  }
  for (int k = 0; k < a.M; k++) {
    const ClusterDesc cd = a.clus[k];
    const double2 *ck = a.coh + (long long)k * 4 * a.R;
    // gradient chunk of a timeslot: t / ceil(tilesz/nchunk)   (robust_lbfgs.c:464-470)
    const int tpc = (a.tilesz + cd.nchunk - 1) / cd.nchunk;
    int i0 = 0;
    while (i0 < TB) {  // runs of timeslots that share a chunk (one run unless hybrid)
      const int chunk = (t0 + i0 < a.tilesz ? t0 + i0 : a.tilesz - 1) / tpc;
      double2 W[16];
#pragma unroll
      for (int z = 0; z < 16; z++) W[z] = make_double2(0.0, 0.0);
      int i1 = i0;
#pragma unroll
      for (int i = 0; i < TB; i++) {
        if (i >= i0 && i == i1) {
          int t = t0 + i;
          int ch = (t < a.tilesz ? t : a.tilesz - 1) / tpc;
          if (ch == chunk) {
            i1 = i + 1;
            if (use[i]) {
              double2 C[4];
#pragma unroll
              for (int c = 0; c < 4; c++) C[c] = ld_stream(ck + (long long)c * a.R + row[i]);
              accum_W(W, Rm[i], C);
            }
          }
        }
      }
      double *gblk = a.g + a.chunk_poff[cd.chunk0 + chunk];
      double2 Jp[4], Jq[4], Gp[4], Gq[4];
#pragma unroll
      for (int c = 0; c < 4; c++) {
        Jp[c] = Jq[c] = Gp[c] = Gq[c] = make_double2(0.0, 0.0);
      }
      if (valid) {
        const double *pblk = a.pp + a.chunk_poff[cd.chunk0 + chunk];
        load_jones(pblk, p, Jp);
        load_jones(pblk, q, Jq);
        contract_W(W, Jp, Jq, Gp, Gq);
      }
      tile_reduce_station_grad(Gp, Gq, gblk, p, q, a.N, p < a.N - 1, sq, a.scale);
      i0 = i1;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// LBFGS gradient over all clusters, TMA-fed: same tile mapping and reductions as k_grad_full, but the
// coherencies of the next cluster(s) are already on their way into shared memory (one ring of bulk
// copies per warp: for a fixed station p the 32 lanes' baselines are one contiguous run of rows)
// while the current cluster is contracted and reduced.  The register-staged version alternates load
// and reduce phases with 8 warps per SM and tops out near 1 TB/s.
// ------------------------------------------------------------------------------------------------
template <int TB, int NST>
__global__ void __launch_bounds__(TILE_THREADS)
k_grad_tma(GradArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  constexpr int STAGE_ELEMS = TB * 4 * 32;  // double2 per stage
  double (*sq)[8][TILE_Q] = reinterpret_cast<double (*)[8][TILE_Q]>(smem_raw);
  double2 *ring = reinterpret_cast<double2 *>(smem_raw + sizeof(double) * TILE_P * 8 * TILE_Q);
  unsigned long long *bars = reinterpret_cast<unsigned long long *>(ring + (size_t)TILE_P * NST * STAGE_ELEMS);
  const TileDesc td = a.tiles[blockIdx.x];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int p = td.pb * TILE_P + w;
  const int q0 = td.qb * TILE_Q;
  const int q = q0 + lane;
  const bool valid = (q > p) && (q < a.N);
  const int t0 = blockIdx.y * TB;
  const int nrows = min(TB, a.tilesz - t0);
  // the warp's run of baselines: stations qs .. qs+nv-1 against p
  const int qs = max(q0, p + 1);
  const int nv = max(0, min(q0 + TILE_Q, a.N) - qs);
  const long long b0 = nv > 0 ? baseline_index(p, qs, a.N) : 0;
  const int el = q - qs;  // slot of this lane inside the run (valid lanes only)
  const long long b = valid ? b0 + el : 0;
  double2 *my_stage = ring + (size_t)w * NST * STAGE_ELEMS;
  unsigned long long *my_bar = bars + w * NST;
  if (lane == 0) {
#pragma unroll
    for (int s = 0; s < NST; s++) mbar_init(&my_bar[s], 1);
    mbar_fence_init();
  }
  __syncwarp();
  auto issue = [&](int k, int s) {
    const unsigned row_bytes = (unsigned)nv * 16u;
    mbar_expect_tx(&my_bar[s], (unsigned)nrows * 4u * row_bytes);
    const double2 *ck = a.coh + (long long)k * 4 * a.R + (long long)t0 * a.Nbase + b0;
    double2 *dst = my_stage + (size_t)s * STAGE_ELEMS;
    for (int i = 0; i < nrows; i++)
#pragma unroll
      for (int c = 0; c < 4; c++)
        bulk_g2s(dst + (i * 4 + c) * 32, ck + (long long)c * a.R + (long long)i * a.Nbase, row_bytes,
                 &my_bar[s]);
  };
  if (lane == 0 && nv > 0) {
#pragma unroll
    for (int s = 0; s < NST - 1; s++)
      if (s < a.M) issue(s, s);
  }

  double2 Rm[TB][4];
  bool use[TB];
#pragma unroll
  for (int i = 0; i < TB; i++) {
    const int t = t0 + i;
    const long long row = (long long)(t < a.tilesz ? t : a.tilesz - 1) * a.Nbase + b;
    use[i] = valid && (t < a.tilesz) && (a.flag[row] == 0);
#pragma unroll
    for (int c = 0; c < 4; c++) {
      double2 e = make_double2(0.0, 0.0);
      if (use[i]) {
        e = ld_stream(a.res + (long long)c * a.R + row);
        if (a.robust) {
          e.x = e.x / (a.nu + e.x * e.x);
          e.y = e.y / (a.nu + e.y * e.y);
        }
      }
      Rm[i][c] = e;
    }
  }
  for (int k = 0; k < a.M; k++) {
    const int s = k % NST;
    if (lane == 0 && nv > 0 && k + NST - 1 < a.M) issue(k + NST - 1, (k + NST - 1) % NST);
    const ClusterDesc cd = a.clus[k];
    // gradient chunk of a timeslot: t / ceil(tilesz/nchunk)   (robust_lbfgs.c:464-470)
    const int tpc = (a.tilesz + cd.nchunk - 1) / cd.nchunk;
    if (nv > 0) mbar_wait(&my_bar[s], (unsigned)((k / NST) & 1));
    const double2 *st = my_stage + (size_t)s * STAGE_ELEMS;
    int i0 = 0;
    while (i0 < TB) {  // runs of timeslots that share a chunk (one run unless hybrid)
      const int chunk = (t0 + i0 < a.tilesz ? t0 + i0 : a.tilesz - 1) / tpc;
      double2 W[16];
#pragma unroll
      for (int z = 0; z < 16; z++) W[z] = make_double2(0.0, 0.0);
      int i1 = i0;
#pragma unroll
      for (int i = 0; i < TB; i++) {
        if (i >= i0 && i == i1) {
          const int t = t0 + i;
          const int ch = (t < a.tilesz ? t : a.tilesz - 1) / tpc;
          if (ch == chunk) {
            i1 = i + 1;
            if (use[i]) {
              double2 C[4];
#pragma unroll
              for (int c = 0; c < 4; c++) C[c] = lds_v2(st + (i * 4 + c) * 32 + el);
              accum_W(W, Rm[i], C);
            }
          }
        }
      }
      double *gblk = a.g + a.chunk_poff[cd.chunk0 + chunk];
      double2 Jp[4], Jq[4], Gp[4], Gq[4];
#pragma unroll
      for (int c = 0; c < 4; c++) Jp[c] = Jq[c] = Gp[c] = Gq[c] = make_double2(0.0, 0.0);
      if (valid) {
        const double *pblk = a.pp + a.chunk_poff[cd.chunk0 + chunk];
        load_jones(pblk, p, Jp);
        load_jones(pblk, q, Jq);
        contract_W(W, Jp, Jq, Gp, Gq);
      }
      // (two CTA barriers inside: every lane is also done with stage s before it is refilled)
      tile_reduce_station_grad(Gp, Gq, gblk, p, q, a.N, p < a.N - 1, sq, a.scale);
      i0 = i1;
    }
  }
}

// sums of four values over the warp with 6 double shuffles instead of 20: halves of the warp trade
// the values they do not keep.  Lane 8*c (c = 0..3) ends up with the warp sum of v[c].
__device__ __forceinline__ double warp_reduce4(double v0, double v1, double v2, double v3, int lane) {
  const bool hi = (lane & 16) != 0;
  double k0 = hi ? v2 : v0, k1 = hi ? v3 : v1;
  k0 += __shfl_xor_sync(0xffffffffu, hi ? v0 : v2, 16);
  k1 += __shfl_xor_sync(0xffffffffu, hi ? v1 : v3, 16);
  const bool h8 = (lane & 8) != 0;
  double kk = h8 ? k1 : k0;
  kk += __shfl_xor_sync(0xffffffffu, h8 ? k0 : k1, 8);
  kk += __shfl_xor_sync(0xffffffffu, kk, 4);
  kk += __shfl_xor_sync(0xffffffffu, kk, 2);
  kk += __shfl_xor_sync(0xffffffffu, kk, 1);
  return kk;
}

// ------------------------------------------------------------------------------------------------
// k_grad_tma with the polarisation split of k_cluster_pass_split: two threads per baseline, thread h
// owns row h of the residual and the half W[i=h] of the accumulator.  16 warps per CTA share the 8
// TMA rings (the two warps of a station p consume the same stages; warp h=0 is the producer, the CTA
// barriers of the per-cluster reduction make a consumed stage reusable).
// threadIdx.x = h*256 + w*32 + lane.
// ------------------------------------------------------------------------------------------------
template <int TB, int NST>
__global__ void __launch_bounds__(2 * TILE_THREADS)
k_grad_tma_split(GradArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  constexpr int STAGE_ELEMS = TB * 4 * 32;  // double2 per stage
  double (*sq)[8][TILE_Q] = reinterpret_cast<double (*)[8][TILE_Q]>(smem_raw);
  double2 *ring = reinterpret_cast<double2 *>(smem_raw + sizeof(double) * 2 * TILE_P * 8 * TILE_Q);
  unsigned long long *bars =
      reinterpret_cast<unsigned long long *>(ring + (size_t)TILE_P * NST * STAGE_ELEMS);
  const TileDesc td = a.tiles[blockIdx.x];
  const int h = threadIdx.x >> 8, w = (threadIdx.x >> 5) & 7, lane = threadIdx.x & 31;
  const int p = td.pb * TILE_P + w;
  const int q0 = td.qb * TILE_Q;
  const int q = q0 + lane;
  const bool valid = (q > p) && (q < a.N);
  const int t0 = blockIdx.y * TB;
  const int nrows = min(TB, a.tilesz - t0);
  const int qs = max(q0, p + 1);
  const int nv = max(0, min(q0 + TILE_Q, a.N) - qs);
  const long long b0 = nv > 0 ? baseline_index(p, qs, a.N) : 0;
  const int el = q - qs;
  const long long b = valid ? b0 + el : 0;
  double2 *my_stage = ring + (size_t)w * NST * STAGE_ELEMS;
  unsigned long long *my_bar = bars + w * NST;
  if (h == 0 && lane == 0) {
#pragma unroll
    for (int s = 0; s < NST; s++) mbar_init(&my_bar[s], 1);
    mbar_fence_init();
  }
  __syncthreads();
  auto issue = [&](int k, int s) {
    const unsigned row_bytes = (unsigned)nv * 16u;
    mbar_expect_tx(&my_bar[s], (unsigned)nrows * 4u * row_bytes);
    const double2 *ck = a.coh + (long long)k * 4 * a.R + (long long)t0 * a.Nbase + b0;
    double2 *dst = my_stage + (size_t)s * STAGE_ELEMS;
    for (int i = 0; i < nrows; i++)
#pragma unroll
      for (int c = 0; c < 4; c++)
        bulk_g2s(dst + (i * 4 + c) * 32, ck + (long long)c * a.R + (long long)i * a.Nbase, row_bytes,
                 &my_bar[s]);
  };
  const bool producer = (h == 0 && lane == 0 && nv > 0);
  if (producer) {
#pragma unroll
    for (int s = 0; s < NST - 1; s++)
      if (s < a.M) issue(s, s);
  }

  double2 Rm[TB][2];
  bool use[TB];
#pragma unroll
  for (int i = 0; i < TB; i++) {
    const int t = t0 + i;
    const long long row = (long long)(t < a.tilesz ? t : a.tilesz - 1) * a.Nbase + b;
    use[i] = valid && (t < a.tilesz) && (a.flag[row] == 0);
#pragma unroll
    for (int j = 0; j < 2; j++) {
      double2 e = make_double2(0.0, 0.0);
      if (use[i]) {
        e = ld_stream(a.res + (long long)(2 * h + j) * a.R + row);
        if (a.robust) {
          e.x = e.x / (a.nu + e.x * e.x);
          e.y = e.y / (a.nu + e.y * e.y);
        }
      }
      Rm[i][j] = e;
    }
  }
  for (int k = 0; k < a.M; k++) {
    const int s = k % NST;
    // stage (k-1)%NST was consumed in iteration k-1 by both warps of this p: its closing CTA barrier
    // has been passed, so the producer may refill it
    if (producer && k + NST - 1 < a.M) issue(k + NST - 1, (k + NST - 1) % NST);
    const ClusterDesc cd = a.clus[k];
    const int tpc = (a.tilesz + cd.nchunk - 1) / cd.nchunk;
    if (nv > 0) mbar_wait(&my_bar[s], (unsigned)((k / NST) & 1));
    const double2 *st = my_stage + (size_t)s * STAGE_ELEMS;
    int i0 = 0;
    while (i0 < TB) {  // runs of timeslots that share a chunk (one run unless hybrid)
      int chunk = 0, i1 = TB;
      double2 W[8];
#pragma unroll
      for (int z = 0; z < 8; z++) W[z] = make_double2(0.0, 0.0);
      if (cd.nchunk == 1) {
        // the common case: no chunk bookkeeping at all
#pragma unroll
        for (int i = 0; i < TB; i++) {
          if (use[i]) {
            double2 C[4];
#pragma unroll
            for (int c = 0; c < 4; c++) C[c] = lds_v2(st + (i * 4 + c) * 32 + el);
#pragma unroll
            for (int j = 0; j < 2; j++)
#pragma unroll
              for (int lm = 0; lm < 4; lm++) cfmac(W[j * 4 + lm], Rm[i][j], C[lm]);
          }
        }
      } else {
        chunk = (t0 + i0 < a.tilesz ? t0 + i0 : a.tilesz - 1) / tpc;
        i1 = i0;
#pragma unroll
        for (int i = 0; i < TB; i++) {
          if (i >= i0 && i == i1) {
            const int t = t0 + i;
            const int ch = (t < a.tilesz ? t : a.tilesz - 1) / tpc;
            if (ch == chunk) {
              i1 = i + 1;
              if (use[i]) {
                double2 C[4];
#pragma unroll
                for (int c = 0; c < 4; c++) C[c] = lds_v2(st + (i * 4 + c) * 32 + el);
#pragma unroll
                for (int j = 0; j < 2; j++)
#pragma unroll
                  for (int lm = 0; lm < 4; lm++) cfmac(W[j * 4 + lm], Rm[i][j], C[lm]);
              }
            }
          }
        }
      }
      double *gblk = a.g + a.chunk_poff[cd.chunk0 + chunk];
      double2 Gp[2], Gq[4];
      Gp[0] = Gp[1] = make_double2(0.0, 0.0);
#pragma unroll
      for (int c = 0; c < 4; c++) Gq[c] = make_double2(0.0, 0.0);
      if (valid) {
        const double *pblk = a.pp + a.chunk_poff[cd.chunk0 + chunk];
        double2 Jr[2], Jq[4];
        const double2 *jp = reinterpret_cast<const double2 *>(pblk + 8 * (long long)p + 4 * h);
        Jr[0] = __ldg(jp);
        Jr[1] = __ldg(jp + 1);
        load_jones(pblk, q, Jq);
#pragma unroll
        for (int l = 0; l < 2; l++)
#pragma unroll
          for (int j = 0; j < 2; j++)
#pragma unroll
            for (int m = 0; m < 2; m++) cfma(Gp[l], Jq[2 * j + m], W[j * 4 + l * 2 + m]);
#pragma unroll
        for (int j = 0; j < 2; j++)
#pragma unroll
          for (int m = 0; m < 2; m++)
#pragma unroll
            for (int l = 0; l < 2; l++) cfmac(Gq[2 * j + m], Jr[l], W[j * 4 + l * 2 + m]);
      }
      // station p: 4 reals per half (components 4h .. 4h+3), lane 8c holds component c
      {
        const double v = warp_reduce4(Gp[0].x, Gp[0].y, Gp[1].x, Gp[1].y, lane);
        if (p < a.N - 1 && (lane & 7) == 0)
          atomicAdd(gblk + 8 * (long long)p + 4 * h + (lane >> 3), a.scale * v);
      }
      // station q: sum over the 16 warps through shared memory
#pragma unroll
      for (int c = 0; c < 4; c++) {
        sq[h * TILE_P + w][2 * c][lane] = Gq[c].x;
        sq[h * TILE_P + w][2 * c + 1][lane] = Gq[c].y;
      }
      __syncthreads();
      if (h == 0) {
        double sacc = 0.0;
#pragma unroll
        for (int ww = 0; ww < 2 * TILE_P; ww++) sacc += sq[ww][w][lane];
        if (q < a.N && sacc != 0.0) atomicAdd(gblk + 8 * (long long)q + w, a.scale * sacc);
      }
      __syncthreads();
      i0 = i1;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// per-cluster E-step pass (LM): one cluster, one hybrid chunk, timeslots [t_begin, t_end)
// ------------------------------------------------------------------------------------------------

// GRAD = false (ADD / SUB passes, ordered-subset trials): no W accumulator, about half the registers
template <bool GRAD>
__global__ void __launch_bounds__(TILE_THREADS)
k_cluster_pass(ClusterPassArgs a) {
  __shared__ double sq[GRAD ? TILE_P : 1][8][TILE_Q];
  const TileDesc td = a.tiles[blockIdx.x];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int p = td.pb * TILE_P + w;
  const int q = td.qb * TILE_Q + lane;
  const bool valid = (q > p) && (q < a.N);
  const int ts = a.t_begin + blockIdx.y * a.tslice;
  const int te = min(ts + a.tslice, a.t_end);
  double cost = 0.0;
  double2 Jp[4], Jq[4], W[GRAD ? 16 : 1];
#pragma unroll
  for (int z = 0; z < (GRAD ? 16 : 1); z++) W[z] = make_double2(0.0, 0.0);
#pragma unroll
  for (int c = 0; c < 4; c++) Jp[c] = Jq[c] = make_double2(0.0, 0.0);
  if (valid) {
    load_jones(a.pblk, p, Jp);
    load_jones(a.pblk, q, Jq);
    double2 Jpo[4], Jqo[4];
    const bool recover = (!GRAD) && a.mode == 3 && a.pblk_old != nullptr;
    const double gamma = recover ? (1.0 - a.beta) / a.beta : 0.0;
    if (recover) {
      load_jones(a.pblk_old, p, Jpo);
      load_jones(a.pblk_old, q, Jqo);
    }
    const long long b = baseline_index(p, q, a.N);
#pragma unroll 2
    for (int t = ts; t < te; t++) {
      const long long row = (long long)t * a.Nbase + b;
      double2 C[4], v[4];
#pragma unroll
      for (int c = 0; c < 4; c++) C[c] = ld_stream(a.coh_k + (long long)c * a.R + row);
#pragma unroll
      for (int c = 0; c < 4; c++) v[c] = ld_stream(a.in + (long long)c * a.R + row);
      const bool fl = a.flag[row] != 0;
      double2 T1[4], m[4];
      mat_ab(Jp, C, T1);
      mat_abh(T1, Jq, m);
      if (fl) {
#pragma unroll
        for (int c = 0; c < 4; c++) m[c] = make_double2(0.0, 0.0);
      }
      double2 e[4];
      if (a.mode == 0) {
#pragma unroll
        for (int c = 0; c < 4; c++) {
          double2 d = cadd(make_double2(a.beta * v[c].x, a.beta * v[c].y), m[c]);
          if (a.write_out) st_stream(a.out + (long long)c * a.R + row, d);
          e[c] = csub(d, m[c]);
        }
      } else if (a.mode == 2) {
#pragma unroll
        for (int c = 0; c < 4; c++)
          st_stream(a.out + (long long)c * a.R + row,
                    cadd(make_double2(a.beta * v[c].x, a.beta * v[c].y), m[c]));
      } else {
        double2 mo[4];
        if (recover) {
          double2 T2[4];
          mat_ab(Jpo, C, T2);
          mat_abh(T2, Jqo, mo);
          if (fl) {
#pragma unroll
            for (int c = 0; c < 4; c++) mo[c] = make_double2(0.0, 0.0);
          }
        }
#pragma unroll
        for (int c = 0; c < 4; c++) {
          e[c] = csub(v[c], m[c]);
          double2 o = e[c];
          if (recover) {
            // + (1-beta) r_old with r_old = (d - f(p_old)) / beta
            o.x = fma(gamma, v[c].x - mo[c].x, o.x);
            o.y = fma(gamma, v[c].y - mo[c].y, o.y);
          } else if (a.mode == 3 && a.in2) {
            const double2 r2 = a.in2[(long long)c * a.R + row];  // may alias out: plain load
            o.x = fma(1.0 - a.beta, r2.x, o.x);
            o.y = fma(1.0 - a.beta, r2.y, o.y);
          }
          if (a.write_out) st_stream(a.out + (long long)c * a.R + row, o);
        }
      }
      if (a.mode <= 1) {
        if (a.wt) {
          // robust LM: e <- wt.e for the cost, J^T (wt.(wt.e)) for the gradient
#pragma unroll
          for (int c = 0; c < 4; c++) {
            const double2 wv = ld_stream(a.wt + (long long)c * a.R + row);
            const double ex = wv.x * e[c].x, ey = wv.y * e[c].y;
            cost = fma(ex, ex, cost);
            cost = fma(ey, ey, cost);
            e[c] = make_double2(wv.x * ex, wv.y * ey);
          }
        } else {
#pragma unroll
          for (int c = 0; c < 4; c++) {
            cost = fma(e[c].x, e[c].x, cost);
            cost = fma(e[c].y, e[c].y, cost);
          }
        }
        if constexpr (GRAD) {
          if (!fl) accum_W(W, e, C);
        }
      }
    }
  }
  if constexpr (GRAD) {
    double2 Gp[4], Gq[4];
#pragma unroll
    for (int c = 0; c < 4; c++) Gp[c] = Gq[c] = make_double2(0.0, 0.0);
    if (valid) contract_W(W, Jp, Jq, Gp, Gq);
    tile_reduce_station_grad(Gp, Gq, a.jte, p, q, a.N, p < a.N - 1, sq, 1.0);
  }
  if (a.mode <= 1) grid_reduce_sum(cost, a.partials, a.cost, a.counter);
}

// ------------------------------------------------------------------------------------------------
// Gradient-carrying passes (INIT, TRIAL), polarisation-split: two threads per baseline, thread h owns
// row h of the 2x2 visibility (components 2h, 2h+1) and the half W[i=h] of the outer-product
// accumulator.  Nothing is computed twice (row h of Jp C Jq^H needs only row h of Jp), the per-thread
// state halves (W: 16 -> 8 complex), and a CTA carries 16 warps instead of 8: these passes run on
// L2-resident data and are latency bound, so resident warps are what they need.
// threadIdx.x = h*256 + w*32 + lane; p = pb*8 + w, q = qb*32 + lane.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(2 * TILE_THREADS)
k_cluster_pass_split(ClusterPassArgs a) {
  __shared__ double sq[2 * TILE_P][8][TILE_Q];
  const TileDesc td = a.tiles[blockIdx.x];
  const int h = threadIdx.x >> 8, w = (threadIdx.x >> 5) & 7, lane = threadIdx.x & 31;
  const int p = td.pb * TILE_P + w;
  const int q = td.qb * TILE_Q + lane;
  const bool valid = (q > p) && (q < a.N);
  const int ts = a.t_begin + blockIdx.y * a.tslice;
  const int te = min(ts + a.tslice, a.t_end);
  double cost = 0.0;
  double2 Jr[2], Jq[4], W[8];
#pragma unroll
  for (int z = 0; z < 8; z++) W[z] = make_double2(0.0, 0.0);
  Jr[0] = Jr[1] = make_double2(0.0, 0.0);
#pragma unroll
  for (int c = 0; c < 4; c++) Jq[c] = make_double2(0.0, 0.0);
  if (valid) {
    {
      const double2 *jp = reinterpret_cast<const double2 *>(a.pblk + 8 * (long long)p + 4 * h);
      Jr[0] = __ldg(jp);
      Jr[1] = __ldg(jp + 1);
    }
    load_jones(a.pblk, q, Jq);
    const long long b = baseline_index(p, q, a.N);
    const long long c0 = (long long)(2 * h) * a.R, c1 = c0 + a.R;
#pragma unroll 2
    for (int t = ts; t < te; t++) {
      const long long row = (long long)t * a.Nbase + b;
      double2 C[4], v[2];
#pragma unroll
      for (int c = 0; c < 4; c++) C[c] = ld_stream(a.coh_k + (long long)c * a.R + row);
      v[0] = ld_stream(a.in + c0 + row);
      v[1] = ld_stream(a.in + c1 + row);
      const bool fl = a.flag[row] != 0;
      // row h of Jp C, then of (Jp C) Jq^H
      const double2 T0 = cdot2(Jr[0], C[0], Jr[1], C[2]);
      const double2 T1 = cdot2(Jr[0], C[1], Jr[1], C[3]);
      double2 m[2];
      m[0] = cdot2c(T0, Jq[0], T1, Jq[1]);
      m[1] = cdot2c(T0, Jq[2], T1, Jq[3]);
      if (fl) m[0] = m[1] = make_double2(0.0, 0.0);
      double2 e[2];
      if (a.mode == 0) {
#pragma unroll
        for (int j = 0; j < 2; j++) {
          const double2 d = cadd(make_double2(a.beta * v[j].x, a.beta * v[j].y), m[j]);
          if (a.write_out) st_stream(a.out + (j ? c1 : c0) + row, d);
          e[j] = csub(d, m[j]);
        }
      } else {
#pragma unroll
        for (int j = 0; j < 2; j++) {
          e[j] = (a.mode == 4) ? v[j] : csub(v[j], m[j]);  // mode 4: the residual is given
          if (a.write_out) st_stream(a.out + (j ? c1 : c0) + row, e[j]);
        }
      }
      if (a.wt) {
        // robust LM: e <- wt.e for the cost, J^T (wt.(wt.e)) for the gradient
#pragma unroll
        for (int j = 0; j < 2; j++) {
          const double2 wv = ld_stream(a.wt + (j ? c1 : c0) + row);
          const double ex = wv.x * e[j].x, ey = wv.y * e[j].y;
          cost = fma(ex, ex, cost);
          cost = fma(ey, ey, cost);
          e[j] = make_double2(wv.x * ex, wv.y * ey);
        }
      } else {
#pragma unroll
        for (int j = 0; j < 2; j++) {
          cost = fma(e[j].x, e[j].x, cost);
          cost = fma(e[j].y, e[j].y, cost);
        }
      }
      if (!fl) {
#pragma unroll
        for (int j = 0; j < 2; j++)
#pragma unroll
          for (int lm = 0; lm < 4; lm++) cfmac(W[j * 4 + lm], e[j], C[lm]);
      }
    }
  }
  // contraction with the Jones: Gp row h complete, Gq partial (the other half adds its share below)
  double2 Gp[2], Gq[4];
  Gp[0] = Gp[1] = make_double2(0.0, 0.0);
#pragma unroll
  for (int c = 0; c < 4; c++) Gq[c] = make_double2(0.0, 0.0);
  if (valid) {
#pragma unroll
    for (int l = 0; l < 2; l++)
#pragma unroll
      for (int j = 0; j < 2; j++)
#pragma unroll
        for (int m = 0; m < 2; m++) cfma(Gp[l], Jq[2 * j + m], W[j * 4 + l * 2 + m]);
#pragma unroll
    for (int j = 0; j < 2; j++)
#pragma unroll
      for (int m = 0; m < 2; m++)
#pragma unroll
        for (int l = 0; l < 2; l++) cfmac(Gq[2 * j + m], Jr[l], W[j * 4 + l * 2 + m]);
  }
  // station p: butterfly over the lanes; 4 reals per half (components 4h .. 4h+3 of station p)
  {
    double vp[4];
    vp[0] = warp_sum(Gp[0].x);
    vp[1] = warp_sum(Gp[0].y);
    vp[2] = warp_sum(Gp[1].x);
    vp[3] = warp_sum(Gp[1].y);
    if (p < a.N - 1 && lane < 4) {
      double v = vp[0];
#pragma unroll
      for (int c = 1; c < 4; c++) v = (lane == c) ? vp[c] : v;
      atomicAdd(a.jte + 8 * (long long)p + 4 * h + lane, v);
    }
  }
  // station q: [half*8 + warp][component][lane] in smem, warp c of half 0 sums component c
#pragma unroll
  for (int c = 0; c < 4; c++) {
    sq[h * TILE_P + w][2 * c][lane] = Gq[c].x;
    sq[h * TILE_P + w][2 * c + 1][lane] = Gq[c].y;
  }
  __syncthreads();
  if (h == 0) {
    double s = 0.0;
#pragma unroll
    for (int ww = 0; ww < 2 * TILE_P; ww++) s += sq[ww][w][lane];
    if (q < a.N && s != 0.0) atomicAdd(a.jte + 8 * (long long)q + w, s);
  }
  grid_reduce_sum(cost, a.partials, a.cost, a.counter);
}

// ------------------------------------------------------------------------------------------------
// Gradient-carrying pass, linear mapping with CTA-wide TMA stages.  A CTA owns 256 CONSECUTIVE
// baselines x a slice of timeslots; per timeslot the 4 coherency products and the 4 visibility
// components of those baselines are 8 contiguous runs of 4 KB, fetched by 8 bulk copies of one elected
// thread into a ring of NST stages (one mbarrier per stage, a CTA barrier frees a stage).  Compared
// with the tile kernels: every lane is busy (the tile mapping idles 43 % of them at N = 62), NST-1
// whole rows per CTA are in flight without costing registers, and the copy engine sees 16x fewer,
// 8x larger requests.  Two threads per baseline as in k_cluster_pass_split (threadIdx.x = h*256 +
// baseline).  Station sums are GATHERED through shared memory (no atomics: thread 8*s+comp adds up
// what the CTA's baselines contribute to station s), written per CTA, and the last time slice of a
// baseline group adds the group's total to J^T e (8 global atomics per entry instead of ~140).
// ------------------------------------------------------------------------------------------------
template <int NST, bool GRAD>
__global__ void __launch_bounds__(512)
k_cluster_pass_lin(ClusterPassArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  constexpr int BL = 256;
  constexpr int STAGE_ELEMS = 8 * BL;  // double2: C00 C01 C10 C11 v0 v1 v2 v3
  double2 *ring = reinterpret_cast<double2 *>(smem_raw);
  double *acc = reinterpret_cast<double *>(ring + (size_t)NST * STAGE_ELEMS);  // [8N] station sums
  unsigned long long *bars = reinterpret_cast<unsigned long long *>(acc + ((8 * a.N + 1) & ~1));
  const int tid = threadIdx.x, h = tid >> 8, bl = tid & (BL - 1);
  const long long b0 = (long long)blockIdx.x * BL;
  const int nvalid = (int)min((long long)BL, (long long)a.Nbase - b0);
  const bool valid = bl < nvalid;
  const int ts = a.t_begin + blockIdx.y * a.tslice;
  const int te = min(ts + a.tslice, a.t_end);
  const int nrow = te - ts;
  if (GRAD)
    for (int i = tid; i < 8 * a.N; i += 512) acc[i] = 0.0;
  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < NST; s++) mbar_init(&bars[s], 1);
    mbar_fence_init();
  }
  __syncthreads();
  auto issue = [&](int j, int s) {
    const unsigned row_bytes = (unsigned)nvalid * 16u;
    const long long row0 = (long long)(ts + j) * a.Nbase + b0;
    double2 *dst = ring + (size_t)s * STAGE_ELEMS;
    mbar_expect_tx(&bars[s], 8u * row_bytes);
#pragma unroll
    for (int c = 0; c < 4; c++) {
      bulk_g2s(dst + c * BL, a.coh_k + (long long)c * a.R + row0, row_bytes, &bars[s]);
      bulk_g2s(dst + (4 + c) * BL, a.in + (long long)c * a.R + row0, row_bytes, &bars[s]);
    }
  };
  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < NST - 1; s++)
      if (s < nrow) issue(s, s);
  }
  int p = 0, q = 0;
  double2 Jr[2], Jq[4], W[8];
#pragma unroll
  for (int z = 0; z < 8; z++) W[z] = make_double2(0.0, 0.0);
  Jr[0] = Jr[1] = make_double2(0.0, 0.0);
#pragma unroll
  for (int c = 0; c < 4; c++) Jq[c] = make_double2(0.0, 0.0);
  unsigned flagbits = 0;  // bit j: row ts+j flagged (slices are at most 32 rows, see the launcher)
  const long long b = b0 + bl;
  // closing pass of a sharded visit: the old residual is recovered from the Jones the visit started
  // with, out = d - f(p) + (1-beta)/beta (d - f(p_old))
  const bool recover = (!GRAD) && a.mode == 3 && a.pblk_old != nullptr;
  const double gamma = recover ? (1.0 - a.beta) / a.beta : 0.0;
  double2 Jro[2], Jqo[4];
  Jro[0] = Jro[1] = make_double2(0.0, 0.0);
#pragma unroll
  for (int c = 0; c < 4; c++) Jqo[c] = make_double2(0.0, 0.0);
  if (valid) {
    const short2 pq = a.blpq[b];
    p = pq.x;
    q = pq.y;
    const double2 *jp = reinterpret_cast<const double2 *>(a.pblk + 8 * (long long)p + 4 * h);
    Jr[0] = __ldg(jp);
    Jr[1] = __ldg(jp + 1);
    load_jones(a.pblk, q, Jq);
    if (recover) {
      const double2 *jo = reinterpret_cast<const double2 *>(a.pblk_old + 8 * (long long)p + 4 * h);
      Jro[0] = __ldg(jo);
      Jro[1] = __ldg(jo + 1);
      load_jones(a.pblk_old, q, Jqo);
    }
    for (int j = 0; j < nrow; j++)
      flagbits |= (a.flag[(long long)(ts + j) * a.Nbase + b] != 0 ? 1u : 0u) << j;
  }
  const long long c0 = (long long)(2 * h) * a.R, c1 = c0 + a.R;
  double cost = 0.0;
  for (int j = 0; j < nrow; j++) {
    const int s = j % NST;
    // stage (j-1)%NST was released by the CTA barrier that closed iteration j-1
    if (tid == 0 && j + NST - 1 < nrow) issue(j + NST - 1, (j + NST - 1) % NST);
    mbar_wait(&bars[s], (unsigned)((j / NST) & 1));
    if (valid) {
      const double2 *st = ring + (size_t)s * STAGE_ELEMS + bl;
      const long long row = (long long)(ts + j) * a.Nbase + b;
      double2 C[4], v[2];
#pragma unroll
      for (int c = 0; c < 4; c++) C[c] = lds_v2(st + c * BL);
      v[0] = lds_v2(st + (4 + 2 * h) * BL);
      v[1] = lds_v2(st + (5 + 2 * h) * BL);
      const bool fl = (flagbits >> j) & 1u;
      const double2 T0 = cdot2(Jr[0], C[0], Jr[1], C[2]);
      const double2 T1 = cdot2(Jr[0], C[1], Jr[1], C[3]);
      double2 m[2];
      m[0] = cdot2c(T0, Jq[0], T1, Jq[1]);
      m[1] = cdot2c(T0, Jq[2], T1, Jq[3]);
      if (fl) m[0] = m[1] = make_double2(0.0, 0.0);
      double2 e[2];
      if (a.mode == 0 || a.mode == 2) {
#pragma unroll
        for (int jj = 0; jj < 2; jj++) {
          const double2 d = cadd(make_double2(a.beta * v[jj].x, a.beta * v[jj].y), m[jj]);
          if (a.write_out) st_stream(a.out + (jj ? c1 : c0) + row, d);
          e[jj] = csub(d, m[jj]);
        }
      } else {
        double2 mo[2];
        if (recover) {
          const double2 U0 = cdot2(Jro[0], C[0], Jro[1], C[2]);
          const double2 U1 = cdot2(Jro[0], C[1], Jro[1], C[3]);
          mo[0] = cdot2c(U0, Jqo[0], U1, Jqo[1]);
          mo[1] = cdot2c(U0, Jqo[2], U1, Jqo[3]);
          if (fl) mo[0] = mo[1] = make_double2(0.0, 0.0);
        }
#pragma unroll
        for (int jj = 0; jj < 2; jj++) {
          e[jj] = csub(v[jj], m[jj]);
          double2 o = e[jj];
          if (recover) {
            o.x = fma(gamma, v[jj].x - mo[jj].x, o.x);
            o.y = fma(gamma, v[jj].y - mo[jj].y, o.y);
          }
          if (a.write_out) st_stream(a.out + (jj ? c1 : c0) + row, o);
        }
      }
      if (a.mode <= 1) {
#pragma unroll
        for (int jj = 0; jj < 2; jj++) {
          cost = fma(e[jj].x, e[jj].x, cost);
          cost = fma(e[jj].y, e[jj].y, cost);
        }
      }
      if (GRAD && !fl) {
#pragma unroll
        for (int jj = 0; jj < 2; jj++)
#pragma unroll
          for (int lm = 0; lm < 4; lm++) cfmac(W[jj * 4 + lm], e[jj], C[lm]);
      }
    }
    __syncthreads();  // every thread is done with stage s
  }
  if (!GRAD) {
    // ADD / SUB / cost-only pass: no station sums
    if (a.mode <= 1) grid_reduce_sum(cost, a.partials, a.cost, a.counter);
    return;
  }
  // contraction with the Jones (see k_cluster_pass_split)
  double2 Gp[2], Gq[4];
  Gp[0] = Gp[1] = make_double2(0.0, 0.0);
#pragma unroll
  for (int c = 0; c < 4; c++) Gq[c] = make_double2(0.0, 0.0);
  if (valid) {
#pragma unroll
    for (int l = 0; l < 2; l++)
#pragma unroll
      for (int jj = 0; jj < 2; jj++)
#pragma unroll
        for (int m = 0; m < 2; m++) cfma(Gp[l], Jq[2 * jj + m], W[jj * 4 + l * 2 + m]);
#pragma unroll
    for (int jj = 0; jj < 2; jj++)
#pragma unroll
      for (int m = 0; m < 2; m++)
#pragma unroll
        for (int l = 0; l < 2; l++) cfmac(Gq[2 * jj + m], Jr[l], W[jj * 4 + l * 2 + m]);
  }
  // Station sums without atomics: every thread parks its 4 + 8 partial values in shared memory (the
  // ring is free now), then thread i = 8*s + comp gathers what the CTA's baselines contribute to
  // component comp of station s, as the q station of (p, s) for the p of this CTA and as the p
  // station of (s, q).  (Shared-memory fp64 atomics for this cost more than the whole pass.)
  double *gq = reinterpret_cast<double *>(ring);  // [512][8]
  double *gp = gq + 512 * 8;                       // [512][4]
#pragma unroll
  for (int c = 0; c < 4; c++) {
    gq[tid * 8 + 2 * c] = Gq[c].x;
    gq[tid * 8 + 2 * c + 1] = Gq[c].y;
  }
  gp[tid * 4 + 0] = Gp[0].x;
  gp[tid * 4 + 1] = Gp[0].y;
  gp[tid * 4 + 2] = Gp[1].x;
  gp[tid * 4 + 3] = Gp[1].y;
  __syncthreads();
  const int pmin = a.blpq[b0].x, pmax = a.blpq[b0 + nvalid - 1].x;
  for (int i = tid; i < 8 * a.N; i += 512) {
    const int sidx = i >> 3, comp = i & 7;
    double tot = 0.0;
    // as station q of baselines (pp, sidx)
    for (int pp = pmin; pp <= pmax && pp < sidx; pp++) {
      const long long bb = baseline_index(pp, sidx, a.N) - b0;
      if (bb >= 0 && bb < nvalid) tot += gq[bb * 8 + comp] + gq[(256 + bb) * 8 + comp];
    }
    // as station p of baselines (sidx, qq): components 4h..4h+3 come from half h
    if (sidx >= pmin && sidx <= pmax) {
      const int hh = comp >> 2, cc = comp & 3;
      long long bb = baseline_index(sidx, sidx + 1, a.N) - b0;
      long long be = bb + (a.N - 1 - sidx);
      if (bb < 0) bb = 0;
      if (be > nvalid) be = nvalid;
      for (; bb < be; bb++) tot += gp[(hh * 256 + bb) * 4 + cc];
    }
    acc[i] = tot;
  }
  // Station sums of this CTA go out with plain stores; the LAST time slice of a baseline group to
  // arrive adds the group's total to J^T e.  (One global atomic per entry and CTA instead: ~140 adds
  // queue up on each of the 8N addresses and cost more than the pass itself.)
  {
    __shared__ bool last_of_group;
    const int n8 = 8 * a.N;
    double *grp = a.jte_part + (size_t)blockIdx.x * gridDim.y * n8;
    double *mine = grp + (size_t)blockIdx.y * n8;
    for (int i = tid; i < n8; i += 512) mine[i] = acc[i];
    __threadfence();
    __syncthreads();
    if (tid == 0) last_of_group = (atomicAdd(a.gcounter + blockIdx.x, 1u) == gridDim.y - 1);
    __syncthreads();
    if (last_of_group) {
      __threadfence();
      for (int i = tid; i < n8; i += 512) {
        double sacc = 0.0;
        for (unsigned c = 0; c < gridDim.y; c++) sacc += __ldcg(grp + (size_t)c * n8 + i);
        if (sacc != 0.0) atomicAdd(a.jte + i, sacc);
      }
      if (tid == 0) a.gcounter[blockIdx.x] = 0;  // re-arm
    }
  }
  grid_reduce_sum(cost, a.partials, a.cost, a.counter);
}

// ------------------------------------------------------------------------------------------------
// time-summed Gram tensor of the coherencies of each baseline:
//   T[b][16] = Hermitian 4x4  sum_t conj(c) c^T,  c = (C00,C01,C10,C11), unflagged rows only
// stored as: 4 real diagonals, then the 6 complex upper off-diagonals (01,02,03,12,13,23)
// grid (ntile, nclusters); the time range of one hybrid chunk / OS subset per launch
// ------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(TILE_THREADS)
k_coh_gram(GramArgs a) {
  const TileDesc td = a.tiles[blockIdx.x];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int p = td.pb * TILE_P + w;
  const int q = td.qb * TILE_Q + lane;
  if (!((q > p) && (q < a.N))) return;
  const long long b = baseline_index(p, q, a.N);
  const double2 *ck = a.coh + (long long)(a.k0 + blockIdx.y) * 4 * a.R;
  double d[4] = {0.0, 0.0, 0.0, 0.0};
  double2 o[6];
#pragma unroll
  for (int z = 0; z < 6; z++) o[z] = make_double2(0.0, 0.0);
#pragma unroll 4
  for (int t = a.t_begin; t < a.t_end; t += a.t_step) {
    const long long row = (long long)t * a.Nbase + b;
    double2 C[4];
#pragma unroll
    for (int c = 0; c < 4; c++) C[c] = ld_stream(ck + (long long)c * a.R + row);
    if (a.flag[row] == 0) {
#pragma unroll
      for (int c = 0; c < 4; c++) {
        d[c] = fma(C[c].x, C[c].x, d[c]);
        d[c] = fma(C[c].y, C[c].y, d[c]);
      }
      cfmacl(o[0], C[0], C[1]);
      cfmacl(o[1], C[0], C[2]);
      cfmacl(o[2], C[0], C[3]);
      cfmacl(o[3], C[1], C[2]);
      cfmacl(o[4], C[1], C[3]);
      cfmacl(o[5], C[2], C[3]);
    }
  }
  double2 *Tb = reinterpret_cast<double2 *>(a.T + ((long long)blockIdx.y * a.Nbase + b) * 16);
  Tb[0] = make_double2(d[0], d[1]);
  Tb[1] = make_double2(d[2], d[3]);
#pragma unroll
  for (int z = 0; z < 6; z++) Tb[2 + z] = o[z];
}

// ------------------------------------------------------------------------------------------------
// host-side launchers
// ------------------------------------------------------------------------------------------------
template <int TB, int NST>
static void launch_grad_tma_split(const GradArgs *a, int ntile, cudaStream_t st) {
  const size_t smem = sizeof(double) * 2 * TILE_P * 8 * TILE_Q +
                      (size_t)TILE_P * NST * TB * 4 * 32 * sizeof(double2) + TILE_P * NST * 8;
  static bool configured = false;
  if (!configured) {
    DB_CHECK(cudaFuncSetAttribute(k_grad_tma_split<TB, NST>,
                                  cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = true;
  }
  dim3 grid(ntile, (a->tilesz + TB - 1) / TB);
  k_grad_tma_split<TB, NST><<<grid, 2 * TILE_THREADS, smem, st>>>(*a);
}
template <int TB, int NST>
static void launch_grad_tma(const GradArgs *a, int ntile, cudaStream_t st) {
  const size_t smem = sizeof(double) * TILE_P * 8 * TILE_Q +
                      (size_t)TILE_P * NST * TB * 4 * 32 * sizeof(double2) + TILE_P * NST * 8;
  static bool configured = false;
  if (!configured) {
    DB_CHECK(cudaFuncSetAttribute(k_grad_tma<TB, NST>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)smem));
    configured = true;
  }
  dim3 grid(ntile, (a->tilesz + TB - 1) / TB);
  k_grad_tma<TB, NST><<<grid, TILE_THREADS, smem, st>>>(*a);
}
extern "C" {

void db_launch_coh_to_planar(const double2 *src, double2 *dst, long long r0, int nr, int M,
                             long long R, cudaStream_t st) {
  dim3 block(32, XP_ROWS), grid((M + 31) / 32, (nr + XP_ROWS - 1) / XP_ROWS);
  k_coh_to_planar<<<grid, block, 0, st>>>(src, dst, r0, nr, M, R);
}
void db_launch_coh_from_planar(const double2 *src, double2 *dst, long long r0, int nr, int M,
                               long long R, cudaStream_t st) {
  dim3 block(32, XP_ROWS), grid((M + 31) / 32, (nr + XP_ROWS - 1) / XP_ROWS);
  k_coh_from_planar<<<grid, block, 0, st>>>(src, dst, r0, nr, M, R);
}
void db_launch_vis_to_planar(const double2 *src, double2 *dst, long long R, cudaStream_t st) {
  long long n = 4 * R;
  k_vis_to_planar<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(src, dst, R);
}
void db_launch_vis_from_planar(const double2 *src, double2 *dst, long long R, cudaStream_t st) {
  long long n = 4 * R;
  k_vis_from_planar<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(src, dst, R);
}

#define PREDICT_TB 4
int db_predict_nblocks(int ntile, int tilesz) { return ntile * ((tilesz + PREDICT_TB - 1) / PREDICT_TB); }
void db_launch_predict_full(const PredictArgs *a, int ntile, cudaStream_t st) {
  dim3 grid(ntile, (a->tilesz + PREDICT_TB - 1) / PREDICT_TB);
  k_predict_full<PREDICT_TB><<<grid, TILE_THREADS, 0, st>>>(*a);
}
void db_launch_grad_full(const GradArgs *a, int ntile, cudaStream_t st) {
  dim3 grid(ntile, (a->tilesz + PREDICT_TB - 1) / PREDICT_TB);
  k_grad_full<PREDICT_TB><<<grid, TILE_THREADS, 0, st>>>(*a);
}
void db_launch_grad_tma(const GradArgs *a, int ntile, cudaStream_t st) {
  static int cfg = -1;
  static const bool unsplit = getenv("DIRAC_B200_CP_UNSPLIT") != nullptr;
  if (!unsplit) {
    static int scfg = -1;
    if (scfg < 0) {
      const char *e = getenv("DIRAC_B200_GRADS_CFG");
      scfg = e ? atoi(e) : 0;
    }
    switch (scfg) {
      case 1: launch_grad_tma_split<2, 2>(a, ntile, st); return;
      case 2: launch_grad_tma_split<2, 3>(a, ntile, st); return;
      case 3: launch_grad_tma_split<4, 3>(a, ntile, st); return;
      case 4: launch_grad_tma_split<8, 2>(a, ntile, st); return;
      case 5: launch_grad_tma_split<1, 4>(a, ntile, st); return;
      default: launch_grad_tma_split<4, 2>(a, ntile, st); return;
    }
  }
  if (cfg < 0) {
    const char *e = getenv("DIRAC_B200_GRAD_CFG");
    cfg = e ? atoi(e) : 0;
  }
  switch (cfg) {
    case 1: launch_grad_tma<2, 3>(a, ntile, st); return;
    case 2: launch_grad_tma<2, 2>(a, ntile, st); return;
    case 3: launch_grad_tma<4, 3>(a, ntile, st); return;
    case 4: launch_grad_tma<3, 2>(a, ntile, st); return;
    default: launch_grad_tma<4, 2>(a, ntile, st); return;
  }
}
int db_cluster_pass_nblocks(int ntile, int nt, int tslice) { return ntile * ((nt + tslice - 1) / tslice); }
void db_launch_cluster_pass(const ClusterPassArgs *a, int ntile, cudaStream_t st) {
  int nt = a->t_end - a->t_begin;
  dim3 grid(ntile, (nt + a->tslice - 1) / a->tslice);
  static const bool no_tma_any = getenv("DIRAC_B200_NO_TMA") != nullptr;
  const bool lin_ok = (size_t)5 * 8 * 256 * sizeof(double2) + sizeof(double) * ((8 * a->N + 1) & ~1) + 40 <=
                          (size_t)200 * 1024 && (a->Nbase + 255) / 256 <= 1024;
  if (!(a->jte != nullptr && a->mode <= 1) && !a->wt && !a->in2 && !no_tma_any && lin_ok &&
      !getenv("DIRAC_B200_ADDSUB_TILE")) {
    // ADD / SUB / cost-only pass in the linear mapping: the same CTA-wide TMA ring as the gradient
    // pass, without the station sums
    constexpr int NST = 5;
    const int nbg = (a->Nbase + 255) / 256;
    int nsl = (db_sm_count() + nbg - 1) / nbg;
    if (nsl > nt) nsl = nt;
    ClusterPassArgs b = *a;
    b.tslice = (nt + nsl - 1) / nsl;
    const int forced = db_opt(DB_OPT_CP_ROWS);
    if (forced > 0) b.tslice = forced;
    if (b.tslice > nt) b.tslice = nt;
    if (b.tslice > 32) b.tslice = 32;
    const size_t smem = (size_t)NST * 8 * 256 * sizeof(double2) + sizeof(double) * ((8 * a->N + 1) & ~1) + NST * 8;
    static bool configured = false;
    if (!configured) {
      DB_CHECK(cudaFuncSetAttribute(k_cluster_pass_lin<NST, false>,
                                    cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
      configured = true;
    }
    dim3 glin(nbg, (nt + b.tslice - 1) / b.tslice);
    k_cluster_pass_lin<NST, false><<<glin, 512, smem, st>>>(b);
    return;
  }
  if (a->jte != nullptr && a->mode == 4) {
    k_cluster_pass_split<<<grid, 2 * TILE_THREADS, 0, st>>>(*a);
    return;
  }
  if (a->jte != nullptr && a->mode <= 1) {
    static const bool unsplit = getenv("DIRAC_B200_CP_UNSPLIT") != nullptr;
    // default: linear mapping with CTA-wide TMA stages; robust weights and DIRAC_B200_NO_TMA take the
    // register-staged tile kernel
    static const bool no_tma = getenv("DIRAC_B200_NO_TMA") != nullptr;
    // the linear-mapped kernel keeps 8N station sums in shared memory next to its ring and one
    // arrival counter per 256-baseline group: arrays too large for either take the tile kernel
    const bool lin_fits = (size_t)5 * 8 * 256 * sizeof(double2) + sizeof(double) * ((8 * a->N + 1) & ~1) + 40 <=
                              (size_t)200 * 1024 && (a->Nbase + 255) / 256 <= 1024;
    if (unsplit) {
      k_cluster_pass<true><<<grid, TILE_THREADS, 0, st>>>(*a);
    } else if (a->wt || no_tma || !lin_fits) {
      k_cluster_pass_split<<<grid, 2 * TILE_THREADS, 0, st>>>(*a);
    } else {
      // linear mapping: 256 baselines per CTA, time sliced to about one CTA per SM (<= 32 rows)
      constexpr int NST = 5;
      const int nbg = (a->Nbase + 255) / 256;
      int nsl = (db_sm_count() + nbg - 1) / nbg;
      if (nsl > nt) nsl = nt;
      ClusterPassArgs b = *a;
      b.tslice = (nt + nsl - 1) / nsl;
      // test hook: rows per CTA forced (drives the multi-row ring on small problems), as long as
      // the slices still fit the per-CTA partial buffer
      const int forced = db_opt(DB_OPT_CP_ROWS);
      if (forced > 0 && (nt + forced - 1) / forced <= db_cp_max_slices(a->Nbase, nt)) b.tslice = forced;
      if (b.tslice > nt) b.tslice = nt;
      if (b.tslice > 32) b.tslice = 32;
      const size_t smem = (size_t)NST * 8 * 256 * sizeof(double2) +
                          sizeof(double) * ((8 * a->N + 1) & ~1) + NST * 8;
      static bool configured = false;
      if (!configured) {
        DB_CHECK(cudaFuncSetAttribute(k_cluster_pass_lin<NST, true>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        configured = true;
      }
      dim3 glin(nbg, (nt + b.tslice - 1) / b.tslice);
      k_cluster_pass_lin<NST, true><<<glin, 512, smem, st>>>(b);
    }
  } else {
    k_cluster_pass<false><<<grid, TILE_THREADS, 0, st>>>(*a);
  }
}
void db_launch_coh_gram(const GramArgs *a, int ntile, int nk, cudaStream_t st) {
  dim3 grid(ntile, nk);
  k_coh_gram<<<grid, TILE_THREADS, 0, st>>>(*a);
}

}  // extern "C"
