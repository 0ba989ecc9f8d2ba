// TMA-pipelined all-cluster passes (Blackwell/Hopper bulk-copy engine feeding a per-warp ring of
// shared-memory stages):
//   MODE 0  model over all clusters, residual / cost      (predict_threadfn_withgain_full,
//           lmfit.c:611-688, plus cost_func / robust_cost_func, robust_lbfgs.c:674-726)
//   MODE 1  line model V0,V1,V2 -> E0,E1,E2 of the LBFGS line search (kernels_line.cu), and on one
//           GPU the per-CTA sums of the Gaussian cost's quartic along the line
//   MODE 2  MODE 0 over a row window [w_lo, w_hi) of the launched timeslots: the cost and residual
//           of the minibatch LBFGS (robust_cost_func_batch, robust_batchmode_lbfgs.c:822-846); rows
//           of the first and last timeslot outside the window are neither written nor summed
//
// Why a ring: a pass that loads the coherencies into registers holds them there until they are
// used, so registers bound it to few resident warps, and each warp waits out the full DRAM latency
// between its dependent load and compute phases.  Here one elected lane per warp issues 1-D bulk
// copies (cp.async.bulk, 16 B x valid lanes = up to 512 B each) for the coherencies of the NEXT
// cluster steps into the warp's private ring of NST shared-memory stages while the warp multiplies
// the current one; no register is held by data in flight, several KB per warp are always in
// flight, completion is tracked by one mbarrier per stage (complete_tx).  The warp is its own
// producer and consumer, so no block-wide barrier appears in the main loop.
//
// Mapping: linear over the canonical baselines (no station reduction is needed by these passes):
// a warp owns 32 consecutive baselines x TB consecutive timeslots and walks all clusters; lane ->
// baseline, so every copy is contiguous and all 32 lanes work (the p x q tile mapping of the
// reducing kernels leaves 38 % of the lanes idle at 62 stations).
#include "internal.cuh"
#include "tma.cuh"

template <int MODE, int TB, int NST, int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
k_stream_all(StreamAllArgs a) {
  // One CTA = one item (32 consecutive baselines x TB timeslots); its WARPS warps split the clusters
  // (k = w, w+WARPS, ...) so that the grid has many small CTAs (little tail on 132 SMs) and every
  // warp runs its own producer/consumer ring.  The partial models are combined through shared
  // memory in warp order (deterministic), warp 0 finishes the rows.
  extern __shared__ __align__(128) unsigned char smem_raw[];
  constexpr int STAGE_ELEMS = TB * 4 * 32;                       // double2 per stage
  constexpr int NACC = (MODE == 1) ? 3 : 1;                       // V0 | V0,V1,V2
  constexpr size_t RING_BYTES = (size_t)WARPS * NST * STAGE_ELEMS * 16;
  constexpr size_t COMB_BYTES = (size_t)(WARPS - 1) * NACC * STAGE_ELEMS * 16;
  constexpr size_t DATA_BYTES = RING_BYTES > COMB_BYTES ? RING_BYTES : COMB_BYTES;
  double2 *ring = reinterpret_cast<double2 *>(smem_raw);
  unsigned long long *bars = reinterpret_cast<unsigned long long *>(smem_raw + DATA_BYTES);
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double2 *my_stage = ring + (size_t)w * NST * STAGE_ELEMS;
  unsigned long long *my_bar = bars + w * NST;
  if (lane == 0) {
#pragma unroll
    for (int s = 0; s < NST; s++) mbar_init(&my_bar[s], 1);
    mbar_fence_init();
  }
  __syncwarp();

  const int nbg = (a.Nbase + 31) >> 5;                 // baseline groups
  const int bg = (int)(blockIdx.x % nbg), tb = (int)(blockIdx.x / nbg);
  const int b0 = bg << 5;
  const int nvalid = min(32, a.Nbase - b0);
  const int t0 = tb * TB;
  const int nrows = min(TB, a.tilesz - t0);
  const bool valid = lane < nvalid;
  const int b = b0 + (valid ? lane : 0);
  const short2 pq = a.blpq[b];
  const int p = pq.x, q = pq.y;
  const unsigned row_bytes = (unsigned)nvalid * 16u;
  const int nk = (a.M - w + WARPS - 1) / WARPS;        // clusters of this warp: w, w+WARPS, ...

  auto issue = [&](int j, int s) {
    // stage s <- rows of cluster (w + j*WARPS): nrows x 4 contiguous runs of nvalid x 16 B
    const int k = w + j * WARPS;
    mbar_expect_tx(&my_bar[s], (unsigned)nrows * 4u * row_bytes);
    const double2 *ck = a.coh + (long long)k * 4 * a.R + (long long)t0 * a.Nbase + b0;
    double2 *dst = my_stage + (size_t)s * STAGE_ELEMS;
    for (int i = 0; i < nrows; i++)
#pragma unroll
      for (int c = 0; c < 4; c++)
        bulk_g2s(dst + (i * 4 + c) * 32, ck + (long long)c * a.R + (long long)i * a.Nbase,
                 row_bytes, &my_bar[s]);
  };
  if (lane == 0) {
#pragma unroll
    for (int s = 0; s < NST - 1; s++)
      if (s < nk) issue(s, s);
  }

  double2 V0[TB][4], V1[TB][4], V2[TB][4];
#pragma unroll
  for (int i = 0; i < TB; i++)
#pragma unroll
    for (int c = 0; c < 4; c++) V0[i][c] = V1[i][c] = V2[i][c] = make_double2(0.0, 0.0);

  double2 Jp[4], Jq[4], Dp[4], Dq[4];
  auto fetch_jones = [&](int j, double2 *jp, double2 *jq, double2 *dp, double2 *dq) {
    const int k = w + j * WARPS;
    const ClusterDesc cd = a.clus[k];
    const long long row = a.row0 + (long long)t0 * a.Nbase + b;
    const int off = a.chunk_poff[cd.chunk0 + row_chunk(row, a.R, cd.nchunk)];
    load_jones(a.pp + off, p, jp);
    load_jones(a.pp + off, q, jq);
    if (MODE == 1) {
      load_jones(a.pk + off, p, dp);
      load_jones(a.pk + off, q, dq);
    }
  };

  for (int j = 0; j < nk; j++) {
    const int s = j % NST;
    if (lane == 0 && j + NST - 1 < nk) issue(j + NST - 1, (j + NST - 1) % NST);
    fetch_jones(j, Jp, Jq, Dp, Dq);
    const int k = w + j * WARPS;
    const ClusterDesc cd = a.clus[k];
    mbar_wait(&my_bar[s], (unsigned)((j / NST) & 1));
    if (valid) {
      const double2 *st = my_stage + (size_t)s * STAGE_ELEMS;
#pragma unroll
      for (int i = 0; i < TB; i++) {
        if (i < nrows) {
          if (cd.nchunk > 1 && i > 0) {
            // hybrid cluster: the chunk (hence the Jones block) may change from row to row
            const long long row = a.row0 + (long long)(t0 + i) * a.Nbase + b;
            const long long row0 = a.row0 + (long long)t0 * a.Nbase + b;
            const int px = row_chunk(row, a.R, cd.nchunk);
            if (px != row_chunk(row0, a.R, cd.nchunk) || i > 1) {
              const int off = a.chunk_poff[cd.chunk0 + px];
              load_jones(a.pp + off, p, Jp);
              load_jones(a.pp + off, q, Jq);
              if (MODE == 1) {
                load_jones(a.pk + off, p, Dp);
                load_jones(a.pk + off, q, Dq);
              }
            }
          }
          double2 C[4];
#pragma unroll
          for (int c = 0; c < 4; c++) C[c] = lds_v2(st + (i * 4 + c) * 32 + lane);
          double2 A[4];
          mat_ab(Jp, C, A);
          mat_abh_acc(A, Jq, V0[i]);
          if (MODE == 1) {
            double2 B[4];
            mat_ab(Dp, C, B);
            mat_abh_acc(B, Jq, V1[i]);
            mat_abh_acc(A, Dq, V1[i]);
            mat_abh_acc(B, Dq, V2[i]);
          }
        }
      }
    }
    __syncwarp();  // every lane is done with stage s before lane 0 refills it (next iteration)
  }

  // combine the partial models of warps 1..WARPS-1 into warp 0 (ring memory is free now)
  __syncthreads();
  double2 *comb = ring;
  if (w > 0) {
#pragma unroll
    for (int i = 0; i < TB; i++)
#pragma unroll
      for (int c = 0; c < 4; c++) {
        double2 *dst = comb + ((size_t)(w - 1) * NACC * TB * 4 + (i * 4 + c)) * 32 + lane;
        dst[0] = V0[i][c];
        if (MODE == 1) {
          dst[(size_t)TB * 4 * 32] = V1[i][c];
          dst[(size_t)2 * TB * 4 * 32] = V2[i][c];
        }
      }
  }
  __syncthreads();
  double cost = 0.0;
  // MODE 1 on one GPU: the Gaussian cost along the line, sum |E0 - a E1 - a^2 E2|^2, is a quartic
  // whose five sums (k_line_poly's) are taken here from the E0, E1, E2 this warp stores
  double cq[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  if (w == 0 && valid) {
    for (int ww = 1; ww < WARPS; ww++)
#pragma unroll
      for (int i = 0; i < TB; i++)
#pragma unroll
        for (int c = 0; c < 4; c++) {
          const double2 *src = comb + ((size_t)(ww - 1) * NACC * TB * 4 + (i * 4 + c)) * 32 + lane;
          V0[i][c] = cadd(V0[i][c], src[0]);
          if (MODE == 1) {
            V1[i][c] = cadd(V1[i][c], src[(size_t)TB * 4 * 32]);
            V2[i][c] = cadd(V2[i][c], src[(size_t)2 * TB * 4 * 32]);
          }
        }
#pragma unroll
    for (int i = 0; i < TB; i++) {
      if (i < nrows) {
        const long long row = (long long)(t0 + i) * a.Nbase + b;
        if (MODE == 2 && (row < a.w_lo || row >= a.w_hi)) continue;
        const bool fl = a.flag[row] != 0;
#pragma unroll
        for (int c = 0; c < 4; c++) {
          const long long ix = (long long)c * a.R + row;
          const double2 z = make_double2(0.0, 0.0);
          const double2 m = fl ? z : V0[i][c];
          if (MODE != 1) {
            double2 xv = z;
            if (a.out_mode == 1 || a.cost_mode) xv = ld_stream(a.x + ix);
            const double2 e = csub(xv, m);
            if (a.out_mode == 1) st_stream(a.out + ix, e);
            if (a.out_mode == 2) st_stream(a.out + ix, m);
            if (a.cost_mode == 1) {
              cost = fma(e.x, e.x, cost);
              cost = fma(e.y, e.y, cost);
            } else if (a.cost_mode == 2) {
              cost += log(1.0 + e.x * e.x * a.inv_nu);
              cost += log(1.0 + e.y * e.y * a.inv_nu);
            }
          } else {
            const double2 xv = ld_stream(a.x + ix);
            const double2 e0 = a.partial ? m : csub(xv, m);
            const double2 e1 = fl ? z : V1[i][c], e2 = fl ? z : V2[i][c];
            st_stream(a.E0 + ix, e0);
            st_stream(a.E1 + ix, e1);
            st_stream(a.E2 + ix, e2);
            if (a.poly_part) {
              cq[0] = fma(e0.x, e0.x, fma(e0.y, e0.y, cq[0]));
              cq[1] = fma(e0.x, e1.x, fma(e0.y, e1.y, cq[1]));
              cq[2] = fma(e1.x, e1.x, fma(e1.y, e1.y, cq[2]));
              cq[2] = fma(-2.0 * e0.x, e2.x, fma(-2.0 * e0.y, e2.y, cq[2]));
              cq[3] = fma(e1.x, e2.x, fma(e1.y, e2.y, cq[3]));
              cq[4] = fma(e2.x, e2.x, fma(e2.y, e2.y, cq[4]));
            }
          }
        }
      }
    }
  }
  if (MODE == 1 && a.poly_part && w == 0) {
    // per-CTA sums in lane order; k_line_poly_finish adds the CTAs in index order (deterministic)
#pragma unroll
    for (int j = 0; j < 5; j++) {
      const double v = warp_sum(cq[j]);
      if (lane == 0) a.poly_part[(size_t)j * gridDim.x + blockIdx.x] = v;
    }
  }
  if (MODE != 1 && a.cost_mode) {
    // deterministic grid reduction (per-CTA partial from warp 0, last CTA sums in index order)
    __shared__ bool is_last;
    cost = warp_sum(cost);
    if (threadIdx.x == 0) {
      a.partials[blockIdx.x] = cost;
      __threadfence();
      is_last = (atomicAdd(a.counter, 1u) == gridDim.x - 1);
    }
    __syncthreads();
    if (is_last && w == 0) {
      double s = 0.0;
      for (unsigned int i = lane; i < gridDim.x; i += 32) s += ((volatile double *)a.partials)[i];
      s = warp_sum(s);
      if (lane == 0) {
        *a.cost = s;
        *a.counter = 0;
      }
    }
  }
}

// ---- launchers ---------------------------------------------------------------------------------------
static int g_line_shape[3] = {-1, -1, -1};  // shape of the last line-model launch (tests)

template <int MODE, int TB, int NST, int WARPS>
static unsigned launch_cfg(const StreamAllArgs *a, cudaStream_t st) {
  if (MODE == 1) {
    g_line_shape[0] = TB;
    g_line_shape[1] = NST;
    g_line_shape[2] = WARPS;
  }
  const int nbg = (a->Nbase + 31) / 32, ntb = (a->tilesz + TB - 1) / TB;
  const unsigned grid = (unsigned)((long long)nbg * ntb);
  constexpr int NACC = (MODE == 1) ? 3 : 1;
  const size_t ring = (size_t)WARPS * NST * TB * 4 * 32 * 16;
  const size_t comb = (size_t)(WARPS - 1) * NACC * TB * 4 * 32 * 16;
  const size_t smem = (ring > comb ? ring : comb) + WARPS * NST * 8;
  static bool configured = false;
  if (!configured) {
    DB_CHECK(cudaFuncSetAttribute(k_stream_all<MODE, TB, NST, WARPS>,
                                  cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = true;
  }
  k_stream_all<MODE, TB, NST, WARPS><<<grid, WARPS * 32, smem, st>>>(*a);
  return grid;
}

extern "C" {
int db_stream_all_nblocks(int Nbase, int tilesz) {
  const int nbg = (Nbase + 31) / 32;
  // upper bound over every compiled shape (one CTA per item, TB >= 1)
  return (int)((long long)nbg * tilesz);
}
void db_launch_predict_tma(const StreamAllArgs *a, cudaStream_t st) {
  launch_cfg<0, 2, 2, 3>(a, st);
}
// the caller shifts the pointers to the first timeslot of the window and sets tilesz to the
// timeslots it touches; the grid, and the cost's grid reduction, cover those timeslots only
void db_launch_cost_window_tma(const StreamAllArgs *a, cudaStream_t st) {
  launch_cfg<2, 2, 2, 3>(a, st);
}
unsigned db_launch_line_setup_tma(const StreamAllArgs *a, cudaStream_t st) {
  // one row per item keeps the three accumulated polynomials of the line model at 24 registers
  // pairs (222 -> ~170 registers: 7.5 % -> 12 % resident warps, ncu r02).  Splitting the clusters
  // of an item over warps only pays while the grid is short of warps (62 stations: 7200 items);
  // a large array has plenty (512 stations: 490 k items) and skips the cross-warp combine.
  const long long items = (long long)((a->Nbase + 31) / 32) * a->tilesz;
  if (items >= 64ll * db_sm_count()) return launch_cfg<1, 1, 4, 1>(a, st);
  return launch_cfg<1, 1, 2, 3>(a, st);
}
void db_line_setup_shape_reset() { g_line_shape[0] = g_line_shape[1] = g_line_shape[2] = -1; }
void db_line_setup_shape(int *shape) {
  for (int i = 0; i < 3; i++) shape[i] = g_line_shape[i];
}
}
