// Channel-batched Student's-t cost / residual pass of the minibatch LBFGS: k_stream_all<0> (kernels_tma.cu)
// over every channel of a band in one launch (robust_cost_func_multifreq, robust_batchmode_lbfgs.c:
// 1096-1139, summed over the channels in one scalar).
//
// Layout: the band's coherencies are [chan][M][4][R] and its data and output [chan][4][R], the planar
// layout of the single-channel passes, one channel after the other.  The grid is the single-channel
// grid (32 baselines x TB timeslots per CTA) times the channels: CTA i works on channel i / nitem,
// whose base pointers are shifted by its stride, so the hybrid chunk of a row comes from its row within
// the channel.  The deterministic grid reduction covers every CTA of every channel.
//
// A kernel of its own rather than a flag of k_stream_all: the existing passes keep their code as it is.
#include "internal.cuh"
#include "tma.cuh"

template <int TB, int NST, int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
k_stream_band(StreamAllArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  constexpr int STAGE_ELEMS = TB * 4 * 32;  // double2 per stage
  constexpr size_t RING_BYTES = (size_t)WARPS * NST * STAGE_ELEMS * 16;
  constexpr size_t COMB_BYTES = (size_t)(WARPS - 1) * STAGE_ELEMS * 16;
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

  const int nbg = (a.Nbase + 31) >> 5;  // baseline groups
  const int nitem = nbg * ((a.tilesz + TB - 1) / TB);
  const long long ch = blockIdx.x / nitem;
  const int item = (int)(blockIdx.x - ch * nitem);
  const double2 *coh = a.coh + ch * a.M * 4 * a.R;
  const double2 *x = a.x + ch * 4 * a.R;
  double2 *out = a.out ? a.out + ch * 4 * a.R : nullptr;
  const int bg = item % nbg, tb = item / nbg;
  const int b0 = bg << 5;
  const int nvalid = min(32, a.Nbase - b0);
  const int t0 = tb * TB;
  const int nrows = min(TB, a.tilesz - t0);
  const bool valid = lane < nvalid;
  const int b = b0 + (valid ? lane : 0);
  const short2 pq = a.blpq[b];
  const int p = pq.x, q = pq.y;
  const unsigned row_bytes = (unsigned)nvalid * 16u;
  const int nk = (a.M - w + WARPS - 1) / WARPS;  // clusters of this warp: w, w+WARPS, ...

  auto issue = [&](int j, int s) {
    const int k = w + j * WARPS;
    mbar_expect_tx(&my_bar[s], (unsigned)nrows * 4u * row_bytes);
    const double2 *ck = coh + (long long)k * 4 * a.R + (long long)t0 * a.Nbase + b0;
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

  double2 V[TB][4];
#pragma unroll
  for (int i = 0; i < TB; i++)
#pragma unroll
    for (int c = 0; c < 4; c++) V[i][c] = make_double2(0.0, 0.0);

  for (int j = 0; j < nk; j++) {
    const int s = j % NST;
    if (lane == 0 && j + NST - 1 < nk) issue(j + NST - 1, (j + NST - 1) % NST);
    const int k = w + j * WARPS;
    const ClusterDesc cd = a.clus[k];
    double2 Jp[4], Jq[4];
    {
      const long long row = (long long)t0 * a.Nbase + b;
      const int off = a.chunk_poff[cd.chunk0 + row_chunk(row, a.R, cd.nchunk)];
      load_jones(a.pp + off, p, Jp);
      load_jones(a.pp + off, q, Jq);
    }
    mbar_wait(&my_bar[s], (unsigned)((j / NST) & 1));
    if (valid) {
      const double2 *st = my_stage + (size_t)s * STAGE_ELEMS;
#pragma unroll
      for (int i = 0; i < TB; i++) {
        if (i < nrows) {
          if (cd.nchunk > 1 && i > 0) {
            // hybrid cluster: the chunk (hence the Jones block) may change from row to row
            const long long row = (long long)(t0 + i) * a.Nbase + b;
            const int off = a.chunk_poff[cd.chunk0 + row_chunk(row, a.R, cd.nchunk)];
            load_jones(a.pp + off, p, Jp);
            load_jones(a.pp + off, q, Jq);
          }
          double2 C[4];
#pragma unroll
          for (int c = 0; c < 4; c++) C[c] = lds_v2(st + (i * 4 + c) * 32 + lane);
          double2 A[4];
          mat_ab(Jp, C, A);
          mat_abh_acc(A, Jq, V[i]);
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
      for (int c = 0; c < 4; c++) comb[((size_t)(w - 1) * TB * 4 + (i * 4 + c)) * 32 + lane] = V[i][c];
  }
  __syncthreads();
  double cost = 0.0;
  if (w == 0 && valid) {
    for (int ww = 1; ww < WARPS; ww++)
#pragma unroll
      for (int i = 0; i < TB; i++)
#pragma unroll
        for (int c = 0; c < 4; c++)
          V[i][c] = cadd(V[i][c], comb[((size_t)(ww - 1) * TB * 4 + (i * 4 + c)) * 32 + lane]);
#pragma unroll
    for (int i = 0; i < TB; i++) {
      if (i < nrows) {
        const long long row = (long long)(t0 + i) * a.Nbase + b;
        const bool fl = a.flag[row] != 0;
#pragma unroll
        for (int c = 0; c < 4; c++) {
          const long long ix = (long long)c * a.R + row;
          const double2 m = fl ? make_double2(0.0, 0.0) : V[i][c];
          const double2 e = csub(ld_stream(x + ix), m);
          if (a.out_mode == 1) st_stream(out + ix, e);
          if (a.cost_mode == 2) {
            cost += log(1.0 + e.x * e.x * a.inv_nu);
            cost += log(1.0 + e.y * e.y * a.inv_nu);
          }
        }
      }
    }
  }
  if (a.cost_mode) {
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

extern "C" {
int db_band_nblocks(int Nbase, int tilesz, int nchan) {
  constexpr int TB = 2;
  return ((Nbase + 31) / 32) * ((tilesz + TB - 1) / TB) * nchan;
}
void db_launch_band_tma(const StreamAllArgs *a, int nchan, cudaStream_t st) {
  constexpr int TB = 2, NST = 2, WARPS = 3;
  const size_t ring = (size_t)WARPS * NST * TB * 4 * 32 * 16;
  const size_t comb = (size_t)(WARPS - 1) * TB * 4 * 32 * 16;
  const size_t smem = (ring > comb ? ring : comb) + WARPS * NST * 8;
  static bool configured = false;
  if (!configured) {
    DB_CHECK(cudaFuncSetAttribute(k_stream_band<TB, NST, WARPS>,
                                  cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = true;
  }
  k_stream_band<TB, NST, WARPS>
      <<<(unsigned)db_band_nblocks(a->Nbase, a->tilesz, nchan), WARPS * 32, smem, st>>>(*a);
}
}
