// Coherency prediction from the sky model on the device.
//
//   k_coherencies        one frequency, every cluster -> resident planar coh[k][4][R]
//                        (replaces precal_threadfn, predict.c:345-497)
//   k_predict_multifreq  sum over clusters per channel with spectral-index fluxes -> x[chan][row][8]
//                        (replaces visibilities_threadfn_multifreq, residual.c:1067-1248)
//
// One thread per row (u,v,w coalesced in, 16-byte planar stores out).  The sources of a direction
// are staged in shared memory by a 1-D TMA bulk copy (cp.async.bulk + mbarrier complete_tx),
// double buffered so the copy of direction k+1 overlaps the trigonometry of direction k.  This
// kernel is SFU/FP64-ALU bound (three sin/cos per source-row), not HBM bound.
#include "internal.cuh"
#include "coh.h"
#include "tma.cuh"

#include "coh_math.cuh"

#define COH_THREADS 128

// MODE 0: coherencies per cluster at freq[0] -> planar coh ; MODE 1: multifreq sum -> xout ;
// MODE 2: xout += sum_k clus_coef[k] J_p C_k J_q^H per channel with the solved Jones, then the
//         optional correction x <- Jinv_p x Jinv_q^H by one cluster's inverse Jones.  The residual
//         passes -1 for clusters with id >= 0 (residual_threadfn_multifreq, residual.c:681-938), the
//         simulation +1 / -1 for the clusters not ignored (predictwithgain_threadfn_multifreq,
//         residual.c:1344-1618); 0 skips a cluster.
template <int MODE>
__global__ void __launch_bounds__(COH_THREADS)
k_sky_predict(CohArgs a) {
  __shared__ __align__(128) DevSource sbuf[2][COH_SEG_MAX];
  __shared__ __align__(8) unsigned long long bar[2];
  const long long r = (long long)blockIdx.x * COH_THREADS + threadIdx.x;
  const bool active = r < a.R;
  if (threadIdx.x == 0) {
    mbar_init(&bar[0], 1);
    mbar_init(&bar[1], 1);
    mbar_fence_init();
  }
  __syncthreads();
  double u = 0.0, v = 0.0, w = 0.0;
  if (active) {
    u = a.u[r];
    v = a.v[r];
    w = a.w[r];
  }
  const int nchan = (MODE == 0) ? 1 : a.Nchan;
  int s1 = 0, s2 = 0, tslot = 0;
  if ((MODE == 2 || a.sta1) && active) {
    s1 = a.sta1[r];
    s2 = a.sta2[r];
  }
  if (a.beam_af || a.beam_E) tslot = (int)(r / a.Nbase);
  // prologue: stage segment 0
  if (threadIdx.x == 0 && a.nseg > 0) {
    const CohSegment sg = a.segs[0];
    const unsigned bytes = (unsigned)sg.count * (unsigned)sizeof(DevSource);
    mbar_expect_tx(&bar[0], bytes);
    if (bytes) bulk_g2s(&sbuf[0][0], a.src + sg.first, bytes, &bar[0]);
  }
  for (int cf = 0; cf < nchan; cf++) {
    // (channels re-walk the segment list; the staging pipeline simply continues)
    double2 X[4];
#pragma unroll
    for (int c = 0; c < 4; c++) X[c] = make_double2(0.0, 0.0);
    const double freq = a.freqs[cf];
    double2 C[4];
#pragma unroll
    for (int c = 0; c < 4; c++) C[c] = make_double2(0.0, 0.0);
    for (int sgi = 0; sgi < a.nseg; sgi++) {
      const int it = cf * a.nseg + sgi;  // global staging iteration
      const int b = it & 1;
      // stage the next segment (of this or the next channel) into the other buffer
      if (threadIdx.x == 0) {
        int nxt = sgi + 1;
        bool more = true;
        if (nxt == a.nseg) {
          nxt = 0;
          more = (cf + 1 < nchan);
        }
        if (more) {
          const CohSegment sn = a.segs[nxt];
          const unsigned bytes = (unsigned)sn.count * (unsigned)sizeof(DevSource);
          mbar_expect_tx(&bar[b ^ 1], bytes);
          if (bytes) bulk_g2s(&sbuf[b ^ 1][0], a.src + sn.first, bytes, &bar[b ^ 1]);
        }
      }
      const CohSegment sg = a.segs[sgi];
      mbar_wait(&bar[b], (unsigned)((it >> 1) & 1));
      if (active) {
        for (int s = 0; s < sg.count; s++) {
          const DevSource &S = sbuf[b][s];
          double2 ph = source_phase(S, a.modes, u, v, w, freq, a.fdelta2);
          // station beams towards this source at this timeslot and channel
          const size_t bt = ((size_t)tslot * nchan + cf) * a.beam_S + (size_t)(sg.first + s);
          if (a.beam_af) {  // array factor of both stations (predict_withbeam.c:336-343)
            const double af = a.beam_af[bt * a.N + s1] * a.beam_af[bt * a.N + s2];
            ph.x *= af;
            ph.y *= af;
          }
          double I = S.sI, Q = S.sQ, U = S.sU, V = S.sV;
          if (MODE >= 1 && S.spec_idx != 0.0) {
            const double fr = log(freq / S.f0);
            const double fr1 = fr * fr, fr2 = fr1 * fr;
            const double tf = S.spec_idx * fr + S.spec_idx1 * fr1 + S.spec_idx2 * fr2;
            I = spec_flux(S.sI0, tf);
            Q = spec_flux(S.sQ0, tf);
            U = spec_flux(S.sU0, tf);
            V = spec_flux(S.sV0, tf);
          }
          if (a.beam_E) {  // E_p (Stokes coherency) E_q^H  (predict_withbeam.c:381-404)
            double2 C0[4], T1[4], E1[4], E2[4];
#pragma unroll
            for (int c = 0; c < 4; c++) {
              C0[c] = make_double2(0.0, 0.0);
              E1[c] = a.beam_E[(bt * a.N + s1) * 4 + c];
              E2[c] = a.beam_E[(bt * a.N + s2) * 4 + c];
            }
            add_stokes(C0, ph, I, Q, U, V);
            mat_ab(E1, C0, T1);
            mat_abh(T1, E2, C0);
#pragma unroll
            for (int c = 0; c < 4; c++) C[c] = cadd(C[c], C0[c]);
          } else {
            add_stokes(C, ph, I, Q, U, V);
          }
        }
        if (sg.last) {
          if (MODE == 0) {
            double2 *ck = a.coh + (long long)sg.cluster * 4 * a.R;
#pragma unroll
            for (int c = 0; c < 4; c++) st_stream(ck + (long long)c * a.R + r, C[c]);
          } else if (MODE == 1) {
#pragma unroll
            for (int c = 0; c < 4; c++) X[c] = cadd(X[c], C[c]);
          } else if (const int coef = a.clus_coef[sg.cluster]) {
            // Jones of this row's hybrid chunk: px = row / ceil(R / nchunk)  (residual.c:717)
            const int nch = a.clus_nchunk[sg.cluster];
            const int px = row_chunk(r, a.R, nch);
            const double *pm = a.p + a.chunk_poff[a.clus_chunk0[sg.cluster] + px];
            double2 G1[4], G2[4], T1[4], T2[4];
            load_jones(pm, s1, G1);
            load_jones(pm, s2, G2);
            mat_ab(G1, C, T1);
            mat_abh(T1, G2, T2);
            // (X - T and X + (-T) round alike: a negative coefficient subtracts bit for bit)
#pragma unroll
            for (int c = 0; c < 4; c++) X[c] = coef < 0 ? csub(X[c], T2[c]) : cadd(X[c], T2[c]);
          }
#pragma unroll
          for (int c = 0; c < 4; c++) C[c] = make_double2(0.0, 0.0);
        }
      }
      __syncthreads();  // everyone is done with sbuf[b] before it is refilled two iterations on
    }
    if (MODE >= 1 && active) {
      double2 *xo = a.xout + ((long long)cf * a.R + r) * 4;
      double2 V[4];
#pragma unroll
      for (int c = 0; c < 4; c++) V[c] = cadd(xo[c], X[c]);
      if (MODE == 2 && a.pinv) {
        const int px = row_chunk(r, a.R, a.pinv_nchunk);
        const double *pm = a.pinv + (size_t)8 * a.N * px;
        double2 G1[4], G2[4], T1[4];
        load_jones(pm, s1, G1);
        load_jones(pm, s2, G2);
        mat_ab(G1, V, T1);
        mat_abh(T1, G2, V);
      }
#pragma unroll
      for (int c = 0; c < 4; c++) xo[c] = V[c];
    }
  }
  if (MODE == 0 && active && a.flag) {
    // uv cut: unflagged rows outside [uvmin, uvmax] get flag 2 (predict.c:488-493).  u u and v v
    // are rounded before they are added, as on the host: a fused multiply-add would move a row that
    // lies on uvmin or uvmax by an ulp to the other side of the limit.
    if (a.flag[r] == 0) {
      const double uvdist = sqrt(__dadd_rn(__dmul_rn(u, u), __dmul_rn(v, v))) * a.freqs[0];
      if (uvdist < a.uvmin || uvdist > a.uvmax) a.flag[r] = 2;
    }
  }
}

// ---- station beam tables: one thread per (timeslot, channel, source, station), coh_math.cuh ---------
__global__ void __launch_bounds__(128) k_beam_tables(BeamArgs a) {
  const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)a.T * a.Nf * a.S * a.N;
  if (gid >= total) return;
  beam_table_entry(a, gid);
}

extern "C" {
void db_launch_beam_tables(const BeamArgs *a, cudaStream_t st) {
  const size_t total = (size_t)a->T * a->Nf * a->S * a->N;
  k_beam_tables<<<(unsigned)((total + 127) / 128), 128, 0, st>>>(*a);
}
void db_launch_coherencies(const CohArgs *a, cudaStream_t st) {
  unsigned grid = (unsigned)((a->R + COH_THREADS - 1) / COH_THREADS);
  k_sky_predict<0><<<grid, COH_THREADS, 0, st>>>(*a);
}
void db_launch_residual_multifreq(const CohArgs *a, cudaStream_t st) {
  unsigned grid = (unsigned)((a->R + COH_THREADS - 1) / COH_THREADS);
  k_sky_predict<2><<<grid, COH_THREADS, 0, st>>>(*a);
}
void db_launch_predict_multifreq(const CohArgs *a, cudaStream_t st) {
  unsigned grid = (unsigned)((a->R + COH_THREADS - 1) / COH_THREADS);
  k_sky_predict<1><<<grid, COH_THREADS, 0, st>>>(*a);
}
}
