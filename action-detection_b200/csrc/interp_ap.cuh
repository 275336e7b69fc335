// The per-class stage of the ActivityNet toolkit's average precision, shared by detection_ap.cu and classification_ap.cu:
// precision and recall of ranked true / false positive flags as the toolkit divides them (eval_detection.py:225-235,
// eval_classification.py:205-210), then interpolated_prec_rec (utils.py:14-23).
#pragma once
#include <cub/cub.cuh>

namespace ssnb {

constexpr int kApSumThreads = 256;

struct ApMaxOp {
  __device__ __forceinline__ double operator()(double a, double b) const { return b > a ? b : a; }
};

// Called by all kApSumThreads threads of one CTA; the result is thread 0's.  f[0 .. n-1]: the class's ranked predictions, 1 =
// true positive.  Ranked prediction e: cum_e = tp count at ranks <= e, prec_e = cum_e / (e + 1) (tp + fp = e + 1 exactly),
// rec_e = cum_e / npos, both double divisions as numpy does them.  interpolated_prec_rec sums (mrec[i] - mrec[i-1]) *
// max(mprec[i:]) over the i where recall changes, which are the true positives (the closing (1 - rec_last) * 0 adds +0).
// Tiles are walked from the last to the first with thread t on rank base + 255 - t, so a prefix over threads is a suffix over
// ranks.  No prediction: mrec = [0, 1], mprec = [0, 0], AP 0; no ground truth and a prediction: rec = 0 / 0, NaN.
__device__ __forceinline__ double interp_ap_cta(const unsigned char* __restrict__ f, int n, int npos) {
  using IScan = cub::BlockScan<int, kApSumThreads>;
  using DScan = cub::BlockScan<double, kApSumThreads>;
  using IRed = cub::BlockReduce<int, kApSumThreads>;
  using DRed = cub::BlockReduce<double, kApSumThreads>;
  __shared__ union {
    typename IScan::TempStorage is;
    typename DScan::TempStorage ds;
    typename IRed::TempStorage ir;
    typename DRed::TempStorage dr;
  } tmp;
  __shared__ int s_total;
  if (n == 0 || npos == 0) return n == 0 ? 0.0 : __longlong_as_double(0x7ff8000000000000LL);
  int mine = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) mine += f[i];
  const int total = IRed(tmp.ir).Sum(mine);
  if (threadIdx.x == 0) s_total = total;
  __syncthreads();
  const int T = s_total;
  const double dn = (double)npos;
  int later = 0;
  double carry = 0.0, acc = 0.0;
  for (int base = ((n - 1) / kApSumThreads) * kApSumThreads; base >= 0; base -= kApSumThreads) {
    const int e = base + kApSumThreads - 1 - threadIdx.x;
    const int flag = e < n ? f[e] : 0;
    int after, tile_tp;
    IScan(tmp.is).ExclusiveSum(flag, after, tile_tp);
    __syncthreads();
    const int cum = T - later - after;
    const double prec = e < n ? (double)cum / (double)(e + 1) : 0.0;
    double smax, tile_max;
    DScan(tmp.ds).InclusiveScan(prec, smax, ApMaxOp(), tile_max);
    __syncthreads();
    smax = ApMaxOp()(smax, carry);
    const double term = flag ? ((double)cum / dn - (double)(cum - 1) / dn) * smax : 0.0;
    const double tile_sum = DRed(tmp.dr).Sum(term);
    __syncthreads();
    acc += tile_sum;                                          // thread 0's value is the one returned
    carry = ApMaxOp()(carry, tile_max);
    later += tile_tp;
  }
  return acc;
}

}  // namespace ssnb
