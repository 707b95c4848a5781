// flow.cu -- N1 (SURVEY 8f): the reference's per-flow feature derivation on device.
//
//   reference traffic_classifier.py:63-78  Flow.updateforward(packets, bytes, curr_time)
//   reference traffic_classifier.py:81-96  Flow.updatereverse(...)       (same arithmetic, other block)
//   reference traffic_classifier.py:104    feature order handed to model.predict
//
// One thread per flow applies one poll sample.  Counters are integers carried in float64 (exact below
// 2^53) and the divisions are IEEE fp64 divisions, as Python's int/float(int) is, so the features are
// bit-identical to the reference's.  The guards `curr_time != time_start` / `!= last_time` keep the
// previous rate when no time has passed, exactly like the reference.
#include "common.h"

namespace tcsdn {

template <typename F>
__global__ void flow_update_kernel(double *__restrict__ state, const double *__restrict__ packets,
                                   const double *__restrict__ bytes, const double *__restrict__ curr_time,
                                   const uint8_t *__restrict__ dir, int64_t n, F *__restrict__ feat) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        double *st = state + i * TCSDN_FLOW_STATE;
        const uint8_t dr = dir[i];
        if (dr < 2) {
            double *b = st + (dr ? 9 : 0);
            const double t0 = st[18], p = packets[i], by = bytes[i], now = curr_time[i];
            b[2] = p - b[0];
            b[0] = p;
            if (now != t0) b[5] = p / (now - t0);
            if (now != b[8]) b[4] = b[2] / (now - b[8]);
            b[3] = by - b[1];
            b[1] = by;
            if (now != t0) b[7] = by / (now - t0);
            if (now != b[8]) b[6] = b[3] / (now - b[8]);
            b[8] = now;
        }
        if (feat) {
            F *f = feat + i * 12;
#pragma unroll
            for (int j = 0; j < 6; ++j) {
                f[j] = static_cast<F>(st[2 + j]);
                f[6 + j] = static_cast<F>(st[11 + j]);
            }
        }
    }
}

int launch_flow_update(double *state, const double *packets, const double *bytes, const double *curr_time,
                       const uint8_t *dir, int64_t n, void *features_out, int feat_dtype, cudaStream_t st) {
    if (n == 0) return TCSDN_OK;
    int64_t blocks = (n + 255) / 256;
    if (blocks > 132 * 8) blocks = 132 * 8;
    if (feat_dtype == TCSDN_F32)
        flow_update_kernel<float><<<(unsigned)blocks, 256, 0, st>>>(state, packets, bytes, curr_time, dir, n,
                                                                    static_cast<float *>(features_out));
    else
        flow_update_kernel<double><<<(unsigned)blocks, 256, 0, st>>>(state, packets, bytes, curr_time, dir, n,
                                                                     static_cast<double *>(features_out));
    TCSDN_CUDA(cudaGetLastError());
    return TCSDN_OK;
}

}  // namespace tcsdn
