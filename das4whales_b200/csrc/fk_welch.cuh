// fk_welch.cuh -- segment staging of the f-k Welch spectrum (d4w_fk_segment_stage, d4w_fk_welch.cu).
//
// A batch of segments of one [nx x ns] float32 record, all on the same channel range [c0, c0 + lx): segment s covers time
// samples [t0 + s * step, t0 + s * step + l).  Each is written as its own contiguous [lx x l] matrix at out + s * seg_stride,
// ready for the f-k spectrum's column pass (which takes a row pitch equal to its row length only):
//   out[s][c][t] = (x[c0 + c][t0 + s * step + t] - mean_cs) * wx[c] * wt[t]
// mean_cs is the mean of the row's l samples (accumulated in double, subtracted in double) when `detrend` is set, else 0:
// SciPy's per-segment detrend='constant' along time, applied before the window.
//
// One CTA per (segment, row) = (blockIdx.x, blockIdx.y), so that CTAs issued together read neighbouring segments of the
// same channel and overlapping samples are served by L2.  Two routes for a row, chosen per launch (StageParams::smem_row):
//   smem row  the row is read from HBM once into shared memory while the mean accumulates, then written from there;
//   re-read   the mean pass reads the row, the write pass reads it again (from L2 in practice: the row was just read).
// The body is __host__ __device__ with (block, tid, nthr, smem) loops, so tests/host_emul/fk_welch_emul.cu runs it on the CPU.
#pragma once
#include "fft_smem.cuh"

namespace d4w {

struct StageParams {
    int ns;                 // row pitch of the source, samples
    int c0, t0, step;       // first channel, first segment's first sample, samples between segment starts
    int lx, l;              // segment shape
    size_t seg_stride;      // floats between staged segments
    int detrend;            // 1: subtract each row's mean over the segment
    int smem_row;           // 1: keep the row in shared memory between the mean and the write (with detrend only)
};

// shared memory of one CTA: [row: l floats, rounded up to 4 (smem route)][partial sums: nthr doubles][mean: 1 double]
__host__ __device__ inline size_t fk_stage_row_floats(int l, int smem_row) { return smem_row ? (size_t)(l + 3) / 4 * 4 : 0; }
__host__ __device__ inline size_t fk_stage_smem_bytes(int l, int nthr, int smem_row) {
    return fk_stage_row_floats(l, smem_row) * sizeof(float) + (size_t)(nthr + 1) * sizeof(double);
}

__host__ __device__ inline void body_fk_segment_stage(const StageParams& sp, const float* __restrict__ x, const float* __restrict__ wx,
                                                      const float* __restrict__ wt, float* __restrict__ out, long long seg, int row,
                                                      int tid, int nthr, void* smem) {
    float* buf = static_cast<float*>(smem);
    double* part = reinterpret_cast<double*>(buf + fk_stage_row_floats(sp.l, sp.smem_row));
    double* mean = part + nthr;
    const int l = sp.l;
    const float* src = x + (size_t)(sp.c0 + row) * sp.ns + (size_t)sp.t0 + (size_t)seg * sp.step;
    float* dst = out + (size_t)seg * sp.seg_stride + (size_t)row * l;
    if (sp.detrend) {
        double acc = 0.0;
        for (int i = tid; i < l; i += nthr) {
            const float v = src[i];
            if (sp.smem_row) buf[i] = v;
            acc += (double)v;
        }
        part[tid] = acc;
        D4W_SYNC();
        if (tid == 0) {                                  // fixed summation order: the same mean on every run
            double s = 0.0;
            for (int j = 0; j < nthr; ++j) s += part[j];
            *mean = s / l;
        }
        D4W_SYNC();
    }
    const double mu = sp.detrend ? *mean : 0.0;
    const bool from_smem = sp.detrend && sp.smem_row;
    const float w = wx[row];
    if (l % 4 == 0) {
        // 16-byte stores (d4w_fk_segment_stage keeps every staged row and wt 16-byte aligned when l % 4 == 0); the source
        // row has no alignment, so it is read by scalars
        const float4* wt4 = reinterpret_cast<const float4*>(wt);
        float4* dst4 = reinterpret_cast<float4*>(dst);
        for (int i = tid; i < l / 4; i += nthr) {
            float4 v;
            if (from_smem) v = reinterpret_cast<const float4*>(buf)[i];
            else v = make_float4(src[4 * i], src[4 * i + 1], src[4 * i + 2], src[4 * i + 3]);
            const float4 g = wt4[i];
            dst4[i] = make_float4((float)((double)v.x - mu) * (w * g.x), (float)((double)v.y - mu) * (w * g.y),
                                  (float)((double)v.z - mu) * (w * g.z), (float)((double)v.w - mu) * (w * g.w));
        }
    } else {
        for (int i = tid; i < l; i += nthr) {
            const float v = from_smem ? buf[i] : src[i];
            dst[i] = (float)((double)v - mu) * (w * wt[i]);
        }
    }
}

}  // namespace d4w
