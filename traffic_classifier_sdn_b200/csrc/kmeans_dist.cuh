// kmeans_dist.cuh -- the one squared distance of KMeans.transform, KMeans.score and the k-means++ seeding
// (scorers.cu, kmeanspp.cu).
//
// scikit-learn's _euclidean_dense_dense (sk:cluster/_k_means_common.pyx:16-43) in fp64: the features in groups of four,
// each group ((d0 d0 + d1 d1) + d2 d2) + d3 d3 with d_j = x_j - c_j added to the running result, then the remaining
// features one at a time.  Every operation is an explicitly rounded __d*_rn, so nvcc cannot contract a product and a sum
// into an FMA: the result equals _euclidean_dense_dense_wrapper on the widened rows bit for bit.
#pragma once

namespace tcsdn {

// x(j), c(j): feature j of the row and of the centre, as fp64
template <typename XF, typename CF>
__device__ __forceinline__ double km_sqdist(int d, const XF &x, const CF &c) {
    double s = 0.0;
    const int d4 = d & ~3;
#pragma unroll
    for (int j = 0; j < d4; j += 4) {
        const double a0 = __dsub_rn(x(j), c(j)), a1 = __dsub_rn(x(j + 1), c(j + 1));
        const double a2 = __dsub_rn(x(j + 2), c(j + 2)), a3 = __dsub_rn(x(j + 3), c(j + 3));
        const double g = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(a0, a0), __dmul_rn(a1, a1)), __dmul_rn(a2, a2)), __dmul_rn(a3, a3));
        s = __dadd_rn(s, g);
    }
#pragma unroll
    for (int j = d4; j < d; ++j) {
        const double a = __dsub_rn(x(j), c(j));
        s = __dadd_rn(s, __dmul_rn(a, a));
    }
    return s;
}

}  // namespace tcsdn
