// tgen.cu — node dynamics of the temporal graph generators: rand_temporal_radius_graph (GNNGraphs/src/generate.jl:
// 265-284) and rand_temporal_hyperbolic_graph (generate.jl:287-297, 340-380).  The edges of every snapshot come from one
// count and one fill of knn.cu over the T snapshots as T segments (radius: the Euclidean test on fp32 points,
// hyperbolic: its pair-test policy on the records written here).
//
// One thread per node keeps the node's state in fp64 registers, loops over the T snapshots and writes each snapshot's
// row; the arithmetic restates the reference's line by line, every mul / add / sub rounded on its own.  The draws are
// the counter-based stream of include/gnnb200.h: u(i, τ, k) = (splitmix64(K + c) >> 11) 2^-53, K = splitmix64(seed),
// c = ((τ n + i) << 1) | k, so a call is reproducible on any GPU and a numpy statement of it can be compared.
#include "common.cuh"

namespace gnnb {
namespace tgen {

constexpr double TWO_PI = 2.0 * 3.141592653589793;     // Julia's 2 * pi

__device__ __forceinline__ double draw(uint64_t K, int64_t n, int64_t tau, int64_t i, int k) {
    const uint64_t c = ((uint64_t)(tau * n + i) << 1) | (uint64_t)k;
    return (double)(splitmix64(K + c) >> 11) * 0x1.0p-53;
}

// 1 - |1 - |v||: generate.jl:280-281
__device__ __forceinline__ double reflect(double v) { return __dsub_rn(1.0, fabs(__dsub_rn(1.0, fabs(v)))); }

__global__ void radius_points_kernel(int64_t n, int T, double speed, uint64_t K, float* __restrict__ pts) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double two_speed = 2.0 * speed;
    double x = draw(K, n, 0, i, 0), y = draw(K, n, 0, i, 1);
    for (int t = 0; t < T; ++t) {
        if (t > 0) {
            const double rho = __dsub_rn(__dmul_rn(two_speed, draw(K, n, t, i, 0)), speed);
            const double th = __dmul_rn(TWO_PI, draw(K, n, t, i, 1));
            double s, c;
            sincos(th, &s, &c);
            x = reflect(__dadd_rn(x, __dmul_rn(rho, c)));
            y = reflect(__dadd_rn(y, __dmul_rn(rho, s)));
        }
        float* row = pts + 2 * ((int64_t)t * n + i);
        row[0] = __double2float_rn(x);
        row[1] = __double2float_rn(y);
    }
}

// cm1 = cosh(αR) - 1 and inv_alpha = 1/α come from the host (generate.jl:362-363 evaluates them once too)
__global__ void hyperbolic_records_kernel(int64_t n, int T, double inv_alpha, double cm1, double speed, double zeta,
                                          uint64_t K, double* __restrict__ rec) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double two_speed = 2.0 * speed;
    double p = draw(K, n, 0, i, 0);
    double th = __dmul_rn(TWO_PI, draw(K, n, 0, i, 1));
    for (int t = 0; t < T; ++t) {
        if (t > 0) {                                                  // generate.jl:371-376
            p = __dadd_rn(p, __dsub_rn(__dmul_rn(two_speed, draw(K, n, t, i, 0)), speed));
            if (p > 1.0) p = __dsub_rn(1.0, fmod(p, 1.0));
            if (p < 0.0) p = fabs(p);
            th = __dadd_rn(th, __dsub_rn(__dmul_rn(two_speed, draw(K, n, t, i, 1)), speed));
        }
        const double r = __dmul_rn(inv_alpha, acosh(__dadd_rn(1.0, __dmul_rn(cm1, p))));
        const double zr = __dmul_rn(zeta, r);
        double s, c;
        sincos(th, &s, &c);
        double* out = rec + 4 * ((int64_t)t * n + i);
        out[0] = cosh(zr);
        out[1] = sinh(zr);
        out[2] = c;
        out[3] = s;
    }
}

static int check_sizes(const char* who, int64_t n, int64_t T, const void* out) {
    if (n < 0 || T < 0) GNNB_FAIL(GNNB_EINVAL, "%s: n = %lld and T = %lld must be >= 0", who, (long long)n, (long long)T);
    const int64_t lim = (int64_t)1 << 31;
    if (n >= lim || T >= lim || n * T >= lim)
        GNNB_FAIL(GNNB_ESIZE, "%s: T * n = %lld * %lld must be < 2^31", who, (long long)T, (long long)n);
    if (n * T > 0 && !out) GNNB_FAIL(GNNB_EINVAL, "%s: the output is NULL", who);
    return GNNB_OK;
}

static bool finite(double v) { return v == v && v - v == 0.0; }

}  // namespace tgen
}  // namespace gnnb

using namespace gnnb;

extern "C" {

int gnnb_temporal_radius_points(int64_t n, int64_t T, double speed, uint64_t seed, float* pts, void* stream) {
    GNNB_TRY(tgen::check_sizes("gnnb_temporal_radius_points", n, T, pts));
    if (!tgen::finite(speed)) GNNB_FAIL(GNNB_EINVAL, "gnnb_temporal_radius_points: speed = %g is not finite", speed);
    if (n * T == 0) return GNNB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    tgen::radius_points_kernel<<<(unsigned)ceil_div(n, 128), 128, 0, st>>>(n, (int)T, speed, splitmix64(seed), pts);
    GNNB_LAUNCHED();
    GNNB_CUDA(cudaStreamSynchronize(st));
    return GNNB_OK;
}

int gnnb_temporal_hyperbolic_records(int64_t n, int64_t T, double alpha, double R, double speed, double zeta,
                                     uint64_t seed, double* rec, void* stream) {
    const char* who = "gnnb_temporal_hyperbolic_records";
    GNNB_TRY(tgen::check_sizes(who, n, T, rec));
    if (!tgen::finite(alpha) || !(alpha > 0)) GNNB_FAIL(GNNB_EINVAL, "%s: α = %g must be > 0 and finite", who, alpha);
    if (!tgen::finite(R) || R < 0) GNNB_FAIL(GNNB_EINVAL, "%s: R = %g must be >= 0 and finite", who, R);
    if (!tgen::finite(zeta) || !(zeta > 0)) GNNB_FAIL(GNNB_EINVAL, "%s: ζ = %g must be > 0 and finite", who, zeta);
    if (!tgen::finite(speed)) GNNB_FAIL(GNNB_EINVAL, "%s: speed = %g is not finite", who, speed);
    const double ch = cosh(alpha * R);
    if (!tgen::finite(ch)) GNNB_FAIL(GNNB_EINVAL, "%s: cosh(α R) = cosh(%g) overflows", who, alpha * R);
    if (n * T == 0) return GNNB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    tgen::hyperbolic_records_kernel<<<(unsigned)ceil_div(n, 128), 128, 0, st>>>(n, (int)T, 1.0 / alpha, ch - 1.0, speed,
                                                                              zeta, splitmix64(seed), rec);
    GNNB_LAUNCHED();
    GNNB_CUDA(cudaStreamSynchronize(st));
    return GNNB_OK;
}

}  // extern "C"
