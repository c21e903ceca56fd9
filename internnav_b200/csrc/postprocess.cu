// Action tail of a System-1 step on the GPU: 32 sampled trajectories per environment -> mean path -> greedy pure-pursuit
// discretisation -> action ids.  Replaces the host tail of the reference (internnav/model/utils/vln_utils.py L63-136
// `traj_to_actions`: `/= 4`, float32 cumsum, float64 mean over the samples, `trajectory_to_discrete_actions_close_to_goal`)
// and the per-step device->host copy of all trajectories (786 KB at 64 envs) by a copy of the ids (1 KB).
//
// The result is integer, so the arithmetic restates numpy's operation by operation -- which operations are fused matters:
//   * `dp_actions[:, :, :2] /= 4` and np.cumsum run in float32, sequentially over time;
//   * np.mean(axis=0) adds the 32 samples sequentially in float64, then divides by 32;
//   * np.linalg.norm of a 1-D vector is sqrt(dot(x, x)) and the BLAS dot accumulates with a fused multiply-add
//     (verified against numpy in this image); np.linalg.norm(axis=1) is sqrt(x0*x0 + x1*x1) with separate roundings;
//   * Python's `%` on floats is fmod with the sign fix of npy_divmod; round() is round-half-to-even.
// Every multiply/add below is therefore an explicit __dmul_rn / __dadd_rn / __fma_rn (nvcc would otherwise contract).
// atan2 / sin / cos come from the CUDA math library (<= 2 ulp; glibc's are <= 1 ulp): the ids can differ from numpy's only
// when a decision sits within an ulp of its threshold.
#include <math.h>

#include "n1_ops.h"

namespace n1 {
namespace {

__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
// np.linalg.norm(v) for a 2-vector: sqrt(ddot(v, v)), ddot = fma(v1, v1, v0 * v0)
__device__ __forceinline__ double norm_dot(double a, double b) { return sqrt(__fma_rn(b, b, dmul(a, a))); }
// np.linalg.norm(M, axis=1) row: sqrt(add.reduce(M * M))
__device__ __forceinline__ double norm_axis(double a, double b) { return sqrt(dadd(dmul(a, a), dmul(b, b))); }
__device__ __forceinline__ double py_mod(double a, double b) {  // b > 0
  double m = fmod(a, b);
  if (m != 0.0) {
    if (m < 0.0) m = dadd(m, b);
  } else {
    m = 0.0;
  }
  return m;
}
__device__ __forceinline__ double normalize_angle(double a) {
  const double pi = 3.141592653589793;
  return dsub(py_mod(dadd(a, pi), dmul(2.0, pi)), pi);
}

// one block per environment; blockDim = 64 * ceil(...): threads (sample, channel) build the cumulative sums, threads
// (t, channel) the mean, thread 0 walks the path.  ids == NULL: the mean path alone (mean_out), no walk.
__global__ void traj_actions_kernel(const float* __restrict__ traj, int Ns, int T, double turn_rad, double step_size,
                                    int lookahead, int max_actions, int cap, int* __restrict__ ids,
                                    int* __restrict__ count, double* __restrict__ mean_out) {
  extern __shared__ double sm[];
  double* xy = sm;                               // [Ns][T + 1][2]
  double* mean = sm + (size_t)Ns * (T + 1) * 2;  // [T + 1][2]
  const int env = blockIdx.x, tid = threadIdx.x;
  for (int i = tid; i < Ns * 2; i += blockDim.x) {
    const int s = i >> 1, c = i & 1;
    const float* p = traj + ((size_t)(env * Ns + s) * T) * 3 + c;
    float acc = 0.f;
    xy[((size_t)s * (T + 1)) * 2 + c] = 0.0;
    for (int t = 0; t < T; ++t) {
      const float a = __fdiv_rn(p[(size_t)t * 3], 4.0f);
      acc = t == 0 ? a : __fadd_rn(acc, a);
      xy[((size_t)s * (T + 1) + t + 1) * 2 + c] = (double)acc;
    }
  }
  __syncthreads();
  for (int i = tid; i < (T + 1) * 2; i += blockDim.x) {
    double m = xy[i];
    for (int s = 1; s < Ns; ++s) m = dadd(m, xy[(size_t)s * (T + 1) * 2 + i]);
    m = m / (double)Ns;
    mean[i] = m;
    if (mean_out) mean_out[(size_t)env * (T + 1) * 2 + i] = m;
  }
  if (ids == nullptr) return;
  __syncthreads();
  if (tid != 0) return;
  int n = 0;
  int* out = ids + (size_t)env * cap;
  double yaw = 0.0, px = mean[0], py = mean[1];
  const double gx = mean[T * 2], gy = mean[T * 2 + 1];
  auto push = [&](int id) {
    if (n < cap) out[n] = id;
    ++n;
  };
  for (int guard = 0; guard < 4096; ++guard) {
    const double dgoal = norm_dot(dsub(px, gx), dsub(py, gy));
    if (!(dgoal > 0.2)) break;
    if (max_actions > 0 && n >= max_actions) break;
    int best = 0;
    double bd = norm_axis(dsub(mean[0], px), dsub(mean[1], py));
    for (int i = 1; i <= T; ++i) {
      const double d = norm_axis(dsub(mean[i * 2], px), dsub(mean[i * 2 + 1], py));
      if (d < bd) bd = d, best = i;
    }
    const int ti = min(best + lookahead, T);
    const double tx = dsub(mean[ti * 2], px), ty = dsub(mean[ti * 2 + 1], py);
    if (norm_dot(tx, ty) < 1e-6) break;
    const double dyaw = normalize_angle(dsub(atan2(ty, tx), yaw));
    const long nt = (long)rint(dyaw / turn_rad);
    for (long k = 0; k < nt; ++k) push(2);
    for (long k = 0; k < -nt; ++k) push(3);
    yaw = normalize_angle(dadd(yaw, dmul((double)nt, turn_rad)));
    const double nx = dadd(px, dmul(step_size, cos(yaw))), ny = dadd(py, dmul(step_size, sin(yaw)));
    if (norm_dot(dsub(nx, gx), dsub(ny, gy)) > dgoal) break;
    push(1);
    px = nx, py = ny;
  }
  count[env] = n;
  for (int i = n; i < cap; ++i) out[i] = 0;
}

}  // namespace

static void launch_traj_kernel(const float* traj, int B, int Ns, int T, double turn_rad, double step_size, int lookahead,
                               int max_actions, int cap, int* ids, int* count, double* mean_out, cudaStream_t s) {
  const size_t smem = ((size_t)Ns * (T + 1) * 2 + (size_t)(T + 1) * 2) * sizeof(double);
  N1_CHECK(smem <= 200 * 1024, "traj_to_actions: Ns * (T + 1) too large for shared memory");
  static size_t attr = 48 * 1024;
  if (smem > attr) {
    N1_CUDA(cudaFuncSetAttribute(traj_actions_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = smem;
  }
  traj_actions_kernel<<<B, 64, smem, s>>>(traj, Ns, T, turn_rad, step_size, lookahead, max_actions, cap, ids, count, mean_out);
  prof_count_launch();
  N1_CUDA(cudaGetLastError());
}

void traj_to_actions(const float* traj, int B, int Ns, int T, double turn_rad, double step_size, int lookahead,
                     int max_actions, int cap, int* ids, int* count, double* mean_out, cudaStream_t s) {
  N1_CHECK(traj && ids && count && B > 0 && Ns > 0 && T > 0 && cap > 0, "traj_to_actions: bad arguments");
  launch_traj_kernel(traj, B, Ns, T, turn_rad, step_size, lookahead, max_actions, cap, ids, count, mean_out, s);
}

void traj_mean_path(const float* traj, int B, int Ns, int T, double* mean_out, cudaStream_t s) {
  N1_CHECK(traj && mean_out && B > 0 && Ns > 0 && T > 0, "traj_mean_path: bad arguments");
  launch_traj_kernel(traj, B, Ns, T, 0.0, 0.0, 0, 0, 0, nullptr, nullptr, mean_out, s);
}

}  // namespace n1
