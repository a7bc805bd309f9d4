// geom_harness.cu — test-only C surface over the device geometry headers, for tests/test_device_geometry.py:
// csrc/ba_math.cuh (quaternions, SE3 maps, pose_oplus, huber, edge_jacobians), csrc/sim3.cuh (g2o's Sim3) and
// csrc/jacobi.cuh (OpenCV's Jacobi SVD at every shape its callers instantiate).  It is not part of libb200slam.so.
//
// The test compiles it once per flag set that an including object is built with (build.py's NVCC_FLAGS and NO_FMAD) and
// defines GEOM_SIM3 / GEOM_JACOBI only in the builds whose flags an includer of that header really uses: ba_math.cuh is
// built with FMA contraction (localba.o, gba.o) and without (essential.o, sim3opt.o); sim3.cuh and jacobi.cuh only
// without.
//
// Every entry takes n cases as host arrays, copies them to the device, runs one thread per case that calls the header
// function, and copies the results back.  Return codes: 0 ok, 1 bad argument, 3 CUDA error.
#include <cuda_runtime.h>

#include <vector>

#include "ba_math.cuh"
#ifdef GEOM_SIM3
#include "sim3.cuh"
#endif
#ifdef GEOM_JACOBI
#include "jacobi.cuh"
#endif

using namespace b2s;

namespace {

enum { OK = 0, BAD_ARG = 1, CUDA_ERR = 3 };

struct Arg {
  const void* h;  // host array of n * bytes
  size_t bytes;   // per case
  bool out;       // copied back after the launch (inputs are copied in either way)
};

template <typename Op>
__global__ void k_each(Op op, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) op(i);
}

// Copy the arguments in, launch op over n cases (bind receives the device pointers and returns the functor), copy the
// outputs back.
template <typename Bind>
int run(int n, std::vector<Arg> args, Bind bind) {
  if (n < 0) return BAD_ARG;
  for (const Arg& a : args)
    if (!a.h) return BAD_ARG;
  if (n == 0) return OK;
  std::vector<void*> d(args.size(), nullptr);
  cudaError_t e = cudaSuccess;
  for (size_t k = 0; k < args.size() && e == cudaSuccess; k++) {
    e = cudaMalloc(&d[k], n * args[k].bytes);
    if (e == cudaSuccess) e = cudaMemcpy(d[k], args[k].h, n * args[k].bytes, cudaMemcpyHostToDevice);
  }
  if (e == cudaSuccess) {
    k_each<<<(n + 127) / 128, 128>>>(bind(d), n);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  for (size_t k = 0; k < args.size() && e == cudaSuccess; k++)
    if (args[k].out) e = cudaMemcpy((void*)args[k].h, d[k], n * args[k].bytes, cudaMemcpyDeviceToHost);
  for (void* p : d)
    if (p) cudaFree(p);
  return e == cudaSuccess ? OK : CUDA_ERR;
}

// ------------------------------------------------------------------------------------------------ ba_math.cuh
struct QuatFromR {
  const double* R;
  double* q;
  __device__ void operator()(int i) const {
    double m[3][3];
    for (int r = 0; r < 9; r++) m[r / 3][r % 3] = R[9 * i + r];
    quat_from_R(m, q + 4 * i);
  }
};
struct NormalizeRot {
  double* q;
  __device__ void operator()(int i) const { normalize_rot(q + 4 * i); }
};
struct FromTcw {
  const float* T;
  double* P;
  __device__ void operator()(int i) const { se3quat_from_Tcw(T + 16 * i, P + POSE_STRIDE * i); }
};
struct ToTcw {
  const double* P;
  float* T;
  __device__ void operator()(int i) const { se3quat_to_Tcw(P + POSE_STRIDE * i, T + 16 * i); }
};
struct PoseOplus {
  double* P;
  const double* upd;
  __device__ void operator()(int i) const { pose_oplus(P + POSE_STRIDE * i, upd + 6 * i); }
};
struct Huber {
  const double* ed;  // e, delta
  double* rho;       // rho0, rho1
  __device__ void operator()(int i) const { huber(ed[2 * i], ed[2 * i + 1], rho[2 * i], rho[2 * i + 1]); }
};
struct EdgeJacobians {
  const double* P;    // POSE_STRIDE
  const double* Xc;   // X, fx, fy, bf, stereo flag (0 / 1): 7
  double* out;        // Xc 3, A 9, B 18
  __device__ void operator()(int i) const {
    const double* c = Xc + 7 * i;
    EdgeJac J;
    edge_jacobians(P + POSE_STRIDE * i, c, c[6] != 0.0, c[3], c[4], c[5], J);
    double* o = out + 30 * i;
    for (int r = 0; r < 3; r++) o[r] = J.Xc[r];
    for (int r = 0; r < 9; r++) o[3 + r] = J.A[r / 3][r % 3];
    for (int r = 0; r < 18; r++) o[12 + r] = J.B[r / 6][r % 6];
  }
};

#ifdef GEOM_SIM3
// ------------------------------------------------------------------------------------------------ sim3.cuh
struct S3Mul {
  const double *a, *b;
  double* o;
  __device__ void operator()(int i) const { s3_mul(a + 8 * i, b + 8 * i, o + 8 * i); }
};
struct S3Inv {
  const double* a;
  double* o;
  __device__ void operator()(int i) const { s3_inv(a + 8 * i, o + 8 * i); }
};
struct S3Map {
  const double *a, *X;
  double* o;
  __device__ void operator()(int i) const { s3_map(a + 8 * i, X + 3 * i, o + 3 * i); }
};
struct S3Exp {
  const double* u;
  double* o;
  __device__ void operator()(int i) const { s3_exp(u + 7 * i, o + 8 * i); }
};
struct S3Log {
  const double* a;
  double* o;
  __device__ void operator()(int i) const { s3_log(a + 8 * i, o + 7 * i); }
};
#endif

#ifdef GEOM_JACOBI
// ------------------------------------------------------------------------------------------------ jacobi.cuh
// One case: At max(n, n1) rows of m (row stride m), W n, Vt n x n, in place as the callers hold them.
template <int NMAX, typename T>
struct Jacobi {
  T *At, *W, *Vt;
  int m, n, n1;
  __device__ void operator()(int i) const {
    const int rows = n > n1 ? n : n1;
    jacobi_svd<NMAX, T>(At + (size_t)i * rows * m, m, W + (size_t)i * n, Vt + (size_t)i * n * n, m, n, n1);
  }
};
template <int NMAX, typename T>
int jacobi_run(int count, int m, int n, int n1, T* At, T* W, T* Vt) {
  const size_t rows = n > n1 ? n : n1, e = sizeof(T);
  return run(count, {{At, rows * m * e, true}, {W, n * e, true}, {Vt, (size_t)n * n * e, true}},
             [&](std::vector<void*>& d) { return Jacobi<NMAX, T>{(T*)d[0], (T*)d[1], (T*)d[2], m, n, n1}; });
}
#endif

}  // namespace

// The number of visible CUDA devices (0 with the return code 3 when there is no driver or device).
extern "C" int geom_device_count(int* n) {
  *n = 0;
  return cudaGetDeviceCount(n) == cudaSuccess ? OK : CUDA_ERR;
}

extern "C" int geom_quat_from_R(int n, const double* R, double* q) {
  return run(n, {{R, 72, false}, {q, 32, true}},
             [](std::vector<void*>& d) { return QuatFromR{(const double*)d[0], (double*)d[1]}; });
}
extern "C" int geom_normalize_rot(int n, double* q) {
  return run(n, {{q, 32, true}}, [](std::vector<void*>& d) { return NormalizeRot{(double*)d[0]}; });
}
extern "C" int geom_se3quat_from_Tcw(int n, const float* T, double* P) {
  return run(n, {{T, 64, false}, {P, 8 * POSE_STRIDE, true}},
             [](std::vector<void*>& d) { return FromTcw{(const float*)d[0], (double*)d[1]}; });
}
extern "C" int geom_se3quat_to_Tcw(int n, const double* P, float* T) {
  return run(n, {{P, 8 * POSE_STRIDE, false}, {T, 64, true}},
             [](std::vector<void*>& d) { return ToTcw{(const double*)d[0], (float*)d[1]}; });
}
// P (POSE_STRIDE doubles per case) is updated in place
extern "C" int geom_pose_oplus(int n, double* P, const double* upd) {
  return run(n, {{P, 8 * POSE_STRIDE, true}, {upd, 48, false}},
             [](std::vector<void*>& d) { return PoseOplus{(double*)d[0], (const double*)d[1]}; });
}
extern "C" int geom_huber(int n, const double* e_delta, double* rho) {
  return run(n, {{e_delta, 16, false}, {rho, 16, true}},
             [](std::vector<void*>& d) { return Huber{(const double*)d[0], (double*)d[1]}; });
}
extern "C" int geom_edge_jacobians(int n, const double* P, const double* X_cam_st, double* out) {
  return run(n, {{P, 8 * POSE_STRIDE, false}, {X_cam_st, 56, false}, {out, 240, true}}, [](std::vector<void*>& d) {
    return EdgeJacobians{(const double*)d[0], (const double*)d[1], (double*)d[2]};
  });
}

#ifdef GEOM_SIM3
extern "C" int geom_s3_mul(int n, const double* a, const double* b, double* o) {
  return run(n, {{a, 64, false}, {b, 64, false}, {o, 64, true}},
             [](std::vector<void*>& d) { return S3Mul{(const double*)d[0], (const double*)d[1], (double*)d[2]}; });
}
extern "C" int geom_s3_inv(int n, const double* a, double* o) {
  return run(n, {{a, 64, false}, {o, 64, true}},
             [](std::vector<void*>& d) { return S3Inv{(const double*)d[0], (double*)d[1]}; });
}
extern "C" int geom_s3_map(int n, const double* a, const double* X, double* o) {
  return run(n, {{a, 64, false}, {X, 24, false}, {o, 24, true}},
             [](std::vector<void*>& d) { return S3Map{(const double*)d[0], (const double*)d[1], (double*)d[2]}; });
}
extern "C" int geom_s3_exp(int n, const double* u, double* o) {
  return run(n, {{u, 56, false}, {o, 64, true}},
             [](std::vector<void*>& d) { return S3Exp{(const double*)d[0], (double*)d[1]}; });
}
extern "C" int geom_s3_log(int n, const double* a, double* o) {
  return run(n, {{a, 64, false}, {o, 56, true}},
             [](std::vector<void*>& d) { return S3Log{(const double*)d[0], (double*)d[1]}; });
}
#endif

#ifdef GEOM_JACOBI
// The (NMAX, m, n, n1) that initializer.cu instantiates: svd_square<3> (3 x 3, n1 3), Triangulate's svd_square<4>
// (4 x 4, n1 0), ComputeH21 (16 x 9, n1 0), ComputeF21 (8 x 9 transposed: m 9, n 8, n1 9).
extern "C" int geom_jacobi_f32(int count, int m, int n, int n1, float* At, float* W, float* Vt) {
  if (m == 3 && n == 3 && n1 == 3) return jacobi_run<3>(count, m, n, n1, At, W, Vt);
  if (m == 4 && n == 4 && n1 == 0) return jacobi_run<4>(count, m, n, n1, At, W, Vt);
  if (m == 16 && n == 9 && n1 == 0) return jacobi_run<9>(count, m, n, n1, At, W, Vt);
  if (m == 9 && n == 8 && n1 == 9) return jacobi_run<8>(count, m, n, n1, At, W, Vt);
  return BAD_ARG;
}
// The ones pnpsolver.cu instantiates: svd_at<3> (3 x 3), svd_at<12> (12 x 12), solve6_svd<N> (6 rows, N = 3, 4, 5);
// each with n1 = n.
extern "C" int geom_jacobi_f64(int count, int m, int n, int n1, double* At, double* W, double* Vt) {
  if (n1 != n) return BAD_ARG;
  if (m == 3 && n == 3) return jacobi_run<3>(count, m, n, n1, At, W, Vt);
  if (m == 12 && n == 12) return jacobi_run<12>(count, m, n, n1, At, W, Vt);
  if (m == 6 && n == 3) return jacobi_run<3>(count, m, n, n1, At, W, Vt);
  if (m == 6 && n == 4) return jacobi_run<4>(count, m, n, n1, At, W, Vt);
  if (m == 6 && n == 5) return jacobi_run<5>(count, m, n, n1, At, W, Vt);
  return BAD_ARG;
}
#endif
