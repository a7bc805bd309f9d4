// chol_harness.cu — test-only C surface over csrc/chol.cuh (the tiled envelope Cholesky, the substitutions, the tile
// envelope and the deterministic sums shared by gba.cu and essential.cu), for tests/test_chol.py.  It is compiled by the
// test with the product's flags, once with FMA contraction (as gba.o) and once with --fmad=false (as essential.o); it is
// not part of libb200slam.so.
//
// Return codes: 0 ok, 1 bad argument (also: a COO entry outside the lower envelope — a test mistake is reported on the
// host and never becomes an out-of-bounds device write), 2 over the context's capacity, 3 CUDA error.
#include "chol.cuh"

using namespace b2s::chol;

namespace {

enum { OK = 0, BAD_ARG = 1, CAPACITY = 2, CUDA_ERR = 3 };
enum { FLAG_POISON = 1, FLAG_KEEP_FAIL = 2 };

struct Ctx {
  long long maxTiles = 0;
  int maxNpPad = 0;
  double *tiles = nullptr, *linv = nullptr, *rhs = nullptr, *ybuf = nullptr, *x = nullptr;
  int *envT = nullptr, *rows = nullptr, *fail = nullptr;
  long long* tileOff = nullptr;
  cudaStream_t s = nullptr;
};

bool envelope_ok(const int* envBlk, int nBlk, int B) {
  if (nBlk < 1 || B < 1 || (long long)nBlk * B > (1 << 30)) return false;
  for (int i = 0; i < nBlk; i++)
    if (envBlk[i] < 0 || envBlk[i] > i) return false;
  return true;
}

}  // namespace

// tile_envelope of block rows starting at block column envBlk[i]; rows holds at most rowsCap entries.  Returns the
// number of stored tiles, or -1 (bad argument / rows too small).
extern "C" long long chol_envelope(const int* envBlk, int nBlk, int B, int* envT, long long* off, int* rowOff, int* rows,
                                   long long rowsCap, long long* nRows) {
  if (!envelope_ok(envBlk, nBlk, B)) return -1;
  std::vector<int> e(envBlk, envBlk + nBlk), T, ro, r;
  std::vector<long long> o;
  const long long nTiles = tile_envelope(e, nBlk, B, T, o, ro, r);
  *nRows = (long long)r.size();
  if ((long long)r.size() > rowsCap) return -1;
  std::copy(T.begin(), T.end(), envT);
  std::copy(o.begin(), o.end(), off);
  std::copy(ro.begin(), ro.end(), rowOff);
  std::copy(r.begin(), r.end(), rows);
  return nTiles;
}

extern "C" void chol_ctx_destroy(void* p) {
  Ctx* c = (Ctx*)p;
  if (!c) return;
  if (c->s) cudaStreamSynchronize(c->s);
  for (void* q : {(void*)c->tiles, (void*)c->linv, (void*)c->rhs, (void*)c->ybuf, (void*)c->x, (void*)c->envT,
                  (void*)c->rows, (void*)c->fail, (void*)c->tileOff})
    if (q) cudaFree(q);
  if (c->s) cudaStreamDestroy(c->s);
  delete c;
}

// A context whose device buffers hold up to maxTiles stored tiles and maxNpPad padded scalar rows, kept across calls.
extern "C" void* chol_ctx_create(long long maxTiles, int maxNpPad) {
  if (maxTiles < 1 || maxNpPad < TS || maxNpPad % TS) return nullptr;
  Ctx* c = new Ctx;
  c->maxTiles = maxTiles;
  c->maxNpPad = maxNpPad;
  const size_t nT = (size_t)maxNpPad / TS;
  cudaError_t e = cudaStreamCreateWithFlags(&c->s, cudaStreamNonBlocking);
  auto A = [&](void* pp, size_t bytes) {
    if (e == cudaSuccess) e = cudaMalloc((void**)pp, bytes);
  };
  A(&c->tiles, (size_t)maxTiles * TT * 8);
  A(&c->linv, nT * TT * 8);
  A(&c->rhs, (size_t)maxNpPad * 8);
  A(&c->ybuf, (size_t)maxNpPad * 8);
  A(&c->x, (size_t)maxNpPad * 8);
  A(&c->envT, nT * 4);
  A(&c->tileOff, (nT + 1) * 8);
  A(&c->rows, (size_t)maxTiles * 4);
  A(&c->fail, 4);
  if (e == cudaSuccess) e = cudaMemset(c->fail, 0, 4);
  if (e == cudaSuccess) e = set_smem_limits();
  if (e != cudaSuccess) {
    chol_ctx_destroy(c);
    return nullptr;
  }
  return c;
}

// Factorise the symmetric system given by its lower-triangle COO entries (row >= col; duplicates are summed) over the
// envelope envBlk of nBlk blocks of B scalars, and solve it for b (n = nBlk * B entries).  As the solvers do: tiles
// zeroed and filled, padded rhs zero, fail reset (unless FLAG_KEEP_FAIL), then factor_solve on a stream.  FLAG_POISON
// fills linv, ybuf and x with NaN first.  Outputs: x_out (npPad), *fail_out, and optionally the factored tiles
// (nTiles x 64 x 64: L below the diagonal tiles, the updated A on them) and linv (nT x 64 x 64).
extern "C" int chol_ctx_solve(void* p, int nBlk, int B, const int* envBlk, long long nnz, const int* row, const int* col,
                              const double* val, const double* b, int flags, double* x_out, int* fail_out,
                              double* tiles_out, double* linv_out) {
  Ctx* c = (Ctx*)p;
  if (!c || !envelope_ok(envBlk, nBlk, B) || nnz < 0) return BAD_ARG;
  const int np = nBlk * B, nT = (np + TS - 1) / TS, npPad = nT * TS;
  std::vector<int> envT, rowOff, rows;
  std::vector<long long> off;
  const long long nTiles = tile_envelope(std::vector<int>(envBlk, envBlk + nBlk), nBlk, B, envT, off, rowOff, rows);
  if (nTiles > c->maxTiles || npPad > c->maxNpPad) return CAPACITY;
  std::vector<double> hTiles((size_t)nTiles * TT, 0.0);
  for (long long q = 0; q < nnz; q++) {
    const int r = row[q], k = col[q];
    if (r < 0 || r >= np || k < 0 || k > r) return BAD_ARG;
    const int I = r / TS, K = k / TS;
    if (K < envT[(size_t)I]) return BAD_ARG;
    hTiles[(size_t)(off[(size_t)I] + K - envT[(size_t)I]) * TT + (size_t)(r % TS) * TS + (k % TS)] += val[q];
  }
  cudaStream_t s = c->s;
#define H_CUDA(call)                 \
  do {                               \
    if ((call) != cudaSuccess) {     \
      cudaStreamSynchronize(s);      \
      return CUDA_ERR;               \
    }                                \
  } while (0)
  if (flags & FLAG_POISON) {  // all-ones bytes are a NaN double
    H_CUDA(cudaMemsetAsync(c->linv, 0xFF, (size_t)c->maxNpPad / TS * TT * 8, s));
    H_CUDA(cudaMemsetAsync(c->ybuf, 0xFF, (size_t)c->maxNpPad * 8, s));
    H_CUDA(cudaMemsetAsync(c->x, 0xFF, (size_t)c->maxNpPad * 8, s));
  }
  H_CUDA(cudaMemcpyAsync(c->envT, envT.data(), (size_t)nT * 4, cudaMemcpyHostToDevice, s));
  H_CUDA(cudaMemcpyAsync(c->tileOff, off.data(), (size_t)(nT + 1) * 8, cudaMemcpyHostToDevice, s));
  if (!rows.empty()) H_CUDA(cudaMemcpyAsync(c->rows, rows.data(), rows.size() * 4, cudaMemcpyHostToDevice, s));
  H_CUDA(cudaMemcpyAsync(c->tiles, hTiles.data(), hTiles.size() * 8, cudaMemcpyHostToDevice, s));
  H_CUDA(cudaMemsetAsync(c->rhs, 0, (size_t)npPad * 8, s));
  H_CUDA(cudaMemcpyAsync(c->rhs, b, (size_t)np * 8, cudaMemcpyHostToDevice, s));
  if (!(flags & FLAG_KEEP_FAIL)) H_CUDA(cudaMemsetAsync(c->fail, 0, 4, s));
  const TileSys ts = {np, c->envT, c->tileOff, c->tiles, c->linv, c->rhs, c->ybuf, c->x, c->fail};
  factor_solve(ts, nT, envT, rowOff, c->rows, s);
  H_CUDA(cudaGetLastError());
  H_CUDA(cudaMemcpyAsync(x_out, c->x, (size_t)npPad * 8, cudaMemcpyDeviceToHost, s));
  H_CUDA(cudaMemcpyAsync(fail_out, c->fail, 4, cudaMemcpyDeviceToHost, s));
  if (tiles_out) H_CUDA(cudaMemcpyAsync(tiles_out, c->tiles, (size_t)nTiles * TT * 8, cudaMemcpyDeviceToHost, s));
  if (linv_out) H_CUDA(cudaMemcpyAsync(linv_out, c->linv, (size_t)nT * TT * 8, cudaMemcpyDeviceToHost, s));
  H_CUDA(cudaStreamSynchronize(s));
#undef H_CUDA
  return OK;
}

// reduce<0> (op 0: the fixed-order sum) or reduce<1> (op 1: max |v|) of v[0, n) on a device copy of v.
extern "C" int chol_reduce(int op, const double* v, long long n, double* out) {
  if ((op != 0 && op != 1) || n < 0) return BAD_ARG;
  double *dv = nullptr, *part = nullptr, *dout = nullptr;
  cudaError_t e = cudaMalloc(&dv, (size_t)std::max(n, 1LL) * 8);
  if (e == cudaSuccess) e = cudaMalloc(&part, RED_BLOCKS * 8);
  if (e == cudaSuccess) e = cudaMalloc(&dout, 8);
  if (e == cudaSuccess && n) e = cudaMemcpy(dv, v, (size_t)n * 8, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) {
    if (op == 0)
      reduce<0>(dv, n, part, dout, 0);
    else
      reduce<1>(dv, n, part, dout, 0);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpy(out, dout, 8, cudaMemcpyDeviceToHost);
  for (double* q : {dv, part, dout})
    if (q) cudaFree(q);
  return e == cudaSuccess ? OK : CUDA_ERR;
}
