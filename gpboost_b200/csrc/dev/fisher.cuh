// Fisher information of the covariance parameters of the Gaussian Vecchia model, stochastic trace branch. Included at the end of
// dev_api.cu after laplace.cuh: it reuses the engine struct, the CSC view of B, the Laplace engine's multi-vector operators and
// its polling triangular solves.
//
// Replaces CalcStdDevCovPar (include/GPBoost/re_model_template.h:10788-10815) up to the 3 x 3 matrix: the factor and its
// derivatives on the original scale (CalcCovFactor(false, sigma2), CalcGradientVecchia(false, sigma2, true)) and
// CalcFisherInformation_Vecchia with transf_scale = false, include_error_var = true, no weights (:10145-10230):
//   W1 = B^-T Z,  W2 = B^-1 D W1,  S_k = B^T D^-1 (-dB_k W2 + dD_k W1) - dB_k^T W1,  S_0 = B^T D^-1 B Z,
//   FI(a, b) = mean over the probe columns of sum_rows S_a .* S_b / 2,   order (sigma2, sigma1^2, rho).
// Everything is formed on the transformed scale of the engine (Psi = Sigma~ / sigma2, s = sigma1^2 / sigma2, rho_t): B is the
// same, D = sigma2 D_Psi, and with the factor kernel's derivatives w.r.t. log s and log rho_t (dA = -dB)
//   S_0 = T_0 / sigma2,  S_1 = -T_1 / sigma1^2,  S_2 = (d log rho_t / d rho) T_2
// where  T_0 = B^T U0, U0 = D_Psi^-1 B Z;  T_k = B^T H_k + Bg_k^T V1,  H_k = D_Psi^-1 (Bg_k V2 - dD_k V1),  Bg_k = -dA_k,
//        V1 = B^-T Z,  V2 = B^-1 D_Psi V1   (T_k = -[B^T D_Psi^-1 (dA_k V2 + dD_k V1) + dA_k^T V1]).
// The six column products T_a . T_b come from one fused pass over B's columns (fi_contract_kernel) that forms H_k at every
// gathered row on the fly: no S or H matrix is written. Probe counts above gpl::kMaxCols run in column blocks whose column sums
// are added on the host in column order, so two calls give bitwise the same result.

namespace gpl {

// One unit = (column j, 32 probe columns), the scheme of mv_Bt_kernel. Per warp: partial[(slot * 6 + q) * kMaxCols + c] for
// q = 00, 01, 02, 11, 12, 22 of the products T_a[j, c] T_b[j, c] summed over this warp's columns j.
__global__ void __launch_bounds__(kBlock) fi_contract_kernel(const double* __restrict__ A, const double* __restrict__ dA0,
                                                             const double* __restrict__ dA1, const int32_t* __restrict__ colptr,
                                                             const int32_t* __restrict__ csc_pos, int m, int64_t n, int t, int G,
                                                             const double* __restrict__ Dinv, const double* __restrict__ dD0,
                                                             const double* __restrict__ dD1, const double* __restrict__ U0,
                                                             const double* __restrict__ Y0, const double* __restrict__ Y1,
                                                             const double* __restrict__ V1, double* __restrict__ partial,
                                                             const int32_t* __restrict__ order) {
  const Unit u = make_unit(t, G);
  double pr[6] = {0., 0., 0., 0., 0., 0.};
  for (int64_t p = u.r0; p < n; p += u.rstep) {
    const int64_t j = order ? (int64_t)order[p] : p;
    // unit diagonal of B (Bg has none)
    const double vj = V1[j * t + u.cc], dj = Dinv[j];
    double t0 = U0[j * t + u.cc];
    double t1 = dj * (Y0[j * t + u.cc] - dD0[j] * vj);
    double t2 = dj * (Y1[j * t + u.cc] - dD1[j] * vj);
    const int e0 = colptr[j], e1 = colptr[j + 1];
    for (int eb = e0; eb < e1; eb += 32) {
      const int e = eb + u.lane;
      const bool real = e < e1;
      const int32_t pos = real ? csc_pos[e] : 0;
      const int64_t rowp = real ? pos / m : j;  // idle slots: zero coefficients, any valid row
      const double ap = real ? A[pos] : 0., g0 = real ? dA0[pos] : 0., g1 = real ? dA1[pos] : 0.;
      const double di = real ? Dinv[rowp] : 0.;
      const double c0 = real ? di * dD0[rowp] : 0., c1 = real ? di * dD1[rowp] : 0.;
      const int cnt = min(32, e1 - eb);
      for (int hb = 0; hb < cnt; hb += 8) {
        double vu[8], vy0[8], vy1[8], vv[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const int64_t r = __shfl_sync(0xffffffffu, rowp, hb + q);
          vu[q] = U0[r * t + u.cc]; vy0[q] = Y0[r * t + u.cc]; vy1[q] = Y1[r * t + u.cc]; vv[q] = V1[r * t + u.cc];
        }
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const int s = hb + q;
          const double a = __shfl_sync(0xffffffffu, ap, s), d = __shfl_sync(0xffffffffu, di, s);
          const double ga = __shfl_sync(0xffffffffu, g0, s), gb = __shfl_sync(0xffffffffu, g1, s);
          const double ca = __shfl_sync(0xffffffffu, c0, s), cb = __shfl_sync(0xffffffffu, c1, s);
          t0 -= a * vu[q];
          t1 -= a * (d * vy0[q] - ca * vv[q]) + ga * vv[q];
          t2 -= a * (d * vy1[q] - cb * vv[q]) + gb * vv[q];
        }
      }
    }
    pr[0] += t0 * t0; pr[1] += t0 * t1; pr[2] += t0 * t2;
    pr[3] += t1 * t1; pr[4] += t1 * t2; pr[5] += t2 * t2;
  }
  if (u.active) {
#pragma unroll
    for (int q = 0; q < 6; ++q) partial[(u.pslot * 6 + q) * kMaxCols + u.c] = pr[q];
  }
}

}  // namespace gpl

namespace {

// device buffers of one Fisher-information call (freed on every exit path)
struct FisherBufs {
  double *A = nullptr, *Dinv = nullptr, *w = nullptr, *dA0 = nullptr, *dD0 = nullptr, *dA1 = nullptr, *dD1 = nullptr;
  double *ones = nullptr, *Pcm = nullptr, *Z = nullptr, *V1 = nullptr, *V2 = nullptr, *U0 = nullptr, *Y0 = nullptr, *Y1 = nullptr;
  double *partial = nullptr, *colsum = nullptr;
  ~FisherBufs() {
    double* b[] = {A, Dinv, w, dA0, dD0, dA1, dD1, ones, Pcm, Z, V1, V2, U0, Y0, Y1, partial, colsum};
    for (double* p : b) cudaFree(p);
  }
};

// The Gaussian factor (nugget 1 on the transformed scale) with both derivative pairs, into the call's own buffers: the engine's
// A, D^-1, u and its "STORE state" (launch_eval) are left exactly as they were, so later passes are not affected.
int fisher_factor(gpbdev_vecchia* h, int cov_type, double var, double range, FisherBufs& f) {
  CUDA_TRY(cudaMemcpyToSymbolAsync(gpb::g_factor_dA, &f.dA1, sizeof(double*), 0, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(cudaMemcpyToSymbolAsync(gpb::g_factor_dD, &f.dD1, sizeof(double*), 0, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(cudaMemcpyToSymbolAsync(gpb::g_factor_dA0, &f.dA0, sizeof(double*), 0, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(cudaMemcpyToSymbolAsync(gpb::g_factor_dD0, &f.dD0, sizeof(double*), 0, cudaMemcpyHostToDevice, h->stream));
  gpb::FactorArgs a;
  a.coords = h->coords; a.nn = h->nn; a.y = h->y;
  a.A = f.A; a.Dinv = f.Dinv; a.w = f.w;
  a.partials = h->partials;  // per-warp sums are not reduced: the engine's last sums stay as they are
  a.n = h->n; a.row_begin = 0; a.row_end = h->n;
  a.m = h->m; a.d = h->d; a.var = var; a.range = range;
  a.diag_nb = var + 1.; a.diag_obs = var + 1.;
  FactorKernel k = pick_kernel(cov_type, gpb::MODE_STORE_GRAD2, h->d, h->m);
  const size_t smem = sizeof(double) * gpb::kWarpsPerBlock * (32 * gpb::kLd + 32 * h->d + 64);
  CUDA_TRY(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CUDA_TRY(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  int per_sm = 0;
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, gpb::kWarpsPerBlock * 32, smem));
  const int grid = std::min(std::max(per_sm, 1) * h->num_sms, h->grid_cap);
  k<<<grid, gpb::kWarpsPerBlock * 32, smem, h->stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  return 0;
}

}  // namespace

extern "C" {

int gpbdev_vecchia_fisher_info(gpbdev_vecchia_t h, int cov_type, double sigma2, double var, double range, const double* probes_colmajor,
                               int t, double* FI9) {
  if (!h || !probes_colmajor || !FI9) return fail("gpbdev_vecchia_fisher_info: null argument");
  if (cov_type < 0 || cov_type > 3) return fail("gpbdev_vecchia_fisher_info: unknown covariance id");
  if (!(sigma2 > 0.) || !(var > 0.) || !(range > 0.)) return fail("gpbdev_vecchia_fisher_info: covariance parameters must be positive");
  if (t < 1) return fail("gpbdev_vecchia_fisher_info: need at least one probe vector");
  if (h->row_begin != 0 || h->row_end != h->n) return fail("gpbdev_vecchia_fisher_info: row-sharded engines are not supported");
  if (h->m > gpl::kM) return fail("gpbdev_vecchia_fisher_info: num_neighbors must be <= 30");
  CUDA_TRY(cudaSetDevice(h->device));
  if (laplace_ensure(h)) return -1;
  if (ensure_csc(h)) return -1;
  gpb_laplace_state* L = h->lap;
  const int64_t n = h->n;
  const int m = h->m;
  const int tb_max = std::min(t, gpl::kMaxCols);
  const size_t nb = sizeof(double) * (size_t)n, blk = nb * (size_t)tb_max;
  const int slots = lap_grid(L->grid_mv, 1) * (gpl::kBlock / 32);  // upper bound of the partial rows at any G
  FisherBufs f;
  CUDA_TRY(cudaMalloc(&f.A, nb * m)); CUDA_TRY(cudaMalloc(&f.dA0, nb * m)); CUDA_TRY(cudaMalloc(&f.dA1, nb * m));
  CUDA_TRY(cudaMalloc(&f.Dinv, nb)); CUDA_TRY(cudaMalloc(&f.w, nb)); CUDA_TRY(cudaMalloc(&f.dD0, nb)); CUDA_TRY(cudaMalloc(&f.dD1, nb));
  CUDA_TRY(cudaMalloc(&f.ones, nb));
  double** mv[] = {&f.Pcm, &f.Z, &f.V1, &f.V2, &f.U0, &f.Y0, &f.Y1};
  for (double** p : mv) CUDA_TRY(cudaMalloc(p, blk));
  CUDA_TRY(cudaMalloc(&f.partial, sizeof(double) * (size_t)slots * 6 * gpl::kMaxCols));
  CUDA_TRY(cudaMemsetAsync(f.partial, 0, sizeof(double) * (size_t)slots * 6 * gpl::kMaxCols, h->stream));
  CUDA_TRY(cudaMalloc(&f.colsum, sizeof(double) * 6 * gpl::kMaxCols));
  const int eb = (int)std::min<int64_t>((n + 255) / 256, (int64_t)h->num_sms * 16);
  fill_kernel<<<eb, 256, 0, h->stream>>>(f.ones, n, 1.);
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  if (fisher_factor(h, cov_type, var, range, f)) return -1;
  CUDA_TRY(cudaMemsetAsync(L->err, 0, sizeof(int), h->stream));
  // column sums of the six products, accumulated over the column blocks in column order
  double tot[6] = {0., 0., 0., 0., 0., 0.};
  std::vector<double> cs(6 * gpl::kMaxCols);
  for (int c0 = 0; c0 < t; c0 += gpl::kMaxCols) {
    const int tb = std::min(gpl::kMaxCols, t - c0);
    const int64_t len = n * tb;
    const int lb = (int)std::min<int64_t>((len + 255) / 256, (int64_t)h->num_sms * 16);
    const int G = lap_groups(tb), gridg = lap_grid(L->grid_mv, G), prow = gridg * (gpl::kBlock / 32) / G;
    CUDA_TRY(cudaMemcpyAsync(f.Pcm, probes_colmajor + (size_t)c0 * n, sizeof(double) * (size_t)len, cudaMemcpyHostToDevice, h->stream));
    gpl::scale_transpose_kernel<<<lb, 256, 0, h->stream>>>(n, tb, f.Pcm, f.ones, f.Z);  // Z, n x tb row-major
    gpl::fill_sentinel_kernel<<<lb, 256, 0, h->stream>>>(f.V1, len);
    gpl::fill_sentinel_kernel<<<lb, 256, 0, h->stream>>>(f.V2, len);
    CUDA_TRY(cudaGetLastError());
    h->launches += 3;
    // V1 = B^-T Z, V2 = B^-1 (V1 / D^-1) (the VADU solves with dw = D^-1; their column dots are not used)
    {
      const double* Ac = f.A; const int32_t* colptr = h->colptr; const int32_t* csc = h->csc_pos; const int32_t* nnp = h->nn;
      int mm = m; int64_t nn_ = n; int tt = tb; int GG = G; const double* Zc = f.Z; const double* dwc = f.Dinv;
      const double* V1c = f.V1; double* V1 = f.V1; double* V2 = f.V2; double* part = L->partial; int* err = L->err;
      const int grid = lap_grid(L->grid, G);
      if (coop_launch(h, grid, gpl::trs_bwd_kernel, Ac, colptr, csc, mm, nn_, tt, GG, Zc, V1, err)) return -1;
      if (coop_launch(h, grid, gpl::trs_fwd_kernel, Ac, nnp, mm, nn_, tt, GG, dwc, V1c, Zc, V2, part, err)) return -1;
    }
    // U0 = D^-1 B Z,  Y_k = Bg_k V2
    gpl::mv_B_kernel<<<gridg, gpl::kBlock, 0, h->stream>>>(f.A, h->nn, m, n, tb, G, f.Dinv, f.Z, f.U0, L->order);
    gpl::mv_Bg_kernel<<<gridg, gpl::kBlock, 0, h->stream>>>(f.dA0, h->nn, m, n, tb, G, f.V2, f.Y0);
    gpl::mv_Bg_kernel<<<gridg, gpl::kBlock, 0, h->stream>>>(f.dA1, h->nn, m, n, tb, G, f.V2, f.Y1);
    gpl::fi_contract_kernel<<<gridg, gpl::kBlock, 0, h->stream>>>(f.A, f.dA0, f.dA1, h->colptr, h->csc_pos, m, n, tb, G, f.Dinv, f.dD0,
                                                                  f.dD1, f.U0, f.Y0, f.Y1, f.V1, f.partial, L->order);
    gpl::col_reduce_kernel<<<6 * gpl::kMaxCols, gpl::kBlock, 0, h->stream>>>(f.partial, prow, 6 * gpl::kMaxCols, f.colsum);
    CUDA_TRY(cudaGetLastError());
    h->launches += 5;
    CUDA_TRY(cudaMemcpyAsync(cs.data(), f.colsum, sizeof(double) * 6 * gpl::kMaxCols, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(cudaStreamSynchronize(h->stream));
    for (int q = 0; q < 6; ++q)
      for (int c = 0; c < tb; ++c) tot[q] += cs[(size_t)q * gpl::kMaxCols + c];
  }
  if (lap_check_err(h)) return -1;
  // back to the original scale: S_0 = T_0 / sigma2, S_1 = -T_1 / sigma1^2, S_2 = -(d log rho_t / d rho) T_2 with
  // rho_t = c / rho (Matern family, exponential) or 1 / rho^2 (Gaussian kernel): d log rho_t / d rho = -1 / rho resp. -2 / rho
  double rho;
  switch (cov_type) {
    case gpb::COV_EXPONENTIAL: rho = 1. / range; break;
    case gpb::COV_MATERN15: rho = std::sqrt(3.) / range; break;
    case gpb::COV_MATERN25: rho = std::sqrt(5.) / range; break;
    default: rho = 1. / std::sqrt(range); break;
  }
  const double fac[3] = {1. / sigma2, -1. / (sigma2 * var), (cov_type == gpb::COV_GAUSSIAN ? 2. : 1.) / rho};
  const int qa[6] = {0, 0, 0, 1, 1, 2}, qb[6] = {0, 1, 2, 1, 2, 2};
  for (int q = 0; q < 6; ++q) {
    const double v = tot[q] / (double)t / 2. * fac[qa[q]] * fac[qb[q]];
    FI9[qa[q] * 3 + qb[q]] = v;
    FI9[qb[q] * 3 + qa[q]] = v;
  }
  return 0;
}

}  // extern "C"
