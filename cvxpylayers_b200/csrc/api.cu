// api.cu -- the C ABI of libbcone.so (declared in include/bcone.h): handle management,
// structure upload, launch geometry, and the five entry points the reference-side binding
// calls.  No torch types, no exceptions across the boundary.
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include <cstdlib>
#include "common.cuh"

namespace {
// One kernel's launch plan: its address (from the bc_*_kernel lookup of its file), block size, dynamic shared memory and the
// CTAs one SM keeps resident (>= 1 once configured).
struct Plan { const void *fn = nullptr; int threads = 0; size_t smem = 0; int ctas = 0; };
cudaError_t configure(Plan &p) {
  if (!p.fn) return cudaErrorInvalidDeviceFunction;   // no such instantiation
  const cudaError_t e = cudaFuncSetAttribute(p.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem);
  if (e != cudaSuccess) return e;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&p.ctas, p.fn, p.threads, p.smem) != cudaSuccess || p.ctas < 1) p.ctas = 1;
  return cudaSuccess;
}
// args: the kernel's one argument block (FwdArgs / BwdArgs)
cudaError_t launch(const Plan &p, int grid, const void *args, cudaStream_t st) {
  void *argv[] = {const_cast<void *>(args)};
  cudaLaunchKernel(p.fn, dim3(grid), dim3(p.threads), argv, p.smem, st);
  return cudaGetLastError();   // (read and cleared: not left for the caller's next CUDA call)
}
int grid_for(const Plan &p, int B, int num_sms) { return std::min(B, num_sms * p.ctas); }

// A generic kernel's plan.  <= 256-thread instances have a second build of the generic kernels for four resident CTAs per SM
// (64 registers).  It wins when the batch exceeds what the 128-register build keeps resident (more CTAs overlap each other's
// stalls: exp-cone workload) and loses when every instance is resident anyway and only its own latency counts (SDP at B = 256),
// so the choice is made per launch from the batch size.  BCONE_SMALL_CTA=0 disables, =2 forces.
struct TieredPlan {
  Plan big, small;
  bool has_small = false;
  int indirect = 0;        // forward, large instances: CG instead of Cholesky, vectors in a global slab
  int factor_global = 0;   // forward, in between: values on chip, vectors + packed Cholesky factor in the slab (direct solve from L2 / HBM)
  int p_in_smem = 0, vec_global = 0;   // LSQR: P staged in shared memory; large instances: vectors in a global slab
  // values off chip (the tier after every on-chip option): the forward copies each instance's CSR values into its CTA's slab,
  // the backward / forward-mode LSQR reads them in place from A_vals.  Only 512-thread builds exist for it (no small variant).
  int vals_global = 0;
  size_t ws_stride = 0;    // doubles of slab per CTA
};
// the 4-CTA/SM build only when the batch does not fit the resident capacity of the 128-register build
const Plan &pick(const TieredPlan &t, int B, int num_sms, int small_mode) {
  return t.has_small && (small_mode == 2 || B > num_sms * t.big.ctas) ? t.small : t.big;
}
// CTAs of the largest grid either build launches: what the per-CTA slabs are sized for
size_t max_grid(const TieredPlan &t, int num_sms) { return (size_t)num_sms * std::max(t.big.ctas, t.has_small ? t.small.ctas : 0); }

// The backward plans of one least-squares method (settings.lsmr: [0] LSQR, [1] LSMR), each with a flag saying it exists.
// gen / jvp: the generic kernel (bwd.cu) as the adjoint and as the forward mode; fast: the fused single-pass adjoint (bwd_fast.cu;
// dense A, polyhedral cones, dense-or-no P), which runs instead of gen where it exists; block: the KKT-block preconditioned
// adjoint (bwd_block.cu, lsqr_precond = 2), whose rejected instances take a second pass on fast, else gen.
struct LsPlans {
  TieredPlan gen, jvp;
  Plan fast, block;
  bool gen_ok = false, jvp_ok = false, fast_ok = false, block_ok = false;
};

struct Handle {
  DevStruct S{};
  int device = 0, max_batch = 0, num_sms = 0;
  std::vector<void *> allocs;
  static constexpr int RING = 16;  // concurrent calls on different streams each get their own work-queue counters
  int *counters = nullptr;  // RING x {fwd queue, bwd queue, fail count, fallback queue}
  int slot = 0;
  int nnz_aug = 0, nb = 0;
  int *d_gather = nullptr, *d_bidx = nullptr;
  int *d_gatherP = nullptr; int nnzP_b = -1;   // boundary rows of P_eval feeding the engine's upper-triangular slots (bcone_set_boundary_quad)
  // parameter -> matrix maps (bcone_set_param_maps): CSR [rows x P1] per boundary tensor, device copies
  struct PMap { int *ptr = nullptr, *col = nullptr; double *val = nullptr; int rows = 0; };
  PMap pmA, pmq, pmP;
  int P1 = 0;
  int tma_ok = 0, psd_total = 0;
  // Launch plans, chosen once in bcone_create.  The generic forward (fwd.cu) has a TieredPlan; fast_fwd says where the
  // register-tiled forward runs instead.  The backward plans are per least-squares method.
  TieredPlan fwd;
  Plan fwd_fast;    // fast_fwd: dense A, polyhedral cones, direct mode: register-tiled forward (fwd_fast.cu)
  int fast_fwd = 0;
  LsPlans ls[2];
  // solution polishing: planned only for zero + nonneg cones; otherwise polish_why says why.  Tier 0 (polish.cu): on chip, for
  // n <= 128 when it fits; tier 1 (polish_large.cu): everything else, with each CTA's working set in a slab of global memory.
  Plan polish;
  int polish_ok = 0, polish_tier = -1;
  long long polish_stage = 0;   // tier 0: doubles of its staging buffer (live rows of A, then W and S)
  long long polish_slab = 0;    // tier 1: doubles of slab per CTA
  int polish_ctas = 0;          // tier 1: CTAs of the grid (the SM count, fewer when the slabs would exceed the budget)
  int p_diag = 1;               // no P, or only diagonal entries (the slab tier's L_P is then a vector)
  std::string polish_why;
  // solution refinement (refine.cu): the forward mode's tiers with the refinement kernel's sizes; refine_why when it does not fit
  TieredPlan refine;
  int refine_ok = 0, refine_last_small = -1;   // (the build the last bcone_refine launch took: bcone_refine_info)
  std::string refine_why;
  int small_mode = 1;   // BCONE_SMALL_CTA: 0 disables the 4-CTA/SM builds, 2 forces them
  // Per-stream scratch slabs (one per CTA of the grid): launches on different streams may overlap, launches on one
  // stream cannot, so the stream is the unit of ownership.  Allocated on first use.
  // shared matrices: setup = the batch's one set-up record of the register-tiled forward (+ the outputs of its set-up launch),
  // srec / part = the adjoint's per-instance r, pi_y records and the reduction's partial sums (shared.cu)
  // bwd / jvp: the generic backward's vector slabs, per least-squares method
  struct StreamWs { cudaStream_t s; double *fwd = nullptr, *aa = nullptr, *park = nullptr; size_t aa_cap = 0;
                    double *bwd[2] = {nullptr, nullptr}, *jvp[2] = {nullptr, nullptr}, *refine = nullptr, *polish = nullptr;
                    double *setup = nullptr, *srec = nullptr, *part = nullptr; size_t srec_cap = 0, part_cap = 0; };
  std::vector<StreamWs> sws;
  int *fail_list[RING] = {nullptr}; int fail_cap[RING] = {0};
  long long launches = 0;
  int last_block_slot = -1;   // ring slot of the last block-preconditioned vjp (its fallback counter is read by bcone_fallback_count)
  unsigned long long *prof = nullptr;   // device [32] phase cycle counters (bcone_set_profile)
  std::string err;
  bool upload_failed = false;   // set by upload(), read and cleared by upload_status()
};
thread_local std::string g_create_err;

int fail(Handle *h, int code, const std::string &msg) {
  if (h) h->err = msg; else g_create_err = msg;
  return code;
}
int cuda_fail(Handle *h, cudaError_t e, const char *where) {
  return fail(h, BCONE_ECUDA, std::string(where) + ": " + cudaGetErrorString(e));
}
// Device copy of v (nullptr for an empty one).  A failed allocation or copy returns nullptr too and is recorded on the handle:
// callers upload everything they need and then ask upload_status() once.
template <class T>
T *upload(Handle *h, const std::vector<T> &v) {
  if (v.empty()) return nullptr;
  void *p = nullptr;
  cudaError_t e = cudaMalloc(&p, v.size() * sizeof(T));
  if (e == cudaSuccess) {
    h->allocs.push_back(p);
    e = cudaMemcpy(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice);
  }
  if (e == cudaSuccess) return (T *)p;
  cudaGetLastError();   // (not left for the next launch check)
  h->upload_failed = true;
  h->err = std::string("upload of ") + std::to_string(v.size() * sizeof(T)) + " B failed: " + cudaGetErrorString(e);
  return nullptr;
}
// BCONE_ENOMEM (message in h->err) if an upload since the last call failed
int upload_status(Handle *h) {
  const bool failed = h->upload_failed;
  h->upload_failed = false;
  return failed ? BCONE_ENOMEM : BCONE_OK;
}
Handle::StreamWs *stream_ws(Handle *h, cudaStream_t s) {
  for (auto &w : h->sws) if (w.s == s) return &w;
  Handle::StreamWs w; w.s = s;
  h->sws.push_back(w);
  return &h->sws.back();
}
// slab of `doubles` per CTA for `ctas` CTAs; *cap tracks the current size in doubles (0: fixed-size slab)
bool ensure_slab(Handle *h, double **p, size_t *cap, size_t doubles) {
  if (*p && (!cap || *cap >= doubles)) return true;
  double *q = nullptr;
  if (cudaMalloc((void **)&q, doubles * sizeof(double)) != cudaSuccess) { cudaGetLastError(); return false; }   // (not left for the next launch check)
  h->allocs.push_back(q);   // (an outgrown slab stays alive until destroy: a kernel in flight may still use it)
  *p = q;
  if (cap) *cap = doubles;
  return true;
}
}  // namespace

extern "C" void bcone_default_settings(bcone_settings *st) {
  st->eps_abs = 1e-4; st->eps_rel = 1e-4; st->eps_infeas = 1e-7;
  st->alpha = 1.5; st->rho_x = 1e-6; st->scale = 0.1;
  st->lsqr_atol = 1e-8; st->lsqr_btol = 1e-8; st->lsqr_conlim = 1e8;
  st->max_iters = 100000; st->normalize = 1; st->adaptive_scale = 1; st->check_interval = 25;
  st->ruiz_passes = 10; st->lsqr_iter_lim = -1; st->lsqr_precond = 0; st->adaptive_check = 0;
  st->acceleration_lookback = 10; st->acceleration_interval = 10;   // SCS defaults
  st->lsmr = 0;
}

extern "C" const char *bcone_last_error(void *handle) {
  return handle ? ((Handle *)handle)->err.c_str() : g_create_err.c_str();
}

namespace {
// The BCONE_EINVAL checks of bcone_create: nothing is allocated before they pass.  nullptr = valid.
const char *validate(const bcone_desc *d) {
  if (d->n <= 0 || d->m < 0 || d->nnzA < 0 || !d->A_indptr || (d->nnzA > 0 && !d->A_indices)) return "bad dimensions / missing A structure";
  if (d->ep < 0 || d->ed < 0) return "negative cone count";
  const int n = d->n, m = d->m;
  long long rows = d->z + d->l + 3LL * (d->ep + d->ed);
  for (int i = 0; i < d->nq; i++) rows += d->q[i];
  for (int i = 0; i < d->ns; i++) rows += (long long)d->s[i] * (d->s[i] + 1) / 2;
  if (rows != m) return "cone dimensions do not add up to m";
  if (d->A_indptr[0] != 0 || d->A_indptr[m] != d->nnzA) return "A_indptr inconsistent with nnzA";
  for (int i = 0; i < m; i++) {
    if (d->A_indptr[i + 1] < d->A_indptr[i] || d->A_indptr[i + 1] > d->nnzA) return "A_indptr not monotone";   // (it ends at nnzA)
    for (int k = d->A_indptr[i]; k < d->A_indptr[i + 1]; k++)
      if (d->A_indices[k] < 0 || d->A_indices[k] >= n) return "A column index out of range";
  }
  if (d->P_indptr && d->nnzP > 0)
    for (int i = 0; i < n; i++) for (int k = d->P_indptr[i]; k < d->P_indptr[i + 1]; k++)
      if (d->P_indices[k] < i || d->P_indices[k] >= n) return "P must be upper triangular CSR";
  return nullptr;
}

// Host-side structure analysis (CSR -> CSC views, dense-pattern detection, cone block table) and its upload into h->S.
// The caller checks upload_status() afterwards.
void analyse_and_upload(Handle *h, const bcone_desc *d) {
  const int n = d->n, m = d->m;
  DevStruct &S = h->S;
  S.n = n; S.m = m; S.nnzA = d->nnzA; S.nnzP = d->P_indptr ? d->nnzP : 0;
  S.z = d->z; S.l = d->l; S.nq = d->nq; S.ns = d->ns;
  S.ep = d->ep; S.ed = d->ed;
  std::vector<int> indptr(d->A_indptr, d->A_indptr + m + 1), indices(d->A_indices, d->A_indices + d->nnzA);
  std::vector<int> rowof(d->nnzA), colptr(n + 1, 0), rowidx(d->nnzA), perm(d->nnzA);
  bool dense = (long long)d->nnzA == (long long)m * n && d->nnzA > 0;
  for (int i = 0; i < m; i++) {
    for (int k = indptr[i]; k < indptr[i + 1]; k++) {
      int j = indices[k];
      rowof[k] = i; colptr[j + 1]++;
      if (dense && j != k - indptr[i]) dense = false;
    }
    if (dense && indptr[i + 1] - indptr[i] != n) dense = false;
  }
  for (int j = 0; j < n; j++) colptr[j + 1] += colptr[j];
  {
    std::vector<int> fill(colptr.begin(), colptr.end() - 1);
    for (int k = 0; k < d->nnzA; k++) { int p = fill[indices[k]]++; rowidx[p] = rowof[k]; perm[p] = k; }
  }
  S.dense = dense ? 1 : 0;
  std::vector<int> ctype, cstart, csize, corder;
  int off = d->z + d->l;
  for (int i = 0; i < d->nq; i++) { ctype.push_back(BC_CSOC); cstart.push_back(off); csize.push_back(d->q[i]); corder.push_back(0); off += d->q[i]; }
  for (int i = 0; i < d->ns; i++) {
    int k = d->s[i], sz = k * (k + 1) / 2;
    ctype.push_back(BC_CPSD); cstart.push_back(off); csize.push_back(sz); corder.push_back(k); off += sz;
    S.max_psd = std::max(S.max_psd, k); h->psd_total += k * k + k;
  }
  S.exp_start = off;
  S.ncones = (int)ctype.size();
  S.A_indptr = upload(h, indptr); S.A_indices = upload(h, indices); S.A_rowof = upload(h, rowof);
  S.At_colptr = upload(h, colptr); S.At_rowidx = upload(h, rowidx); S.At_perm = upload(h, perm);
  S.cone_type = upload(h, ctype); S.cone_start = upload(h, cstart); S.cone_size = upload(h, csize); S.cone_order = upload(h, corder);
  if (S.nnzP > 0) {
    std::vector<int> pptr(d->P_indptr, d->P_indptr + n + 1), pidx(d->P_indices, d->P_indices + S.nnzP), prow(S.nnzP);
    for (int i = 0; i < n; i++) for (int k = pptr[i]; k < pptr[i + 1]; k++) { prow[k] = i; if (pidx[k] != i) h->p_diag = 0; }
    S.P_indptr = upload(h, pptr); S.P_indices = upload(h, pidx); S.P_rowof = upload(h, prow);
    // CSC view of the upper triangle + dense-pattern detection (row-major full upper triangle)
    std::vector<int> pc(n + 1, 0), pr(S.nnzP), pp(S.nnzP);
    bool pd = (long long)S.nnzP == (long long)n * (n + 1) / 2;
    for (int i = 0; i < n; i++) {
      if (pd && pptr[i + 1] - pptr[i] != n - i) pd = false;
      for (int k = pptr[i]; k < pptr[i + 1]; k++) { pc[pidx[k] + 1]++; if (pd && pidx[k] != i + (k - pptr[i])) pd = false; }
    }
    for (int j = 0; j < n; j++) pc[j + 1] += pc[j];
    { std::vector<int> fill(pc.begin(), pc.end() - 1); for (int k = 0; k < S.nnzP; k++) { int p = fill[pidx[k]]++; pr[p] = prow[k]; pp[p] = k; } }
    S.Pt_colptr = upload(h, pc); S.Pt_rowidx = upload(h, pr); S.Pt_perm = upload(h, pp);
    S.p_dense = pd ? 1 : 0;
  }
}

// What the tier searches start from, besides the structure in h->S.
struct Limits {
  size_t smem_cap;   // opt-in shared memory per block: must hold what a tier keeps on chip
  int threads;       // by problem size; the searches halve it down to 64
  // Last tier, for instances whose CSR values do not fit next to the rest: the values in global memory (L2 when the grid's
  // working set fits, HBM otherwise), the same rule for everything else.  Tried only after every on-chip option has failed;
  // BCONE_VALUES_GLOBAL=1 selects it for every generic kernel of a structure that would fit on chip (a test hook).
  int vals_lo;
};
Limits limits(const Handle *h, size_t smem_cap) {
  const DevStruct &S = h->S;
  int threads = S.nnzA >= 8192 ? 512 : (S.nnzA >= 1024 ? 256 : 128);
  while (threads < 512 && threads < S.n) threads *= 2;  // transposed products want one lane per column
  const char *vgv = getenv("BCONE_VALUES_GLOBAL");
  return {smem_cap, threads, (vgv && atoi(vgv)) ? 1 : 0};
}

// Configures t.big (its fn, threads and smem are set) and, where it applies and keeps more CTAs resident, the 4-CTA/SM build.
cudaError_t configure_tiers(const Handle *h, TieredPlan &t, const void *small_fn) {
  const cudaError_t e = configure(t.big);
  if (e != cudaSuccess) return e;
  if (h->small_mode != 0 && !t.vals_global && t.big.threads <= 256 && t.big.smem <= 56 * 1024) {
    t.small = t.big; t.small.fn = small_fn;
    t.has_small = configure(t.small) == cudaSuccess && t.small.ctas > t.big.ctas;
  }
  return cudaSuccess;
}

// Forward: BCONE_OK, BCONE_EUNSUPPORTED (no tier fits) or BCONE_ECUDA (message set).
int plan_forward(Handle *h, const Limits &L) {
  const DevStruct &S = h->S;
  const int n = S.n, m = S.m, nexp = S.ep + S.ed;
  // DIRECT (everything on chip) if the instance fits; else values on chip with the vectors and the packed Cholesky factor
  // in a per-CTA slab of global memory (two triangular products per iteration read it from L2: n <= 512, i.e. <= 1 MB
  // per CTA); else INDIRECT (conjugate gradients, SCS's "indirect" mode).  BCONE_FWD_MODE=indirect forces the last one.
  const char *fm = getenv("BCONE_FWD_MODE");
  const bool force_indirect = fm && std::string(fm) == "indirect";
  TieredPlan &t = h->fwd;
  for (int vals = L.vals_lo; vals <= 1 && !t.big.threads; vals++)
    for (int ind = 0; ind <= 1 && !t.big.threads; ind++)
      for (int tt = L.threads; tt >= 64; tt /= 2) {
        size_t sm = bc_fwd_smem_bytes(n, m, S.nnzA, tt, S.max_psd, ind, S.ns, nexp, vals);
        if (sm <= L.smem_cap) {
          t.big.threads = tt; t.big.smem = sm; t.indirect = ind; t.vals_global = vals;
          // (n <= 512: one thread per column in the transposed triangular product; on the sparse LP with n = 1000 the slab mode
          //  streams 8 MB of factor per iteration and CTA from HBM and loses to conjugate gradients, while at n = 101 the factor
          //  stays in L2 and the slab mode wins by a wide margin)
          if (ind && !force_indirect && n <= 512) { t.indirect = 0; t.factor_global = 1; }
          break;
        }
      }
  if (!t.big.threads) return BCONE_EUNSUPPORTED;
  // register-tiled forward (fwd_fast.cu) when the structure allows it; BCONE_NO_FAST_FWD=1 keeps the generic kernel
  if (S.dense && S.ncones == 0 && nexp == 0 && !t.indirect && !t.factor_global && bc_fwdf_eligible(n, m) &&
      bc_fwdf_smem_bytes(n, m) <= L.smem_cap && !(getenv("BCONE_NO_FAST_FWD") && atoi(getenv("BCONE_NO_FAST_FWD")))) {
    h->fwd_fast = Plan{bc_fwdf_kernel(n, m), bc_fwdf_threads(), bc_fwdf_smem_bytes(n, m)};
    if (configure(h->fwd_fast) == cudaSuccess) { h->fast_fwd = 1; t = TieredPlan(); return BCONE_OK; }   // (the generic kernel is then never launched)
  }
  t.big.fn = bc_fwd_kernel(S.dense, t.indirect, 0, t.vals_global);
  const cudaError_t e = configure_tiers(h, t, bc_fwd_kernel(S.dense, t.indirect, 1, t.vals_global));
  if (e != cudaSuccess) return cuda_fail(nullptr, e, "cudaFuncSetAttribute");
  if (t.indirect || t.factor_global || t.vals_global)
    t.ws_stride = bc_fwd_ws_doubles(n, m, t.indirect || t.factor_global, t.factor_global, t.vals_global ? S.nnzA : 0);
  return BCONE_OK;
}

// Generic LSQR kernel (bwd.cu), as the adjoint or as the forward mode, or its LSMR variant (lsmr = 1), or the refinement
// kernel (refine = 1: the forward mode's kernel with the refinement's vectors, refine.cu): prefer P staged in shared memory, then
// vectors on chip, then vectors in L2; values off chip last.  BCONE_OK, BCONE_EUNSUPPORTED (no tier fits) or BCONE_ECUDA
// (message set).
int plan_lsqr(Handle *h, const Limits &L, TieredPlan &t, int jvp, int lsmr, int refine = 0) {
  const DevStruct &S = h->S;
  const int npoly = S.z + S.l;
  auto smem = [&](int psm, int tt, int vg, int vals) {
    const int nnzP = psm ? S.nnzP : 0, nexp = S.ep + S.ed;
    return refine ? bc_refine_smem_bytes(S.n, S.m, npoly, S.nnzA, nnzP, tt, S.max_psd, h->psd_total, nexp, vg, vals)
                  : bc_bwd_smem_bytes(S.n, S.m, npoly, S.nnzA, nnzP, tt, S.max_psd, h->psd_total, nexp, vg, vals, lsmr);
  };
  auto kernel = [&](int small) { return refine ? bc_refine_kernel(S.dense, small, t.vals_global) : bc_lsqr_kernel(S.dense, small, jvp, t.vals_global, lsmr); };
  for (int vals = L.vals_lo; vals <= 1 && !t.big.threads; vals++)
    for (int vg = 0; vg <= 1 && !t.big.threads; vg++)
      for (int psm = (S.nnzP > 0 ? 1 : 0); psm >= 0 && !t.big.threads; psm--)
        for (int tt = L.threads; tt >= 64; tt /= 2) {
          size_t sm = smem(psm, tt, vg, vals);
          if (sm <= L.smem_cap) { t.big.threads = tt; t.big.smem = sm; t.p_in_smem = psm; t.vec_global = vg; t.vals_global = vals; break; }
          if (psm) break;  // do not trade threads for P residency
        }
  if (!t.big.threads) return BCONE_EUNSUPPORTED;
  t.big.fn = kernel(0);
  const cudaError_t e = configure_tiers(h, t, kernel(1));
  if (e != cudaSuccess) return cuda_fail(nullptr, e, "cudaFuncSetAttribute");
  if (t.vec_global) t.ws_stride = refine ? bc_refine_ws_doubles(S.n, S.m, npoly) : bc_bwd_ws_doubles(S.n, S.m, npoly, lsmr);
  return BCONE_OK;
}

// The backward plans of one least-squares method (lsmr: LSMR, whose kernels keep one more N-vector), planned after LSQR's.
// The fused adjoint where the structure allows it and it fits (needing N more doubles at the same thread count, LSMR's exists
// only where LSQR's does); the block-preconditioned adjoint on top of LSQR's fused one, for strongly convex QPs (LSMR's where
// LSQR's configured: its shared memory does not depend on the method); the generic adjoint where there is no fused one; the
// generic forward mode always.  Returns the adjoint's BCONE_OK, BCONE_EUNSUPPORTED (no tier fits) or BCONE_ECUDA (message set);
// only LSQR's adjoint is required (bcone_create fails without it), so for LSMR a missing fused plan falls back to the generic
// one, and a missing adjoint disables the block pass (there is no pass for the instances it rejects).
int plan_backward(Handle *h, const Limits &L, int lsmr) {
  const DevStruct &S = h->S;
  const int n = S.n, m = S.m;
  LsPlans &p = h->ls[lsmr];
  if (S.dense && S.ncones == 0 && S.ep + S.ed == 0 && n <= 128 && (n % 2) == 0 && (S.nnzP == 0 || S.p_dense))
    for (int tt = L.threads; tt >= 64; tt /= 2) {
      const size_t sm = bc_bwdf_smem_bytes(n, m, S.nnzA, S.nnzP, tt, lsmr);
      if (sm <= L.smem_cap) {
        p.fast = Plan{bc_bwdf_kernel(n, lsmr), tt, sm};
        const cudaError_t e = configure(p.fast);
        if (e != cudaSuccess && !lsmr) return cuda_fail(nullptr, e, "cudaFuncSetAttribute");
        p.fast_ok = e == cudaSuccess;
        break;
      }
    }
  if (h->ls[0].fast_ok && (!lsmr || h->ls[0].block_ok) && S.nnzP > 0 && 6 * (n + m + 1) >= 8 * n + 72)
    for (int tt = L.threads; tt >= 128; tt /= 2) {
      const size_t sm = bc_bwdb_smem_bytes(n, m, tt);
      if (sm <= L.smem_cap) { p.block = Plan{bc_bwdb_kernel(lsmr), tt, sm}; p.block_ok = configure(p.block) == cudaSuccess; break; }
    }
  const int rc = p.fast_ok ? BCONE_OK : plan_lsqr(h, L, p.gen, 0, lsmr);
  if (rc != BCONE_OK && !lsmr) return rc;
  p.gen_ok = !p.fast_ok && rc == BCONE_OK;
  if (rc != BCONE_OK) p.block_ok = false;
  p.jvp_ok = plan_lsqr(h, L, p.jvp, 1, lsmr) == BCONE_OK;
  return rc;
}

// Solution polishing, slab tier: one 512-thread CTA per SM, each with a slab of global memory for the instance's live rows,
// vectors, L_P^{-1}, W and S (bc_polish_large_slab_doubles).  The slabs of the grid stay within min(4 GB, half the device memory
// free at bcone_create): fewer CTAs when they would not, no plan when one slab alone would not.
void plan_polish_slab(Handle *h) {
  const DevStruct &S = h->S;
  const int tt = bc_polish_large_threads();
  const long long per = bc_polish_large_slab_doubles(S.n, S.m, tt, h->p_diag);
  size_t free_b = 0, total_b = 0;
  if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) { cudaGetLastError(); free_b = 0; }
  const size_t budget = std::min((size_t)4 << 30, free_b / 2), bytes = (size_t)per * sizeof(double);
  if (bytes > budget) {
    h->polish_why = "polish: the working set of one instance needs " + std::to_string(bytes) + " B of global memory, more than the budget of " +
                    std::to_string(budget) + " B (min(4 GB, half the free device memory))";
    return;
  }
  Plan p{bc_polish_large_kernel(S.dense), tt, bc_polish_large_smem_bytes(tt)};
  if (configure(p) != cudaSuccess) { h->polish_why = "polish: kernel configuration failed"; return; }
  h->polish = p; h->polish_ok = 1; h->polish_tier = 1; h->polish_slab = per;
  h->polish_ctas = (int)std::max<size_t>(1, std::min<size_t>((size_t)h->num_sms * p.ctas, budget / bytes));
}

// Solution polishing: zero + nonneg cones (a finite active set).  On chip (polish.cu) for n <= 128 (W = L^{-1} A_L' is formed
// with 8 rows of A in a warp's registers): the staging buffer holds the live rows (at most min(m, n)), then W and S; it is as
// large as that needs or as what is left of the opt-in shared memory, and an instance whose W and S do not fit it is not
// attempted.  Every other such structure takes the slab tier.  Sets h->polish_ok, or h->polish_why.  Never fails bcone_create.
void plan_polish(Handle *h, const Limits &L) {
  const DevStruct &S = h->S;
  const int n = S.n, m = S.m;
  if (S.ncones > 0 || S.ep + S.ed > 0) { h->polish_why = "polish: only structures with zero and nonneg cones have a finite active set to polish (this one has SOC, PSD or exponential cones)"; return; }
  if (n <= 128) {
    const long long k = std::min(m, n), full = k * n + k * (k + 1) / 2;
    for (int tt = L.threads; tt >= 128; tt /= 2) {
      const size_t base = bc_polish_smem_bytes(n, m, tt, 0);
      if (base > L.smem_cap) continue;
      const long long cap = std::min(full, (long long)((L.smem_cap - base) / sizeof(double)) & ~1LL);
      if (cap < std::min(full, (long long)n + 1)) continue;   // (not even one live row)
      h->polish = Plan{bc_polish_kernel(S.dense), tt, bc_polish_smem_bytes(n, m, tt, cap)};
      if (configure(h->polish) != cudaSuccess) { h->polish_why = "polish: kernel configuration failed"; return; }
      h->polish_ok = 1; h->polish_stage = cap; h->polish_tier = 0;
      return;
    }
  }
  plan_polish_slab(h);
}

// Solution refinement: the forward mode's tier search with the refinement kernel's sizes (every cone type has one).  Sets
// h->refine_ok, or h->refine_why.  Never fails bcone_create: refinement is optional like the forward-mode plans.
void plan_refine(Handle *h, const Limits &L) {
  const int rc = plan_lsqr(h, L, h->refine, 1, 0, 1);
  h->refine_ok = rc == BCONE_OK;
  if (rc == BCONE_EUNSUPPORTED) h->refine_why = "refine: the instance does not fit the refinement kernel, even with the values and vectors in global memory";
  else if (rc != BCONE_OK) h->refine_why = "refine: kernel configuration failed (" + g_create_err + ")";
}

// With values and vectors off chip, what is left in shared memory is the per-CTA scratch: the cone scratch (per-warp PSD
// scratch, persistent eigenvectors, exp-cone slots) and the 8 n column partials.  Name the largest PSD order that would fit.
std::string explain_no_fit(const Handle *h, const bcone_desc *d, size_t smem_cap) {
  const DevStruct &S = h->S;
  const int n = S.n, m = S.m, max_psd = S.max_psd;
  auto need = [&](int k, size_t *f, size_t *b) {
    int pt = 0;
    for (int i = 0; i < d->ns; i++) { const int kk = std::min(d->s[i], k); pt += kk * kk + kk; }
    *f = bc_fwd_smem_bytes(n, m, d->nnzA, 64, k, 1, k > 0 ? d->ns : 0, d->ep + d->ed, 1);
    *b = bc_bwd_smem_bytes(n, m, S.z + S.l, d->nnzA, 0, 64, k, pt, d->ep + d->ed, 1, 1, 0);
    return *f <= smem_cap && *b <= smem_cap;
  };
  size_t fb = 0, bb = 0, f2 = 0, b2 = 0;
  need(max_psd, &fb, &bb);
  int kfit = -1;
  for (int k = max_psd; k >= 0 && kfit < 0; k--) if (need(k, &f2, &b2)) kfit = k;
  char buf[512];
  if (max_psd > 0 && kfit >= 0)
    snprintf(buf, sizeof buf, "instance does not fit the engine: even with the CSR values and the vectors in global memory, the on-chip cone scratch "
             "(per-warp PSD scratch and persistent eigenvectors of PSD order %d) needs fwd %zu B / bwd %zu B, %zu B per CTA available; "
             "the largest PSD order that fits is %d", max_psd, fb, bb, smem_cap, kfit);
  else
    snprintf(buf, sizeof buf, "instance does not fit the engine: even with the CSR values and the vectors in global memory, the on-chip scratch "
             "(cone scratch and 8 n = %d column partials) needs fwd %zu B / bwd %zu B, %zu B per CTA available", 8 * n, fb, bb, smem_cap);
  return buf;
}
}  // namespace

extern "C" int bcone_create(const bcone_desc *d, void **out) {
  if (!d || !out) return fail(nullptr, BCONE_EINVAL, "null argument");
  *out = nullptr;
  if (const char *bad = validate(d)) return fail(nullptr, BCONE_EINVAL, bad);
  if (cudaSetDevice(d->device) != cudaSuccess) return fail(nullptr, BCONE_ECUDA, "cudaSetDevice failed (no CUDA device?)");
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, d->device) != cudaSuccess) return fail(nullptr, BCONE_ECUDA, "cudaGetDeviceProperties failed");

  Handle *h = new Handle();
  h->device = d->device; h->max_batch = d->max_batch; h->num_sms = prop.multiProcessorCount;
  // from here on: an error leaves through this, with the message kept past the handle
  auto give_up = [&](int code, std::string msg) { bcone_destroy(h); return fail(nullptr, code, msg); };
  analyse_and_upload(h, d);
  if (upload_status(h) != BCONE_OK) return give_up(BCONE_ENOMEM, h->err);
  if (cudaMalloc((void **)&h->counters, Handle::RING * 4 * sizeof(int)) != cudaSuccess) return give_up(BCONE_ENOMEM, "cudaMalloc counters");
  h->allocs.push_back(h->counters);

  // --- launch geometry: threads by problem size, shared memory must hold the whole instance ---
  const Limits L = limits(h, prop.sharedMemPerBlockOptin);
  const char *sc = getenv("BCONE_SMALL_CTA");
  h->small_mode = sc ? atoi(sc) : 1;
  int rc = plan_forward(h, L);
  const int rb = plan_backward(h, L, 0);
  if (rc == BCONE_OK || rb == BCONE_EUNSUPPORTED) rc = rb;   // "does not fit" comes before a CUDA error
  if (rc == BCONE_EUNSUPPORTED) return give_up(rc, explain_no_fit(h, d, L.smem_cap));
  if (rc != BCONE_OK) return give_up(rc, g_create_err);
  h->tma_ok = (d->nnzA > 0 && (d->nnzA % 2) == 0 && (size_t)d->nnzA * 8 < (1u << 20)) ? 1 : 0;
  // A structure without an LSMR adjoint or without a forward-mode geometry (either method) is still accepted; only the calls
  // that need them refuse it.
  plan_backward(h, L, 1);
  plan_polish(h, L);
  plan_refine(h, L);
  cudaGetLastError();   // (a refused configuration is not an error of this call)
  *out = h;
  return BCONE_OK;
}

extern "C" void bcone_destroy(void *handle) {
  if (!handle) return;
  Handle *h = (Handle *)handle;
  cudaSetDevice(h->device);
  for (void *p : h->allocs) cudaFree(p);
  delete h;
}

extern "C" int bcone_set_boundary(void *handle, int32_t nnz_aug, const int32_t *gather, int32_t nb, const int32_t *b_idx) {
  Handle *h = (Handle *)handle;
  if (!h) return BCONE_EINVAL;
  if (nnz_aug != h->S.nnzA + nb || (h->S.nnzA > 0 && !gather) || (nb > 0 && !b_idx)) return fail(h, BCONE_EINVAL, "set_boundary: inconsistent sizes");
  for (int k = 0; k < h->S.nnzA; k++) if (gather[k] < 0 || gather[k] >= h->S.nnzA) return fail(h, BCONE_EINVAL, "set_boundary: gather out of range");
  for (int r = 0; r < nb; r++) if (b_idx[r] < 0 || b_idx[r] >= h->S.m) return fail(h, BCONE_EINVAL, "set_boundary: b_idx out of range");
  cudaSetDevice(h->device);
  h->nnz_aug = h->nb = 0;   // (until the maps are in place: ingest then asks for this call again)
  h->d_gather = upload(h, std::vector<int>(gather, gather + h->S.nnzA));
  h->d_bidx = upload(h, std::vector<int>(b_idx, b_idx + nb));
  if (upload_status(h) != BCONE_OK) return BCONE_ENOMEM;
  h->nnz_aug = nnz_aug; h->nb = nb;
  return BCONE_OK;
}

extern "C" int bcone_set_boundary_quad(void *handle, int32_t nnzP_boundary, const int32_t *gatherP) {
  Handle *h = (Handle *)handle;
  if (!h) return BCONE_EINVAL;
  if (h->S.nnzP > 0 && (!gatherP || nnzP_boundary < 1)) return fail(h, BCONE_EINVAL, "set_boundary_P: missing gather map");
  for (int k = 0; k < h->S.nnzP; k++) if (gatherP[k] < 0 || gatherP[k] >= nnzP_boundary) return fail(h, BCONE_EINVAL, "set_boundary_P: gather out of range");
  cudaSetDevice(h->device);
  h->nnzP_b = -1;
  h->d_gatherP = h->S.nnzP > 0 ? upload(h, std::vector<int>(gatherP, gatherP + h->S.nnzP)) : nullptr;
  if (upload_status(h) != BCONE_OK) return BCONE_ENOMEM;
  h->nnzP_b = nnzP_boundary;
  return BCONE_OK;
}

#define CK(call, where) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return cuda_fail(h, e_, where); } while (0)

// ---- parameter -> matrix affine map fused into ingest / emit (SURVEY.md 8f.1) ----
extern "C" int bcone_set_param_maps(void *handle, int32_t P1, const int32_t *A_ptr, const int32_t *A_col, const double *A_val,
                                    const int32_t *q_ptr, const int32_t *q_col, const double *q_val,
                                    const int32_t *P_ptr, const int32_t *P_col, const double *P_val) {
  Handle *h = (Handle *)handle;
  if (!h || P1 <= 0 || !A_ptr || !q_ptr) return fail(h, BCONE_EINVAL, "set_param_maps: null argument");
  if (h->nnz_aug == 0 && h->S.nnzA + h->nb != 0) return fail(h, BCONE_EINVAL, "set_param_maps: call bcone_set_boundary first");
  const DevStruct &S = h->S;
  const int rowsA = h->nnz_aug, rowsq = S.n + 1, rowsP = (P_ptr && S.nnzP > 0) ? (h->nnzP_b > 0 ? h->nnzP_b : S.nnzP) : 0;
  const int32_t *ptrs[3] = {A_ptr, q_ptr, P_ptr}, *colsv[3] = {A_col, q_col, P_col};
  const double *valsv[3] = {A_val, q_val, P_val};
  const int rows[3] = {rowsA, rowsq, rowsP};
  std::vector<int> count(P1, 0);
  for (int w = 0; w < 3; w++) {
    if (!rows[w]) continue;
    if (ptrs[w][0] != 0) return fail(h, BCONE_EINVAL, "set_param_maps: row pointer must start at 0");
    for (int r = 0; r < rows[w]; r++) if (ptrs[w][r + 1] < ptrs[w][r]) return fail(h, BCONE_EINVAL, "set_param_maps: row pointer not monotone");
    const int nz = ptrs[w][rows[w]];
    if (nz > 0 && (!colsv[w] || !valsv[w])) return fail(h, BCONE_EINVAL, "set_param_maps: missing column / value array");
    for (int e = 0; e < nz; e++) {
      if (colsv[w][e] < 0 || colsv[w][e] >= P1) return fail(h, BCONE_EINVAL, "set_param_maps: parameter index out of range");
      count[colsv[w][e]]++;
    }
  }
  cudaSetDevice(h->device);
  Handle::PMap *dst[3] = {&h->pmA, &h->pmq, &h->pmP};
  h->P1 = 0;   // (until all three maps are in place)
  for (int w = 0; w < 3; w++) {
    *dst[w] = Handle::PMap();
    if (!rows[w]) continue;
    const int nz = ptrs[w][rows[w]];
    std::vector<int> ptr(ptrs[w], ptrs[w] + rows[w] + 1), col(std::max(nz, 1), 0);
    std::vector<double> val(std::max(nz, 1), 0.0);
    for (int e = 0; e < nz; e++) { col[e] = colsv[w][e] | (count[colsv[w][e]] == 1 ? 0x40000000 : 0); val[e] = valsv[w][e]; }   // bit 30: exclusive column
    dst[w]->ptr = upload(h, ptr); dst[w]->col = upload(h, col); dst[w]->val = upload(h, val); dst[w]->rows = rows[w];
    if (upload_status(h) != BCONE_OK) return BCONE_ENOMEM;
  }
  h->P1 = P1;
  return BCONE_OK;
}

// shared: A_vals / P_vals from column 0 of p_stack only (one copy for the batch), b and c from every column
static int ingest_params(Handle *h, int32_t B, const double *p_stack, double *A_vals, double *P_vals, double *b, double *c, int shared, void *stream) {
  if (!h || B <= 0 || !p_stack || !A_vals || !b || !c) return fail(h, BCONE_EINVAL, "ingest_params: null argument");
  if (h->P1 <= 0) return fail(h, BCONE_EINVAL, "ingest_params: call bcone_set_param_maps first");
  cudaStream_t st = (cudaStream_t)stream;
  const DevStruct &S = h->S;
  const int BM = shared ? 1 : B;   // instances of the matrix values
  CK(bc_p2e(p_stack, h->pmA.ptr, h->pmA.col, h->pmA.val, A_vals, S.nnzA, BM, S.nnzA, 0, h->d_gather, nullptr, -1.0, B, st), "ingest_params A");
  CK(cudaMemsetAsync(b, 0, (size_t)B * S.m * sizeof(double), st), "ingest_params b memset");
  CK(bc_p2e(p_stack, h->pmA.ptr, h->pmA.col, h->pmA.val, b, h->nb, B, S.m, S.nnzA, nullptr, h->d_bidx, 1.0, B, st), "ingest_params b");
  CK(bc_p2e(p_stack, h->pmq.ptr, h->pmq.col, h->pmq.val, c, S.n, B, S.n, 0, nullptr, nullptr, 1.0, B, st), "ingest_params c");
  h->launches += 3;
  if (P_vals && S.nnzP > 0) {
    if (!h->pmP.rows) return fail(h, BCONE_EINVAL, "ingest_params: structure has P but no parameter map for it");
    CK(bc_p2e(p_stack, h->pmP.ptr, h->pmP.col, h->pmP.val, P_vals, S.nnzP, BM, S.nnzP, 0, h->d_gatherP, nullptr, 1.0, B, st), "ingest_params P");
    h->launches++;
  }
  return BCONE_OK;
}
extern "C" int bcone_ingest_params(void *handle, int32_t B, const double *p_stack, double *A_vals, double *P_vals, double *b, double *c, void *stream) {
  return ingest_params((Handle *)handle, B, p_stack, A_vals, P_vals, b, c, 0, stream);
}
extern "C" int bcone_ingest_params_shared(void *handle, int32_t B, const double *p_stack, double *A_vals, double *P_vals, double *b, double *c,
                                          void *stream) {
  return ingest_params((Handle *)handle, B, p_stack, A_vals, P_vals, b, c, 1, stream);
}

// shared: dA_vals / dP_vals are the batch sums [nnzA] / [nnzP], written into column 0 of dp_stack; db, dc into every column
static int emit_params(Handle *h, int32_t B, const double *dA_vals, const double *dP_vals, const double *db, const double *dc, double *dp_stack,
                       int shared, void *stream) {
  if (!h || B <= 0 || !dA_vals || !db || !dc || !dp_stack) return fail(h, BCONE_EINVAL, "emit_params: null argument");
  if (h->P1 <= 0) return fail(h, BCONE_EINVAL, "emit_params: call bcone_set_param_maps first");
  cudaStream_t st = (cudaStream_t)stream;
  const DevStruct &S = h->S;
  const int skip = h->P1 - 1;   // the constant-1 row of p_stack is not a parameter
  CK(cudaMemsetAsync(dp_stack, 0, (size_t)h->P1 * B * sizeof(double), st), "emit_params memset");
  const int BM = shared ? 1 : B;
  CK(bc_e2p(dA_vals, h->pmA.ptr, h->pmA.col, h->pmA.val, dp_stack, S.nnzA, BM, S.nnzA, 0, nullptr, h->d_gather, -1.0, skip, B, st), "emit_params dA");
  CK(bc_e2p(db, h->pmA.ptr, h->pmA.col, h->pmA.val, dp_stack, h->nb, B, S.m, S.nnzA, h->d_bidx, nullptr, 1.0, skip, B, st), "emit_params db");
  CK(bc_e2p(dc, h->pmq.ptr, h->pmq.col, h->pmq.val, dp_stack, S.n, B, S.n, 0, nullptr, nullptr, 1.0, skip, B, st), "emit_params dc");
  h->launches += 3;
  if (dP_vals && S.nnzP > 0 && h->pmP.rows) {
    CK(bc_e2p(dP_vals, h->pmP.ptr, h->pmP.col, h->pmP.val, dp_stack, S.nnzP, BM, S.nnzP, 0, nullptr, h->d_gatherP, 1.0, skip, B, st), "emit_params dP");
    h->launches++;
  }
  return BCONE_OK;
}
extern "C" int bcone_emit_params(void *handle, int32_t B, const double *dA_vals, const double *dP_vals, const double *db, const double *dc,
                                 double *dp_stack, void *stream) {
  return emit_params((Handle *)handle, B, dA_vals, dP_vals, db, dc, dp_stack, 0, stream);
}
extern "C" int bcone_emit_params_shared(void *handle, int32_t B, const double *dA_sum, const double *dP_sum, const double *db, const double *dc,
                                        double *dp_stack, void *stream) {
  return emit_params((Handle *)handle, B, dA_sum, dP_sum, db, dc, dp_stack, 1, stream);
}

extern "C" int bcone_ingest_pitched(void *handle, int32_t B, int64_t ldb, const double *A_eval, const double *q_eval, const double *P_eval,
                                    double *A_vals, double *P_vals, double *b, double *c, void *stream) {
  Handle *h = (Handle *)handle;
  if (!h || B <= 0 || ldb < B || !A_eval || !q_eval || !A_vals || !b || !c) return fail(h, BCONE_EINVAL, "ingest: null argument / bad pitch");
  if (h->nnz_aug == 0 && h->S.nnzA + h->nb != 0) return fail(h, BCONE_EINVAL, "ingest: call bcone_set_boundary first");
  cudaStream_t st = (cudaStream_t)stream;
  const DevStruct &S = h->S;
  CK(bc_b2e(A_eval, A_vals, S.nnzA, B, S.nnzA, 0, h->d_gather, nullptr, -1.0, ldb, st), "ingest A");
  CK(cudaMemsetAsync(b, 0, (size_t)B * S.m * sizeof(double), st), "ingest b memset");
  CK(bc_b2e(A_eval, b, h->nb, B, S.m, S.nnzA, nullptr, h->d_bidx, 1.0, ldb, st), "ingest b");
  CK(bc_b2e(q_eval, c, S.n, B, S.n, 0, nullptr, nullptr, 1.0, ldb, st), "ingest c");
  h->launches += 3;
  if (P_eval && P_vals && S.nnzP > 0) { CK(bc_b2e(P_eval, P_vals, S.nnzP, B, S.nnzP, 0, h->d_gatherP, nullptr, 1.0, ldb, st), "ingest P"); h->launches++; }
  return BCONE_OK;
}
extern "C" int bcone_ingest(void *handle, int32_t B, const double *A_eval, const double *q_eval, const double *P_eval,
                            double *A_vals, double *P_vals, double *b, double *c, void *stream) {
  return bcone_ingest_pitched(handle, B, B, A_eval, q_eval, P_eval, A_vals, P_vals, b, c, stream);
}

extern "C" int bcone_emit_pitched(void *handle, int32_t B, int64_t ldb, const double *dA_vals, const double *dP_vals, const double *db,
                                  const double *dc, double *dA_eval, double *dq_eval, double *dP_eval, void *stream) {
  Handle *h = (Handle *)handle;
  if (!h || B <= 0 || ldb < B || !dA_vals || !db || !dc || !dA_eval || !dq_eval) return fail(h, BCONE_EINVAL, "emit: null argument / bad pitch");
  cudaStream_t st = (cudaStream_t)stream;
  const DevStruct &S = h->S;
  CK(bc_e2b(dA_vals, dA_eval, S.nnzA, B, S.nnzA, 0, nullptr, h->d_gather, -1.0, ldb, st), "emit dA");
  CK(bc_e2b(db, dA_eval, h->nb, B, S.m, S.nnzA, h->d_bidx, nullptr, 1.0, ldb, st), "emit db");
  CK(bc_e2b(dc, dq_eval, S.n, B, S.n, 0, nullptr, nullptr, 1.0, ldb, st), "emit dc");
  CK(cudaMemset2DAsync(dq_eval + (size_t)S.n * ldb, (size_t)ldb * sizeof(double), 0, (size_t)B * sizeof(double), 1, st), "emit dq tail");
  h->launches += 3;
  if (dP_vals && dP_eval && S.nnzP > 0) {
    // boundary rows without an engine slot (the lower triangle of a full symmetric pattern) get a zero gradient:
    // the engine reads the upper triangle only, so that is the derivative of what was computed
    if (h->d_gatherP && h->nnzP_b != S.nnzP)
      CK(cudaMemset2DAsync(dP_eval, (size_t)ldb * sizeof(double), 0, (size_t)B * sizeof(double), (size_t)h->nnzP_b, st), "emit dP memset");
    CK(bc_e2b(dP_vals, dP_eval, S.nnzP, B, S.nnzP, 0, nullptr, h->d_gatherP, 1.0, ldb, st), "emit dP"); h->launches++;
  }
  return BCONE_OK;
}
extern "C" int bcone_emit(void *handle, int32_t B, const double *dA_vals, const double *dP_vals, const double *db,
                          const double *dc, double *dA_eval, double *dq_eval, double *dP_eval, void *stream) {
  return bcone_emit_pitched(handle, B, B, dA_vals, dP_vals, db, dc, dA_eval, dq_eval, dP_eval, stream);
}

// ---- layer prologue / epilogue (SURVEY.md 8f.3): index maps instead of the reference's reshape / permute / cat chains ----
// All pointers are DEVICE pointers (maps: int32, scales: double); no handle, no state.  op: 0 identity, 1 exp, 2 log.
#define CKG(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { g_create_err = std::string(__func__) + ": " + cudaGetErrorString(e_); return BCONE_ECUDA; } } while (0)
extern "C" int bcone_rows_from_param(const double *param, int64_t stride, const int32_t *map, int32_t K, int32_t B, int32_t op, double *rows, void *stream) {
  if (!param || !rows || K < 0 || B < 0) return BCONE_EINVAL;
  CKG(bc_rows_from_param(param, stride, map, K, B, op, rows, (cudaStream_t)stream));
  return BCONE_OK;
}
extern "C" int bcone_param_from_rows(const double *grows, const double *param, int64_t stride, const int32_t *map, int32_t K, int32_t B, int32_t op,
                                     double *gparam, void *stream) {
  if (!grows || !gparam || K < 0 || B < 0 || (op == 2 && !param)) return BCONE_EINVAL;
  CKG(bc_param_from_rows(grows, param, stride, map, K, B, op, gparam, (cudaStream_t)stream));
  return BCONE_OK;
}
extern "C" int bcone_gather_cols(const double *in, int64_t ld, const int32_t *map, const double *scale, int32_t K, int32_t B, int32_t op, double *out, void *stream) {
  if (!in || !out || !map || K < 0 || B < 0) return BCONE_EINVAL;
  CKG(bc_gather_cols(in, ld, map, scale, K, B, op, out, (cudaStream_t)stream));
  return BCONE_OK;
}
extern "C" int bcone_scatter_cols(const double *gout, const double *out, int64_t ld, const int32_t *map, const double *scale, int32_t K, int32_t B, int32_t op,
                                  double *gin, void *stream) {
  if (!gout || !gin || !map || K < 0 || B < 0 || (op == 1 && !out)) return BCONE_EINVAL;
  CKG(bc_scatter_cols(gout, out, ld, map, scale, K, B, op, gin, (cudaStream_t)stream));
  return BCONE_OK;
}

// ---- peer exchange: a buffer on one GPU that every rank of the node can write (CUDA IPC over NVLink) -----------------------
extern "C" int bcone_peer_alloc(int32_t device, int64_t bytes, void **ptr, void *ipc_handle64) {
  if (!ptr || !ipc_handle64 || bytes <= 0) return BCONE_EINVAL;
  if (cudaSetDevice(device) != cudaSuccess) return BCONE_ECUDA;
  void *p = nullptr;
  cudaError_t e = cudaMalloc(&p, (size_t)bytes);
  if (e != cudaSuccess) { g_create_err = std::string("bcone_peer_alloc: ") + cudaGetErrorString(e); return BCONE_ENOMEM; }
  cudaIpcMemHandle_t hnd;
  e = cudaIpcGetMemHandle(&hnd, p);
  if (e != cudaSuccess) { cudaFree(p); g_create_err = std::string("bcone_peer_alloc (ipc handle): ") + cudaGetErrorString(e); return BCONE_ECUDA; }
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "ipc handle size");
  memcpy(ipc_handle64, &hnd, 64);
  *ptr = p;
  return BCONE_OK;
}
extern "C" int bcone_peer_open(int32_t device, const void *ipc_handle64, void **ptr) {
  if (!ptr || !ipc_handle64) return BCONE_EINVAL;
  if (cudaSetDevice(device) != cudaSuccess) return BCONE_ECUDA;
  cudaIpcMemHandle_t hnd;
  memcpy(&hnd, ipc_handle64, 64);
  cudaError_t e = cudaIpcOpenMemHandle(ptr, hnd, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) { g_create_err = std::string("bcone_peer_open: ") + cudaGetErrorString(e); cudaGetLastError(); return BCONE_ECUDA; }
  return BCONE_OK;
}
extern "C" int bcone_peer_close(void *ptr) { return cudaIpcCloseMemHandle(ptr) == cudaSuccess ? BCONE_OK : BCONE_ECUDA; }
extern "C" int bcone_peer_free(void *ptr) { return cudaFree(ptr) == cudaSuccess ? BCONE_OK : BCONE_ECUDA; }
// dst / src: any device pointers of this process' address space (local or peer-mapped); pitches and width in bytes.
// height = 1 is a plain copy.  Runs on the copy engines: no SM is taken from a solve that is in flight.
extern "C" int bcone_copy2d_async(void *dst, int64_t dpitch, const void *src, int64_t spitch, int64_t width, int64_t height, void *stream) {
  cudaError_t e = height <= 1 ? cudaMemcpyAsync(dst, src, (size_t)width, cudaMemcpyDefault, (cudaStream_t)stream)
                              : cudaMemcpy2DAsync(dst, (size_t)dpitch, src, (size_t)spitch, (size_t)width, (size_t)height, cudaMemcpyDefault, (cudaStream_t)stream);
  if (e != cudaSuccess) { g_create_err = std::string("bcone_copy2d_async: ") + cudaGetErrorString(e); return BCONE_ECUDA; }
  return BCONE_OK;
}

extern "C" int bcone_solve_cached(void *handle, int32_t B, const double *A_vals, const double *P_vals, const double *b, const double *c,
                                  const double *x0, const double *y0, const double *s0, double *x, double *y, double *s, int32_t *status,
                                  int32_t *iters, double *resid, void *cache, int32_t reuse, const bcone_settings *stg, void *stream);
extern "C" int bcone_solve_warm(void *handle, int32_t B, const double *A_vals, const double *P_vals, const double *b, const double *c,
                                const double *x0, const double *y0, const double *s0, double *x, double *y, double *s, int32_t *status,
                                int32_t *iters, double *resid, const bcone_settings *stg, void *stream) {
  return bcone_solve_cached(handle, B, A_vals, P_vals, b, c, x0, y0, s0, x, y, s, status, iters, resid, nullptr, 0, stg, stream);
}
extern "C" size_t bcone_cache_bytes(void *handle, int32_t B) {
  Handle *h = (Handle *)handle;
  if (!h || B <= 0 || !h->fast_fwd) return 0;
  return (size_t)B * bc_fwdf_cache_doubles(h->S.n, h->S.m) * sizeof(double);
}
extern "C" int bcone_solve(void *handle, int32_t B, const double *A_vals, const double *P_vals, const double *b,
                           const double *c, double *x, double *y, double *s, int32_t *status, int32_t *iters,
                           double *resid, const bcone_settings *stg, void *stream) {
  return bcone_solve_warm(handle, B, A_vals, P_vals, b, c, nullptr, nullptr, nullptr, x, y, s, status, iters, resid, stg, stream);
}
// shared: A_vals [nnzA] / P_vals [nnzP] are one copy for the whole batch (stride 0); with the register-tiled kernel the batch
// then also shares one set-up (caller's cache must be NULL)
static int solve_impl(Handle *h, int32_t B, const double *A_vals, const double *P_vals, const double *b, const double *c,
                      const double *x0, const double *y0, const double *s0, double *x, double *y, double *s, int32_t *status,
                      int32_t *iters, double *resid, void *cache, int32_t reuse, int shared, const bcone_settings *stg, void *stream) {
  if (h && cache && !h->fast_fwd) return fail(h, BCONE_EINVAL, "solve: this structure has no cached set-up path (bcone_cache_bytes() is 0)");
  if (h && cache && ((uintptr_t)cache & 15)) return fail(h, BCONE_EINVAL, "solve: cache must be 16-byte aligned");
  if (h && ((x0 != nullptr) != (y0 != nullptr) || (x0 != nullptr) != (s0 != nullptr))) return fail(h, BCONE_EINVAL, "solve: warm start needs x0, y0 and s0 together");
  if (!h || B <= 0 || !A_vals || !b || !c || !x || !y || !s || !status || !iters || !stg) return fail(h, BCONE_EINVAL, "solve: null argument");
  if (h->S.nnzP > 0 && !P_vals) return fail(h, BCONE_EINVAL, "solve: structure has P but P_vals is NULL");
  if (stg->check_interval <= 0 || stg->max_iters <= 0) return fail(h, BCONE_EINVAL, "solve: check_interval and max_iters must be positive");
  if (stg->acceleration_lookback > BC_AA_MAXMEM || stg->acceleration_lookback < -BC_AA_MAXMEM)
    return fail(h, BCONE_EINVAL, "solve: |acceleration_lookback| must be <= 16");
  cudaStream_t st = (cudaStream_t)stream;
  CK(cudaSetDevice(h->device), "solve set device");
  FwdArgs a;
  a.S = h->S; a.B = B; a.A_vals = A_vals; a.P_vals = h->S.nnzP > 0 ? P_vals : nullptr; a.b = b; a.c = c;
  a.x = x; a.y = y; a.s = s; a.status = status; a.iters = iters; a.resid = resid; a.st = kernel_settings(*stg);
  a.x0 = x0; a.y0 = y0; a.s0 = s0;
  a.cache = (double *)cache; a.cache_stride = h->fast_fwd ? (long long)bc_fwdf_cache_doubles(h->S.n, h->S.m) : 0; a.cache_reuse = cache && reuse;
  a.sA = shared ? 0 : h->S.nnzA; a.sP = shared ? 0 : h->S.nnzP;
  int *ctr = h->counters + 4 * (h->slot++ % Handle::RING);
  a.counter = ctr; a.use_tma = h->tma_ok && (((uintptr_t)A_vals & 15) == 0);
  const Plan &plan = h->fast_fwd ? h->fwd_fast : pick(h->fwd, B, h->num_sms, h->small_mode);
  const int grid = grid_for(plan, B, h->num_sms);
  const size_t slabs = h->fast_fwd ? (size_t)h->num_sms * plan.ctas : max_grid(h->fwd, h->num_sms);
  Handle::StreamWs *sw = stream_ws(h, st);
  a.ws = nullptr; a.ws_stride = (long long)h->fwd.ws_stride; a.prof = h->prof;
  a.slab_vectors = h->fwd.indirect || h->fwd.factor_global;
  if (h->fwd.indirect || h->fwd.factor_global || h->fwd.vals_global) {
    if (!ensure_slab(h, &sw->fwd, nullptr, h->fwd.ws_stride * slabs)) {
      char buf[160];
      snprintf(buf, sizeof buf, "cudaMalloc forward workspace (%zu B: %zu B per CTA x %zu CTAs)", h->fwd.ws_stride * slabs * sizeof(double),
               h->fwd.ws_stride * sizeof(double), slabs);
      return fail(h, BCONE_ENOMEM, buf);
    }
    a.ws = sw->fwd;
  }
  a.aa_ws = nullptr; a.aa_stride = 0;
  if (stg->acceleration_lookback != 0 && stg->max_iters > 1) {
    const int mem = std::abs(stg->acceleration_lookback);
    a.aa_stride = (long long)((aa_ws_doubles(h->S.n + h->S.m + 1, mem) + 1) & ~(size_t)1);
    if (!ensure_slab(h, &sw->aa, &sw->aa_cap, (size_t)a.aa_stride * slabs)) return fail(h, BCONE_ENOMEM, "cudaMalloc acceleration workspace");
    a.aa_ws = sw->aa;
  }
  a.park = nullptr;
  if (h->fast_fwd) {   // where the register tile waits while a termination check or an acceleration event runs (128 KB per CTA, L2)
    if (!ensure_slab(h, &sw->park, nullptr, (size_t)32 * 512 * slabs)) return fail(h, BCONE_ENOMEM, "cudaMalloc tile parking slab");
    a.park = sw->park;
  }
  if (shared && h->fast_fwd) {
    // One set-up for the batch: a launch of one CTA builds the record (E, D, K^-1 at the initial scale) by the cached set-up's
    // own code -- it stops after the first iteration, so the record is never refreshed at another scale -- and the batch
    // reads it with record stride 0, as with reuse = 1.  Its solution of instance 0 goes to scratch behind the record.
    const size_t rec = bc_fwdf_cache_doubles(h->S.n, h->S.m), extra = (size_t)h->S.n + 2 * (size_t)h->S.m + 4;
    if (!ensure_slab(h, &sw->setup, nullptr, rec + extra)) return fail(h, BCONE_ENOMEM, "cudaMalloc shared set-up record");
    FwdArgs u = a;
    double *o = sw->setup + rec;
    u.B = 1; u.x0 = u.y0 = u.s0 = nullptr; u.x = o; u.y = o + h->S.n; u.s = o + h->S.n + h->S.m; u.resid = nullptr;
    u.status = (int *)(o + h->S.n + 2 * h->S.m); u.iters = u.status + 2;
    u.st.max_iters = 1; u.st.acceleration_lookback = 0; u.aa_ws = nullptr; u.aa_stride = 0;
    u.cache = sw->setup; u.cache_stride = (long long)rec; u.cache_reuse = 0;
    int *uctr = h->counters + 4 * (h->slot++ % Handle::RING);
    u.counter = uctr;
    CK(cudaMemsetAsync(uctr, 0, sizeof(int), st), "solve counter (set-up)");
    CK(launch(plan, 1, &u, st), "solve launch (shared set-up)");
    h->launches++;
    a.cache = sw->setup; a.cache_stride = 0; a.cache_reuse = 1;
  }
  CK(cudaMemsetAsync(ctr, 0, sizeof(int), st), "solve counter");
  CK(launch(plan, grid, &a, st), h->fast_fwd ? "solve launch (fast)" : "solve launch");
  h->launches++;
  return BCONE_OK;
}
extern "C" int bcone_solve_cached(void *handle, int32_t B, const double *A_vals, const double *P_vals, const double *b, const double *c,
                                  const double *x0, const double *y0, const double *s0, double *x, double *y, double *s, int32_t *status,
                                  int32_t *iters, double *resid, void *cache, int32_t reuse, const bcone_settings *stg, void *stream) {
  return solve_impl((Handle *)handle, B, A_vals, P_vals, b, c, x0, y0, s0, x, y, s, status, iters, resid, cache, reuse, 0, stg, stream);
}
extern "C" int bcone_solve_shared(void *handle, int32_t B, const double *A_vals, const double *P_vals, const double *b, const double *c,
                                  const double *x0, const double *y0, const double *s0, double *x, double *y, double *s, int32_t *status,
                                  int32_t *iters, double *resid, const bcone_settings *stg, void *stream) {
  return solve_impl((Handle *)handle, B, A_vals, P_vals, b, c, x0, y0, s0, x, y, s, status, iters, resid, nullptr, 0, 1, stg, stream);
}

// shared: A_vals / P_vals one copy for the batch; dA_vals [nnzA] / dP_vals [nnzP] receive the batch sums
static int vjp_impl(Handle *h, int32_t B, const double *A_vals, const double *P_vals, const double *b,
                    const double *c, const double *x, const double *y, const double *s, const double *dx,
                    const double *dy, double *dA_vals, double *dP_vals, double *db, double *dc,
                    int32_t *lsqr_iters, int shared, const bcone_settings *stg, void *stream) {
  if (!h || B <= 0 || !A_vals || !b || !c || !x || !y || !s || !dx || !dy || !dA_vals || !db || !dc || !stg)
    return fail(h, BCONE_EINVAL, "vjp: null argument");
  if (h->S.nnzP > 0 && !P_vals) return fail(h, BCONE_EINVAL, "vjp: structure has P but P_vals is NULL");
  const int lsmr = stg->lsmr != 0;   // the LSQR or the LSMR kernels
  const LsPlans &p = h->ls[lsmr];
  if (!p.fast_ok && !p.gen_ok) return fail(h, BCONE_EUNSUPPORTED, "vjp: the instance does not fit the LSMR kernels");   // (LSQR's exist)
  const TieredPlan &gen = p.gen;
  cudaStream_t st = (cudaStream_t)stream;
  BwdArgs a;
  a.S = h->S; a.B = B; a.A_vals = A_vals; a.P_vals = h->S.nnzP > 0 ? P_vals : nullptr; a.b = b; a.c = c;
  a.x = x; a.y = y; a.s = s; a.dx = dx; a.dy = dy; a.dA = dA_vals; a.dP = dP_vals; a.db = db; a.dc = dc;
  a.sA = shared ? 0 : h->S.nnzA; a.sP = shared ? 0 : h->S.nnzP; a.srec = nullptr;
  a.tA = a.tP = a.tb = a.tc = nullptr; a.tx = a.ty = a.ts = nullptr;
  Handle::StreamWs *sw = stream_ws(h, st);
  if (shared) {
    const size_t R = (size_t)bc_srec_doubles(h->S.n, h->S.m);
    if (!ensure_slab(h, &sw->srec, &sw->srec_cap, R * B) || !ensure_slab(h, &sw->part, &sw->part_cap, bc_shared_part_doubles(&h->S, B)))
      return fail(h, BCONE_ENOMEM, "cudaMalloc shared-matrix adjoint scratch");
    a.srec = sw->srec; a.dA = nullptr; a.dP = nullptr;
  }
  // batch-summed dA / dP from the records (same stream: after the kernels that wrote them)
  auto reduce = [&]() -> int {
    if (shared) {
      CK(bc_shared_grad(&h->S, sw->srec, x, B, dA_vals, h->S.nnzP > 0 ? dP_vals : nullptr, sw->part, st), "vjp shared reduction");
      h->launches += (h->S.nnzA > 0 ? 2 : 0) + (h->S.nnzP > 0 && dP_vals ? 2 : 0);   // two stages per matrix
    }
    return BCONE_OK;
  };
  const int slot = h->slot++ % Handle::RING;
  int *ctr = h->counters + 4 * slot;
  a.lsqr_iters = lsqr_iters; a.st = kernel_settings(*stg); a.counter = ctr + 1;
  // (values off chip: nothing of A is staged, use_tma only allows the bulk copy of P)
  a.use_tma = gen.vals_global || (h->tma_ok && (((uintptr_t)A_vals & 15) == 0)); a.psd_total = h->psd_total; a.p_in_smem = gen.p_in_smem;
  CK(cudaSetDevice(h->device), "vjp set device");
  a.ws = nullptr; a.ws_stride = (long long)gen.ws_stride;
  if (gen.vec_global) {
    if (!ensure_slab(h, &sw->bwd[lsmr], nullptr, gen.ws_stride * max_grid(gen, h->num_sms))) return fail(h, BCONE_ENOMEM, "cudaMalloc backward workspace");
    a.ws = sw->bwd[lsmr];
  }
  a.inst_list = nullptr; a.B_dev = nullptr; a.fail_list = nullptr; a.fail_count = nullptr; a.prof = h->prof;
  if (p.block_ok && stg->lsqr_precond == 2) {
    // pass 1: block-preconditioned solve; pass 2: equilibrated LSQR on the instances it rejected
    if (h->fail_cap[slot] < B) {
      int *q = nullptr;
      CK(cudaMalloc((void **)&q, (size_t)B * sizeof(int)), "vjp fail list");
      h->allocs.push_back(q); h->fail_list[slot] = q; h->fail_cap[slot] = B;
    }
    CK(cudaMemsetAsync(ctr + 1, 0, 3 * sizeof(int), st), "vjp counters");
    h->last_block_slot = slot;
    a.fail_list = h->fail_list[slot]; a.fail_count = ctr + 2;
    CK(launch(p.block, std::min(B, h->num_sms), &a, st), "vjp launch (block)");
    BwdArgs f = a;
    f.st.lsqr_precond = 1; f.counter = ctr + 3; f.inst_list = h->fail_list[slot]; f.B_dev = ctr + 2;
    f.fail_list = nullptr; f.fail_count = nullptr;
    const Plan &second = p.fast_ok ? p.fast : pick(gen, B, h->num_sms, h->small_mode);   // (LSQR: always the fused kernel)
    CK(launch(second, grid_for(second, B, h->num_sms), &f, st), "vjp launch (fallback)");
    h->launches += 2;
    return reduce();
  }
  if (a.st.lsqr_precond == 2) a.st.lsqr_precond = 1;   // block factorisation not available for this structure
  CK(cudaMemsetAsync(ctr + 1, 0, sizeof(int), st), "vjp counter");
  const Plan &plan = p.fast_ok ? p.fast : pick(gen, B, h->num_sms, h->small_mode);
  CK(launch(plan, grid_for(plan, B, h->num_sms), &a, st), p.fast_ok ? "vjp launch (fast)" : "vjp launch");
  h->launches++;
  return reduce();
}
extern "C" int bcone_vjp(void *handle, int32_t B, const double *A_vals, const double *P_vals, const double *b,
                         const double *c, const double *x, const double *y, const double *s, const double *dx,
                         const double *dy, double *dA_vals, double *dP_vals, double *db, double *dc,
                         int32_t *lsqr_iters, const bcone_settings *stg, void *stream) {
  return vjp_impl((Handle *)handle, B, A_vals, P_vals, b, c, x, y, s, dx, dy, dA_vals, dP_vals, db, dc, lsqr_iters, 0, stg, stream);
}
extern "C" int bcone_vjp_shared(void *handle, int32_t B, const double *A_vals, const double *P_vals, const double *b,
                                const double *c, const double *x, const double *y, const double *s, const double *dx,
                                const double *dy, double *dA_sum, double *dP_sum, double *db, double *dc,
                                int32_t *lsqr_iters, const bcone_settings *stg, void *stream) {
  return vjp_impl((Handle *)handle, B, A_vals, P_vals, b, c, x, y, s, dx, dy, dA_sum, dP_sum, db, dc, lsqr_iters, 1, stg, stream);
}

// shared: A_vals / P_vals and the tangents dA_vals / dP_vals are one copy for the batch
static int jvp_impl(Handle *h, int32_t B, const double *A_vals, const double *P_vals, const double *b, const double *c,
                    const double *x, const double *y, const double *s, const double *dA_vals, const double *dP_vals,
                    const double *db, const double *dc, double *dx, double *dy, double *ds, int32_t *lsqr_iters, int shared,
                    const bcone_settings *stg, void *stream) {
  if (!h || B <= 0 || !A_vals || !b || !c || !x || !y || !s || !dA_vals || !db || !dc || !dx || !dy || !stg)
    return fail(h, BCONE_EINVAL, "jvp: null argument");
  if (h->S.nnzP > 0 && !P_vals) return fail(h, BCONE_EINVAL, "jvp: structure has P but P_vals is NULL");
  const int lsmr = stg->lsmr != 0;   // the LSQR or the LSMR kernel
  if (!h->ls[lsmr].jvp_ok)
    return fail(h, BCONE_EUNSUPPORTED, lsmr ? "jvp: the instance does not fit the generic LSMR kernel" : "jvp: the instance does not fit the generic LSQR kernel");
  const TieredPlan &gen = h->ls[lsmr].jvp;
  cudaStream_t st = (cudaStream_t)stream;
  BwdArgs a{};
  a.S = h->S; a.B = B; a.A_vals = A_vals; a.P_vals = h->S.nnzP > 0 ? P_vals : nullptr; a.b = b; a.c = c;
  a.x = x; a.y = y; a.s = s;
  a.tA = dA_vals; a.tP = h->S.nnzP > 0 ? dP_vals : nullptr; a.tb = db; a.tc = dc; a.tx = dx; a.ty = dy; a.ts = ds;
  a.sA = shared ? 0 : h->S.nnzA; a.sP = shared ? 0 : h->S.nnzP;
  int *ctr = h->counters + 4 * (h->slot++ % Handle::RING);
  a.lsqr_iters = lsqr_iters; a.st = kernel_settings(*stg); a.counter = ctr + 1;
  if (a.st.lsqr_precond == 2) a.st.lsqr_precond = 1;   // no block-preconditioned forward mode
  a.use_tma = gen.vals_global || (h->tma_ok && (((uintptr_t)A_vals & 15) == 0)); a.psd_total = h->psd_total; a.p_in_smem = gen.p_in_smem;
  CK(cudaSetDevice(h->device), "jvp set device");
  a.ws_stride = (long long)gen.ws_stride;
  if (gen.vec_global) {
    Handle::StreamWs *sw = stream_ws(h, st);
    if (!ensure_slab(h, &sw->jvp[lsmr], nullptr, gen.ws_stride * max_grid(gen, h->num_sms))) return fail(h, BCONE_ENOMEM, "cudaMalloc jvp workspace");
    a.ws = sw->jvp[lsmr];
  }
  a.prof = h->prof;
  CK(cudaMemsetAsync(ctr + 1, 0, sizeof(int), st), "jvp counter");
  const Plan &plan = pick(gen, B, h->num_sms, h->small_mode);
  CK(launch(plan, grid_for(plan, B, h->num_sms), &a, st), "jvp launch");
  h->launches++;
  return BCONE_OK;
}
extern "C" int bcone_jvp(void *handle, int32_t B, const double *A_vals, const double *P_vals, const double *b, const double *c,
                         const double *x, const double *y, const double *s, const double *dA_vals, const double *dP_vals,
                         const double *db, const double *dc, double *dx, double *dy, double *ds, int32_t *lsqr_iters,
                         const bcone_settings *stg, void *stream) {
  return jvp_impl((Handle *)handle, B, A_vals, P_vals, b, c, x, y, s, dA_vals, dP_vals, db, dc, dx, dy, ds, lsqr_iters, 0, stg, stream);
}
extern "C" int bcone_jvp_shared(void *handle, int32_t B, const double *A_vals, const double *P_vals, const double *b, const double *c,
                                const double *x, const double *y, const double *s, const double *dA, const double *dP,
                                const double *db, const double *dc, double *dx, double *dy, double *ds, int32_t *lsqr_iters,
                                const bcone_settings *stg, void *stream) {
  return jvp_impl((Handle *)handle, B, A_vals, P_vals, b, c, x, y, s, dA, dP, db, dc, dx, dy, ds, lsqr_iters, 1, stg, stream);
}

// shared: A_vals [nnzA] / P_vals [nnzP] one copy for the batch
static int polish_impl(Handle *h, int32_t B, const double *A_vals, const double *P_vals, const double *b, const double *c, double *x,
                       double *y, double *s, const int32_t *status, int32_t *polished, double *resid, int shared, const bcone_settings *stg,
                       void *stream) {
  if (!h || B <= 0 || !A_vals || !b || !c || !x || !y || !s || !status || !polished || !stg) return fail(h, BCONE_EINVAL, "polish: null argument");
  if (h->S.nnzP > 0 && !P_vals) return fail(h, BCONE_EINVAL, "polish: structure has P but P_vals is NULL");
  if (!h->polish_ok) return fail(h, BCONE_EUNSUPPORTED, h->polish_why);
  cudaStream_t st = (cudaStream_t)stream;
  CK(cudaSetDevice(h->device), "polish set device");
  PolishArgs a;
  a.S = h->S; a.B = B; a.A_vals = A_vals; a.P_vals = h->S.nnzP > 0 ? P_vals : nullptr; a.b = b; a.c = c;
  a.x = x; a.y = y; a.s = s; a.status = status; a.polished = polished; a.resid = resid;
  a.sA = shared ? 0 : h->S.nnzA; a.sP = shared ? 0 : h->S.nnzP;
  a.use_tma = h->S.dense && (h->S.n % 2) == 0 && (((uintptr_t)A_vals & 15) == 0);
  a.stage_cap = h->polish_stage;
  a.delta = 1e-6; a.refine = 3;   // OSQP's defaults
  int *ctr = h->counters + 4 * (h->slot++ % Handle::RING);
  a.counter = ctr;
  PolishLargeArgs g{};
  if (h->polish_tier == 1) {
    Handle::StreamWs *sw = stream_ws(h, st);
    if (!ensure_slab(h, &sw->polish, nullptr, (size_t)h->polish_slab * h->polish_ctas)) return fail(h, BCONE_ENOMEM, "cudaMalloc polish workspace");
    a.use_tma = 0; a.stage_cap = 0;
    g.a = a; g.ws = sw->polish; g.ws_stride = h->polish_slab; g.p_diag = h->p_diag;
  }
  CK(cudaMemsetAsync(ctr, 0, sizeof(int), st), "polish counter");
  if (h->polish_tier == 1) CK(launch(h->polish, std::min(B, h->polish_ctas), &g, st), "polish launch (slab)");
  else CK(launch(h->polish, grid_for(h->polish, B, h->num_sms), &a, st), "polish launch");
  h->launches++;
  return BCONE_OK;
}
extern "C" int bcone_polish_supported(void *handle) {
  Handle *h = (Handle *)handle;
  if (!h) return BCONE_EINVAL;
  return h->polish_ok ? BCONE_OK : fail(h, BCONE_EUNSUPPORTED, h->polish_why);
}
extern "C" int bcone_polish_info(void *handle, int32_t *tier, int32_t *threads, int32_t *ctas, int64_t *slab_bytes_per_cta) {
  Handle *h = (Handle *)handle;
  if (!h) return BCONE_EINVAL;
  const int tr = h->polish_ok ? h->polish_tier : -1;
  if (tier) *tier = tr;
  if (threads) *threads = tr >= 0 ? h->polish.threads : 0;
  if (ctas) *ctas = tr == 1 ? h->polish_ctas : (tr == 0 ? h->num_sms * h->polish.ctas : 0);
  if (slab_bytes_per_cta) *slab_bytes_per_cta = tr == 1 ? (int64_t)h->polish_slab * (int64_t)sizeof(double) : 0;
  return BCONE_OK;
}
extern "C" int bcone_polish(void *handle, int32_t B, const double *A_vals, const double *P_vals, const double *b, const double *c, double *x,
                            double *y, double *s, const int32_t *status, int32_t *polished, double *resid, const bcone_settings *st, void *stream) {
  return polish_impl((Handle *)handle, B, A_vals, P_vals, b, c, x, y, s, status, polished, resid, 0, st, stream);
}
extern "C" int bcone_polish_shared(void *handle, int32_t B, const double *A_vals, const double *P_vals, const double *b, const double *c,
                                   double *x, double *y, double *s, const int32_t *status, int32_t *polished, double *resid,
                                   const bcone_settings *st, void *stream) {
  return polish_impl((Handle *)handle, B, A_vals, P_vals, b, c, x, y, s, status, polished, resid, 1, st, stream);
}

// shared: A_vals [nnzA] / P_vals [nnzP] one copy for the batch
static int refine_impl(Handle *h, int32_t B, const double *A_vals, const double *P_vals, const double *b, const double *c, double *x,
                       double *y, double *s, const int32_t *status, int32_t *refined, double *resid, int32_t steps, int shared,
                       const bcone_settings *stg, void *stream) {
  if (!h || B <= 0 || !A_vals || !b || !c || !x || !y || !s || !status || !refined || !stg) return fail(h, BCONE_EINVAL, "refine: null argument");
  if (h->S.nnzP > 0 && !P_vals) return fail(h, BCONE_EINVAL, "refine: structure has P but P_vals is NULL");
  if (steps < 1 || steps > 10) return fail(h, BCONE_EINVAL, "refine: steps must be 1 ... 10 (got " + std::to_string(steps) + ")");
  if (!h->refine_ok) return fail(h, BCONE_EUNSUPPORTED, h->refine_why);
  const TieredPlan &gen = h->refine;
  cudaStream_t st = (cudaStream_t)stream;
  RefineArgs ra{};
  BwdArgs &a = ra.a;
  a.S = h->S; a.B = B; a.A_vals = A_vals; a.P_vals = h->S.nnzP > 0 ? P_vals : nullptr; a.b = b; a.c = c;
  a.x = x; a.y = y; a.s = s; a.tx = x; a.ty = y; a.ts = s;
  a.sA = shared ? 0 : h->S.nnzA; a.sP = shared ? 0 : h->S.nnzP;
  int *ctr = h->counters + 4 * (h->slot++ % Handle::RING);
  a.st = kernel_settings(*stg); a.counter = ctr + 1;
  if (a.st.lsqr_precond == 2) a.st.lsqr_precond = 1;   // (as for the forward mode)
  a.use_tma = gen.vals_global || (h->tma_ok && (((uintptr_t)A_vals & 15) == 0)); a.psd_total = h->psd_total; a.p_in_smem = gen.p_in_smem;
  ra.status = status; ra.flags = refined; ra.resid = resid; ra.steps = steps;
  CK(cudaSetDevice(h->device), "refine set device");
  a.ws_stride = (long long)gen.ws_stride;
  if (gen.vec_global) {
    Handle::StreamWs *sw = stream_ws(h, st);
    if (!ensure_slab(h, &sw->refine, nullptr, gen.ws_stride * max_grid(gen, h->num_sms))) return fail(h, BCONE_ENOMEM, "cudaMalloc refine workspace");
    a.ws = sw->refine;
  }
  a.prof = h->prof;
  CK(cudaMemsetAsync(ctr + 1, 0, sizeof(int), st), "refine counter");
  const Plan &plan = pick(gen, B, h->num_sms, h->small_mode);
  h->refine_last_small = &plan == &gen.small;
  CK(launch(plan, grid_for(plan, B, h->num_sms), &ra, st), "refine launch");
  h->launches++;
  return BCONE_OK;
}
extern "C" int bcone_refine_supported(void *handle) {
  Handle *h = (Handle *)handle;
  if (!h) return BCONE_EINVAL;
  return h->refine_ok ? BCONE_OK : fail(h, BCONE_EUNSUPPORTED, h->refine_why);
}
extern "C" int bcone_refine_info(void *handle, int32_t *threads, int32_t *ctas_per_sm, int32_t *small_ctas_per_sm, int32_t *vals_global,
                                 int32_t *vec_global, int32_t *num_sms, int32_t *last_small) {
  Handle *h = (Handle *)handle;
  if (!h) return BCONE_EINVAL;
  const TieredPlan &t = h->refine;
  if (threads) *threads = h->refine_ok ? t.big.threads : 0;
  if (ctas_per_sm) *ctas_per_sm = h->refine_ok ? t.big.ctas : 0;
  if (small_ctas_per_sm) *small_ctas_per_sm = h->refine_ok && t.has_small ? t.small.ctas : 0;
  if (vals_global) *vals_global = t.vals_global;
  if (vec_global) *vec_global = t.vec_global;
  if (num_sms) *num_sms = h->num_sms;
  if (last_small) *last_small = h->refine_last_small;
  return BCONE_OK;
}
extern "C" int bcone_refine(void *handle, int32_t B, const double *A_vals, const double *P_vals, const double *b, const double *c, double *x,
                            double *y, double *s, const int32_t *status, int32_t *refined, double *resid, int32_t steps, const bcone_settings *st,
                            void *stream) {
  return refine_impl((Handle *)handle, B, A_vals, P_vals, b, c, x, y, s, status, refined, resid, steps, 0, st, stream);
}
extern "C" int bcone_refine_shared(void *handle, int32_t B, const double *A_vals, const double *P_vals, const double *b, const double *c,
                                   double *x, double *y, double *s, const int32_t *status, int32_t *refined, double *resid, int32_t steps,
                                   const bcone_settings *st, void *stream) {
  return refine_impl((Handle *)handle, B, A_vals, P_vals, b, c, x, y, s, status, refined, resid, steps, 1, st, stream);
}

// Strided host<->device copy on the caller's stream (cudaMemcpy2DAsync): lets the reference-facing
// call move a batch slice of the [rows, B] boundary tensors without a host-side repack.
extern "C" int bcone_memcpy2d(void *dst, int64_t dpitch, const void *src, int64_t spitch, int64_t width, int64_t height,
                              int32_t to_device, void *stream) {
  cudaError_t e = cudaMemcpy2DAsync(dst, (size_t)dpitch, src, (size_t)spitch, (size_t)width, (size_t)height,
                                    to_device ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToHost, (cudaStream_t)stream);
  if (e != cudaSuccess) { g_create_err = std::string("bcone_memcpy2d: ") + cudaGetErrorString(e); return BCONE_ECUDA; }
  return BCONE_OK;
}

// Debug: enable (on != 0) or read-and-reset the per-phase cycle counters of the forward / block-backward
// kernels.  out (HOST, 16 x uint64) may be NULL.  Phases: 0 load, 1 equilibration, 2 factorisation + g,
// 3 iterations, 4 checks | 8 load, 9 P factor, 10 W, 11 S, 12 S factor, 13 q + LSQR, 14 solve + write.
extern "C" int bcone_set_profile(void *handle, int32_t on, uint64_t *out) {
  Handle *h = (Handle *)handle;
  if (!h) return BCONE_EINVAL;
  cudaSetDevice(h->device);
  if (out && h->prof) { cudaDeviceSynchronize(); cudaMemcpy(out, h->prof, 32 * sizeof(uint64_t), cudaMemcpyDeviceToHost); cudaMemset(h->prof, 0, 32 * sizeof(uint64_t)); }
  if (on && !h->prof) { if (cudaMalloc((void **)&h->prof, 32 * sizeof(uint64_t)) != cudaSuccess) return BCONE_ENOMEM; h->allocs.push_back(h->prof); cudaMemset(h->prof, 0, 32 * sizeof(uint64_t)); }
  if (!on) h->prof = nullptr;
  return BCONE_OK;
}

// Instances of the last block-preconditioned bcone_vjp (lsqr_precond = 2) that the block factorisation rejected and the
// equilibrated LSQR solved instead.  Synchronises the device.  -1: no such call yet.
extern "C" int bcone_fallback_count(void *handle, int32_t *out) {
  Handle *h = (Handle *)handle;
  if (!h || !out) return BCONE_EINVAL;
  *out = -1;
  if (h->last_block_slot < 0) return BCONE_OK;
  cudaSetDevice(h->device);
  if (cudaDeviceSynchronize() != cudaSuccess) return BCONE_ECUDA;
  int v = 0;
  if (cudaMemcpy(&v, h->counters + 4 * h->last_block_slot + 2, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess) return BCONE_ECUDA;
  *out = v;
  return BCONE_OK;
}

extern "C" int64_t bcone_launch_count(void *handle) { return handle ? ((Handle *)handle)->launches : 0; }

extern "C" int bcone_path_info(void *handle, int32_t *fwd_path, int32_t *bwd_path) {
  Handle *h = (Handle *)handle;
  if (!h) return BCONE_EINVAL;
  if (fwd_path) {
    if (h->fast_fwd) *fwd_path = 2;
    else if (h->fwd.vals_global) *fwd_path = h->fwd.indirect ? 6 : (h->fwd.factor_global ? 5 : 4);
    else *fwd_path = h->fwd.indirect ? 1 : (h->fwd.factor_global ? 3 : 0);
  }
  const LsPlans &p = h->ls[0];   // (the LSQR plans)
  if (bwd_path) *bwd_path = p.block_ok ? 2 : (p.fast_ok ? 1 : (p.gen.vals_global ? 3 : 0));
  return BCONE_OK;
}

extern "C" int bcone_small_cta_info(void *handle, int32_t *fwd_small_ctas, int32_t *bwd_small_ctas) {
  Handle *h = (Handle *)handle;
  if (!h) return BCONE_EINVAL;
  if (fwd_small_ctas) *fwd_small_ctas = h->fwd.has_small ? h->fwd.small.ctas : 0;
  if (bwd_small_ctas) *bwd_small_ctas = h->ls[0].gen.has_small ? h->ls[0].gen.small.ctas : 0;   // (the LSQR plans)
  return BCONE_OK;
}

extern "C" int bcone_kernel_info(void *handle, int32_t *ft, int32_t *fs, int32_t *fc, int32_t *bt, int32_t *bs, int32_t *bcx) {
  Handle *h = (Handle *)handle;
  if (!h) return BCONE_EINVAL;
  const LsPlans &p = h->ls[0];   // (the LSQR plans)
  const Plan &f = h->fast_fwd ? h->fwd_fast : h->fwd.big, &b = p.fast_ok ? p.fast : p.gen.big;
  if (ft) *ft = f.threads; if (fs) *fs = (int32_t)f.smem; if (fc) *fc = f.ctas;
  if (bt) *bt = b.threads; if (bs) *bs = (int32_t)b.smem; if (bcx) *bcx = b.ctas;
  return BCONE_OK;
}
