// engine.cu -- the H100-native ADMM iteration engine behind include/cosmo_b200.h.
//
// Host-side driver of the hot loop of COSMO.optimize! (reference
// src/solver.jl:125-167, restated in SURVEY.md Appendix A) plus the C ABI.
// All arithmetic runs in the hand-written sm_90a kernels of spmv.cuh,
// vector_kernels.cuh and psd.cuh; the host only sequences launches, reads
// back a handful of scalars at the reference's own decision points
// (termination / infeasibility / rho-adaptation checks, CG convergence) and
// never touches vector data.  There is no CPU fallback: without a CUDA device
// every entry point fails with COSMO_B200_ERR_CUDA.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <functional>
#include <thread>
#include <chrono>
#include <string>
#include <vector>

#include "../../include/cosmo_b200.h"
#include "common.cuh"
#include "host.cuh"
#include "psd.cuh"
#include "cone3.cuh"
#include "aa.cuh"
#include "spmv.cuh"
#include "vector_kernels.cuh"
#include "ruiz.cuh"
#include "cg_persistent.cuh"
#include "ldl.cuh"
#include "ldl_sn.cuh"
#include "chordal_rev.cuh"
#include "chordal_fwd.cuh"
#include "mat_update.cuh"
#include "custom_cone.cuh"

namespace cosmo {

static thread_local std::string g_create_error;

static inline double now_s() {
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// ---- NCCL through dlopen (the single-GPU path has no NCCL dependency) --------
struct NcclUniqueId { char internal[128]; };
typedef void* NcclComm;
struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(NcclUniqueId*) = nullptr;
  int (*CommInitRank)(NcclComm*, int, NcclUniqueId, int) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, NcclComm, cudaStream_t) = nullptr;
  int (*CommDestroy)(NcclComm) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  bool load(std::string& err) {
    if (lib) return true;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* nm : names) {
      lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
      if (lib) break;
    }
    if (!lib) { err = std::string("cannot dlopen libnccl: ") + dlerror(); return false; }
    GetUniqueId = (int (*)(NcclUniqueId*))dlsym(lib, "ncclGetUniqueId");
    CommInitRank = (int (*)(NcclComm*, int, NcclUniqueId, int))dlsym(lib, "ncclCommInitRank");
    AllReduce = (int (*)(const void*, void*, size_t, int, int, NcclComm, cudaStream_t))dlsym(lib, "ncclAllReduce");
    CommDestroy = (int (*)(NcclComm))dlsym(lib, "ncclCommDestroy");
    GetErrorString = (const char* (*)(int))dlsym(lib, "ncclGetErrorString");
    if (!GetUniqueId || !CommInitRank || !AllReduce || !CommDestroy) { err = "libnccl lacks required symbols"; return false; }
    return true;
  }
};
static NcclApi g_nccl;
constexpr int kNcclFloat32 = 7, kNcclFloat64 = 8, kNcclSum = 0, kNcclMax = 2;

// ---- phase timers (ResultTimes.proj_time / kkt_time, types.jl:26-41) ------------
// CUDA events on the engine stream around a phase; elapsed times are harvested in batches so that the loop never
// waits for a timer (one event synchronisation per kCap phases).
struct PhaseTimer {
  static constexpr int kCap = 64;
  Event a[kCap], b[kCap];
  int n = 0;
  bool on = false;
  double total_ms = 0.0;
  void enable(bool e) {
    on = e;
    if (on) for (int i = 0; i < kCap; ++i) { a[i].create(); b[i].create(); }
    n = 0; total_ms = 0.0;
  }
  void begin(cudaStream_t st) { if (on) cudaEventRecord(a[n], st); }
  void end(cudaStream_t st) {
    if (!on) return;
    cudaEventRecord(b[n], st);
    if (++n == kCap) harvest();
  }
  void harvest() {
    if (!on || n == 0) return;
    cudaEventSynchronize(b[n - 1]);
    for (int i = 0; i < n; ++i) { float ms = 0.f; cudaEventElapsedTime(&ms, a[i], b[i]); total_ms += ms; }
    n = 0;
  }
};

template <typename T>
struct DevCsr {
  int nrows = 0, ncols = 0;
  long long nnz = 0;
  DevBuf<int> rowptr, col;
  DevBuf<T> val;
  int lanes = 32;
  // column-windowed copy (spmv_win_kernel); absent when the rows are too short to pay off
  bool windowed = false;
  int nwin = 0, W = 0, nctas = 0;
  DevBuf<int> w_rowptr, w_cta_rows;
  DevBuf<unsigned short> w_col;   // 10 B layout
  DevBuf<T> w_val;
  bool packed = false;            // 9 B layout (fp64 only, win_pack.h): w_word + w_colhi + w_esc replace w_val + w_col
  int ebase = 0;
  DevBuf<unsigned long long> w_word;
  DevBuf<unsigned char> w_colhi;
  DevBuf<double> w_esc;
  long long w_elems = 0, w_nesc = 0;
  bool packable = false;          // the 9 B layout may hold this slab (fp64, 15-bit columns)
  // where every stored value comes from (cosmo_b200_update_matrices): CSR position -> CSC index (none when the CSR is
  // the CSC order itself, as for A'), slab column position -> CSC index of the matrix or -1 for padding.  Device copies
  // made by the first update (upload_value_maps); h_src holds the CSR(P) map from create until then.
  std::vector<int> h_src;
  DevBuf<int> d_src, d_wsrc;
  WcsrView<T> wview() const {
    return WcsrView<T>{w_rowptr.p, w_col.p, w_val.p, w_word.p, w_colhi.p, w_esc.p, winpack::exp_offset(ebase), w_cta_rows.p,
                       nwin, W, nrows, ncols};
  }
  CsrView<T> view() const { return CsrView<T>{rowptr.p, col.p, val.p}; }
  double spmv_bytes() const {  // SURVEY.md 8d: 12 nnz + 4 (rows+1) + 8 cols + 8 rows   (fp64)
    return (double)nnz * (sizeof(T) + 4) + 4.0 * (nrows + 1) + (double)sizeof(T) * ncols + (double)sizeof(T) * nrows;
  }
};

static int pick_lanes(double mean_row) {
  if (mean_row > 24.0) return 32;
  if (mean_row > 3.0) return 8;
  return 2;
}

// a sparsity pattern; the values go to the device separately (mat_update.cuh)
struct HostCsr {
  int nrows = 0, ncols = 0;
  std::vector<int> rowptr, col;
  std::vector<int> src;     // CSR position -> CSC index (csr_transpose; empty for the CSC pattern itself)
};

class EngineBase {
 public:
  virtual ~EngineBase() {}
  std::string err;
  virtual void update_settings(const cosmo_b200_settings& st) = 0;
  virtual void warm_start(const void* x, const void* s, const void* mu) = 0;
  virtual void update_qb(const void* q, const void* b) = 0;
  virtual void update_matrices(const void* Px, long long nnzP, const void* Ax, long long nnzA, const void* q, const void* b) = 0;
  virtual void update_rho(const void* rho_vec, double rho) = 0;
  virtual void reset() = 0;
  virtual void solve(cosmo_b200_result* out) = 0;
  virtual void project(const void* ws, void* s_out) = 0;
  virtual void kkt_solve(const void* rhs, void* sol, int64_t* inner) = 0;
  virtual void residuals(const void* x, const void* s, const void* mu, int ignore_scaling, double* out) = 0;
  virtual void spmv(int which, const void* x, void* y) = 0;
  virtual void spmv_bench(int which, int reps, double* ms, double* bytes) = 0;
  virtual void get_rho_vec(void* out) = 0;
  virtual void get_w(void* out) = 0;
  virtual void psd_stats(int64_t* out8) = 0;
  virtual void get_scaling(void* D, void* E, double* c) = 0;
  virtual void comm_init(int nranks, int rank, const void* id128) = 0;
  virtual void p2p_export(void* blob128) = 0;
  virtual void p2p_attach(const void* blobs, int nranks) = 0;
  virtual void set_accelerator(const cosmo_b200_accelerator* acc) = 0;
  virtual void accelerator_stats(int64_t* out6) = 0;
  virtual void infeasibility_test(int which, const void* delta, double* out8) = 0;
  virtual void psd_lambda_max(const void* v, double* lam) = 0;
  virtual void ldl_stats(double* out8) = 0;
  virtual void ldl_sn_stats(int64_t* out8) = 0;
  virtual void set_decomposition(const cosmo_b200_decomposition* d, bool traditional) = 0;
  virtual void set_forward_map(const cosmo_b200_forward_map* f) = 0;
  virtual void update_matrices_original(const void* Px, long long nnzP, const void* Ax, long long nnzA_orig, const void* q,
                                        const void* b) = 0;
  virtual void reverse_decomposition(int complete_dual, void* x, void* s, void* mu, int64_t* stats4) = 0;
  virtual void custom_cone_stats(int64_t* out4) = 0;
  virtual void set_caller_stream(void* stream) = 0;
  virtual void update_qb_original(const double* q, const double* b) = 0;
  virtual void original_qb(double* q, double* b) = 0;
  virtual void solution(int complete_dual, double* x, double* y, double* s) = 0;
  virtual void rescale_iterates() = 0;
};

template <typename T>
class Engine : public EngineBase {
 public:
  Engine(const cosmo_b200_problem& p, const cosmo_b200_settings& st);
  ~Engine() override;
  void update_settings(const cosmo_b200_settings& st) override {
    if (st.sigma != st_.sigma) {   // sigma is baked into the captured kernel arguments
      destroy_cg_graphs();
      destroy_ldl_factor_graph();
      ldl_dirty_ = true;
      sn_factor_graph_.reset();
      sn_dirty_ = true;
    }
    st_ = st;
  }
  void warm_start(const void* x, const void* s, const void* mu) override;
  void update_qb(const void* q, const void* b) override;
  void update_matrices(const void* Px, long long nnzP, const void* Ax, long long nnzA, const void* q, const void* b) override;
  void update_rho(const void* rho_vec, double rho) override;
  void reset() override;
  void solve(cosmo_b200_result* out) override;
  void project(const void* ws, void* s_out) override;
  void kkt_solve(const void* rhs, void* sol, int64_t* inner) override;
  void residuals(const void* x, const void* s, const void* mu, int ignore_scaling, double* out) override;
  void spmv(int which, const void* x, void* y) override;
  void spmv_bench(int which, int reps, double* ms, double* bytes) override;
  void get_rho_vec(void* out) override;
  void get_w(void* out) override;
  void psd_stats(int64_t* out8) override;
  void get_scaling(void* D, void* E, double* c) override;
  void equilibrate();
  void comm_init(int nranks, int rank, const void* id128) override;
  void p2p_export(void* blob128) override;
  void p2p_attach(const void* blobs, int nranks) override;
  void set_accelerator(const cosmo_b200_accelerator* acc) override;
  void accelerator_stats(int64_t* out6) override;
  void infeasibility_test(int which, const void* delta, double* out8) override;
  void psd_lambda_max(const void* v, double* lam) override;
  void ldl_stats(double* out8) override;
  void ldl_sn_stats(int64_t* out8) override;
  void set_decomposition(const cosmo_b200_decomposition* d, bool traditional) override;
  void set_forward_map(const cosmo_b200_forward_map* f) override;
  void update_matrices_original(const void* Px, long long nnzP, const void* Ax, long long nnzA_orig, const void* q,
                                const void* b) override;
  void reverse_decomposition(int complete_dual, void* x, void* s, void* mu, int64_t* stats4) override;
  void custom_cone_stats(int64_t* out4) override {
    out4[0] = (int64_t)cust_types_.size(); out4[1] = n_cust_; out4[2] = cust_compiled_; out4[3] = cust_hits_;
  }
  void set_caller_stream(void* stream) override {
    single_gpu("set_caller_stream");
    caller_stream_ = static_cast<cudaStream_t>(stream);
  }
  void update_qb_original(const double* q, const double* b) override;
  void original_qb(double* q, double* b) override;
  void solution(int complete_dual, double* x, double* y, double* s) override;
  void rescale_iterates() override;

 private:
  // ---- problem ----
  int n_ = 0, m_ = 0, device_ = 0;
  double create_time_ = 0.0;      // engine construction (the device part of setup!)
  bool device_scaled_ = false;    // D, E, c are computed here (equilibrate), not handed over by the host
  int auto_rho_interval_ = 0;     // adaptive_rho_interval chosen by the automatic rule (kept across solves like settings)
  cosmo_b200_settings st_;
  bool scaled_ = false;
  double c_ = 1.0;
  DevCsr<T> A_, At_, P_;
  DevBuf<T> q_, b_, D_, Dinv_, E_, Einv_;
  // cones
  DevBuf<unsigned char> row_class_, rho_class_;
  DevBuf<int> row_cone_;
  DevBuf<T> box_l_, box_u_;       // m-length, +-inf outside Box rows
  DevBuf<T> box_l0_, box_u0_;     // the unscaled Box bounds of an equilibrating engine (Ruiz restarts from them)
  DevBuf<int> rect_off_, rect_dim_;   // cones that rectify_set_scalings! scales by one scalar (equilibrating engine)
  int n_soc_ = 0, n_soc_chunks_ = 0;
  DevBuf<int> soc_off_, soc_dim_, soc_chunk_start_, soc_chunk_len_, soc_cone_chunk_ptr_;
  DevBuf<T> soc_norm_, soc_chunk_sum_, soc_norm2_;
  PsdBatch<T> psd_;
  PhaseTimer t_proj_, t_kkt_;
  DevBuf<T> proj_w_, proj_s_;     // scratch of the plugin-level project() entry point
  int n_c3_ = 0;             // exponential / power cones and their duals (cone3.cuh)
  DevBuf<int> c3_off_, c3_maxit_;
  DevBuf<unsigned char> c3_kind_;
  DevBuf<T> c3_alpha_, c3_tol_;
  Cone3Table<T> c3_table() const {
    return Cone3Table<T>{n_c3_, c3_off_.p, c3_kind_.p, c3_alpha_.p, c3_maxit_.p, c3_tol_.p};
  }
  // custom cones (custom_cone.cuh): one table of all of them, grouped by type; one slice of it per type
  std::vector<custom::TypeSlice> cust_types_;
  int n_cust_ = 0;
  DevBuf<int> cust_off_, cust_dim_, cust_flag_;
  DevBuf<T> cust_params_, cust_tmp_;
  long long cust_compiled_ = 0, cust_hits_ = 0;   // types this create compiled / found in the process-wide cache
  void custom_project(const T* ws);
  void custom_certificates(const T* v, T eps, int which);
  // ---- accelerator (aa.cuh) ----
  DevBuf<T> aaG_, aaQ_, aaR_, aa_eta_, aa_glast_, aa_f_, aa_flast_, aa_sc_;
  PinnedBuf<T> h_aa_;          // mirror of aa_sc_
  int aa_mem_ = 0;             // allocated history length (min(mem, dim)), 0 = not allocated
  int aa_iter_ = 0;            // columns filled since the last restart
  bool aa_init_ = true, aa_success_ = false, aa_active_ = false;
  long long aa_accelerated_ = 0, aa_declined_ = 0;
  // variant and activation reason (cosmo_b200_set_accelerator); the default is the QR variant above
  cosmo_b200_accelerator acc_{COSMO_B200_AA_TYPE2_QR, COSMO_B200_AA_RESTARTED_MEMORY, COSMO_B200_AA_NO_REGULARIZER,
                              COSMO_B200_AA_IMMEDIATE, 0.0, 2, 0.0};
  long long aa_rejected_ = 0, aa_rho_restarts_ = 0, aa_mem_restarts_ = 0, aa_activated_at_ = 0;
  // normal-equation variants: F is stored in aaQ_, M in aaR_ (row-major, leading dimension aa_mem_)
  DevBuf<T> aaX_, aa_xlast_, aa_nrm_, aa_gsc_, aa_gpart_;
  int aa_j_ = 0;               // column written by the last aa_update
  bool aa_fresh_ = false;      // aa_update wrote a column that aa_accelerate has not used yet
  bool aa_qr() const { return acc_.type == COSMO_B200_AA_TYPE2_QR; }
  void aa_prepare();
  void aa_restart() { aa_iter_ = 0; aa_init_ = true; aa_fresh_ = false; }
  void aa_update(const T* g, const T* x);
  bool aa_accelerate(T* g);
  // ---- state ----
  DevBuf<T> W_[2];           // operator variable, ping-pong (w / w_prev)
  int cur_ = 0, prev_ = 1;
  DevBuf<T> xs_, s_, mu_;    // warm-start / exit copies of x; s; mu
  DevBuf<T> rho_vec_;
  double rho_ = 0.1;
  std::vector<double> rho_updates_;
  bool have_solution_ = false;   // xs_, s_, mu_ hold what the last solve() returned (cleared by reset / warm_start)
  rev::Reverse rev_;             // map of a chordal decomposition (cosmo_b200_set_decomposition)
  fwd::Forward fwd_;             // where the values of the decomposed problem come from (cosmo_b200_set_forward_map)
  rev::Reverse ident_;           // the identity map: cosmo_b200_solution of a handle without a decomposition map
  // q and b of the last update_qb_original, fp64 in the original coordinates (allocated on first use)
  DevBuf<double> q0_, b0_;
  bool have_q0_ = false, have_b0_ = false;
  // caller arrays in device memory are ordered on caller_stream_ (cosmo_b200_set_caller_stream)
  cudaStream_t caller_stream_ = nullptr;
  Event caller_ev_;
  unsigned caller_arrays(std::initializer_list<const void*> ptrs);
  void caller_written();
  void single_gpu(const char* what) const {
    if (nranks_ > 1) throw EngineError{COSMO_B200_ERR_UNSUPPORTED, std::string(what) + ": a sharded handle holds only a slice of the data"};
  }
  // KKT (reduced CG)
  DevBuf<T> ls_, t0_, tm_, xsol_, rhsb_, cb_, r_, u_, nu_;
  DevBuf<T> mr_[6], mr_x_, mr_c_, mr_b_;   // MINRES Lanczos / direction vectors, solution, operator output, rhs
  int cur_maxit_ = -1;
  // CUDA graphs of 1, 2, 4, 8 CG iterations (the inner loop is launch-bound for small problems)
  GraphExec cg_graph_[4];
  // persistent cooperative CG kernel for launch-latency-bound (small / medium, non-windowed) problems
  int persist_grid_ = 0, persist_lanes_ = 0;
  DevBuf<T> persist_part_;
  long long persist_solves_ = 0;
  bool persistent_cg_ok();
  void launch_persistent_cg(double tol_num);
  void cg_iteration_launches(const int* done);
  void build_cg_graphs(const int* done);
  void destroy_cg_graphs();
  // direct LDL' plugin (ldl.cuh): symbolic analysis on the host, factor and solves as captured graphs
  bool ldl_ready_ = false;
  bool ldl_dirty_ = true;          // rho_vec_ or sigma changed since the last factorisation
  std::vector<ldl::Segment> ldl_fseg_, ldl_bseg_;
  std::vector<int> ldl_fptr_h_, ldl_bptr_h_;
  int ldl_N_ = 0, ldl_ws_ctas_ = 1, ldl_solve_nodes_ = 0, ldl_factor_nodes_ = 0;
  long long ldl_nnzK_ = 0, ldl_nnzL_ = 0, ldl_factorizations_ = 0;
  double ldl_symbolic_s_ = 0.0, ldl_factor_s_ = 0.0;
  DevBuf<int64_t> ldl_Kp_, ldl_Ksp_, ldl_Ksrc_, ldl_Lp_, ldl_Rp_, ldl_Rmap_;
  DevBuf<int> ldl_Ki_, ldl_Li_, ldl_Rj_, ldl_fcols_, ldl_fptr_, ldl_bcols_, ldl_bptr_, ldl_perm_, ldl_flags_;
  DevBuf<T> ldl_Kx_, ldl_Lx_, ldl_Rx_, ldl_D_, ldl_Dinv_, ldl_ws_, ldl_y_;
  GraphExec ldl_factor_graph_, ldl_solve_graph_;
  Event ldl_ev_[2];
  void ldl_setup();
  void ldl_factor();
  void ldl_solve();
  void destroy_ldl_factor_graph() { ldl_factor_graph_.reset(); }
  bool direct_kkt() const { return st_.kkt_solver == COSMO_B200_KKT_LDL || st_.kkt_solver == COSMO_B200_KKT_LDL_SUPERNODAL; }
  void direct_factor() {
    if (st_.kkt_solver == COSMO_B200_KKT_LDL) ldl_factor();
    else if (st_.kkt_solver == COSMO_B200_KKT_LDL_SUPERNODAL) sn_factor();
  }
  // supernodal LDL' plugin (ldl_sn.cuh): host analysis, factor and solves as captured graphs
  struct SnBig { int s; int64_t groups, chunk; };
  struct SnLevel { int small0 = 0, small1 = 0; size_t smem = 0; std::vector<SnBig> big; };
  bool sn_ready_ = false;
  bool sn_dirty_ = true;           // rho_vec_ or sigma changed since the last factorisation
  ldl_sn::Symbolic sn_;            // the analysis; the graphs are built from it
  std::vector<SnLevel> sn_levels_;
  int sn_solve_nodes_ = 0, sn_factor_nodes_ = 0, sn_small_count_ = 0, sn_tiled_count_ = 0;
  long long sn_factorizations_ = 0;
  double sn_symbolic_s_ = 0.0, sn_factor_s_ = 0.0;
  DevBuf<int64_t> sn_rptr_, sn_off_, sn_uptr_, sn_Ksp_, sn_Ksrc_, sn_Kpos_, sn_gptr_;
  DevBuf<int> sn_sptr_, sn_rows_, sn_ud_, sn_up0_, sn_up1_, sn_gd_, sn_gi_, sn_perm_, sn_small_, sn_lrows_, sn_lcols_,
      sn_bcols_, sn_flags_;
  DevBuf<T> sn_Lx_, sn_D_, sn_Dinv_, sn_part_, sn_y_;
  GraphExec sn_factor_graph_, sn_solve_graph_;
  void sn_setup();
  void sn_factor();
  void sn_solve();
  long long kkt_counter_ = 1;   // S.iteration_counter
  int last_cg_iters_ = 1;
  // tm_ = rho .* (A xsol_), stored by the fused ADMM tail: the next CG solve of the same solve() starts from it instead
  // of recomputing the product.  It never outlives one solve() call: solve() and kkt_solve() clear it on entry (so
  // warm_start, reset, update_qb/update_rho/update_settings in between cannot leave it stale), a rho adaptation clears
  // it, and kkt_core consumes it and sets it again only from a tail that stored tm_ for the chained CG loop.
  bool tm_valid_ = false;
  long long total_inner_ = 0, total_mults_ = 0;
  // scratch
  DevBuf<T> vec_m_, vec_n_, vec_n2_, dy_, dx_, ypart_;
  DevBuf<unsigned> chunk_ticket_;
  int num_sms_ = 132;
  DevBuf<T> sc_;       // device scalars
  DevBuf<int> isc_;
  DevBuf<T> partials_;
  DevBuf<unsigned> ticket_;
  PinnedBuf<T> h_sc_;  // host mirrors
  PinnedBuf<int> h_isc_;
  cudaStream_t stream_ = nullptr;
  Event ev0_, ev1_;
  long long launches_ = 0;
  // multi-GPU
  int nranks_ = 1, rank_ = 0;
  NcclComm comm_ = nullptr;
  // peer-memory exchange of the reduced-KKT operator partials (replaces the per-application allreduce)
  bool p2p_ = false;
  P2pView<T> xv_;
  DevBuf<T> xchg_data_;
  DevBuf<unsigned> xchg_flags_, xchg_seq_, xchg_arrive_;
  std::vector<void*> ipc_opened_;

  // ---- helpers ----
  RedBuf<T> red(int out_slot) { return RedBuf<T>{partials_.p, sc_.p + out_slot, ticket_.p}; }
  RedBuf<T> red_ptr(T* out) { return RedBuf<T>{partials_.p, out, ticket_.p}; }
  // K5 + K7 pass over w: the projection (do_proj) and / or the right-hand side of admm_x! from ws_rhs (do_rhs).
  // 128-bit kernel for fp64 when every (n+m)-vector's m-part is 16-byte aligned (n even; ws_rhs too)
  void launch_proj_rhs(const T* w, const T* ws_rhs, bool do_proj, bool do_rhs) {
    ProjRhsArgs<T> a;
    a.n = n_; a.m = m_; a.w = w; a.ws_rhs = ws_rhs;
    a.q = q_.p; a.b = b_.p; a.rho = rho_vec_.p; a.box_l = box_l_.p; a.box_u = box_u_.p;
    a.row_class = row_class_.p; a.row_cone = row_cone_.p;
    a.soc = SocTable<T>{soc_off_.p, soc_norm_.p};
    a.s = s_.p; a.ls = ls_.p; a.t0 = t0_.p; a.sigma = (T)st_.sigma;
    a.do_proj = do_proj ? 1 : 0; a.do_rhs = do_rhs ? 1 : 0;
    if constexpr (std::is_same<T, double>::value) {
      if ((a.n & 1) == 0 && ((reinterpret_cast<uintptr_t>(a.ws_rhs) & 15) == 0) && ((reinterpret_cast<uintptr_t>(a.w) & 15) == 0)) {
        const long long pairs = (a.n >> 1) + ((a.m + 1) >> 1);
        proj_rhs_vec2_kernel<<<vgrid(pairs), kBlock, 0, stream_>>>(a);
        check_launch("proj_rhs_vec2");
        return;
      }
    }
    proj_rhs_kernel<T><<<vgrid((long long)a.n + a.m), kBlock, 0, stream_>>>(a);
    check_launch("proj_rhs");
  }
  static int vgrid(long long n) { return (int)std::min<long long>(std::max<long long>((n + kBlock - 1) / kBlock, 1), kMaxGrid); }
  static int sgrid(long long rows, int lanes) {
    long long per = kBlock / lanes;
    return (int)std::min<long long>(std::max<long long>((rows + per - 1) / per, 1), kMaxGrid);
  }
  void check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) throw EngineError{COSMO_B200_ERR_CUDA, std::string("launch of ") + what + " failed: " + cudaGetErrorString(e)};
    ++launches_;
  }
  void sync() { CUDA_TRY(cudaStreamSynchronize(stream_)); }
  void upload_vec(DevBuf<T>& dst, const void* host, size_t count);
  void download_vec(void* host, const T* src, size_t count);
  void build_csr(DevCsr<T>& dst, const HostCsr& h);
  void build_windows(DevCsr<T>& dst, const HostCsr& h, const int* src);
  void write_values(const void* Px, const void* Ax, const void* q, const void* b);
  void upload_values(const void* Px, const void* Ax, const void* q, const void* b, DevBuf<T>& px);
  void values_placed(const T* Px, bool A, bool b);
  void finish_update(const T* Px, bool A, bool b, double t0);
  void gather_csr(DevCsr<T>& M, const T* v);
  int exponent_window();
  void update_slab(DevCsr<T>& M, int ebase);
  void upload_value_maps();
  bool maps_ready_ = false;        // d_src / d_wsrc of A_, At_, P_ are on the device
  void classify_and_set_rho(bool reset_rho);
  void write_rho_vec();
  void allreduce_sum(T* buf, size_t count);
  void allreduce_max(T* buf, size_t count);

  template <typename Epi>
  void launch_spmv(const DevCsr<T>& M1, const T* x1, const DevCsr<T>* M2, const T* x2, int nrows, const Epi& epi,
                   RedBuf<T> rb, const char* name, T* pbuf = nullptr);
  template <typename Epi, int PL>
  void launch_win(const DevCsr<T>& M1, const T* x1, CsrView<T> v2, const T* x2, const Epi& epi, RedBuf<T> rb, T* pbuf);
  template <typename Epi, int PL, bool PACKED>
  void launch_win_layout(const DevCsr<T>& M1, const T* x1, CsrView<T> v2, const T* x2, const Epi& epi, RedBuf<T> rb, T* pbuf);
  void project_device(const T* w, bool with_rhs, const T* ws_rhs);
  void soc_norms(const T* ws, T* norm_out);
  void kkt_core(bool fused_tail, const T* w_src, T* w_dst);
  void kkt_op_stage2(const int* done, const T* u, const T* t_in, T* c_out, bool exchange = false);
  void kkt_cg(const int* done, bool tm_ready);
  void kkt_minres(bool full);
  // get_tolerance (kktsolver_indirect.jl:168-170): tol_constant / k^tol_exponent for the k-th inner solve
  double inner_tol() const { return st_.tol_constant / pow((double)kkt_counter_, st_.tol_exponent); }
  template <typename Enqueue>
  int poll_inner(const Enqueue& enqueue);
  void set_maxit(int v);
  void compute_residuals(const T* x, const T* s, const T* mu, bool ignore_scaling, double out[5]);
  bool adapt_rho(const T* x);
  bool primal_infeasible();
  bool dual_infeasible();
  int cone_certificates(const T* v, T eps, int which);
  double inf_rec_[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // what the last primal_infeasible / dual_infeasible computed
  void recover_mu(const T* w_prev) {
    recover_mu_kernel<T><<<vgrid(m_), kBlock, 0, stream_>>>(m_, rho_vec_.p, w_prev + n_, s_.p, mu_.p);
    check_launch("recover_mu");
  }
  void read_scalars(int first, int count) {
    CUDA_TRY(cudaMemcpyAsync(h_sc_.p + first, sc_.p + first, count * sizeof(T), cudaMemcpyDeviceToHost, stream_));
    sync();
  }
};

// ---------------------------------------------------------------------------
template <typename T>
void Engine<T>::upload_vec(DevBuf<T>& dst, const void* host, size_t count) {
  if (count == 0) return;
  CUDA_TRY(cudaMemcpyAsync(dst.p, host, count * sizeof(T), cudaMemcpyDefault, stream_));
}
template <typename T>
void Engine<T>::download_vec(void* host, const T* src, size_t count) {
  if (count == 0) return;
  CUDA_TRY(cudaMemcpyAsync(host, src, count * sizeof(T), cudaMemcpyDefault, stream_));
}

template <typename T>
void Engine<T>::build_csr(DevCsr<T>& dst, const HostCsr& h) {
  dst.nrows = h.nrows;
  dst.ncols = h.ncols;
  dst.nnz = (long long)h.col.size();
  dst.lanes = pick_lanes(h.nrows ? (double)dst.nnz / h.nrows : 0.0);
  dst.rowptr.alloc(h.nrows + 1, false);
  dst.col.alloc(dst.nnz + 4, true);   // +4: the vector path never reads past nnz, padding keeps ASAN-style tools quiet
  dst.val.alloc(dst.nnz + 4, true);
  dst.rowptr.upload(h.rowptr.data(), h.nrows + 1, stream_);
  dst.col.upload(h.col.data(), dst.nnz, stream_);
  sync();
}

// Column-windowed storage for spmv_win_kernel (see spmv.cuh).
//
// Inside one 256-entry step of a row segment, lane l / slot i reads entry l*8+i, and the
// shared-memory gather of slot i is issued per half-warp: the 16 lanes of a half-warp hit
// distinct 8-byte banks iff their window-local columns differ mod 16.  The order of the
// nonzeros inside a row is ours to choose (a dot product does not care), so the builder
// deals the entries of every residue class (col mod 16) over the (step, half-warp, slot)
// groups such that a group holds at most one entry per class whenever that is possible:
// the gathers become (nearly) bank-conflict free.
namespace {
struct WinGroupScratch {
  std::vector<int> cap, load;
  std::vector<unsigned short> used;
  std::vector<std::vector<int>> members;
  std::vector<int> bucket[16];
};
}  // namespace

static void win_fill_segment(const int* cols, const int* src, const int* idx, int k, int wbase, long long start,
                             unsigned short* wc, int* wsrc, WinGroupScratch& S) {
  constexpr int GL = 16;                // lanes that share one shared-memory wavefront: a half-warp
  const int kpad = (k + 7) & ~7;
  if (kpad == 0) return;
  const int lanes_total = kpad / 8;
  const int steps = (lanes_total + 31) / 32;
  const int SUB = 32 / GL;              // lane groups per step
  const int GPS = SUB * 8;              // (lane group, slot) groups per step
  const int G = steps * GPS;
  S.cap.assign(G, 0); S.load.assign(G, 0); S.used.assign(G, 0);
  if ((int)S.members.size() < G) S.members.resize(G);
  for (int g = 0; g < G; ++g) S.members[g].clear();
  for (int st = 0; st < steps; ++st) {
    const int ls = std::min(32, lanes_total - 32 * st);
    for (int h = 0; h < SUB; ++h) {
      const int cap = std::max(0, std::min(GL, ls - GL * h));
      for (int i = 0; i < 8; ++i) S.cap[st * GPS + h * 8 + i] = cap;
    }
  }
  for (int r = 0; r < 16; ++r) S.bucket[r].clear();
  for (int e = 0; e < k; ++e) S.bucket[(cols[idx[e]] - wbase) & 15].push_back(idx[e]);
  int cls[16];
  for (int r = 0; r < 16; ++r) cls[r] = r;
  std::sort(cls, cls + 16, [&](int a, int b) { return S.bucket[a].size() > S.bucket[b].size(); });
  int cursor = 0;   // rotating start keeps the scan short and the loads balanced
  for (int ci = 0; ci < 16; ++ci) {
    const int r = cls[ci];
    for (int e : S.bucket[r]) {
      int best = -1, best_free = 0, fallback = -1, fb_free = 0;
      // bounded scan from the rotating cursor (long rows have hundreds of groups: an unbounded scan made the build
      // quadratic in the row length -- 15 s for the 10 000-entry rows of config C3); a second, unbounded pass only if
      // the window found no free slot at all
      const int scan = std::min(G, 96);
      for (int pass = 0; pass < 2 && best < 0 && fallback < 0; ++pass) {
        const int lim = pass == 0 ? scan : G;
        for (int t = 0; t < lim; ++t) {
          const int g = (cursor + t) % G;
          const int free_slots = S.cap[g] - S.load[g];
          if (free_slots <= 0) continue;
          if (!((S.used[g] >> r) & 1)) { if (free_slots > best_free) { best = g; best_free = free_slots; if (free_slots == GL) break; } }
          else if (free_slots > fb_free) { fallback = g; fb_free = free_slots; }
        }
      }
      const int g = best >= 0 ? best : fallback;
      S.members[g].push_back(e);
      S.used[g] |= (unsigned short)(1u << r);
      S.load[g]++;
      cursor = (g + 1) % G;
    }
  }
  for (int g = 0; g < G; ++g) {
    const int st = g / GPS, h = (g % GPS) / 8, i = g % 8;
    const int nl = S.cap[g];
    for (int t = 0; t < nl; ++t) {
      // column position: lane-contiguous (one 16-byte load per lane); the value of the same entry sits at its
      // instruction-coalesced position (matup::value_pos)
      const int lane = GL * h + t;
      const long long pos_c = start + (long long)st * 256 + (long long)lane * 8 + i;
      if (t < S.load[g]) {
        const int e = S.members[g][t];
        if (wc) wc[pos_c] = (unsigned short)(cols[e] - wbase);
        wsrc[pos_c] = src ? src[e] : e;
      } else {   // padding: zero value on a bank this group does not use yet
        int r0 = 0;
        while (r0 < 15 && ((S.used[g] >> r0) & 1)) ++r0;
        S.used[g] |= (unsigned short)(1u << r0);
        if (wc) wc[pos_c] = (unsigned short)r0;
        wsrc[pos_c] = -1;
      }
    }
  }
}

// fn(a, b) on contiguous ranges [a, b) of nr rows, one host thread each
static void parallel_rows(int nr, const std::function<void(int, int)>& fn) {
  const int nthreads = (int)std::max(1u, std::min(32u, std::thread::hardware_concurrency()));
  std::vector<std::thread> th;
  const int chunk = (nr + nthreads - 1) / nthreads;
  for (int t = 0; t < nthreads; ++t) {
    const int a = t * chunk, b = std::min(nr, a + chunk);
    if (a < b) th.emplace_back(fn, a, b);
  }
  for (auto& x : th) x.join();
}

// Pass 2 of build_windows: the bank-aware placement of every row segment of a CSR (rowptr, col) into the slab laid out
// by rp: wc[slot] = the window-local column (or a free bank for padding), wsrc[slot] = src[k] (k itself when src is
// null), -1 for padding.  It depends on the pattern alone, so the first update_matrices runs it again (wc = nullptr) to
// recover the slot maps that create released.
static void win_place(const int* rowptr, const int* col, const int* src, int nr, int nwin, int W,
                      const std::vector<int>& rp, unsigned short* wc, int* wsrc) {
  parallel_rows(nr, [&](int a, int b) {
    WinGroupScratch S;
    std::vector<std::vector<int>> seg(nwin);
    for (int r = a; r < b; ++r) {
      for (int w = 0; w < nwin; ++w) seg[w].clear();
      for (int k = rowptr[r]; k < rowptr[r + 1]; ++k) seg[col[k] / W].push_back(k);
      for (int w = 0; w < nwin; ++w)
        win_fill_segment(col, src, seg[w].data(), (int)seg[w].size(), w * W, rp[(size_t)w * (nr + 1) + r], wc, wsrc, S);
    }
  });
}

// the slab layout line of COSMO_B200_SETUP_DEBUG (create and update_matrices)
template <typename T>
static void report_windows(const DevCsr<T>& d) {
  if (getenv("COSMO_B200_SETUP_DEBUG") == nullptr) return;
  const double bytes = (double)d.w_elems * (d.packed ? 9 : sizeof(T) + 2) + 8.0 * d.w_nesc;
  fprintf(stderr, "[setup] windows %d x %d, %d rows: %s layout, ebase %d, %lld escapes, slab %.1f MB\n", d.nwin, d.W, d.nrows,
          d.packed ? "9 B" : sizeof(T) == 8 ? "10 B" : "6 B", d.ebase, d.w_nesc, bytes / 1e6);
}

template <typename T>
void Engine<T>::build_windows(DevCsr<T>& dst, const HostCsr& h, const int* src) {
  dst.windowed = false;
  dst.packed = false;
  if (h.nrows == 0 || h.ncols == 0) return;
  const long long nnz = (long long)h.col.size();
  const int Wmax = (int)(204800 / sizeof(T));
  const int nwin = (h.ncols + Wmax - 1) / Wmax;
  if (nwin > 16) return;
  const double per_seg = (double)nnz / ((double)h.nrows * nwin);
  if (per_seg < 24.0) return;                     // short rows: padding + per-row overhead would dominate
  int W = (h.ncols + nwin - 1) / nwin;
  W = (W + 31) & ~31;
  if (W > 65536) return;                          // 16-bit window-local indices
  const int nr = h.nrows;
  std::vector<int> rp((size_t)nwin * (nr + 1), 0);
  std::vector<long long> row_cost(nr, 0);
  // pass 1: padded segment lengths
  parallel_rows(nr, [&](int a, int b) {
    std::vector<int> cnt(nwin);
    for (int r = a; r < b; ++r) {
      std::fill(cnt.begin(), cnt.end(), 0);
      for (int k = h.rowptr[r]; k < h.rowptr[r + 1]; ++k) cnt[h.col[k] / W]++;
      for (int w = 0; w < nwin; ++w) {
        const int padded = (cnt[w] + 7) & ~7;
        rp[(size_t)w * (nr + 1) + r + 1] = padded;
        row_cost[r] += padded + 48;   // per-row latency overhead measured at ~40 streamed entries (C3: 40k one-entry rows)
      }
    }
  });
  // window-major layout: all rows of window 0, then window 1, ...
  long long run = 0;
  for (int w = 0; w < nwin; ++w) {
    int* p = rp.data() + (size_t)w * (nr + 1);
    long long prev = run;
    for (int r = 0; r < nr; ++r) { const int len = p[r + 1]; p[r] = (int)prev; prev += len; if (prev >= (1LL << 31) - 16) return; }
    p[nr] = (int)prev;
    run = prev;
  }
  const long long total = run;
  std::vector<unsigned short> wc((size_t)total + 8, 0);
  std::vector<int> wsrc((size_t)total + 8, -1);
  win_place(h.rowptr.data(), h.col.data(), src, nr, nwin, W, rp, wc.data(), wsrc.data());
  // contiguous row chunks per CTA, balanced by padded nnz (+ per-row overhead)
  // one CTA per (row chunk, window): chunks are contiguous row ranges balanced by padded nnz
  const int nchunks = std::max(1, num_sms_ / nwin);
  const int nctas = nchunks * nwin;
  std::vector<int> cta_rows(nchunks + 1, nr);
  long long all_cost = 0;
  for (int r = 0; r < nr; ++r) all_cost += row_cost[r];
  cta_rows[0] = 0;
  long long acc = 0;
  int g = 1;
  for (int r = 0; r < nr && g < nchunks; ++r) {
    acc += row_cost[r];
    while (g < nchunks && acc * nchunks >= all_cost * g) { cta_rows[g] = r + 1; ++g; }
  }
  for (; g < nchunks; ++g) cta_rows[g] = nr;
  cta_rows[nchunks] = nr;
  dst.nwin = nwin; dst.W = W; dst.nctas = nctas; dst.w_elems = total;
  dst.w_rowptr.upload(rp, stream_);
  dst.w_cta_rows.upload(cta_rows, stream_);
  // the values go in later (update_slab), through the slot map
  dst.w_col.upload(wc, stream_);
  dst.d_wsrc.upload(wsrc, stream_);
  sync();
  // fp64: the 9 B layout when the window-local columns fit its column bits, unless the values need too many escapes
  // (update_slab)
  dst.packable = sizeof(T) == sizeof(double) && W - 1 <= (int)winpack::kMaxCol;
  dst.windowed = true;
}

// CSR of a matrix from the CSR of its transpose (its CSC pattern): stable counting-sort transposition, with
// csr.src[k] = the CSC index of the entry at CSR position k
static void csr_transpose(const HostCsr& csr_t, HostCsr& csr) {
  const long long nr = csr_t.ncols, nc = csr_t.nrows, nnz = (long long)csr_t.col.size();
  csr.nrows = (int)nr; csr.ncols = (int)nc;
  csr.rowptr.assign(nr + 1, 0);
  csr.col.resize(nnz);
  csr.src.resize(nnz);
  // Parallel over column blocks: thread t counts the rows of its columns, a prefix over (row, thread) gives every thread
  // its own slots in every row, so the scatter needs no synchronisation and the entries of a row stay ordered by column
  // whatever the thread count (deterministic).
  const int nt = (int)std::max<long long>(1, std::min<long long>(std::min<long long>(32, (long long)std::thread::hardware_concurrency()),
                                                                  std::min<long long>(nnz / 200000 + 1, nc ? nc : 1)));
  std::vector<long long> cb(nt + 1, 0);                    // column block boundaries, balanced by nnz
  for (int t = 1; t < nt; ++t) {
    const long long target = nnz * t / nt;
    cb[t] = std::lower_bound(csr_t.rowptr.begin(), csr_t.rowptr.end(), (int)target) - csr_t.rowptr.begin();
    if (cb[t] > nc) cb[t] = nc;
    if (cb[t] < cb[t - 1]) cb[t] = cb[t - 1];
  }
  cb[nt] = nc;
  std::vector<std::vector<int>> cnt(nt);
  auto run = [&](const std::function<void(int)>& fn) {
    if (nt == 1) { fn(0); return; }
    std::vector<std::thread> th;
    for (int t = 0; t < nt; ++t) th.emplace_back(fn, t);
    for (auto& x : th) x.join();
  };
  run([&](int t) {
    cnt[t].assign(nr, 0);
    for (long long k = csr_t.rowptr[cb[t]]; k < csr_t.rowptr[cb[t + 1]]; ++k) cnt[t][csr_t.col[k]]++;
  });
  for (long long r = 0; r < nr; ++r) {
    int run_sum = csr.rowptr[r];
    for (int t = 0; t < nt; ++t) { const int c = cnt[t][r]; cnt[t][r] = run_sum; run_sum += c; }   // cnt -> first slot of (t, r)
    csr.rowptr[r + 1] = run_sum;
  }
  run([&](int t) {
    std::vector<int>& next = cnt[t];
    for (long long j = cb[t]; j < cb[t + 1]; ++j)
      for (int k = csr_t.rowptr[j]; k < csr_t.rowptr[j + 1]; ++k) {
        const int dstk = next[csr_t.col[k]]++;
        csr.col[dstk] = (int)j;
        csr.src[dstk] = k;
      }
  });
}

// Julia CSC pattern -> (a) CSR of the transpose (zero conversion: same arrays, rebased)
//                      (b) CSR of the matrix itself, with its CSR -> CSC map (csr_transpose)
static void csc_to_host_csrs(const cosmo_b200_csc& M, int base, HostCsr& csr, HostCsr& csr_t) {
  const long long nr = M.nrows, nc = M.ncols;
  if (nr < 0 || nc < 0 || nr >= (1LL << 31) - 8 || nc >= (1LL << 31) - 8)
    throw EngineError{COSMO_B200_ERR_INVALID, "matrix dimensions out of int32 range"};
  const long long nnz = nc ? (M.colptr[nc] - base) : 0;
  if (nnz < 0 || nnz >= (1LL << 31) - 8) throw EngineError{COSMO_B200_ERR_INVALID, "nnz out of int32 range"};
  csr_t.nrows = (int)nc; csr_t.ncols = (int)nr;
  csr_t.rowptr.resize(nc + 1);
  csr_t.col.resize(nnz);
  for (long long j = 0; j <= nc; ++j) {
    long long v = nc ? M.colptr[j] - base : 0;
    if (v < 0 || v > nnz || (j > 0 && v < csr_t.rowptr[j - 1])) throw EngineError{COSMO_B200_ERR_INVALID, "colptr not monotone"};
    csr_t.rowptr[j] = (int)v;
  }
  std::atomic<bool> bad{false};
  parallel_rows((int)nc, [&](int a, int b) {
    for (long long k = csr_t.rowptr[a]; k < csr_t.rowptr[b]; ++k) {
      const long long r = M.rowval[k] - base;
      if (r < 0 || r >= nr) { bad = true; return; }
      csr_t.col[k] = (int)r;
    }
  });
  if (bad) throw EngineError{COSMO_B200_ERR_INVALID, "rowval out of range"};
  csr_transpose(csr_t, csr);
}

template <typename T>
Engine<T>::Engine(const cosmo_b200_problem& p, const cosmo_b200_settings& st) : st_(st) {
  if (p.m < 0 || p.n < 0 || p.m >= (1LL << 31) - 8 || p.n >= (1LL << 31) - 8)
    throw EngineError{COSMO_B200_ERR_INVALID, "model size out of range"};
  n_ = (int)p.n; m_ = (int)p.m; device_ = p.device;
  if (p.A.nrows != p.m || p.A.ncols != p.n) throw EngineError{COSMO_B200_ERR_INVALID, "A must be m x n"};
  if (p.P.nrows != p.n || p.P.ncols != p.n) throw EngineError{COSMO_B200_ERR_INVALID, "P must be n x n"};
  if (st.adaptive_rho && st.adaptive_rho_interval < 0) throw EngineError{COSMO_B200_ERR_INVALID, "adaptive_rho_interval < 0"};
  const double t_ctor0 = now_s();
  int ndev = 0;
  cudaError_t de = cudaGetDeviceCount(&ndev);
  if (de != cudaSuccess || ndev == 0)
    throw EngineError{COSMO_B200_ERR_CUDA, "no CUDA device available: the COSMO H100 engine has no CPU fallback"};
  if (device_ < 0 || device_ >= ndev) throw EngineError{COSMO_B200_ERR_INVALID, "bad device ordinal"};
  CUDA_TRY(cudaSetDevice(device_));
  CUDA_TRY(cudaDeviceGetAttribute(&num_sms_, cudaDevAttrMultiProcessorCount, device_));
  if (num_sms_ < 1 || num_sms_ > kMaxGrid) num_sms_ = 132;
  CUDA_TRY(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
  ev0_.create();
  ev1_.create();
  h_sc_.alloc(SC_COUNT);
  h_isc_.alloc(ISC_COUNT);

  // ---- sets -> row tables -------------------------------------------------
  long long off = 0;
  std::vector<unsigned char> row_class(m_);
  std::vector<int> row_cone(m_, 0);
  std::vector<T> box_l(m_, T(-INFINITY)), box_u(m_, T(INFINITY));
  std::vector<int> rect_off, rect_dim;
  std::vector<int> soc_off, soc_dim;
  std::vector<PsdConeDesc> psd_descs;
  std::vector<int> c3_off, c3_maxit;
  std::vector<unsigned char> c3_kind;
  std::vector<T> c3_alpha, c3_tol;
  std::map<custom::Key, int> cust_index;           // type -> position in cust_keys (first appearance order)
  std::vector<custom::Key> cust_keys;
  std::vector<std::vector<int>> cust_off, cust_dim;
  std::vector<std::vector<T>> cust_par;
  for (long long k = 0; k < p.n_sets; ++k) {
    const cosmo_b200_set& sdesc = p.sets[k];
    if (sdesc.dim < 0 || off + sdesc.dim > m_) throw EngineError{COSMO_B200_ERR_INVALID, "set dimensions exceed m"};
    unsigned char cls;
    switch (sdesc.type) {
      case COSMO_B200_ZERO: cls = ROW_ZERO; break;
      case COSMO_B200_NONNEG: cls = ROW_NONNEG; break;
      case COSMO_B200_BOX: {
        cls = ROW_BOX;
        if (!sdesc.l || !sdesc.u) throw EngineError{COSMO_B200_ERR_INVALID, "Box set without bounds"};
        const T* l = static_cast<const T*>(sdesc.l);
        const T* u = static_cast<const T*>(sdesc.u);
        for (long long i = 0; i < sdesc.dim; ++i) {
          if (l[i] > u[i]) throw EngineError{COSMO_B200_ERR_INVALID, "Box set: inconsistent lower/upper bounds"};
          box_l[off + i] = l[i]; box_u[off + i] = u[i];
        }
        break;
      }
      case COSMO_B200_SOC:
        cls = ROW_SOC;
        for (long long i = 0; i < sdesc.dim; ++i) row_cone[off + i] = (int)soc_off.size();
        if (sdesc.dim > 0) { soc_off.push_back((int)off); soc_dim.push_back((int)sdesc.dim); }
        break;
      case COSMO_B200_PSD_SQUARE:
      case COSMO_B200_PSD_TRIANGLE: {
        cls = ROW_PSD;
        long long N;
        if (sdesc.type == COSMO_B200_PSD_SQUARE) {
          N = (long long)llround(sqrt((double)sdesc.dim));
          if (N * N != sdesc.dim) throw EngineError{COSMO_B200_ERR_INVALID, "PsdCone: dimension must be a square"};
        } else {
          N = ((long long)floor(sqrt(1.0 + 8.0 * (double)sdesc.dim)) - 1) / 2;
          while (N * (N + 1) / 2 < sdesc.dim) ++N;
          if (N * (N + 1) / 2 != sdesc.dim) throw EngineError{COSMO_B200_ERR_INVALID, "PsdConeTriangle: dimension must be N(N+1)/2"};
        }
        for (long long i = 0; i < sdesc.dim; ++i) row_cone[off + i] = (int)psd_descs.size();
        if (sdesc.dim > 0) psd_descs.push_back(PsdConeDesc{(int)off, (int)N, sdesc.type == COSMO_B200_PSD_TRIANGLE ? 1 : 0});
        break;
      }
      case COSMO_B200_PSD_TRIANGLE_COMPLEX: {
        cls = ROW_PSD;
        const long long Nc = (long long)llround(sqrt((double)sdesc.dim));
        if (Nc * Nc != sdesc.dim) throw EngineError{COSMO_B200_ERR_INVALID, "complex PsdConeTriangle: dimension must be a square"};
        if (2 * Nc >= (1LL << 15)) throw EngineError{COSMO_B200_ERR_INVALID, "complex PsdConeTriangle: N too large"};
        for (long long i = 0; i < sdesc.dim; ++i) row_cone[off + i] = (int)psd_descs.size();
        // N = 1: project! is max(x, 0) (convexset.jl:404-405), the real 1 x 1 case
        if (sdesc.dim == 1) psd_descs.push_back(PsdConeDesc{(int)off, 1, 1});
        else if (sdesc.dim > 0) psd_descs.push_back(PsdConeDesc{(int)off, (int)(2 * Nc), 2});
        break;
      }
      case COSMO_B200_EXP:
      case COSMO_B200_DUAL_EXP:
      case COSMO_B200_POW:
      case COSMO_B200_DUAL_POW: {
        cls = ROW_CONE3;
        if (sdesc.dim != 3) throw EngineError{COSMO_B200_ERR_INVALID, "exponential / power cones have dimension 3"};
        const bool is_pow = (sdesc.type == COSMO_B200_POW || sdesc.type == COSMO_B200_DUAL_POW);
        if (is_pow && !(sdesc.alpha > 0.0 && sdesc.alpha < 1.0))
          throw EngineError{COSMO_B200_ERR_INVALID, "The exponent alpha of the power cone has to be in (0, 1)."};
        for (int i = 0; i < 3; ++i) row_cone[off + i] = (int)c3_off.size();
        c3_off.push_back((int)off);
        c3_kind.push_back((unsigned char)(sdesc.type - COSMO_B200_EXP));
        c3_alpha.push_back(is_pow ? (T)sdesc.alpha : T(0.5));
        c3_maxit.push_back(sdesc.max_iter > 0 ? sdesc.max_iter : (is_pow ? 20 : 100));   // convexset.jl:503, 631
        c3_tol.push_back(sdesc.tol > 0.0 ? (T)sdesc.tol : (T)1e-8);
        break;
      }
      case COSMO_B200_CUSTOM: {
        cls = ROW_CUSTOM;
        const custom::Key key = custom::make_key(static_cast<const cosmo_b200_custom_cone*>(sdesc.u),
                                                 sizeof(T) == sizeof(double) ? COSMO_B200_F64 : COSMO_B200_F32);
        if (key.n_params > 0 && !sdesc.l)
          throw EngineError{COSMO_B200_ERR_INVALID, "custom cone " + key.name + ": n_params > 0 but the set has no parameters (l)"};
        if (sdesc.alpha != 0.0 || sdesc.tol != 0.0 || sdesc.max_iter != 0)
          throw EngineError{COSMO_B200_ERR_INVALID, "custom cone " + key.name + ": alpha, tol and max_iter must be 0"};
        if (sdesc.dim == 0) break;
        auto it = cust_index.find(key);
        const int t = it != cust_index.end() ? it->second : (int)cust_keys.size();
        if (it == cust_index.end()) {
          cust_index[key] = t;
          cust_keys.push_back(key);
          cust_off.emplace_back(); cust_dim.emplace_back(); cust_par.emplace_back();
        }
        cust_off[t].push_back((int)off);
        cust_dim[t].push_back((int)sdesc.dim);
        const T* par = static_cast<const T*>(sdesc.l);
        cust_par[t].insert(cust_par[t].end(), par, par + key.n_params);
        break;
      }
      default:
        throw EngineError{COSMO_B200_ERR_UNSUPPORTED, "unsupported cone type (complex PSD): fall back to the host loop"};
    }
    for (long long i = 0; i < sdesc.dim; ++i) row_class[off + i] = cls;
    // rectify_set_scalings! (scaling.jl:129-142) gives every other cone one scalar scaling
    if (cls != ROW_ZERO && cls != ROW_NONNEG && cls != ROW_BOX && sdesc.dim > 0) {
      rect_off.push_back((int)off);
      rect_dim.push_back((int)sdesc.dim);
    }
    off += sdesc.dim;
  }
  if (off != m_) throw EngineError{COSMO_B200_ERR_INVALID, "sum of set dimensions != m"};

  // ---- matrices -----------------------------------------------------------
  const bool dbg = getenv("COSMO_B200_SETUP_DEBUG") != nullptr;
  double tp = now_s();
  auto lap = [&](const char* what) {
    if (dbg) { const double t = now_s(); fprintf(stderr, "[setup] %-22s %.3f s\n", what, t - tp); tp = t; }
  };
  lap("cone tables");
  {
    // The host lays out the patterns and the value maps; write_values fills every copy on the device below, the way
    // update_matrices does, and the maps are released after it (an engine that never updates does not keep them).
    HostCsr a, at, pp, ppt;
    csc_to_host_csrs(p.A, p.index_base, a, at);
    lap("csc -> csr (A, A')");
    build_csr(A_, a);
    build_csr(At_, at);
    A_.d_src.upload(a.src, stream_);
    lap("csr A, A'");
    build_windows(A_, a, a.src.data());
    lap("windows A");
    build_windows(At_, at, nullptr);
    lap("windows A'");
    // P's CSC order is not resident: its CSR -> CSC map stays on the host for update_matrices (A's is derived from A')
    csc_to_host_csrs(p.P, p.index_base, pp, ppt);
    build_csr(P_, pp);
    P_.d_src.upload(pp.src, stream_);
    P_.h_src.swap(pp.src);
    lap("P");
    // A' and P rows are traversed by the same lane group in the fused operator kernel
    double mean = n_ ? (double)(At_.nnz + P_.nnz) / n_ : 0.0;
    At_.lanes = pick_lanes(mean);
  }
  // ---- vectors ------------------------------------------------------------
  auto up = [&](DevBuf<T>& d, const void* h, size_t cnt) { d.alloc(cnt); if (h) upload_vec(d, h, cnt); };
  q_.alloc(n_);
  b_.alloc(m_);
  scaled_ = (p.D && p.Dinv && p.E && p.Einv);
  c_ = p.c;
  if (scaled_) { up(D_, p.D, n_); up(Dinv_, p.Dinv, n_); up(E_, p.E, m_); up(Einv_, p.Einv, m_); }
  // scaling requested but no scaling matrices handed over: the data are unscaled, equilibrate them here
  // (setup.jl:27-33 -> scale_ruiz!); the host reads D, E, c back with cosmo_b200_get_scaling
  device_scaled_ = (p.flags & COSMO_B200_PROBLEM_EQUILIBRATE) && st_.scaling != 0;
  if (device_scaled_ && scaled_)
    throw EngineError{COSMO_B200_ERR_INVALID, "COSMO_B200_PROBLEM_EQUILIBRATE expects D = Dinv = E = Einv = NULL"};
  row_class_.alloc(m_); row_cone_.alloc(m_); rho_class_.alloc(m_);
  if (m_) {
    CUDA_TRY(cudaMemcpyAsync(row_class_.p, row_class.data(), m_, cudaMemcpyHostToDevice, stream_));
    CUDA_TRY(cudaMemcpyAsync(row_cone_.p, row_cone.data(), m_ * sizeof(int), cudaMemcpyHostToDevice, stream_));
  }
  box_l_.alloc(m_); box_u_.alloc(m_);
  upload_vec(box_l_, box_l.data(), m_);
  upload_vec(box_u_, box_u.data(), m_);
  if (device_scaled_) {
    box_l0_.alloc(m_, false); box_u0_.alloc(m_, false);
    upload_vec(box_l0_, box_l.data(), m_);
    upload_vec(box_u0_, box_u.data(), m_);
    rect_off_.upload(rect_off, stream_); rect_dim_.upload(rect_dim, stream_);
  }
  sync();
  // SOC tables (chunks of <= 8192 tail rows)
  n_soc_ = (int)soc_off.size();
  if (n_soc_) {
    const int CH = 8192;
    std::vector<int> cs, cl, ptr(1, 0);
    for (int k = 0; k < n_soc_; ++k) {
      int start = soc_off[k] + 1, len = soc_dim[k] - 1;
      for (int o = 0; o < len; o += CH) { cs.push_back(start + o); cl.push_back(std::min(CH, len - o)); }
      ptr.push_back((int)cs.size());
    }
    n_soc_chunks_ = (int)cs.size();
    soc_off_.upload(soc_off, stream_); soc_dim_.upload(soc_dim, stream_);
    soc_chunk_start_.upload(cs, stream_); soc_chunk_len_.upload(cl, stream_); soc_cone_chunk_ptr_.upload(ptr, stream_);
    soc_norm_.alloc(n_soc_); soc_norm2_.alloc(n_soc_); soc_chunk_sum_.alloc(2 * std::max(n_soc_chunks_, 1));   // (scaled sum, exponent) per chunk
    sync();
  }
  psd_.init(psd_descs, stream_);
  n_c3_ = (int)c3_off.size();
  if (n_c3_) {
    c3_off_.upload(c3_off, stream_); c3_kind_.upload(c3_kind, stream_); c3_alpha_.upload(c3_alpha, stream_);
    c3_maxit_.upload(c3_maxit, stream_); c3_tol_.upload(c3_tol, stream_);
    sync();
  }
  // custom cones: compile (or find) and load every type, then one table of all cones, type by type
  if (!cust_keys.empty()) {
    std::vector<int> offs, dims;
    std::vector<T> pars;
    for (size_t t = 0; t < cust_keys.size(); ++t) {
      bool compiled = false;
      custom::Entry* e = custom::cache().get(cust_keys[t], &compiled);
      ++(compiled ? cust_compiled_ : cust_hits_);
      custom::cache().load(e);
      custom::TypeSlice ts;
      ts.entry = e; ts.first = (int)offs.size(); ts.n = (int)cust_off[t].size(); ts.param_first = (long long)pars.size();
      cust_types_.push_back(ts);
      offs.insert(offs.end(), cust_off[t].begin(), cust_off[t].end());
      dims.insert(dims.end(), cust_dim[t].begin(), cust_dim[t].end());
      pars.insert(pars.end(), cust_par[t].begin(), cust_par[t].end());
    }
    n_cust_ = (int)offs.size();
    cust_off_.upload(offs, stream_); cust_dim_.upload(dims, stream_);
    if (!pars.empty()) cust_params_.upload(pars, stream_);
    cust_flag_.alloc(n_cust_);
    cust_tmp_.alloc(m_);
    sync();
  }
  write_values(p.P.nzval, p.A.nzval, p.q, p.b);
  A_.d_src.release(); P_.d_src.release(); A_.d_wsrc.release(); At_.d_wsrc.release();
  lap("values");

  // ---- state / scratch ------------------------------------------------------
  W_[0].alloc(n_ + m_); W_[1].alloc(n_ + m_);
  xs_.alloc(n_); s_.alloc(m_); mu_.alloc(m_); rho_vec_.alloc(m_);
  ls_.alloc(n_ + m_); t0_.alloc(m_); tm_.alloc(m_); xsol_.alloc(n_);
  rhsb_.alloc(n_ + 8); cb_.alloc(n_ + 8); r_.alloc(n_); u_.alloc(n_); nu_.alloc(m_);
  vec_m_.alloc(m_); vec_n_.alloc(n_ + 8); vec_n2_.alloc(n_); dy_.alloc(m_); dx_.alloc(n_);
  ypart_.alloc((size_t)std::max(n_, m_) * 16);   // nwin <= 16 per-window partial sums
  chunk_ticket_.alloc(kMaxGrid);
  sc_.alloc(SC_COUNT); isc_.alloc(ISC_COUNT);
  partials_.alloc((size_t)kMaxGrid * kMaxRed); ticket_.alloc(1);
  {
    int h[ISC_COUNT] = {0};
    h[ISC_MAXIT] = n_;   // IterativeSolvers default maxiter = size(A, 2)
    CUDA_TRY(cudaMemcpyAsync(isc_.p, h, sizeof(h), cudaMemcpyHostToDevice, stream_));
    sync();
  }
  memset(&xv_, 0, sizeof(xv_));
  rho_ = st_.rho;
  classify_and_set_rho(true);
  sync();
  // QdldlKKTSolver's constructor factors K (kktsolver.jl:293-306): a non-convex P or a singular K fails the create
  if (direct_kkt()) direct_factor();
  create_time_ = now_s() - t_ctor0;
  auto_rho_interval_ = 0;
}

template <typename T>
void Engine<T>::destroy_cg_graphs() {
  for (auto& g : cg_graph_) g.reset();
}

template <typename T>
Engine<T>::~Engine() {
  for (void* p : ipc_opened_) cudaIpcCloseMemHandle(p);
  if (comm_ && g_nccl.CommDestroy) g_nccl.CommDestroy(comm_);
  if (stream_) cudaStreamDestroy(stream_);
}

// classify_constraints! (setup.jl:75-85; convexset.jl:62-69, 831-842) on the resident b and Box bounds, then
// set_rho_vec! / update_rho_vec! (parameters.jl:3-13, 75-81)
template <typename T>
void Engine<T>::classify_and_set_rho(bool reset_rho) {
  rho_class_kernel<T><<<vgrid(m_), kBlock, 0, stream_>>>(m_, row_class_.p, b_.p, box_l_.p, box_u_.p,
                                                         st_.COSMO_INFTY * st_.MIN_SCALING, st_.RHO_TOL, rho_class_.p);
  check_launch("rho_class");
  if (reset_rho) {
    rho_ = st_.rho;
    rho_updates_.clear();
    rho_updates_.push_back(rho_);
  }
  write_rho_vec();
}

// rho_vec_ from rho_class_ and the current rho_; the LDL factor follows it before the next KKT solve
template <typename T>
void Engine<T>::write_rho_vec() {
  rho_vec_kernel<T><<<vgrid(m_), kBlock, 0, stream_>>>(m_, rho_class_.p, (T)rho_, (T)st_.RHO_EQ_OVER_RHO_INEQ, (T)st_.RHO_MIN, rho_vec_.p);
  check_launch("rho_vec");
  ldl_dirty_ = true;
  sn_dirty_ = true;
}

// scale_ruiz! (scaling.jl:21-116) on the resident data; see ruiz.cuh
template <typename T>
void Engine<T>::equilibrate() {
  const int n = n_, m = m_;
  const T lo = (T)st_.MIN_SCALING, hi = (T)(st_.MAX_SCALING > 0.0 ? st_.MAX_SCALING : 1e4);
  D_.alloc(n, false); Dinv_.alloc(n, false); E_.alloc(m, false); Einv_.alloc(m, false);
  DevBuf<T> cdev;
  cdev.alloc(1, false);
  ruiz_fill_kernel<T><<<vgrid(n), kBlock, 0, stream_>>>(n, D_.p, T(1));
  check_launch("ruiz_fill");
  ruiz_fill_kernel<T><<<vgrid(m), kBlock, 0, stream_>>>(m, E_.p, T(1));
  check_launch("ruiz_fill");
  ruiz_fill_kernel<T><<<1, 32, 0, stream_>>>(1, cdev.p, T(1));
  check_launch("ruiz_fill");
  T* Dw = Dinv_.p;   // the inverse scalings double as work vectors, like in the reference (scaling.jl:37-41)
  T* Ew = Einv_.p;
  auto wgrid = [&](long long rows) { return (int)std::min<long long>((rows * 32 + kBlock - 1) / kBlock + 1, kMaxGrid); };
  for (int it = 0; it < st_.scaling; ++it) {
    // kkt_col_norms! (scaling.jl:3-8)
    ruiz_row_inf_kernel<T><<<wgrid(n), kBlock, 0, stream_>>>(n, P_.view(), D_.p, D_.p, cdev.p, Dw, 0);
    check_launch("ruiz_row_inf");
    ruiz_row_inf_kernel<T><<<wgrid(n), kBlock, 0, stream_>>>(n, At_.view(), D_.p, E_.p, (const T*)nullptr, Dw, 1);
    check_launch("ruiz_row_inf");
    ruiz_row_inf_kernel<T><<<wgrid(m), kBlock, 0, stream_>>>(m, A_.view(), E_.p, D_.p, (const T*)nullptr, Ew, 0);
    check_launch("ruiz_row_inf");
    ruiz_update_kernel<T><<<vgrid(n), kBlock, 0, stream_>>>(n, Dw, D_.p, lo, hi);
    check_launch("ruiz_update");
    ruiz_update_kernel<T><<<vgrid(m), kBlock, 0, stream_>>>(m, Ew, E_.p, lo, hi);
    check_launch("ruiz_update");
    // cost scaling (scaling.jl:73-90): column norms of the newly scaled P, |q|_inf
    ruiz_row_inf_kernel<T><<<wgrid(n), kBlock, 0, stream_>>>(n, P_.view(), D_.p, D_.p, cdev.p, Dw, 0);
    check_launch("ruiz_row_inf");
    ruiz_cost_kernel<T><<<1, 1024, 0, stream_>>>(n, Dw, q_.p, D_.p, cdev.p, lo, hi);
    check_launch("ruiz_cost");
  }
  // rectify_set_scalings! (scaling.jl:129-142): one scalar per cone of the table the constructor built
  if (rect_off_.n) {
    ruiz_rectify_kernel<T><<<(int)rect_off_.n, kBlock, 0, stream_>>>(rect_off_.p, rect_dim_.p, E_.p);
    check_launch("ruiz_rectify");
  }
  // apply D, E, c to the CSR copies (A and A' both scale an entry by the product D_j E_i, so they stay equal bit for
  // bit), q, b and the Box bounds; write_values fills the slabs from the scaled A' afterwards
  ruiz_apply_csr_kernel<T><<<wgrid(m), kBlock, 0, stream_>>>(m, A_.rowptr.p, A_.col.p, A_.val.p, E_.p, D_.p, (const T*)nullptr);
  check_launch("ruiz_apply_csr");
  ruiz_apply_csr_kernel<T><<<wgrid(n), kBlock, 0, stream_>>>(n, At_.rowptr.p, At_.col.p, At_.val.p, D_.p, E_.p, (const T*)nullptr);
  check_launch("ruiz_apply_csr");
  ruiz_apply_csr_kernel<T><<<wgrid(n), kBlock, 0, stream_>>>(n, P_.rowptr.p, P_.col.p, P_.val.p, D_.p, D_.p, cdev.p);
  check_launch("ruiz_apply_csr");
  ruiz_finish_n_kernel<T><<<vgrid(n), kBlock, 0, stream_>>>(n, q_.p, D_.p, Dinv_.p, cdev.p);
  check_launch("ruiz_finish_n");
  ruiz_finish_m_kernel<T><<<vgrid(m), kBlock, 0, stream_>>>(m, b_.p, E_.p, Einv_.p, row_class_.p, box_l_.p, box_u_.p);
  check_launch("ruiz_finish_m");
  T ch = T(1);
  CUDA_TRY(cudaMemcpyAsync(&ch, cdev.p, sizeof(T), cudaMemcpyDeviceToHost, stream_));
  sync();
  c_ = (double)ch;
  scaled_ = true;
}

template <typename T>
void Engine<T>::get_scaling(void* D, void* E, double* c) {
  if (!scaled_) {
    std::vector<T> one_n(n_, T(1)), one_m(m_, T(1));
    if (D) memcpy(D, one_n.data(), (size_t)n_ * sizeof(T));
    if (E) memcpy(E, one_m.data(), (size_t)m_ * sizeof(T));
    if (c) *c = 1.0;
    return;
  }
  if (D) download_vec(D, D_.p, n_);
  if (E) download_vec(E, E_.p, m_);
  sync();
  if (c) *c = c_;
}

template <typename T>
void Engine<T>::warm_start(const void* x, const void* s, const void* mu) {
  caller_arrays({x, s, mu});
  have_solution_ = false;
  if (x) upload_vec(xs_, x, n_);
  if (s) upload_vec(s_, s, m_);
  if (mu) upload_vec(mu_, mu, m_);
  sync();
}

template <typename T>
void Engine<T>::update_qb(const void* q, const void* b) {
  caller_arrays({q, b});
  if (q) upload_vec(q_, q, n_);
  if (b) {
    upload_vec(b_, b, m_);
    classify_and_set_rho(false);
  }
  sync();
}

// New values of P and/or A on the resident pattern, left in the state a create with the new data and the current
// settings leaves (mat_update.cuh): same scaling, rho vector, zero iterates, KKT call counter at 1, a fresh factor.
template <typename T>
void Engine<T>::update_matrices(const void* Px, long long nnzP, const void* Ax, long long nnzA, const void* q, const void* b) {
  if (nranks_ > 1) throw EngineError{COSMO_B200_ERR_UNSUPPORTED, "update_matrices: a sharded handle holds only a slice of the data"};
  if ((Px && nnzP != P_.nnz) || (Ax && nnzA != At_.nnz))
    throw EngineError{COSMO_B200_ERR_INVALID, "update_matrices: nnz differs from the pattern given at create (a new pattern needs a new engine)"};
  // Ruiz restarts from identity on the unscaled data, and the engine keeps only the scaled values
  if (device_scaled_ && !(Px && Ax && q && b))
    throw EngineError{COSMO_B200_ERR_INVALID, "update_matrices: an equilibrating engine needs the unscaled P, A, q and b"};
  caller_arrays({Px, Ax, q, b});
  const double t0 = now_s();
  DevBuf<T> px;
  upload_values(Px, Ax, q, b, px);
  finish_update(Px ? px.p : nullptr, Ax != nullptr, b != nullptr, t0);
}

// The same update from values in the coordinates of the problem a chordal decomposition started from: they are staged on
// the device, gathered through the forward map (chordal_fwd.cuh) into the resident arrays of the decomposed problem,
// and take the value path of update_matrices from there.  Nothing is written before every check has passed.
template <typename T>
void Engine<T>::update_matrices_original(const void* Px, long long nnzP, const void* Ax, long long nnzA_orig, const void* q,
                                         const void* b) {
  if (nranks_ > 1) throw EngineError{COSMO_B200_ERR_UNSUPPORTED, "update_matrices_original: a sharded handle holds only a slice of the data"};
  if (!fwd_.has_map()) throw EngineError{COSMO_B200_ERR_INVALID, "update_matrices_original: no forward map (cosmo_b200_set_forward_map)"};
  if ((Px && nnzP != P_.nnz) || (Ax && nnzA_orig != fwd_.nnzA_orig()))
    throw EngineError{COSMO_B200_ERR_INVALID, "update_matrices_original: nnz differs from the pattern the decomposition was made for (a new pattern needs a new engine)"};
  if (device_scaled_ && !(Px && Ax && q && b))
    throw EngineError{COSMO_B200_ERR_INVALID, "update_matrices_original: an equilibrating engine needs the unscaled P, A, q and b"};
  caller_arrays({Px, Ax, q, b});
  const double t0 = now_s();
  DevBuf<T> px, ax, b0;
  if (Px) px.alloc((size_t)P_.nnz, false);
  if (Ax) ax.alloc((size_t)fwd_.nnzA_orig(), false);
  if (b) {
    b0.alloc((size_t)fwd_.m_orig(), false);
    upload_vec(b0, b, (size_t)fwd_.m_orig());
    const long long bad = fwd_.count_uncovered<T>(b0.p, stream_);
    launches_ += 2;
    if (bad)
      throw EngineError{COSMO_B200_ERR_INVALID, "update_matrices_original: b is nonzero in " + std::to_string(bad) +
                                                    " rows of a decomposed cone that no clique holds (the sparsity pattern, and with it the decomposition, changes: a new engine is needed)"};
  }
  if (Px) upload_vec(px, Px, (size_t)P_.nnz);   // P' = blockdiag(P, 0): P's values in P's order
  if (Ax) {
    upload_vec(ax, Ax, (size_t)fwd_.nnzA_orig());
    fwd_.gather_values<T>(ax.p, At_.val.p, stream_);
    ++launches_;
  }
  if (q) {   // q' = [q; 0]
    upload_vec(q_, q, (size_t)fwd_.n_orig());
    if (n_ > fwd_.n_orig()) CUDA_TRY(cudaMemsetAsync(q_.p + fwd_.n_orig(), 0, (size_t)(n_ - fwd_.n_orig()) * sizeof(T), stream_));
  }
  if (b) {
    fwd_.gather_b<T>(b0.p, b_.p, stream_);
    ++launches_;
  }
  sync();   // the staged host arrays have been read
  finish_update(Px ? px.p : nullptr, Ax != nullptr, b != nullptr, t0);
}

// What follows the new values on the device, for both updates: every resident copy (values_placed), then the state of a
// new engine.
template <typename T>
void Engine<T>::finish_update(const T* Px, bool A, bool b, double t0) {
  upload_value_maps();
  values_placed(Px, A, b);
  destroy_cg_graphs();   // the slab and escape-table pointers they captured may have changed
  reset();
  auto_rho_interval_ = 0;
  direct_factor();   // reset() marked the factor dirty; a non-convex P fails here
  create_time_ = now_s() - t0;
}

// Host values of P, A, q and b (null: keep the current ones) to the device: A's into At_.val (CSR(A') is the CSC order of
// A), q and b into place, P's CSC values into the scratch `px` (P's CSC order is not resident).
template <typename T>
void Engine<T>::upload_values(const void* Px, const void* Ax, const void* q, const void* b, DevBuf<T>& px) {
  if (Px) {
    px.alloc((size_t)P_.nnz, false);
    upload_vec(px, Px, (size_t)P_.nnz);
  }
  if (Ax) upload_vec(At_.val, Ax, (size_t)At_.nnz);
  if (q) upload_vec(q_, q, n_);
  if (b) upload_vec(b_, b, m_);
  sync();
}

// The values of P, A, q and b from host arrays, for create.
template <typename T>
void Engine<T>::write_values(const void* Px, const void* Ax, const void* q, const void* b) {
  DevBuf<T> px;
  upload_values(Px, Ax, q, b, px);
  values_placed(Px ? px.p : nullptr, Ax != nullptr, b != nullptr);
}

// The one value path of create and of both updates, from sources in device memory: `Px` holds P's new CSC values (null:
// keep P), At_.val the new CSC values of A when `A` is set, b_ the new b when `b` is set (q_ needs nothing more).  They
// go through the value maps of mat_update.cuh into the CSR copies.  An equilibrating engine scales the CSR copies, q, b
// and its unscaled Box bounds first; the slabs come last, gathered from the final A' values, so every resident copy of A
// holds the same numbers.
template <typename T>
void Engine<T>::values_placed(const T* Px, bool A, bool b) {
  if (A) gather_csr(A_, At_.val.p);
  if (Px) gather_csr(P_, Px);
  if (device_scaled_) {
    CUDA_TRY(cudaMemcpyAsync(box_l_.p, box_l0_.p, (size_t)m_ * sizeof(T), cudaMemcpyDeviceToDevice, stream_));
    CUDA_TRY(cudaMemcpyAsync(box_u_.p, box_u0_.p, (size_t)m_ * sizeof(T), cudaMemcpyDeviceToDevice, stream_));
    equilibrate();
  }
  if (A) {
    const int ebase = A_.packable || At_.packable ? exponent_window() : 0;   // one exponent window for A and A'
    update_slab(A_, ebase);
    update_slab(At_, ebase);
  }
  sync();
}

// CSR values through the CSR -> CSC map M.d_src: M.val[k] = v[src[k]]
template <typename T>
void Engine<T>::gather_csr(DevCsr<T>& M, const T* v) {
  matup::gather_kernel<T><<<vgrid(M.nnz), kBlock, 0, stream_>>>(M.nnz, M.d_src.p, v, M.val.p);
  check_launch("gather_csr");
  sync();
}

// The window base of the packed slabs of A and A' (win_pack.h): the kCodes binades that hold the most finite normal
// values of A, from its values in At_.val.  Integer histogram on the device, window picked on the host.
template <typename T>
int Engine<T>::exponent_window() {
  if constexpr (sizeof(T) != sizeof(double)) {
    return 0;
  } else {
    DevBuf<unsigned long long> hist;
    hist.alloc(2048);
    matup::exp_hist_kernel<<<std::min(vgrid(At_.nnz), 4 * num_sms_), kBlock, 0, stream_>>>(At_.nnz, At_.val.p, hist.p);
    check_launch("exp_hist");
    std::vector<long long> h(2048);
    CUDA_TRY(cudaMemcpyAsync(h.data(), hist.p, 2048 * sizeof(long long), cudaMemcpyDeviceToHost, stream_));
    sync();
    return winpack::pick_ebase(h.data());
  }
}

// The value maps of update_matrices, made by the first update and kept on the device.  Creating an engine keeps only
// the CSR(P) map (P's CSC order is not resident); the others are derived again from the resident pattern with the
// functions create used: CSR(A) position -> CSC index by csr_transpose of A' (the CSC pattern itself), and slab slot ->
// CSC index, -1 for padding, by win_place on the same CSR pattern and row layout.  Padding cannot be told from a stored
// zero by its content, but the placement is a function of the pattern, so it places every entry where create placed
// it.  Engines that never update pay nothing for the maps, in time or memory.
template <typename T>
void Engine<T>::upload_value_maps() {
  if (maps_ready_) return;
  auto down = [&](std::vector<int>& v, const int* d, size_t cnt) {
    v.resize(cnt);
    if (cnt) CUDA_TRY(cudaMemcpyAsync(v.data(), d, cnt * sizeof(int), cudaMemcpyDeviceToHost, stream_));
  };
  HostCsr a, at;
  at.nrows = n_; at.ncols = m_;
  down(at.rowptr, At_.rowptr.p, (size_t)n_ + 1);
  down(at.col, At_.col.p, (size_t)At_.nnz);
  sync();
  csr_transpose(at, a);
  A_.d_src.upload(a.src, stream_);
  P_.d_src.upload(P_.h_src, stream_);
  auto slab = [&](DevCsr<T>& M, const HostCsr& h, const int* src) {
    if (!M.windowed) return;
    std::vector<int> rp;
    down(rp, M.w_rowptr.p, (size_t)M.nwin * (M.nrows + 1));
    sync();
    std::vector<int> wsrc((size_t)M.w_elems + 8, -1);
    win_place(h.rowptr.data(), h.col.data(), src, M.nrows, M.nwin, M.W, rp, nullptr, wsrc.data());
    M.d_wsrc.upload(wsrc, stream_);
    sync();
  };
  slab(A_, a, a.src.data());
  slab(At_, at, nullptr);
  sync();
  std::vector<int>().swap(P_.h_src);
  maps_ready_ = true;
}

// Slab values of a windowed matrix from the CSC values in At_.val, in the layout their escapes call for (win_pack.h).
// create calls it on a fresh slab, which holds the columns (w_col) and no values yet; an update on a filled one, in
// either layout.
template <typename T>
void Engine<T>::update_slab(DevCsr<T>& M, int ebase) {
  if (!M.windowed) return;
  const long long nseg = (long long)M.nwin * M.nrows;
  const int grid = (int)std::min<long long>((nseg * 32 + kBlock - 1) / kBlock, kMaxGrid);
  if constexpr (sizeof(T) == sizeof(double)) {
    if (M.packable) {
      DevBuf<int> cnt;
      cnt.alloc((size_t)nseg, false);
      matup::slab_esc_count_kernel<<<grid, kBlock, 0, stream_>>>(M.nwin, M.nrows, M.w_rowptr.p, M.d_wsrc.p, At_.val.p, ebase, cnt.p);
      check_launch("slab_esc_count");
      std::vector<int> hc((size_t)nseg);
      CUDA_TRY(cudaMemcpyAsync(hc.data(), cnt.p, (size_t)nseg * sizeof(int), cudaMemcpyDeviceToHost, stream_));
      sync();
      std::vector<long long> off((size_t)nseg + 1, 0);   // escape slots in slab order: window, row, entry
      for (long long g = 0; g < nseg; ++g) off[g + 1] = off[g] + hc[g];
      const long long nesc = off.back();
      if (nesc * winpack::kEscDen <= M.w_elems) {
        DevBuf<long long> doff;
        doff.upload(off, stream_);
        if ((long long)M.w_esc.n < nesc) M.w_esc.alloc((size_t)nesc, false);
        if (!M.packed) {   // 10 B (or fresh) -> 9 B: the columns come from w_col
          M.w_word.alloc((size_t)M.w_elems + 8);
          M.w_colhi.alloc((size_t)M.w_elems + 8);
          matup::slab_encode_kernel<true><<<grid, kBlock, 0, stream_>>>(M.nwin, M.nrows, M.w_rowptr.p, M.d_wsrc.p, At_.val.p, ebase,
                                                                       doff.p, M.w_col.p, M.w_word.p, M.w_colhi.p, M.w_esc.p);
          check_launch("slab_encode");
          sync();
          M.w_col.release();
          M.w_val.release();
        } else {
          matup::slab_encode_kernel<false><<<grid, kBlock, 0, stream_>>>(M.nwin, M.nrows, M.w_rowptr.p, M.d_wsrc.p, At_.val.p, ebase,
                                                                        doff.p, nullptr, M.w_word.p, M.w_colhi.p, M.w_esc.p);
          check_launch("slab_encode");
          sync();
        }
        M.packed = true;
        M.ebase = ebase;
        M.w_nesc = nesc;
        report_windows(M);
        return;
      }
      if (M.packed) {   // 9 B -> 10 B: decode the columns before the words go
        M.w_col.alloc((size_t)M.w_elems + 8);
        matup::slab_unpack_col_kernel<<<grid, kBlock, 0, stream_>>>(M.nwin, M.nrows, M.w_rowptr.p, M.w_word.p, M.w_colhi.p, M.w_col.p);
        check_launch("slab_unpack_col");
        sync();
        M.w_word.release();
        M.w_colhi.release();
        M.w_esc.release();
        M.packed = false;
        M.ebase = 0;
        M.w_nesc = 0;
      }
    }
  }
  if (!M.w_val.p) M.w_val.alloc((size_t)M.w_elems + 8);   // a fresh slab, or one that was 9 B
  matup::slab_gather_kernel<T><<<grid, kBlock, 0, stream_>>>(M.nwin, M.nrows, M.w_rowptr.p, M.d_wsrc.p, At_.val.p, M.w_val.p);
  check_launch("slab_gather");
  sync();
  report_windows(M);
}

template <typename T>
void Engine<T>::update_rho(const void* rho_vec, double rho) {
  if (rho_vec) upload_vec(rho_vec_, rho_vec, m_);
  rho_ = rho;
  ldl_dirty_ = true;   // update_rho! -> refactor! (kktsolver.jl:310-313), done before the next KKT solve
  sn_dirty_ = true;
  sync();
}

template <typename T>
void Engine<T>::reset() {
  CUDA_TRY(cudaMemsetAsync(xs_.p, 0, std::max(n_, 1) * sizeof(T), stream_));
  CUDA_TRY(cudaMemsetAsync(s_.p, 0, std::max(m_, 1) * sizeof(T), stream_));
  CUDA_TRY(cudaMemsetAsync(mu_.p, 0, std::max(m_, 1) * sizeof(T), stream_));
  CUDA_TRY(cudaMemsetAsync(xsol_.p, 0, std::max(n_, 1) * sizeof(T), stream_));
  CUDA_TRY(cudaMemsetAsync(W_[0].p, 0, std::max(n_ + m_, 1) * sizeof(T), stream_));
  CUDA_TRY(cudaMemsetAsync(W_[1].p, 0, std::max(n_ + m_, 1) * sizeof(T), stream_));
  if (mr_x_.p) CUDA_TRY(cudaMemsetAsync(mr_x_.p, 0, mr_x_.n * sizeof(T), stream_));
  kkt_counter_ = 1;
  last_cg_iters_ = 1;
  have_solution_ = false;
  psd_.reset_warm_start();
  classify_and_set_rho(true);
  sync();
}

template <typename T>
void Engine<T>::allreduce_sum(T* buf, size_t count) {
  if (nranks_ <= 1) return;
  int rc = g_nccl.AllReduce(buf, buf, count, sizeof(T) == 8 ? kNcclFloat64 : kNcclFloat32, kNcclSum, comm_, stream_);
  if (rc != 0) throw EngineError{COSMO_B200_ERR_NCCL, "ncclAllReduce(sum) failed"};
}
template <typename T>
void Engine<T>::allreduce_max(T* buf, size_t count) {
  if (nranks_ <= 1) return;
  int rc = g_nccl.AllReduce(buf, buf, count, sizeof(T) == 8 ? kNcclFloat64 : kNcclFloat32, kNcclMax, comm_, stream_);
  if (rc != 0) throw EngineError{COSMO_B200_ERR_NCCL, "ncclAllReduce(max) failed"};
}

template <typename T>
void Engine<T>::comm_init(int nranks, int rank, const void* id128) {
  if (nranks < 1 || rank < 0 || rank >= nranks) throw EngineError{COSMO_B200_ERR_INVALID, "bad rank / nranks"};
  if (direct_kkt())
    throw EngineError{COSMO_B200_ERR_UNSUPPORTED, "the direct LDL' KKT solver is single-GPU (use CG or reduced MINRES when sharded)"};
  nranks_ = nranks; rank_ = rank;
  if (nranks == 1) return;
  std::vector<int>().swap(P_.h_src);   // update_matrices refuses sharded handles
  std::string e;
  if (!g_nccl.load(e)) throw EngineError{COSMO_B200_ERR_NCCL, e};
  NcclUniqueId id;
  memcpy(&id, id128, sizeof(id));
  CUDA_TRY(cudaSetDevice(device_));
  int rc = g_nccl.CommInitRank(&comm_, nranks, id, rank);
  if (rc != 0) throw EngineError{COSMO_B200_ERR_NCCL, std::string("ncclCommInitRank failed: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "?")};
}

// Peer-memory exchange set-up: every rank exports its exchange buffer + flag array as two CUDA IPC
// handles (64 B each); the host plumbing all-gathers the blobs; attach() maps the peers' buffers.
template <typename T>
void Engine<T>::p2p_export(void* blob128) {
  CUDA_TRY(cudaSetDevice(device_));
  const size_t stride = ((size_t)n_ + 8 + 15) & ~(size_t)15;
  xchg_data_.alloc(2 * (size_t)kMaxRanks * stride);   // [slot][source rank][stride]
  xchg_flags_.alloc(2 * kMaxRanks);
  xchg_seq_.alloc(1);
  xchg_arrive_.alloc(kMaxRanks);
  xv_.stride = stride;
  cudaIpcMemHandle_t hd, hf;
  CUDA_TRY(cudaIpcGetMemHandle(&hd, xchg_data_.p));
  CUDA_TRY(cudaIpcGetMemHandle(&hf, xchg_flags_.p));
  memcpy(blob128, &hd, 64);
  memcpy(static_cast<char*>(blob128) + 64, &hf, 64);
}

template <typename T>
void Engine<T>::p2p_attach(const void* blobs, int nranks) {
  if (nranks != nranks_ || nranks > kMaxRanks) throw EngineError{COSMO_B200_ERR_INVALID, "p2p_attach: rank count mismatch (max 8)"};
  if (!xchg_data_.p) throw EngineError{COSMO_B200_ERR_INVALID, "p2p_attach before p2p_export"};
  CUDA_TRY(cudaSetDevice(device_));
  for (int r = 0; r < nranks; ++r) {
    if (r == rank_) {
      xv_.peer_data[r] = xchg_data_.p;
      xv_.peer_flags[r] = xchg_flags_.p;
      continue;
    }
    cudaIpcMemHandle_t hd, hf;
    memcpy(&hd, static_cast<const char*>(blobs) + (size_t)r * 128, 64);
    memcpy(&hf, static_cast<const char*>(blobs) + (size_t)r * 128 + 64, 64);
    void *pd = nullptr, *pf = nullptr;
    CUDA_TRY(cudaIpcOpenMemHandle(&pd, hd, cudaIpcMemLazyEnablePeerAccess));
    CUDA_TRY(cudaIpcOpenMemHandle(&pf, hf, cudaIpcMemLazyEnablePeerAccess));
    ipc_opened_.push_back(pd);
    ipc_opened_.push_back(pf);
    xv_.peer_data[r] = static_cast<T*>(pd);
    xv_.peer_flags[r] = static_cast<unsigned*>(pf);
  }
  for (int r = nranks; r < kMaxRanks; ++r) { xv_.peer_data[r] = nullptr; xv_.peer_flags[r] = nullptr; }
  xv_.local_flags = xchg_flags_.p;
  xv_.seq = xchg_seq_.p;
  xv_.nranks = nranks;
  xv_.rank = rank_;
  destroy_cg_graphs();
  p2p_ = true;
}

// ---------------------------------------------------------------------------
template <typename T>
template <typename Epi>
void Engine<T>::launch_spmv(const DevCsr<T>& M1, const T* x1, const DevCsr<T>* M2, const T* x2, int nrows,
                            const Epi& epi, RedBuf<T> rb, const char* name, T* pbuf) {
  const CsrView<T> v2 = M2 ? M2->view() : CsrView<T>{nullptr, nullptr, nullptr};
  if (M1.windowed) {
    // a second matrix on the windowed path: the P rows of the reduced KKT operator, summed with P's own lane count
    // into pbuf (M2 must be plain CSR)
    if (M2 == nullptr) {
      launch_win<Epi, 0>(M1, x1, v2, x2, epi, rb, nullptr);
    } else if constexpr (std::is_same<Epi, EpiKktOp<T>>::value) {
      if (M2->windowed || pbuf == nullptr) throw EngineError{COSMO_B200_ERR_INVALID, "windowed SpMV: P rows need plain CSR and a buffer"};
      if (M2->lanes == 32) launch_win<Epi, 32>(M1, x1, v2, x2, epi, rb, pbuf);
      else if (M2->lanes == 8) launch_win<Epi, 8>(M1, x1, v2, x2, epi, rb, pbuf);
      else launch_win<Epi, 2>(M1, x1, v2, x2, epi, rb, pbuf);
    } else {
      throw EngineError{COSMO_B200_ERR_INVALID, "windowed SpMV: a second matrix is only folded into the KKT operator"};
    }
    check_launch(name);
    return;
  }
  const int lanes = M1.lanes;
  const int grid = sgrid(nrows, lanes);
  auto kernel = lanes == 32 ? spmv_kernel<T, 32, Epi> : lanes == 8 ? spmv_kernel<T, 8, Epi> : spmv_kernel<T, 2, Epi>;
  launch_pdl(kernel, grid, kBlock, 0, stream_, M1.view(), x1, v2, x2, nrows, epi, rb);
  check_launch(name);
}

template <typename T>
template <typename Epi, int PL>
void Engine<T>::launch_win(const DevCsr<T>& M1, const T* x1, CsrView<T> v2, const T* x2, const Epi& epi, RedBuf<T> rb,
                           T* pbuf) {
  if constexpr (sizeof(T) == sizeof(double)) {
    if (M1.packed) {
      launch_win_layout<Epi, PL, true>(M1, x1, v2, x2, epi, rb, pbuf);
      return;
    }
  }
  launch_win_layout<Epi, PL, false>(M1, x1, v2, x2, epi, rb, pbuf);
}

template <typename T>
template <typename Epi, int PL, bool PACKED>
void Engine<T>::launch_win_layout(const DevCsr<T>& M1, const T* x1, CsrView<T> v2, const T* x2, const Epi& epi,
                                  RedBuf<T> rb, T* pbuf) {
  const size_t smem = (size_t)M1.W * sizeof(T);
  // function attributes are per device: one flag per (T, PACKED, Epi, PL) instantiation AND device ordinal
  static bool configured[64] = {false};
  const int dev_slot = device_ & 63;
  if (!configured[dev_slot] || device_ >= 64) {
    CUDA_TRY(cudaFuncSetAttribute(spmv_win_kernel<T, PACKED, Epi, PL>, cudaFuncAttributeMaxDynamicSharedMemorySize, 204800));
    configured[dev_slot] = true;
  }
  launch_pdl(spmv_win_kernel<T, PACKED, Epi, PL>, M1.nctas, kWinThreads, smem, stream_, M1.wview(), x1, v2, x2, epi, rb, ypart_.p,
             chunk_ticket_.p, pbuf);
}

template <typename T>
void Engine<T>::soc_norms(const T* ws, T* norm_out) {
  if (!n_soc_) return;
  if (n_soc_chunks_) {
    soc_chunk_kernel<T><<<n_soc_chunks_, kBlock, 0, stream_>>>(ws, soc_chunk_start_.p, soc_chunk_len_.p, soc_chunk_sum_.p);
    check_launch("soc_chunk");
  }
  soc_final_kernel<T><<<(n_soc_ + 127) / 128, 128, 0, stream_>>>(soc_chunk_sum_.p, soc_cone_chunk_ptr_.p, n_soc_, norm_out);
  check_launch("soc_final");
}

// admm_z! (solver.jl:7-21) [+ rhs of admm_x!, solver.jl:50-51]
template <typename T>
void Engine<T>::project_device(const T* w, bool with_rhs, const T* ws_rhs) {
  soc_norms(w + n_, soc_norm_.p);
  psd_.project(w + n_, s_.p, stream_, st_.psd_max_sweeps, launches_);
  if (n_c3_) {
    cone3_project_kernel<T><<<(n_c3_ + 127) / 128, 128, 0, stream_>>>(c3_table(), w + n_, s_.p);
    check_launch("cone3_project");
  }
  if (n_cust_) custom_project(w + n_);
  launch_proj_rhs(w, ws_rhs ? ws_rhs : w + n_, true, with_rhs);
}

// s = Pi_K(w_s) on the rows of every custom cone: one launch of the type's compiled projection kernel per type
template <typename T>
void Engine<T>::custom_project(const T* ws) {
  for (const custom::TypeSlice& t : cust_types_) {
    dim3 grid, block;
    custom::launch_dims(t.entry->key.granularity, t.n, grid, block);
    int n = t.n;
    const int* off = cust_off_.p + t.first;
    const int* dim = cust_dim_.p + t.first;
    const T* par = t.entry->key.n_params ? cust_params_.p + t.param_first : nullptr;
    T* s = s_.p;
    void* args[] = {&n, &off, &dim, &par, &ws, &s};
    CUDA_TRY(cudaLaunchKernel((const void*)t.entry->project, grid, block, args, 0, stream_));
    check_launch("custom_project");
  }
}

// The custom-cone certificates on v into SC_TMP6 (1: some cone is not certified): in_dual(-v) for the primal test
// (which = 0), in_pol_recc(v) for the dual one; a type without the hook certifies none of its cones
template <typename T>
void Engine<T>::custom_certificates(const T* v, T eps, int which) {
  for (const custom::TypeSlice& t : cust_types_) {
    dim3 grid, block;
    custom::launch_dims(t.entry->key.granularity, t.n, grid, block);
    int n = t.n, w = which;
    const int* off = cust_off_.p + t.first;
    const int* dim = cust_dim_.p + t.first;
    const T* par = t.entry->key.n_params ? cust_params_.p + t.param_first : nullptr;
    T* tmp = cust_tmp_.p;
    int* flag = cust_flag_.p + t.first;
    void* args[] = {&n, &off, &dim, &par, &v, &tmp, &eps, &w, &flag};
    CUDA_TRY(cudaLaunchKernel((const void*)t.entry->cert, grid, block, args, 0, stream_));
    check_launch("custom_cert");
  }
  custom_flag_fold_kernel<T><<<1, kBlock, 0, stream_>>>(n_cust_, cust_flag_.p, sc_.p + SC_TMP6);
  check_launch("custom_fold");
}

// c = A' tm + P u + sigma u ; cb[n] = u'c   (second half of reduced_mul!, kktsolver_indirect.jl:61-65)
// Rank 0 alone adds the replicated P / sigma terms of a row-sharded run.
template <typename T>
void Engine<T>::kkt_op_stage2(const int* done, const T* u, const T* t_in, T* c_out, bool exchange) {
  const bool lead = (rank_ == 0);
  const bool px = exchange && p2p_;
  const T sig = lead ? (T)st_.sigma : (T)0;
  const DevCsr<T>* M2 = nullptr;
  const T* pu = nullptr;
  if (At_.windowed) {
    // P u lands in vec_n2_ and enters through the epilogue's `add`: the slab kernel sums the P rows of each chunk
    // (spread over the chunk's window CTAs) before streaming; a column-windowed P keeps its own launch
    if (lead && P_.nnz > 0) {
      pu = vec_n2_.p;
      if (P_.windowed)
        launch_spmv(P_, u, (const DevCsr<T>*)nullptr, (const T*)nullptr, n_, EpiStore<T>{done, vec_n2_.p}, red(SC_TMP0), "spmv_P");
      else
        M2 = &P_;
    }
  } else if (lead) {
    M2 = &P_;
  }
  launch_spmv(At_, t_in, M2, u, n_, EpiKktOp<T>{done, c_out, u, sig, pu}, red_ptr(cb_.p + n_), "spmv_kkt_op", vec_n2_.p);
  if (px) {
    // one-shot allreduce over NVLink: push [c; u'c] into every peer's exchange buffer (coalesced 16-byte remote
    // stores), the consumers (cg_init / cg_update_xr) wait for the flags and sum their local segments in rank order
    if (c_out != cb_.p) throw EngineError{COSMO_B200_ERR_INVALID, "peer exchange expects the operator output in cb_"};
    const int len = n_ + 1;
    const int gx = std::max(1, std::min(16, (len * (int)sizeof(T) + 32767) / 32768));
    p2p_push_kernel<T><<<dim3(gx, nranks_), kBlock, 0, stream_>>>(xv_, cb_.p, len, done, xchg_arrive_.p);
    check_launch("p2p_push");
  }
}

template <typename T>
void Engine<T>::set_maxit(int v) {
  if (cur_maxit_ == v) return;
  h_isc_[ISC_MAXIT] = v;
  CUDA_TRY(cudaMemcpyAsync(isc_.p + ISC_MAXIT, h_isc_.p + ISC_MAXIT, sizeof(int), cudaMemcpyHostToDevice, stream_));
  sync();
  cur_maxit_ = v;
}

// solve!(S::IndirectReducedKKTSolver, y, x) with CG (kktsolver_indirect.jl:36-88).
// Inputs: ls_ = [x1; x2], t0_ = rho .* x2.  Output: xsol_ = y1; then either
//   fused_tail: w_dst = admm_w!(...) computed in the epilogue of the last SpMV, or
//   plain:      nu_ = y2 = rho .* (A y1 - x2).
template <typename T>
void Engine<T>::kkt_core(bool fused_tail, const T* w_src, T* w_dst) {
  const bool lead = (rank_ == 0);
  const bool full = (st_.kkt_solver == COSMO_B200_KKT_MINRES);
  const bool direct = direct_kkt();
  if (st_.kkt_solver != COSMO_B200_KKT_CG && st_.kkt_solver != COSMO_B200_KKT_MINRES_REDUCED && !full && !direct)
    throw EngineError{COSMO_B200_ERR_UNSUPPORTED, "unknown kkt_solver"};
  if (full && nranks_ > 1)
    throw EngineError{COSMO_B200_ERR_UNSUPPORTED, "full-KKT MINRES is single-GPU in this build (use CG or reduced MINRES when sharded)"};
  const bool tm_ready = tm_valid_;
  tm_valid_ = false;
  if (full || direct) {
    if (direct && st_.kkt_solver == COSMO_B200_KKT_LDL) ldl_solve();   // xsol_ = y1, nu_ = y2
    else if (direct) sn_solve();
    else kkt_minres(true);
    if (fused_tail) {
      admm_tail_kernel<T><<<vgrid(m_), kBlock, 0, stream_>>>(m_, nu_.p, rho_vec_.p, s_.p, w_src + n_, w_dst + n_, (T)st_.alpha);
      check_launch("admm_tail");
    }
    return;
  }
  // reduced system: rhs = x1 + A' (rho .* x2)   (kktsolver_indirect.jl:50-54)
  launch_spmv(At_, t0_.p, (const DevCsr<T>*)nullptr, (const T*)nullptr, n_,
              EpiAddVec<T>{nullptr, rhsb_.p, lead ? ls_.p : nullptr}, red(SC_TMP0), "spmv_rhs");
  allreduce_sum(rhsb_.p, n_);
  const bool cg = (st_.kkt_solver == COSMO_B200_KKT_CG);
  if (cg) kkt_cg(isc_.p + ISC_DONE, tm_ready);
  else kkt_minres(false);
  kkt_counter_ += 1;
  if (fused_tail) {
    // the tail also keeps tm = rho .* (A xsol) for the warm start of the next CG solve of the chained loop (the
    // persistent CG kernel computes its own; reduced MINRES uses tm_ as scratch)
    const bool keep_tm = cg && !persistent_cg_ok();
    launch_spmv(A_, xsol_.p, (const DevCsr<T>*)nullptr, (const T*)nullptr, m_,
                EpiAdmmTail<T>{nullptr, ls_.p + n_, rho_vec_.p, s_.p, w_src + n_, w_dst + n_, (T)st_.alpha,
                               keep_tm ? tm_.p : nullptr},
                red(SC_TMP0), "spmv_admm_tail");
    tm_valid_ = keep_tm;
  } else {
    launch_spmv(A_, xsol_.p, (const DevCsr<T>*)nullptr, (const T*)nullptr, m_,
                EpiY2<T>{nullptr, nu_.p, ls_.p + n_, rho_vec_.p}, red(SC_TMP0), "spmv_y2");
  }
}

// cg!(previous_solution, L, y1; abstol = tol_k/|y1|, reltol = 0) (kktsolver_indirect.jl:70)
template <typename T>
void Engine<T>::kkt_cg(const int* done, bool tm_ready) {
  set_maxit(n_);   // IterativeSolvers default maxiter = size(A, 2)
  if (persistent_cg_ok()) {
    launch_persistent_cg(inner_tol());
    return;
  }
  // c = L x0 (warm start => one product for the initial residual); tm = rho .* (A x0) is left by the previous
  // iteration's fused tail when nothing changed since (the product is still counted: the reference computes it)
  if (!tm_ready)
    launch_spmv(A_, xsol_.p, (const DevCsr<T>*)nullptr, (const T*)nullptr, m_, EpiScale<T>{nullptr, tm_.p, rho_vec_.p},
                red(SC_TMP0), "spmv_A_scale");
  kkt_op_stage2(nullptr, xsol_.p, tm_.p, cb_.p, true);
  if (!p2p_) allreduce_sum(cb_.p, n_ + 1);
  launch_pdl(cg_init_kernel<T>, vgrid(n_), kBlock, 0, stream_, n_, (const T*)rhsb_.p, (const T*)cb_.p, r_.p, u_.p, red(SC_RES2),
             CgInitFin<T>{sc_.p, isc_.p, (T)inner_tol(), p2p_ ? xchg_seq_.p : nullptr}, p2p_, xv_);
  check_launch("cg_init");
  // NCCL collectives are capturable too: sharded runs replay the same graphs
  if (!cg_graph_[0]) build_cg_graphs(done);
  total_mults_ += 1 + poll_inner([&](int k) {
    for (int b = 3; b >= 0; --b)
      while (k >= (1 << b)) {
        CUDA_TRY(cudaGraphLaunch(cg_graph_[b], stream_));
        launches_ += (long long)(1 << b) * (At_.windowed && P_.windowed && P_.nnz > 0 && rank_ == 0 ? 5 : 4);
        k -= (1 << b);
      }
  });
}

// The host loop of both iterative KKT solvers: enqueue(k) enqueues k iterations, which stop themselves on the device
// once converged; the first chunk is the previous solve's count, then one iteration at a time until ISC_DONE is set.
// Records the count in last_cg_iters_ and total_inner_ and returns it.
template <typename T>
template <typename Enqueue>
int Engine<T>::poll_inner(const Enqueue& enqueue) {
  int chunk = std::max(last_cg_iters_, 0);
  for (;;) {
    enqueue(chunk);
    CUDA_TRY(cudaMemcpyAsync(h_isc_.p, isc_.p, 2 * sizeof(int), cudaMemcpyDeviceToHost, stream_));
    sync();
    if (h_isc_[ISC_DONE]) break;
    chunk = 1;
  }
  const int iters = h_isc_[ISC_IT];
  last_cg_iters_ = iters;
  total_inner_ += iters;
  return iters;
}

template <typename T>
bool Engine<T>::persistent_cg_ok() {
  if (nranks_ != 1 || A_.windowed || At_.windowed) return false;
  const long long work = A_.nnz + At_.nnz + P_.nnz + 4LL * ((long long)n_ + m_);
  if (work > 6000000LL) return false;           // bigger problems are bandwidth-bound: separate kernels win
  if (persist_grid_ == 0) {
    int coop = 0;
    CUDA_TRY(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, device_));
    if (!coop) { persist_grid_ = -1; return false; }
    const int la = std::max(A_.lanes, At_.lanes);
    persist_lanes_ = la;
    int nb = 0;
    if (la == 32) CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, cg_persistent_kernel<T, 32>, kBlock, 0));
    else if (la == 8) CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, cg_persistent_kernel<T, 8>, kBlock, 0));
    else CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, cg_persistent_kernel<T, 2>, kBlock, 0));
    const long long per = kBlock / la;
    const long long need = std::max<long long>(1, (std::max(n_, m_) + per - 1) / per);
    // a grid barrier costs more the more CTAs take part: at most two CTAs per SM
    persist_grid_ = (int)std::max<long long>(1, std::min<long long>(std::min<long long>((long long)nb, 2) * num_sms_, need));
    if (nb <= 0) { persist_grid_ = -1; return false; }
    persist_part_.alloc((size_t)persist_grid_ * 4);
  }
  return persist_grid_ > 0;
}

template <typename T>
void Engine<T>::launch_persistent_cg(double tol_num) {
  CgPersistArgs<T> a;
  a.A = A_.view(); a.At = At_.view(); a.P = P_.view();
  a.n = n_; a.m = m_;
  a.rhs = rhsb_.p; a.rho = rho_vec_.p; a.x = xsol_.p; a.r = r_.p; a.u = u_.p; a.tm = tm_.p; a.c = cb_.p;
  a.partA = persist_part_.p; a.partB = persist_part_.p + (size_t)persist_grid_ * 2;
  a.sc = sc_.p; a.isc = isc_.p; a.sigma = (T)st_.sigma; a.tol_num = (T)tol_num;
  void* args[] = {&a};
  const void* fn = persist_lanes_ == 32 ? (const void*)cg_persistent_kernel<T, 32>
                 : persist_lanes_ == 8 ? (const void*)cg_persistent_kernel<T, 8> : (const void*)cg_persistent_kernel<T, 2>;
  CUDA_TRY(cudaLaunchCooperativeKernel(fn, dim3(persist_grid_), dim3(kBlock), args, 0, stream_));
  check_launch("cg_persistent");
  ++persist_solves_;
}

// one CG iteration: u = r + beta u ; c = L u ; alpha = res^2/u'c ; x += alpha u ; r -= alpha c
template <typename T>
void Engine<T>::cg_iteration_launches(const int* done) {
  launch_pdl(cg_update_u_kernel<T>, vgrid(n_), kBlock, 0, stream_, n_, (const T*)r_.p, u_.p, (const T*)sc_.p, (const int*)isc_.p);
  check_launch("cg_update_u");
  launch_spmv(A_, u_.p, (const DevCsr<T>*)nullptr, (const T*)nullptr, m_, EpiScale<T>{done, tm_.p, rho_vec_.p}, red(SC_TMP0),
              "spmv_A_scale");
  kkt_op_stage2(done, u_.p, tm_.p, cb_.p, true);
  if (!p2p_) allreduce_sum(cb_.p, n_ + 1);
  launch_pdl(cg_update_xr_kernel<T>, vgrid(n_), kBlock, 0, stream_, n_, (const T*)u_.p, (const T*)cb_.p, (const T*)cb_.p + n_,
             xsol_.p, r_.p, (const T*)sc_.p, (const int*)isc_.p, red(SC_RES2),
             CgStepFin<T>{sc_.p, isc_.p, p2p_ ? xchg_seq_.p : nullptr}, p2p_, xv_);
  check_launch("cg_update_xr");
}

// Stream-capture 1, 2, 4 and 8 CG iterations into executable graphs.  All kernel arguments are
// fixed device pointers (the scalars alpha, beta, tolerance, done flag live on the device), so the
// graphs stay valid for the lifetime of the handle.
template <typename T>
void Engine<T>::build_cg_graphs(const int* done) {
  // make sure one-time function attributes are set outside of the capture
  cg_iteration_launches(done);
  sync();
  const long long saved = launches_;
  for (int b = 0; b < 4; ++b)
    capture_graph(cg_graph_[b], stream_, [&] { for (int i = 0; i < (1 << b); ++i) cg_iteration_launches(done); });
  launches_ = saved;
}

// minres!(previous_solution, L, b; abstol = tol_k/|L x0 - b|, reltol = 0) on the reduced system
// (kktsolver_indirect.jl:72-73) or on the full KKT operator (:123-162).
template <typename T>
void Engine<T>::kkt_minres(bool full) {
  const int npad = (n_ + 3) & ~3;                 // x2 starts 16-byte aligned (TMA bulk copies of v + npad)
  const int L = full ? npad + m_ : n_;
  if (mr_c_.n < (size_t)L) {
    for (auto& b : mr_) b.alloc(L);
    mr_c_.alloc(L);
    if (full) { mr_x_.alloc(L); mr_b_.alloc(L); }
  }
  const int* done = isc_.p + ISC_DONE;
  T* x = full ? mr_x_.p : xsol_.p;
  const T* b = full ? mr_b_.p : rhsb_.p;
  set_maxit(full ? n_ + m_ : n_);
  if (full) {
    CUDA_TRY(cudaMemcpyAsync(mr_b_.p, ls_.p, n_ * sizeof(T), cudaMemcpyDeviceToDevice, stream_));
    CUDA_TRY(cudaMemcpyAsync(mr_b_.p + npad, ls_.p + n_, m_ * sizeof(T), cudaMemcpyDeviceToDevice, stream_));
  }
  // y = L v : reduced (P + sigma I + A' rho A) v  or  full [P + sigma I, A'; A, -1/rho] v
  auto apply = [&](const int* dn, const T* v, T* y) {
    if (full) {
      kkt_op_stage2(dn, v, v + npad, y);                                                        // y1 = A'x2 + P x1 + sigma x1
      launch_spmv(A_, v, (const DevCsr<T>*)nullptr, (const T*)nullptr, m_,
                  EpiKktFullLower<T>{dn, y + npad, v + npad, rho_vec_.p}, red(SC_TMP0), "spmv_kkt_lower");  // y2 = A x1 - x2/rho
    } else {
      launch_spmv(A_, v, (const DevCsr<T>*)nullptr, (const T*)nullptr, m_, EpiScale<T>{dn, tm_.p, rho_vec_.p}, red(SC_TMP0),
                  "spmv_A_scale");
      kkt_op_stage2(dn, v, tm_.p, y);
      allreduce_sum(y, n_);
    }
  };
  T* v_prev = mr_[0].p; T* v_curr = mr_[1].p; T* v_next = mr_[2].p;
  T* w_prev = mr_[3].p; T* w_curr = mr_[4].p; T* w_next = mr_[5].p;
  apply(nullptr, x, mr_c_.p);
  minres_init_kernel<T><<<vgrid(L), kBlock, 0, stream_>>>(L, b, mr_c_.p, v_curr, red(SC_RES2), MinresInitFin<T>{sc_.p, isc_.p, (T)inner_tol()});
  check_launch("minres_init");
  minres_start_kernel<T><<<vgrid(L), kBlock, 0, stream_>>>(L, v_curr, v_prev, w_prev, w_curr, sc_.p);
  check_launch("minres_start");
  int it_host = 0;
  // + init residual + the reference's explicit L*x0 - b (kktsolver_indirect.jl:72,151)
  total_mults_ += 2 + poll_inner([&](int k) {
    for (int i = 0; i < k; ++i) {
      ++it_host;
      apply(done, v_curr, mr_c_.p);
      minres_lanczos1_kernel<T><<<vgrid(L), kBlock, 0, stream_>>>(L, mr_c_.p, v_prev, v_curr, v_next, sc_.p, isc_.p, red(SC_H3));
      check_launch("minres_lanczos1");
      minres_lanczos2_kernel<T><<<vgrid(L), kBlock, 0, stream_>>>(L, v_curr, v_next, sc_.p, isc_.p, red(SC_RES2), MinresStepFin<T>{sc_.p, isc_.p});
      check_launch("minres_lanczos2");
      minres_update_kernel<T><<<vgrid(L), kBlock, 0, stream_>>>(L, it_host, v_curr, v_next, w_prev, w_curr, w_next, x, sc_.p, isc_.p);
      check_launch("minres_update");
      T* t = v_prev; v_prev = v_curr; v_curr = v_next; v_next = t;
      t = w_prev; w_prev = w_curr; w_curr = w_next; w_next = t;
    }
  });
  if (full) {
    CUDA_TRY(cudaMemcpyAsync(xsol_.p, mr_x_.p, n_ * sizeof(T), cudaMemcpyDeviceToDevice, stream_));
    CUDA_TRY(cudaMemcpyAsync(nu_.p, mr_x_.p + npad, m_ * sizeof(T), cudaMemcpyDeviceToDevice, stream_));
    kkt_counter_ += 1;
  }
}

// calculate_residuals! + max_res_component_norm + calculate_cost! (residuals.jl:30-96, 143-147)
template <typename T>
void Engine<T>::compute_residuals(const T* x, const T* s, const T* mu, bool ignore_scaling, double out[5]) {
  const bool unscale = (st_.scaling != 0) && scaled_ && !ignore_scaling;
  launch_spmv(A_, x, (const DevCsr<T>*)nullptr, (const T*)nullptr, m_,
              EpiPrimalRes<T>{nullptr, s, b_.p, unscale ? Einv_.p : nullptr, nullptr}, red(SC_TMP0), "spmv_primal_res");
  allreduce_max(sc_.p + SC_TMP0, 4);
  launch_spmv(At_, mu, (const DevCsr<T>*)nullptr, (const T*)nullptr, n_, EpiStore<T>{nullptr, vec_n_.p}, red(SC_TMP4),
              "spmv_At_mu");
  allreduce_sum(vec_n_.p, n_);
  // slots: [SC_TMP0..3] primal maxes are read first, the dual pass then reuses TMP0.. via a second read
  read_scalars(SC_TMP0, 4);
  const double rp = (double)h_sc_[SC_TMP0], m1 = (double)h_sc_[SC_TMP0 + 1], m2 = (double)h_sc_[SC_TMP0 + 2], m3 = (double)h_sc_[SC_TMP0 + 3];
  // P lanes may differ from A' lanes: P_ has its own
  launch_spmv(P_, x, (const DevCsr<T>*)nullptr, (const T*)nullptr, n_,
              EpiDualRes<T>{nullptr, x, q_.p, vec_n_.p, unscale ? Dinv_.p : nullptr, unscale ? (T)(1.0 / c_) : (T)1},
              red(SC_TMP0), "spmv_dual_res");
  read_scalars(SC_TMP0, 6);
  const double xPx = (double)h_sc_[SC_TMP0], qx = (double)h_sc_[SC_TMP0 + 1];
  const double rd = (double)h_sc_[SC_TMP0 + 2], d1 = (double)h_sc_[SC_TMP0 + 3], d2 = (double)h_sc_[SC_TMP0 + 4], d3 = (double)h_sc_[SC_TMP0 + 5];
  auto nmax = [](double a, double b) { return (a > b || a != a) ? a : b; };
  out[0] = rp;
  out[1] = rd;
  out[2] = nmax(nmax(m1, m2), m3);
  out[3] = nmax(nmax(d1, d2), d3);
  out[4] = (1.0 / c_) * (0.5 * xPx + qx);
}

// adapt_rho_vec! / update_rho_vec! (parameters.jl:53-92)
template <typename T>
bool Engine<T>::adapt_rho(const T* x) {
  double r[5];
  compute_residuals(x, s_.p, mu_.p, true, r);
  double rp = r[0] / (r[2] + 1e-10);
  double rd = r[1] / (r[3] + 1e-10);
  double new_rho = rho_ * sqrt(rp / (rd + 1e-10));
  new_rho = std::min(std::max(new_rho, st_.RHO_MIN), st_.RHO_MAX);
  if (new_rho > st_.adaptive_rho_tolerance * rho_ || new_rho < (1.0 / st_.adaptive_rho_tolerance) * rho_) {
    rho_ = new_rho;
    tm_valid_ = false;
    write_rho_vec();
    rho_updates_.push_back(new_rho);
    return true;
  }
  return false;
}

// is_primal_infeasible! (infeasibility.jl:1-29); dy_ holds delta_y.  inf_rec_ records what the test computed
// (cosmo_b200_infeasibility_test): {verdict, last gate reached (1: norm, 2: A'dy, 4: cone tests), |E dy|_inf,
// |Dinv A'dy|_inf, dy'b (of the normalized -dy / |E dy|_inf), Box support sum, failed families (rows 1, SOC 2, PSD 4,
// Exp/Pow 8), PSD cones whose eigensolver missed psd_max_sweeps}
template <typename T>
bool Engine<T>::primal_infeasible() {
  const T eps = (T)st_.eps_prim_inf;
  double* rec = inf_rec_;
  for (int k = 0; k < 8; ++k) rec[k] = (k == 0 || k >= 6) ? 0.0 : NAN;
  rec[1] = 1;
  scaled_norminf_kernel<T><<<vgrid(m_), kBlock, 0, stream_>>>(m_, scaled_ ? E_.p : nullptr, dy_.p, red(SC_TMP0));
  check_launch("norminf_dy");
  allreduce_max(sc_.p + SC_TMP0, 1);
  read_scalars(SC_TMP0, 1);
  const double norm_dy = (double)h_sc_[SC_TMP0];
  rec[2] = norm_dy;
  if (!(norm_dy > st_.eps_prim_inf)) return false;
  rec[1] = 2;
  launch_spmv(At_, dy_.p, (const DevCsr<T>*)nullptr, (const T*)nullptr, n_, EpiStore<T>{nullptr, vec_n_.p}, red(SC_TMP0), "spmv_At_dy");
  allreduce_sum(vec_n_.p, n_);
  scaled_norminf_kernel<T><<<vgrid(n_), kBlock, 0, stream_>>>(n_, scaled_ ? Dinv_.p : nullptr, vec_n_.p, red(SC_TMP0));
  check_launch("norminf_Atdy");
  read_scalars(SC_TMP0, 1);
  rec[3] = (double)h_sc_[SC_TMP0];
  if (!((double)h_sc_[SC_TMP0] <= st_.eps_prim_inf * norm_dy)) return false;
  rec[1] = 4;
  scal_kernel<T><<<vgrid(m_), kBlock, 0, stream_>>>(m_, (T)(-1.0 / norm_dy), dy_.p);
  check_launch("scal_dy");
  dot_kernel<T><<<vgrid(m_), kBlock, 0, stream_>>>(m_, dy_.p, b_.p, red(SC_TMP0));
  check_launch("dot_dy_b");
  cone_rows_certificate_kernel<T><<<vgrid(m_), kBlock, 0, stream_>>>(m_, 0, dy_.p, row_class_.p, box_l_.p, box_u_.p, eps, red(SC_TMP1));
  check_launch("cone_cert_primal");
  allreduce_sum(sc_.p + SC_TMP0, 2);   // dy'b, box support sum
  const bool cone_bad = cone_certificates(dy_.p, eps, 0) != 0;
  const double dyt_b = (double)h_sc_[SC_TMP0];
  const double box_sum = (double)h_sc_[SC_TMP1];
  rec[4] = dyt_b;
  rec[5] = box_sum;
  const double sF = (cone_bad ? INFINITY : 0.0) + box_sum - dyt_b;
  rec[0] = sF <= st_.eps_prim_inf ? 1.0 : 0.0;
  return sF <= st_.eps_prim_inf;
}

// is_dual_infeasible! (infeasibility.jl:32-68); dx_ holds delta_x.  inf_rec_: {verdict, last gate reached (1: norm,
// 2: q'dx, 3: P dx, 4: cone tests), |D dx|_inf, q'dx, |Dinv P dx|_inf, NaN, failed families, unconverged PSD cones}
template <typename T>
bool Engine<T>::dual_infeasible() {
  const T eps = (T)st_.eps_dual_inf;
  double* rec = inf_rec_;
  for (int k = 0; k < 8; ++k) rec[k] = (k == 0 || k >= 6) ? 0.0 : NAN;
  rec[1] = 1;
  scaled_norminf_kernel<T><<<vgrid(n_), kBlock, 0, stream_>>>(n_, scaled_ ? D_.p : nullptr, dx_.p, red(SC_TMP0));
  check_launch("norminf_dx");
  dot_kernel<T><<<vgrid(n_), kBlock, 0, stream_>>>(n_, q_.p, dx_.p, red(SC_TMP1));
  check_launch("dot_q_dx");
  read_scalars(SC_TMP0, 2);
  const double norm_dx = (double)h_sc_[SC_TMP0];
  rec[2] = norm_dx;
  rec[3] = (double)h_sc_[SC_TMP1];
  if (!(norm_dx > st_.eps_dual_inf)) return false;
  rec[1] = 2;
  if (!((double)h_sc_[SC_TMP1] / (norm_dx * c_) < -st_.eps_dual_inf)) return false;
  rec[1] = 3;
  launch_spmv(P_, dx_.p, (const DevCsr<T>*)nullptr, (const T*)nullptr, n_,
              EpiStoreScaledMax<T>{nullptr, nullptr, scaled_ ? Dinv_.p : nullptr}, red(SC_TMP0), "spmv_P_dx");
  read_scalars(SC_TMP0, 1);
  rec[4] = (double)h_sc_[SC_TMP0];
  if (!((double)h_sc_[SC_TMP0] / (norm_dx * c_) <= st_.eps_dual_inf)) return false;
  rec[1] = 4;
  launch_spmv(A_, dx_.p, (const DevCsr<T>*)nullptr, (const T*)nullptr, m_, EpiStore<T>{nullptr, vec_m_.p}, red(SC_TMP0), "spmv_A_dx");
  if (scaled_) {
    scale_kernel<T><<<vgrid(m_), kBlock, 0, stream_>>>(m_, Einv_.p, vec_m_.p, vec_m_.p);
    check_launch("scale_Adx");
  }
  scal_kernel<T><<<vgrid(m_), kBlock, 0, stream_>>>(m_, (T)(1.0 / norm_dx), vec_m_.p);
  check_launch("scal_Adx");
  cone_rows_certificate_kernel<T><<<vgrid(m_), kBlock, 0, stream_>>>(m_, 1, vec_m_.p, row_class_.p, box_l_.p, box_u_.p, eps, red(SC_TMP1));
  check_launch("cone_cert_dual");
  const bool cone_ok = cone_certificates(vec_m_.p, eps, 1) == 0;
  rec[0] = cone_ok ? 1.0 : 0.0;
  return cone_ok;
}

// The cone tests of both certificates (which = 0: primal, 1: dual) on v, after the row kernel has set the rows flag in
// SC_TMP2: SOC (-v in K*  <=>  |v[2:]| <= tol - v[1]) into SC_TMP3, PSD (-V + tol I positive definite) into SC_TMP4,
// Exp/Pow into SC_TMP5, custom cones into SC_TMP6.  Reads SC_TMP0..5 (and 6) back, records the failed families (rows 1,
// SOC 2, PSD 4, Exp/Pow 8, custom 16) and the PSD cones whose eigensolver missed psd_max_sweeps in inf_rec_[6..7], and
// returns the failed families.
template <typename T>
int Engine<T>::cone_certificates(const T* v, T eps, int which) {
  if (n_soc_) {
    soc_norms(v, soc_norm2_.p);
    soc_cert_kernel<T><<<1, kBlock, 0, stream_>>>(n_soc_, soc_off_.p, soc_norm2_.p, v, eps, sc_.p + SC_TMP3);
    check_launch("soc_cert");
  } else {
    CUDA_TRY(cudaMemsetAsync(sc_.p + SC_TMP3, 0, sizeof(T), stream_));
  }
  if (n_c3_) {
    cone3_cert_kernel<T><<<1, kBlock, 0, stream_>>>(c3_table(), v, eps, sc_.p + SC_TMP5);
    check_launch("cone3_cert");
  } else {
    CUDA_TRY(cudaMemsetAsync(sc_.p + SC_TMP5, 0, sizeof(T), stream_));
  }
  // the custom flag joins the allreduce on every rank of a sharded model, whether or not the rank holds custom cones
  const bool cust_flag = n_cust_ > 0 || nranks_ > 1;
  if (n_cust_) custom_certificates(v, eps, which);
  else if (cust_flag) CUDA_TRY(cudaMemsetAsync(sc_.p + SC_TMP6, 0, sizeof(T), stream_));
  const bool psd_ok = psd_.certificate(v, /*negate=*/true, (double)eps, stream_, st_.psd_max_sweeps, launches_);
  // the PSD verdict is a host bool of THIS rank: put it next to the device flags so that the
  // max-allreduce makes every rank take the same decision
  h_sc_[SC_TMP4] = psd_ok ? T(0) : T(1);
  CUDA_TRY(cudaMemcpyAsync(sc_.p + SC_TMP4, h_sc_.p + SC_TMP4, sizeof(T), cudaMemcpyHostToDevice, stream_));
  allreduce_max(sc_.p + SC_TMP2, 5);   // flags: rows, SOC, PSD, Exp/Pow, custom
  read_scalars(SC_TMP0, cust_flag ? 7 : 6);
  const int failed = (h_sc_[SC_TMP2] != 0 ? 1 : 0) + (h_sc_[SC_TMP3] != 0 ? 2 : 0) + (h_sc_[SC_TMP4] != 0 ? 4 : 0) +
                     (h_sc_[SC_TMP5] != 0 ? 8 : 0) + (cust_flag && h_sc_[SC_TMP6] != 0 ? 16 : 0);
  inf_rec_[6] = failed;
  inf_rec_[7] = psd_.cert_unconverged;
  return failed;
}

// ---------------------------------------------------------------------------
// Accelerator: AndersonAccelerator{T, Type2{QRDecomp} | Type2{NormalEquations} | Type1, ...} (aa.cuh)
// ---------------------------------------------------------------------------
template <typename T>
void Engine<T>::aa_prepare() {   // _make_accelerator!, setup.jl:10-14 (built once per dimension / memory)
  const long long dim = (long long)n_ + m_;
  if (st_.accelerator_mem <= 2) throw EngineError{COSMO_B200_ERR_INVALID, "accelerator: Memory has to be bigger than two."};
  if (st_.accelerator_mem > 32 && dim > 32)
    throw EngineError{COSMO_B200_ERR_UNSUPPORTED, "accelerator_mem > 32 is not supported by the device accelerator"};
  int mem = (int)std::min<long long>(st_.accelerator_mem, std::max<long long>(dim, 1));   // mem = min(mem, dim)
  if (aa_mem_ != mem) {
    aaG_.alloc((size_t)dim * mem, false); aaQ_.alloc((size_t)dim * mem, false);
    aaR_.alloc((size_t)mem * mem); aa_eta_.alloc(32);
    aa_glast_.alloc(dim); aa_f_.alloc(dim); aa_flast_.alloc(dim); aa_sc_.alloc(AA_SC_COUNT);
    if (!h_aa_.p) h_aa_.alloc(AA_SC_COUNT);
    aa_mem_ = mem;
  }
  if (!aa_qr()) {
    if (aa_gsc_.n == 0) {
      aa_gsc_.alloc((size_t)AA_GRAM_MAX_CHUNKS * AA_GRAM_NR);
      aa_gpart_.alloc((size_t)kMaxGrid * AA_GRAM_NR);
      aa_nrm_.alloc(64);
    }
    if (acc_.type == COSMO_B200_AA_TYPE1) {
      if (aa_xlast_.n != (size_t)dim) aa_xlast_.alloc(dim);
      if (aaX_.n != (size_t)dim * mem) aaX_.alloc((size_t)dim * mem, false);
    }
  }
  aa_restart();               // setup.jl:47-49
  aa_active_ = false; aa_success_ = false;
  aa_accelerated_ = aa_declined_ = 0;
  aa_rejected_ = aa_rho_restarts_ = aa_mem_restarts_ = aa_activated_at_ = 0;
}

// CA.update!(aa, g = w, x = w_prev): f = x - g; the first call after a restart only stores (g, f) (and x for Type1);
// otherwise the history columns G_j, F_j (and X_j for Type1, aa.cuh), then for Type2{QRDecomp} the QR update of F by
// modified Gram-Schmidt.  M of the normal-equation variants follows in aa_accelerate.
template <typename T>
void Engine<T>::aa_update(const T* g, const T* x) {
  const int dim = n_ + m_, lo = (rank_ == 0) ? 0 : n_;
  const int grid = vgrid(dim);
  const bool type1 = acc_.type == COSMO_B200_AA_TYPE1;
  const int j = aa_iter_ % aa_mem_;
  // RestartedMemory: the history is full, start again (the QR variant always restarts: set_accelerator refuses rolling)
  if (acc_.memory == COSMO_B200_AA_RESTARTED_MEMORY && j == 0 && aa_iter_ != 0) { aa_iter_ = 0; ++aa_mem_restarts_; }
  T* q = aaQ_.p + (size_t)j * dim;
  aa_hist_kernel<T><<<grid, kBlock, 0, stream_>>>(dim, lo, g, x, aa_f_.p, aa_flast_.p, aa_glast_.p, type1 ? aa_xlast_.p : nullptr,
                                                  aaG_.p + (size_t)j * dim, q, type1 ? aaX_.p + (size_t)j * dim : nullptr,
                                                  aa_init_ ? 1 : 0, red_ptr(aa_sc_.p + AA_F2));
  check_launch("aa_hist");
  allreduce_sum(aa_sc_.p + AA_F2, 1);
  if (aa_init_) { aa_init_ = false; return; }
  if (aa_qr()) {
    T* Rj = aaR_.p + (size_t)j * aa_mem_;        // column j of R
    for (int i = 0; i <= j; ++i) {
      const T* Qp = i > 0 ? aaQ_.p + (size_t)(i - 1) * dim : nullptr;
      const T* Qi = i < j ? aaQ_.p + (size_t)i * dim : nullptr;
      T* out = i < j ? Rj + i : aa_sc_.p + AA_NRM2;
      aa_mgs_kernel<T><<<grid, kBlock, 0, stream_>>>(dim, lo, q, Qp, i > 0 ? Rj + (i - 1) : nullptr, Qi, red_ptr(out));
      check_launch("aa_mgs");
      allreduce_sum(out, 1);
    }
    aa_normalize_kernel<T><<<grid, kBlock, 0, stream_>>>(dim, q, aa_sc_.p + AA_NRM2, Rj + j);
    check_launch("aa_normalize");
  }
  aa_j_ = j;
  ++aa_iter_;
  if (aa_iter_ >= 2 * aa_mem_) aa_iter_ -= aa_mem_;   // RollingMemory: keeps iter mod mem and min(iter, mem)
  aa_fresh_ = true;
}

// CA.accelerate!(g = w, ...): w -= G eta, returns was_successful(aa).  Type2{QRDecomp} solves R eta = Q'f; the
// normal-equation variants refresh row and column j of M in one fused Gram + rhs pass (ceil(l/8) launches, one
// allreduce) and solve with the one-warp LU, which also keeps M current while the window is below min_mem.
template <typename T>
bool Engine<T>::aa_accelerate(T* g) {
  if (!aa_fresh_) return false;
  aa_fresh_ = false;
  const int l = std::min(aa_iter_, aa_mem_);
  const bool solve = l >= std::max(st_.accelerator_min_mem, 1);
  const int dim = n_ + m_, lo = (rank_ == 0) ? 0 : n_;
  const int grid = vgrid(dim);
  if (aa_qr()) {
    if (!solve) return false;
    for (int c0 = 0; c0 < l; c0 += 8) {
      aa_qtf_kernel<T><<<grid, kBlock, 0, stream_>>>(dim, lo, aa_f_.p, aaQ_.p, (size_t)dim, c0, std::min(8, l - c0),
                                                     red_ptr(aa_eta_.p + c0));
      check_launch("aa_qtf");
    }
    allreduce_sum(aa_eta_.p, l);
    aa_solve_kernel<T><<<1, 32, 0, stream_>>>(aaR_.p, aa_mem_, l, aa_eta_.p, aa_sc_.p + AA_FLAG);
    check_launch("aa_solve");
  } else {
    const bool type1 = acc_.type == COSMO_B200_AA_TYPE1;
    const int nch = (l + AA_GRAM_COLS - 1) / AA_GRAM_COLS;
    for (int ch = 0; ch < nch; ++ch) {
      const int c0 = ch * AA_GRAM_COLS, nc = std::min((int)AA_GRAM_COLS, l - c0);
      RedBuf<T> rb{aa_gpart_.p, aa_gsc_.p + (size_t)ch * AA_GRAM_NR, ticket_.p};
      if (type1)
        aa_gram_kernel<T, true><<<grid, kBlock, 0, stream_>>>(dim, lo, aaX_.p, aaQ_.p, (size_t)dim, aa_j_, c0, nc, aa_f_.p, rb);
      else
        aa_gram_kernel<T, false><<<grid, kBlock, 0, stream_>>>(dim, lo, aaQ_.p, aaQ_.p, (size_t)dim, aa_j_, c0, nc, aa_f_.p, rb);
      check_launch("aa_gram");
    }
    allreduce_sum(aa_gsc_.p, (size_t)nch * AA_GRAM_NR);
    aa_ne_solve_kernel<T><<<1, 32, 0, stream_>>>(aa_gsc_.p, aaR_.p, aa_nrm_.p, aa_nrm_.p + aa_mem_, aa_mem_, aa_j_, l, type1 ? 1 : 0,
                                                 acc_.regularizer, (T)acc_.lambda, solve ? 1 : 0, aa_eta_.p, aa_sc_.p + AA_FLAG);
    check_launch("aa_ne_solve");
    if (!solve) return false;
  }
  aa_apply_kernel<T><<<grid, kBlock, 0, stream_>>>(dim, g, aaG_.p, (size_t)dim, l, aa_eta_.p, aa_sc_.p + AA_FLAG);
  check_launch("aa_apply");
  CUDA_TRY(cudaMemcpyAsync(h_aa_.p + AA_FLAG, aa_sc_.p + AA_FLAG, sizeof(T), cudaMemcpyDeviceToHost, stream_));
  sync();
  if (h_aa_[AA_FLAG] == T(0)) { ++aa_rejected_; return false; }
  return true;
}

template <typename T>
void Engine<T>::set_accelerator(const cosmo_b200_accelerator* a) {
  if (!a) {
    acc_ = cosmo_b200_accelerator{COSMO_B200_AA_TYPE2_QR, COSMO_B200_AA_RESTARTED_MEMORY, COSMO_B200_AA_NO_REGULARIZER,
                                  COSMO_B200_AA_IMMEDIATE, 0.0, 2, 0.0};
    return;
  }
  if (a->type < COSMO_B200_AA_TYPE2_QR || a->type > COSMO_B200_AA_TYPE1 || a->memory < 0 || a->memory > 1 ||
      a->regularizer < 0 || a->regularizer > 2 || a->activation < 0 || a->activation > 2)
    throw EngineError{COSMO_B200_ERR_INVALID, "accelerator: unknown type, memory, regularizer or activation"};
  if (!(a->lambda >= 0.0)) throw EngineError{COSMO_B200_ERR_INVALID, "accelerator: lambda must be a non-negative number"};
  if (a->type == COSMO_B200_AA_TYPE2_QR && a->memory == COSMO_B200_AA_ROLLING_MEMORY)
    throw EngineError{COSMO_B200_ERR_UNSUPPORTED, "accelerator: Type2{QRDecomp} with RollingMemory is not supported"};
  if (a->type == COSMO_B200_AA_TYPE2_QR && a->regularizer != COSMO_B200_AA_NO_REGULARIZER)
    throw EngineError{COSMO_B200_ERR_UNSUPPORTED, "accelerator: Type2{QRDecomp} takes no regularizer"};
  acc_ = *a;
}

template <typename T>
void Engine<T>::accelerator_stats(int64_t* out) {
  out[0] = aa_accelerated_; out[1] = aa_declined_; out[2] = aa_rejected_;
  out[3] = aa_rho_restarts_; out[4] = aa_mem_restarts_; out[5] = aa_activated_at_;
}

// ---------------------------------------------------------------------------
// The hot loop: COSMO.optimize!, src/solver.jl:125-167 (SURVEY.md Appendix A)
// ---------------------------------------------------------------------------
template <typename T>
void Engine<T>::solve(cosmo_b200_result* out) {
  const double t_start = now_s();
  const unsigned dev_out = out ? caller_arrays({out->x, out->s, out->mu}) : 0u;
  const int n = n_, m = m_;
  const long long launches0 = launches_;
  total_inner_ = 0; total_mults_ = 0;
  persist_solves_ = 0;
  tm_valid_ = false;
  CUDA_TRY(cudaMemsetAsync(isc_.p + ISC_TOTAL, 0, sizeof(int), stream_));
  int status = COSMO_B200_UNDETERMINED;
  double cost = INFINITY;
  double info[5] = {INFINITY, INFINITY, 0.0, 0.0, INFINITY};
  long long iter = 0;
  bool rho_update_due = false, infeasibility_check_due = false;
  double res_time = 0.0;

  // warm starting the operator variable (solver.jl:128-129): w_x = x, w_s = mu ./ rho + s
  cur_ = 0; prev_ = 1;
  CUDA_TRY(cudaMemcpyAsync(W_[cur_].p, xs_.p, n * sizeof(T), cudaMemcpyDeviceToDevice, stream_));
  ws_from_mu_kernel<T><<<vgrid(m), kBlock, 0, stream_>>>(m, rho_vec_.p, mu_.p, s_.p, W_[cur_].p + n);
  check_launch("ws_from_mu");
  // phase timers: on request (verbose & 2 = settings.verbose_timing) and for every problem that is not latency-bound
  {
    const bool timers = (st_.verbose & 2) != 0 || (long long)n + m >= 20000 || !psd_.large_h.empty();
    t_proj_.enable(timers);
    t_kkt_.enable(timers);
  }
  CUDA_TRY(cudaEventRecord(ev0_, stream_));
  const double iter_start = now_s();
  // setup time as the reference counts it (ws.times.setup_time): the host's figure when it reports one (it then includes
  // the creation of this engine), else the engine's own creation time
  const double setup_time_total = st_.setup_time > 0.0 ? st_.setup_time : create_time_;

  // x-step + w-step reading W[src], writing W[dst]
  auto xw_step = [&](int src, int dst, bool do_proj, const T* ws_override) {
    const T* w = W_[src].p;
    const T* ws_rhs = ws_override ? ws_override : w + n;
    if (do_proj) {
      t_proj_.begin(stream_);
      project_device(w, true, ws_rhs);      // admm_z! fused with the right-hand side of admm_x! (one pass over w)
      t_proj_.end(stream_);
    } else {
      launch_proj_rhs(w, ws_rhs, false, true);
    }
    // the tail reads w_s from ws_rhs's buffer and writes W[dst] (elementwise, may alias)
    T* wd = W_[dst].p;
    t_kkt_.begin(stream_);
    kkt_core(true, ws_override ? (ws_override - n) : w, wd);
    t_kkt_.end(stream_);
    wx_update_kernel<T><<<vgrid(n), kBlock, 0, stream_>>>(n, w, xsol_.p, (T)st_.alpha, wd);
    check_launch("wx_update");
  };

  // one initialisation step (solver.jl:137-138)
  xw_step(cur_, 1 - cur_, false, nullptr);
  cur_ = 1 - cur_; prev_ = 1 - cur_;

  const bool use_aa = (st_.accelerator == COSMO_B200_ACC_ANDERSON);
  long long safeguarding_iter = 0;
  if (use_aa) aa_prepare();
  // update_suggested (solver.jl:284-292): with an Anderson accelerator, rho updates and the infeasibility
  // snapshot wait for the next iteration whose candidate was not accelerated
  auto suggested = [&](bool due) { return due && !(use_aa && aa_success_); };

  while (iter + safeguarding_iter < st_.max_iter) {
    ++iter;
    // acceleration_pre! (accelerator_interface.jl:58-75), ImmediateActivation / IterActivation (:24-33)
    if (use_aa) {
      if (!aa_active_ && ((acc_.activation == COSMO_B200_AA_IMMEDIATE && iter >= 2) ||
                          (acc_.activation == COSMO_B200_AA_ITER && iter >= acc_.start_iter))) {
        aa_active_ = true;
        aa_activated_at_ = iter;
      }
      if (aa_active_) {
        aa_update(W_[cur_].p, W_[prev_].p);
        aa_success_ = aa_accelerate(W_[cur_].p);   // overwrites w with the candidate
        if (aa_success_) ++aa_accelerated_;
      }
    }
    if (suggested(infeasibility_check_due)) {  // solver.jl:145-148
      recover_mu(W_[prev_].p);
      CUDA_TRY(cudaMemcpyAsync(dy_.p, mu_.p, m * sizeof(T), cudaMemcpyDeviceToDevice, stream_));
    }
    // w_prev = w (solver.jl:151): the current buffer becomes w_prev, the other one receives w_{k+1}
    const int src = cur_, dst = 1 - cur_;
    // rho adaptation rules (solver.jl:242-282)
    // automatic interval (solver.jl:244-256): once the loop has run for adaptive_rho_fraction * setup_time, fix the
    // interval at the current iteration count rounded to a multiple of check_termination (at least one multiple)
    if (st_.adaptive_rho && st_.adaptive_rho_interval == 0 && auto_rho_interval_ == 0 &&
        (now_s() - iter_start) > st_.adaptive_rho_fraction * setup_time_total) {
      const long long N = st_.check_termination > 0 ? st_.check_termination : 25;
      const double xr = (double)iter + 0.5 * (double)N;            // round_multiple, algebra.jl:245-247
      const long long rm = (long long)floor(xr - fmod(xr, (double)N));
      auto_rho_interval_ = (int)std::max<long long>(rm, N);
    }
    const int rho_interval = st_.adaptive_rho_interval > 0 ? st_.adaptive_rho_interval : auto_rho_interval_;
    if (st_.adaptive_rho && rho_interval > 0 && (iter % rho_interval) == 0 &&
        (long long)(rho_updates_.size() - 1) < st_.adaptive_rho_max_adaptions)
      rho_update_due = true;
    if (suggested(rho_update_due)) {
      rho_update_due = false;
      t_proj_.begin(stream_);
      project_device(W_[src].p, false, nullptr);          // admm_z!
      t_proj_.end(stream_);
      recover_mu(W_[src].p);                               // w_prev == w here
      const double t0 = now_s();
      const bool adapted = adapt_rho(W_[src].p);
      res_time += now_s() - t0;
      if (adapted) {
        if (use_aa) { aa_restart(); ++aa_rho_restarts_; }   // the operator changed: CA.restart! (solver.jl:272-275)
        // w[n+1:end] = mu ./ rho + s (solver.jl:278), kept apart from w_prev
        ws_from_mu_kernel<T><<<vgrid(m), kBlock, 0, stream_>>>(m, rho_vec_.p, mu_.p, s_.p, W_[dst].p + n);
        check_launch("ws_from_mu");
        xw_step(src, dst, false, W_[dst].p + n);
      } else {
        xw_step(src, dst, false, nullptr);
      }
    } else {
      xw_step(src, dst, true, nullptr);
    }
    prev_ = src; cur_ = dst;
    // acceleration_post! (accelerator_interface.jl:85-114): safeguard the accelerated candidate
    if (use_aa && aa_active_ && aa_success_ && st_.safeguard) {
      const int dim = n + m, lo = (rank_ == 0) ? 0 : n;
      aa_res_kernel<T><<<vgrid(dim), kBlock, 0, stream_>>>(dim, lo, W_[prev_].p, W_[cur_].p, aa_f_.p, red_ptr(aa_sc_.p + AA_FACC2));
      check_launch("aa_res");
      allreduce_sum(aa_sc_.p + AA_FACC2, 1);
      CUDA_TRY(cudaMemcpyAsync(h_aa_.p, aa_sc_.p, 2 * sizeof(T), cudaMemcpyDeviceToHost, stream_));
      sync();
      const double nrm_f = sqrt((double)h_aa_[AA_F2]), nrm_f_acc = sqrt((double)h_aa_[AA_FACC2]);
      if (nrm_f_acc > nrm_f * st_.safeguard_tol) {
        // decline: w_prev = w = g_last, then one plain ADMM step from there (:100-106)
        CUDA_TRY(cudaMemcpyAsync(W_[prev_].p, aa_glast_.p, (size_t)dim * sizeof(T), cudaMemcpyDeviceToDevice, stream_));
        xw_step(prev_, cur_, true, nullptr);
        ++safeguarding_iter;
        ++aa_declined_;
      }
    }

    // check_termination! (solver.jl:303-356)
    if ((st_.check_termination > 0 && iter % st_.check_termination == 0) || iter == 1) {
      const double t0 = now_s();
      recover_mu(W_[prev_].p);
      compute_residuals(W_[prev_].p, s_.p, mu_.p, false, info);
      res_time += now_s() - t0;
      cost = info[4];
      if (fabs(cost) > 1e20) { status = COSMO_B200_UNSOLVED; break; }
      // AccuracyActivation (accelerator_interface.jl:38-46), checked first thing in has_converged (residuals.jl:129)
      if (use_aa && !aa_active_ && acc_.activation == COSMO_B200_AA_ACCURACY) {
        const double tol = acc_.start_accuracy;
        if (info[0] < tol + tol * info[2] && info[1] < tol + tol * info[3]) {
          aa_active_ = true;
          aa_activated_at_ = iter;
        }
      }
      if (st_.verbose & 1) printf("%lld\t%.4e\t%.4e\t%.4e\t%.4e\n", iter, cost, info[0], info[1], rho_);
      // has_converged (residuals.jl:127-140): a known optimal value, when given, must be met as well
      const bool obj_ok = (st_.obj_true != st_.obj_true) || fabs(st_.obj_true - cost) <= st_.obj_true_tol;
      if (info[0] < st_.eps_abs + st_.eps_rel * info[2] && info[1] < st_.eps_abs + st_.eps_rel * info[3] && obj_ok) {
        status = COSMO_B200_SOLVED;
        break;
      }
    }
    if (st_.check_infeasibility > 0 && iter % st_.check_infeasibility == 0) {
      infeasibility_check_due = true;
    } else if (suggested(infeasibility_check_due)) {
      infeasibility_check_due = false;
      recover_mu(W_[prev_].p);
      sub_kernel<T><<<vgrid(m), kBlock, 0, stream_>>>(m, dy_.p, mu_.p, dy_.p);          // dy -= mu
      check_launch("sub_dy");
      sub_kernel<T><<<vgrid(n), kBlock, 0, stream_>>>(n, W_[cur_].p, W_[prev_].p, dx_.p);  // dx = w_x - w_prev_x
      check_launch("sub_dx");
      if (primal_infeasible()) { status = COSMO_B200_PRIMAL_INFEASIBLE; cost = INFINITY; break; }
      if (dual_infeasible()) { status = COSMO_B200_DUAL_INFEASIBLE; cost = -INFINITY; break; }
    }
    // the reference's clock starts before setup! (time_limit_start, solver.jl:119,349)
    if (st_.time_limit != 0 && (now_s() - iter_start) + setup_time_total > st_.time_limit) {
      recover_mu(W_[prev_].p);
      compute_residuals(W_[prev_].p, s_.p, mu_.p, false, info);
      status = COSMO_B200_TIME_LIMIT_REACHED;
      break;
    }
  }
  recover_mu(W_[prev_].p);  // solver.jl:167
  CUDA_TRY(cudaEventRecord(ev1_, stream_));
  sync();
  const double iter_time = now_s() - iter_start;
  float dev_ms = 0.f;
  CUDA_TRY(cudaEventElapsedTime(&dev_ms, ev0_, ev1_));
  if (iter + safeguarding_iter == st_.max_iter && status == COSMO_B200_UNDETERMINED) {  // solver.jl:173-176
    compute_residuals(W_[prev_].p, s_.p, mu_.p, false, info);
    status = COSMO_B200_MAX_ITER_REACHED;
  }
  if (persist_solves_ > 0) {   // inner-iteration statistics of the persistent CG kernel live on the device
    CUDA_TRY(cudaMemcpyAsync(h_isc_.p + ISC_TOTAL, isc_.p + ISC_TOTAL, sizeof(int), cudaMemcpyDeviceToHost, stream_));
    sync();
    total_inner_ += h_isc_[ISC_TOTAL];
    total_mults_ += h_isc_[ISC_TOTAL] + persist_solves_;
  }
  // x = view(w_prev, 1:n): keep it for the next warm start and hand it out
  CUDA_TRY(cudaMemcpyAsync(xs_.p, W_[prev_].p, n * sizeof(T), cudaMemcpyDeviceToDevice, stream_));
  have_solution_ = true;
  if (out) {
    if (out->x) download_vec(out->x, W_[prev_].p, n);
    if (out->s) download_vec(out->s, s_.p, m);
    if (out->mu) download_vec(out->mu, mu_.p, m);
    if (dev_out) caller_written();
    sync();
    out->obj_val = cost;
    out->iter = iter + safeguarding_iter;      // total_iter, solver.jl:195
    out->safeguarding_iter = safeguarding_iter;
    out->status = status;
    out->r_prim = info[0]; out->r_dual = info[1]; out->max_norm_prim = info[2]; out->max_norm_dual = info[3];
    out->rho = rho_;
    out->n_rho_updates = (int64_t)rho_updates_.size();
    if (out->rho_updates)
      for (int64_t i = 0; i < std::min<int64_t>(out->rho_updates_cap, out->n_rho_updates); ++i) out->rho_updates[i] = rho_updates_[i];
    out->setup_time = create_time_;   // the device part of setup!; the host adds its own
    out->iter_time = iter_time;
    out->iter_time_device = dev_ms * 1e-3;
    t_proj_.harvest();
    t_kkt_.harvest();
    out->proj_time = t_proj_.total_ms * 1e-3;   // device time of admm_z! (+ the fused rhs pass); 0 when the timers are off
    out->kkt_time = t_kkt_.total_ms * 1e-3;     // device time of the KKT solves incl. the fused ADMM tail
    out->res_time = res_time;
    out->kkt_inner_iterations = total_inner_;
    out->kkt_multiplications = total_mults_;
    out->kernel_launches = launches_ - launches0;
    out->solver_time = now_s() - t_start;
  }
  sync();
}

// ---- plugin-granularity entry points ---------------------------------------------
template <typename T>
void Engine<T>::project(const void* ws, void* s_out) {
  CUDA_TRY(cudaSetDevice(device_));
  // stage w_s in the s-part of a scratch operator variable of its own and put the slack iterate back afterwards: a
  // caller that projects between two solves must not disturb w_prev or s of the finished one
  if (proj_w_.n < (size_t)n_ + m_) { proj_w_.alloc((size_t)n_ + m_); proj_s_.alloc(std::max(m_, 1), false); }
  upload_vec(vec_m_, ws, m_);
  CUDA_TRY(cudaMemcpyAsync(proj_s_.p, s_.p, m_ * sizeof(T), cudaMemcpyDeviceToDevice, stream_));
  CUDA_TRY(cudaMemcpyAsync(proj_w_.p + n_, vec_m_.p, m_ * sizeof(T), cudaMemcpyDeviceToDevice, stream_));
  project_device(proj_w_.p, false, nullptr);
  download_vec(s_out, s_.p, m_);
  CUDA_TRY(cudaMemcpyAsync(s_.p, proj_s_.p, m_ * sizeof(T), cudaMemcpyDeviceToDevice, stream_));
  sync();
}

template <typename T>
void Engine<T>::kkt_solve(const void* rhs, void* sol, int64_t* inner) {
  CUDA_TRY(cudaSetDevice(device_));
  tm_valid_ = false;
  upload_vec(ls_, rhs, (size_t)n_ + m_);
  scale_kernel<T><<<vgrid(m_), kBlock, 0, stream_>>>(m_, rho_vec_.p, ls_.p + n_, t0_.p);
  check_launch("scale_x2");
  kkt_core(false, nullptr, nullptr);
  download_vec(sol, xsol_.p, n_);
  download_vec(static_cast<T*>(sol) + n_, nu_.p, m_);
  sync();
  if (inner && direct_kkt()) {
    *inner = 0;
  } else if (inner) {
    CUDA_TRY(cudaMemcpyAsync(h_isc_.p, isc_.p, 2 * sizeof(int), cudaMemcpyDeviceToHost, stream_));
    sync();
    *inner = h_isc_[ISC_IT];
  }
}

// ---- direct LDL' plugin (ldl.cuh) -----------------------------------------------------------------------------
// Symbolic analysis of the resident pattern (host), upload of L's structure and the schedules, device buffers.
template <typename T>
void Engine<T>::ldl_setup() {
  CUDA_TRY(cudaSetDevice(device_));
  const double t0 = now_s();
  std::vector<int> Prow(n_ + 1), Pcol(P_.nnz), Arow(n_ + 1), Acol(At_.nnz);
  CUDA_TRY(cudaMemcpyAsync(Prow.data(), P_.rowptr.p, (n_ + 1) * sizeof(int), cudaMemcpyDeviceToHost, stream_));
  CUDA_TRY(cudaMemcpyAsync(Arow.data(), At_.rowptr.p, (n_ + 1) * sizeof(int), cudaMemcpyDeviceToHost, stream_));
  if (P_.nnz) CUDA_TRY(cudaMemcpyAsync(Pcol.data(), P_.col.p, P_.nnz * sizeof(int), cudaMemcpyDeviceToHost, stream_));
  if (At_.nnz) CUDA_TRY(cudaMemcpyAsync(Acol.data(), At_.col.p, At_.nnz * sizeof(int), cudaMemcpyDeviceToHost, stream_));
  sync();
  ldl::Symbolic S;
  ldl::analyze(n_, m_, Prow, Pcol, Arow, Acol, S);
  ldl_symbolic_s_ = now_s() - t0;
  const int N = S.N;
  ldl_N_ = N;
  ldl_nnzK_ = S.nnz_triu_K();
  ldl_nnzL_ = S.nnz_L();
  // one dense workspace of length N per resident factor CTA: as many CTAs as the widest level, at most two per SM
  int maxw = 1;
  for (const ldl::Segment& s : S.fseg)
    if (!s.run) maxw = std::max(maxw, S.fptr[s.l1] - S.fptr[s.l0]);
  ldl_ws_ctas_ = std::max(1, std::min(maxw, 2 * num_sms_));
  const double ts = (double)sizeof(T);
  const double need = (double)ldl_nnzL_ * (2 * ts + 4 + 4 + 8) + (double)ldl_nnzK_ * (ts + 4 + 8) + (double)S.Ksrc.size() * 8 +
                      (double)(N + 1) * 8 * 3 + (double)N * (ts * 3 + 4 * 5) + (double)ldl_ws_ctas_ * N * ts;
  size_t free_b = 0, total_b = 0;
  CUDA_TRY(cudaMemGetInfo(&free_b, &total_b));
  if (need > 0.9 * (double)free_b) {
    char b[256];
    snprintf(b, sizeof(b), "the direct LDL' factor does not fit in device memory: nnz(L) = %lld needs %.2f GB, %.2f GB free",
             ldl_nnzL_, need * 1e-9, (double)free_b * 1e-9);
    throw EngineError{COSMO_B200_ERR_ALLOC, b};
  }
  ldl_Kp_.upload(S.Kp, stream_); ldl_Ki_.upload(S.Ki, stream_); ldl_Ksp_.upload(S.Ksp, stream_); ldl_Ksrc_.upload(S.Ksrc, stream_);
  ldl_Lp_.upload(S.Lp, stream_); ldl_Li_.upload(S.Li, stream_);
  ldl_Rp_.upload(S.Rp, stream_); ldl_Rj_.upload(S.Rj, stream_); ldl_Rmap_.upload(S.Rmap, stream_);
  ldl_fcols_.upload(S.fcols, stream_); ldl_fptr_.upload(S.fptr, stream_);
  ldl_bcols_.upload(S.bcols, stream_); ldl_bptr_.upload(S.bptr, stream_);
  ldl_perm_.upload(S.perm, stream_);
  ldl_Kx_.alloc(std::max<long long>(ldl_nnzK_, 1), false);
  ldl_Lx_.alloc(std::max<long long>(ldl_nnzL_, 1), false);
  ldl_Rx_.alloc(std::max<long long>(ldl_nnzL_, 1), false);
  ldl_D_.alloc(std::max(N, 1)); ldl_Dinv_.alloc(std::max(N, 1)); ldl_y_.alloc(std::max(N, 1));
  ldl_ws_.alloc((size_t)ldl_ws_ctas_ * std::max(N, 1));   // zeroed: every column clears what it touched
  ldl_flags_.alloc(2);
  sync();
  ldl_fseg_ = S.fseg; ldl_bseg_ = S.bseg;
  ldl_fptr_h_ = S.fptr; ldl_bptr_h_ = S.bptr;
  ldl_ev_[0].create();
  ldl_ev_[1].create();
  destroy_ldl_factor_graph();
  ldl_solve_graph_.reset();
  ldl_ready_ = true;
  ldl_dirty_ = true;
}

// Assemble K from the resident (scaled) P_, At_, rho_vec_ and sigma and factor it: one captured graph, replayed on
// every refactorisation.  Reads back the pivot counts (the only host synchronisation of the plugin).
template <typename T>
void Engine<T>::ldl_factor() {
  if (!ldl_ready_) ldl_setup();
  if (!ldl_factor_graph_) {
    int nodes = 0;
    capture_graph(ldl_factor_graph_, stream_, [&] {
      ldl_reset_flags_kernel<<<1, 32, 0, stream_>>>(ldl_flags_.p); ++nodes;
      ldl_assemble_kernel<T><<<vgrid(ldl_nnzK_), kBlock, 0, stream_>>>(ldl_nnzK_, ldl_Ksp_.p, ldl_Ksrc_.p, P_.val.p, At_.val.p,
                                                                       rho_vec_.p, (T)st_.sigma, ldl_Kx_.p);
      ++nodes;
      LdlFactorArgs<T> a;
      a.cols = ldl_fcols_.p; a.lptr = ldl_fptr_.p;
      a.Kp = ldl_Kp_.p; a.Ki = ldl_Ki_.p; a.Kx = ldl_Kx_.p;
      a.Lp = ldl_Lp_.p; a.Li = ldl_Li_.p; a.Lx = ldl_Lx_.p;
      a.Rp = ldl_Rp_.p; a.Rj = ldl_Rj_.p; a.Rmap = ldl_Rmap_.p;
      a.D = ldl_D_.p; a.Dinv = ldl_Dinv_.p; a.ws = ldl_ws_.p; a.N = ldl_N_; a.flags = ldl_flags_.p;
      for (const ldl::Segment& s : ldl_fseg_) {
        a.l0 = s.l0; a.l1 = s.l1;
        const int grid = s.run ? 1 : std::min(ldl_fptr_h_[s.l1] - ldl_fptr_h_[s.l0], ldl_ws_ctas_);
        ldl_factor_kernel<T><<<grid, kBlock, 0, stream_>>>(a);
        ++nodes;
      }
      if (ldl_nnzL_) {
        ldl_csr_gather_kernel<T><<<vgrid(ldl_nnzL_), kBlock, 0, stream_>>>(ldl_nnzL_, ldl_Rmap_.p, ldl_Lx_.p, ldl_Rx_.p);
        ++nodes;
      }
    });
    ldl_factor_nodes_ = nodes;
  }
  int flags[2] = {0, 0};
  CUDA_TRY(cudaEventRecord(ldl_ev_[0], stream_));
  CUDA_TRY(cudaGraphLaunch(ldl_factor_graph_, stream_));
  CUDA_TRY(cudaEventRecord(ldl_ev_[1], stream_));
  CUDA_TRY(cudaMemcpyAsync(flags, ldl_flags_.p, sizeof(flags), cudaMemcpyDeviceToHost, stream_));
  sync();
  launches_ += ldl_factor_nodes_;
  float ms = 0.f;
  CUDA_TRY(cudaEventElapsedTime(&ms, ldl_ev_[0], ldl_ev_[1]));
  ldl_factor_s_ = ms * 1e-3;
  ++ldl_factorizations_;
  if (flags[1] != 0) {
    char b[160];
    snprintf(b, sizeof(b), "LDL' factorisation of the KKT matrix met %d zero or non-finite pivots", flags[1]);
    throw EngineError{COSMO_B200_ERR_NUMERICAL, b};
  }
  // positive_inertia(ldlfact) == n (kktsolver.jl:300-303)
  if (flags[0] != n_) throw EngineError{COSMO_B200_ERR_INVALID, "Objective function is not convex."};
  ldl_dirty_ = false;
}

// [y1; y2] = K \ [x1; x2] with ls_ = [x1; x2], xsol_ = y1, nu_ = y2: forward and backward levels replayed as one graph
template <typename T>
void Engine<T>::ldl_solve() {
  if (nranks_ > 1) throw EngineError{COSMO_B200_ERR_UNSUPPORTED, "the direct LDL' KKT solver is single-GPU"};
  if (!ldl_ready_) ldl_setup();
  if (ldl_dirty_) ldl_factor();
  if (!ldl_solve_graph_) {
    int nodes = 0;
    capture_graph(ldl_solve_graph_, stream_, [&] {
      LdlSolveArgs<T> a;
      a.Dinv = ldl_Dinv_.p; a.perm = ldl_perm_.p; a.rhs = ls_.p; a.y = ldl_y_.p; a.out1 = xsol_.p; a.out2 = nu_.p; a.n = n_;
      auto grid = [&](const std::vector<int>& ptr, const ldl::Segment& s) {
        return s.run ? 1 : (int)std::min<long long>(((long long)ptr[s.l1] - ptr[s.l0] + kWarpsPerBlock - 1) / kWarpsPerBlock, kMaxGrid);
      };
      a.cols = ldl_fcols_.p; a.lptr = ldl_fptr_.p; a.ptr = ldl_Rp_.p; a.idx = ldl_Rj_.p; a.val = ldl_Rx_.p;
      for (const ldl::Segment& s : ldl_fseg_) {
        a.l0 = s.l0; a.l1 = s.l1;
        ldl_forward_kernel<T><<<grid(ldl_fptr_h_, s), kBlock, 0, stream_>>>(a);
        ++nodes;
      }
      a.cols = ldl_bcols_.p; a.lptr = ldl_bptr_.p; a.ptr = ldl_Lp_.p; a.idx = ldl_Li_.p; a.val = ldl_Lx_.p;
      for (const ldl::Segment& s : ldl_bseg_) {
        a.l0 = s.l0; a.l1 = s.l1;
        ldl_backward_kernel<T><<<grid(ldl_bptr_h_, s), kBlock, 0, stream_>>>(a);
        ++nodes;
      }
    });
    ldl_solve_nodes_ = nodes;
  }
  CUDA_TRY(cudaGraphLaunch(ldl_solve_graph_, stream_));
  launches_ += ldl_solve_nodes_;
}

template <typename T>
void Engine<T>::ldl_stats(double* o) {
  if (st_.kkt_solver == COSMO_B200_KKT_LDL_SUPERNODAL) {   // stored entries (explicit zeros included), supernodal levels
    o[0] = sn_.N; o[1] = (double)sn_.nnz_K; o[2] = (double)sn_.stored; o[3] = sn_.levels;
    o[4] = sn_solve_nodes_; o[5] = (double)sn_factorizations_; o[6] = sn_factor_s_; o[7] = sn_symbolic_s_;
    return;
  }
  o[0] = ldl_N_; o[1] = (double)ldl_nnzK_; o[2] = (double)ldl_nnzL_; o[3] = ldl_fptr_h_.empty() ? 0 : (double)ldl_fptr_h_.size() - 1;
  o[4] = ldl_solve_nodes_; o[5] = (double)ldl_factorizations_; o[6] = ldl_factor_s_; o[7] = ldl_symbolic_s_;
}

// ---- supernodal LDL' plugin (ldl_sn.cuh) ------------------------------------------------------------------------
// Symbolic analysis of the resident pattern (host), upload of the panels' structure and the schedules, the choice of
// path per supernode, device buffers.
template <typename T>
void Engine<T>::sn_setup() {
  CUDA_TRY(cudaSetDevice(device_));
  const double t0 = now_s();
  std::vector<int> Prow(n_ + 1), Pcol(P_.nnz), Arow(n_ + 1), Acol(At_.nnz);
  CUDA_TRY(cudaMemcpyAsync(Prow.data(), P_.rowptr.p, (n_ + 1) * sizeof(int), cudaMemcpyDeviceToHost, stream_));
  CUDA_TRY(cudaMemcpyAsync(Arow.data(), At_.rowptr.p, (n_ + 1) * sizeof(int), cudaMemcpyDeviceToHost, stream_));
  if (P_.nnz) CUDA_TRY(cudaMemcpyAsync(Pcol.data(), P_.col.p, P_.nnz * sizeof(int), cudaMemcpyDeviceToHost, stream_));
  if (At_.nnz) CUDA_TRY(cudaMemcpyAsync(Acol.data(), At_.col.p, At_.nnz * sizeof(int), cudaMemcpyDeviceToHost, stream_));
  sync();
  ldl_sn::Symbolic& S = sn_;
  ldl_sn::analyze(n_, m_, Prow, Pcol, Arow, Acol, S);
  sn_symbolic_s_ = now_s() - t0;
  const size_t ts = sizeof(T);
  // path per supernode: the small path when the panel and its relative rows fit one CTA's shared memory; the tiled
  // path's descendant updates split into groups of about kUpdatesPerGroup, the partial sums capped at 256 MB
  constexpr int64_t kUpdatesPerGroup = 16;
  sn_levels_.assign(S.levels, SnLevel());
  std::vector<int> small;
  int64_t part = 0;
  sn_small_count_ = sn_tiled_count_ = 0;
  for (int l = 0; l < S.levels; ++l) {
    SnLevel& L = sn_levels_[l];
    L.small0 = (int)small.size();
    for (int k = S.lptr[l]; k < S.lptr[l + 1]; ++k) {
      const int s = S.lcols[k];
      const int64_t h = S.height(s), w = S.width(s);
      const size_t bytes = (size_t)(h * w) * ts + (size_t)h * sizeof(int);
      if (bytes <= (size_t)sn::kSmallBytes) {
        small.push_back(s);
        L.smem = std::max(L.smem, bytes);
        ++sn_small_count_;
      } else {
        const int64_t nu = S.uptr[s + 1] - S.uptr[s];
        int64_t g = std::max<int64_t>(1, (nu + kUpdatesPerGroup - 1) / kUpdatesPerGroup);
        g = std::max<int64_t>(1, std::min<int64_t>(g, (int64_t)((256u << 20) / (h * w * ts))));
        const int64_t chunk = std::max<int64_t>(1, (nu + g - 1) / g);
        g = std::max<int64_t>(1, (nu + chunk - 1) / chunk);
        L.big.push_back(SnBig{s, g, chunk});
        if (nu) part = std::max(part, g * h * w);
        ++sn_tiled_count_;
      }
    }
    L.small1 = (int)small.size();
  }
  const int64_t N = S.N, entries = S.off.empty() ? 0 : S.off.back();
  const double need = (double)entries * ts + (double)part * ts + (double)S.rows.size() * 4 + (double)S.Kpos.size() * 16 +
                      (double)S.Ksrc.size() * 8 + (double)S.ud.size() * 12 + (double)S.gd.size() * 8 + (double)N * (3 * ts + 24);
  size_t free_b = 0, total_b = 0;
  CUDA_TRY(cudaMemGetInfo(&free_b, &total_b));
  if (need > 0.9 * (double)free_b) {
    char b[256];
    snprintf(b, sizeof(b), "the supernodal LDL' factor does not fit in device memory: %lld stored entries need %.2f GB, %.2f GB free",
             (long long)S.stored, need * 1e-9, (double)free_b * 1e-9);
    throw EngineError{COSMO_B200_ERR_ALLOC, b};
  }
  sn_sptr_.upload(S.sptr, stream_); sn_rptr_.upload(S.rptr, stream_); sn_rows_.upload(S.rows, stream_); sn_off_.upload(S.off, stream_);
  sn_uptr_.upload(S.uptr, stream_); sn_ud_.upload(S.ud, stream_); sn_up0_.upload(S.up0, stream_); sn_up1_.upload(S.up1, stream_);
  sn_Ksp_.upload(S.Ksp, stream_); sn_Ksrc_.upload(S.Ksrc, stream_); sn_Kpos_.upload(S.Kpos, stream_);
  sn_gptr_.upload(S.gptr, stream_); sn_gd_.upload(S.gd, stream_); sn_gi_.upload(S.gi, stream_);
  sn_perm_.upload(S.perm, stream_); sn_small_.upload(small, stream_);
  sn_lrows_.upload(S.lrows, stream_); sn_lcols_.upload(S.lcols, stream_); sn_bcols_.upload(S.bcols, stream_);
  sn_Lx_.alloc(std::max<int64_t>(entries, 1), false);
  sn_part_.alloc(std::max<int64_t>(part, 1), false);
  sn_D_.alloc(std::max<int64_t>(N, 1)); sn_Dinv_.alloc(std::max<int64_t>(N, 1)); sn_y_.alloc(std::max<int64_t>(N, 1));
  sn_flags_.alloc(2);
  sync();
  CUDA_TRY(cudaFuncSetAttribute(sn::sn_small_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, sn::kSmallBytes));
  CUDA_TRY(cudaFuncSetAttribute(sn::sn_fdiag_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, sn::kSmallBytes));
  CUDA_TRY(cudaFuncSetAttribute(sn::sn_backward_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, sn::kSmallBytes));
  ldl_ev_[0].create();
  ldl_ev_[1].create();
  sn_factor_graph_.reset();
  sn_solve_graph_.reset();
  sn_ready_ = true;
  sn_dirty_ = true;
}

template <typename T>
static int sn_lower_tiles(int64_t rows, int64_t cols) {   // tiles (bi >= bj) of a rows x cols panel, kTile square
  const int64_t nrt = (rows + sn::kTile - 1) / sn::kTile, nct = (cols + sn::kTile - 1) / sn::kTile;
  int64_t t = 0;
  for (int64_t bj = 0; bj < nct; ++bj) t += nrt - bj;
  return (int)t;
}

// Assemble the panels from the resident (scaled) P_, At_, rho_vec_ and sigma and factor them level by level: one
// captured graph, replayed on every refactorisation.  Reads back the pivot counts (the plugin's only host sync).
template <typename T>
void Engine<T>::sn_factor() {
  if (!sn_ready_) sn_setup();
  const ldl_sn::Symbolic& S = sn_;
  if (!sn_factor_graph_) {
    int nodes = 0;
    sn::Args<T> a;
    a.sptr = sn_sptr_.p; a.rptr = sn_rptr_.p; a.rows = sn_rows_.p; a.off = sn_off_.p;
    a.uptr = sn_uptr_.p; a.ud = sn_ud_.p; a.up0 = sn_up0_.p; a.up1 = sn_up1_.p;
    a.Lx = sn_Lx_.p; a.D = sn_D_.p; a.Dinv = sn_Dinv_.p; a.flags = sn_flags_.p;
    const int64_t entries = S.off.empty() ? 0 : S.off.back();
    capture_graph(sn_factor_graph_, stream_, [&] {
      ldl_reset_flags_kernel<<<1, 32, 0, stream_>>>(sn_flags_.p); ++nodes;
      if (entries) { CUDA_TRY(cudaMemsetAsync(sn_Lx_.p, 0, entries * sizeof(T), stream_)); ++nodes; }
      if (S.nnz_K) {
        sn::sn_assemble_kernel<T><<<vgrid(S.nnz_K), kBlock, 0, stream_>>>(S.nnz_K, sn_Ksp_.p, sn_Ksrc_.p, sn_Kpos_.p, P_.val.p,
                                                                          At_.val.p, rho_vec_.p, (T)st_.sigma, sn_Lx_.p);
        ++nodes;
      }
      for (const SnLevel& L : sn_levels_) {
        if (L.small1 > L.small0) {
          const int cnt = L.small1 - L.small0;
          sn::sn_small_kernel<T><<<std::min(cnt, kMaxGrid), kBlock, L.smem, stream_>>>(a, sn_small_.p + L.small0, cnt);
          ++nodes;
        }
        for (const SnBig& B : L.big) {
          const int s = B.s, c0 = S.sptr[s], w = S.width(s), h = S.height(s);
          T* F = sn_Lx_.p + S.off[s];
          const int64_t u0 = S.uptr[s], u1 = S.uptr[s + 1];
          if (u1 > u0) {
            sn::sn_tile_update_kernel<T><<<dim3(sn_lower_tiles<T>(h, w), (unsigned)B.groups), kBlock, 0, stream_>>>(
                a, c0, w, h, sn_rows_.p + S.rptr[s], u0, u1, B.chunk, sn_part_.p);
            sn::sn_tile_reduce_kernel<T><<<vgrid((int64_t)h * w), kBlock, 0, stream_>>>(F, sn_part_.p, (int)B.groups, h, w);
            nodes += 2;
          }
          for (int b0 = 0; b0 < w; b0 += sn::kTile) {
            const int nb = std::min(sn::kTile, w - b0), b1 = b0 + nb;
            const int rows = h - b1;
            sn::sn_diag_kernel<T><<<1, kBlock, 0, stream_>>>(a, F, c0, h, b0, nb);
            ++nodes;
            if (rows > 0) {
              sn::sn_panel_kernel<T><<<(rows + sn::kPanelThreads - 1) / sn::kPanelThreads, sn::kPanelThreads, 0, stream_>>>(
                  F, h, b0, nb);
              ++nodes;
            }
            if (b1 < w) {
              sn::sn_trail_kernel<T><<<sn_lower_tiles<T>(h - b1, w - b1), kBlock, 0, stream_>>>(F, sn_D_.p + c0 + b0, h, w, b0, b1);
              ++nodes;
            }
          }
        }
      }
    });
    sn_factor_nodes_ = nodes;
  }
  int flags[2] = {0, 0};
  CUDA_TRY(cudaEventRecord(ldl_ev_[0], stream_));
  CUDA_TRY(cudaGraphLaunch(sn_factor_graph_, stream_));
  CUDA_TRY(cudaEventRecord(ldl_ev_[1], stream_));
  CUDA_TRY(cudaMemcpyAsync(flags, sn_flags_.p, sizeof(flags), cudaMemcpyDeviceToHost, stream_));
  sync();
  launches_ += sn_factor_nodes_;
  float ms = 0.f;
  CUDA_TRY(cudaEventElapsedTime(&ms, ldl_ev_[0], ldl_ev_[1]));
  sn_factor_s_ = ms * 1e-3;
  ++sn_factorizations_;
  if (flags[1] != 0) {
    char b[160];
    snprintf(b, sizeof(b), "supernodal LDL' factorisation of the KKT matrix met %d zero or non-finite pivots", flags[1]);
    throw EngineError{COSMO_B200_ERR_NUMERICAL, b};
  }
  if (flags[0] != n_) throw EngineError{COSMO_B200_ERR_INVALID, "Objective function is not convex."};
  sn_dirty_ = false;
}

// [y1; y2] = K \ [x1; x2] with ls_ = [x1; x2], xsol_ = y1, nu_ = y2: the forward solve by supernodal level, the
// backward solve by depth, replayed as one graph
template <typename T>
void Engine<T>::sn_solve() {
  if (nranks_ > 1) throw EngineError{COSMO_B200_ERR_UNSUPPORTED, "the supernodal LDL' KKT solver is single-GPU"};
  if (!sn_ready_) sn_setup();
  if (sn_dirty_) sn_factor();
  const ldl_sn::Symbolic& S = sn_;
  if (!sn_solve_graph_) {
    int nodes = 0;
    sn::SolveArgs<T> a;
    a.sptr = sn_sptr_.p; a.rptr = sn_rptr_.p; a.rows = sn_rows_.p; a.off = sn_off_.p;
    a.gptr = sn_gptr_.p; a.gd = sn_gd_.p; a.gi = sn_gi_.p;
    a.Lx = sn_Lx_.p; a.Dinv = sn_Dinv_.p; a.perm = sn_perm_.p;
    a.rhs = ls_.p; a.y = sn_y_.p; a.out1 = xsol_.p; a.out2 = nu_.p; a.n = n_;
    // the diagonal solves keep their part of y in shared memory up to kSmallBytes, wider supernodes work on y in place
    auto vec_smem = [&](int wmax) { return (size_t)wmax * sizeof(T) <= (size_t)sn::kSmallBytes ? (size_t)wmax * sizeof(T) : 0; };
    capture_graph(sn_solve_graph_, stream_, [&] {
      for (int l = 0; l < S.levels; ++l) {
        const int r0 = S.lrptr[l], nr = S.lrptr[l + 1] - r0, k0 = S.lptr[l], ns = S.lptr[l + 1] - k0;
        sn::sn_gather_kernel<T><<<(int)std::min<int64_t>((nr + kWarpsPerBlock - 1) / kWarpsPerBlock, kMaxGrid), kBlock, 0, stream_>>>(
            a, sn_lrows_.p + r0, nr);
        ++nodes;
        if (nr > ns) {   // some supernode of the level is wider than one column
          int wmax = 1;
          for (int k = k0; k < k0 + ns; ++k) wmax = std::max(wmax, S.width(S.lcols[k]));
          const size_t sm = vec_smem(wmax);
          sn::sn_fdiag_kernel<T><<<std::min(ns, kMaxGrid), kBlock, sm, stream_>>>(a, sn_lcols_.p + k0, ns, sm > 0);
          ++nodes;
        }
      }
      for (size_t l = 0; l + 1 < S.bptr.size(); ++l) {
        const int k0 = S.bptr[l], ns = S.bptr[l + 1] - k0;
        int wmax = 1;
        for (int k = k0; k < k0 + ns; ++k) wmax = std::max(wmax, S.width(S.bcols[k]));
        const size_t sm = vec_smem(wmax);
        sn::sn_backward_kernel<T><<<std::min(ns, kMaxGrid), kBlock, sm, stream_>>>(a, sn_bcols_.p + k0, ns, sm > 0);
        ++nodes;
      }
    });
    sn_solve_nodes_ = nodes;
  }
  CUDA_TRY(cudaGraphLaunch(sn_solve_graph_, stream_));
  launches_ += sn_solve_nodes_;
}

template <typename T>
void Engine<T>::ldl_sn_stats(int64_t* o) {
  o[0] = sn_.ns; o[1] = sn_.max_width; o[2] = sn_.zeros(); o[3] = sn_.levels;
  o[4] = sn_ready_ ? sn_small_count_ : 0; o[5] = sn_ready_ ? sn_tiled_count_ : 0; o[6] = sn_solve_nodes_;
  o[7] = (int64_t)sn_.update_flops;
}

template <typename T>
void Engine<T>::residuals(const void* x, const void* s, const void* mu, int ignore_scaling, double* out) {
  CUDA_TRY(cudaSetDevice(device_));
  upload_vec(dx_, x, n_);
  upload_vec(vec_m_, s, m_);
  upload_vec(dy_, mu, m_);
  compute_residuals(dx_.p, vec_m_.p, dy_.p, ignore_scaling != 0, out);
}

template <typename T>
void Engine<T>::spmv(int which, const void* x, void* y) {
  CUDA_TRY(cudaSetDevice(device_));
  if (which == 0) {
    upload_vec(dx_, x, n_);
    launch_spmv(A_, dx_.p, (const DevCsr<T>*)nullptr, (const T*)nullptr, m_, EpiStore<T>{nullptr, vec_m_.p}, red(SC_TMP0), "spmv_A");
    download_vec(y, vec_m_.p, m_);
  } else if (which == 1) {
    upload_vec(dy_, x, m_);
    launch_spmv(At_, dy_.p, (const DevCsr<T>*)nullptr, (const T*)nullptr, n_, EpiStore<T>{nullptr, vec_n_.p}, red(SC_TMP0), "spmv_At");
    download_vec(y, vec_n_.p, n_);
  } else if (which == 2) {
    upload_vec(dx_, x, n_);
    launch_spmv(P_, dx_.p, (const DevCsr<T>*)nullptr, (const T*)nullptr, n_, EpiStore<T>{nullptr, vec_n_.p}, red(SC_TMP0), "spmv_P");
    download_vec(y, vec_n_.p, n_);
  } else if (which == 3) {
    // second stage of the reduced KKT operator: y = A' x2 + P x1 + sigma x1, x = [x1; x2] (the CG kernel's pass)
    upload_vec(dx_, x, n_);
    upload_vec(dy_, static_cast<const T*>(x) + n_, m_);
    kkt_op_stage2(nullptr, dx_.p, dy_.p, vec_n_.p);
    download_vec(y, vec_n_.p, n_);
  } else {
    throw EngineError{COSMO_B200_ERR_INVALID, "spmv: which must be 0 (A), 1 (A'), 2 (P) or 3 (A' x2 + P x1 + sigma x1)"};
  }
  sync();
}

template <typename T>
void Engine<T>::spmv_bench(int which, int reps, double* ms, double* bytes) {
  CUDA_TRY(cudaSetDevice(device_));
  if (reps < 1) reps = 1;
  auto one = [&]() {
    if (which == 0)
      launch_spmv(A_, xsol_.p, (const DevCsr<T>*)nullptr, (const T*)nullptr, m_, EpiScale<T>{nullptr, tm_.p, rho_vec_.p}, red(SC_TMP0), "spmv_A_scale");
    else if (which == 1)
      launch_spmv(At_, tm_.p, (const DevCsr<T>*)nullptr, (const T*)nullptr, n_, EpiStore<T>{nullptr, vec_n_.p}, red(SC_TMP0), "spmv_At");
    else if (which == 2)
      launch_spmv(P_, xsol_.p, (const DevCsr<T>*)nullptr, (const T*)nullptr, n_, EpiStore<T>{nullptr, vec_n_.p}, red(SC_TMP0), "spmv_P");
    else  // 3: the reduced-KKT operator stage 2 (A' and P rows + dot)
      kkt_op_stage2(nullptr, xsol_.p, tm_.p, cb_.p);
  };
  for (int i = 0; i < 3; ++i) one();
  CUDA_TRY(cudaEventRecord(ev0_, stream_));
  for (int i = 0; i < reps; ++i) one();
  CUDA_TRY(cudaEventRecord(ev1_, stream_));
  sync();
  float t = 0.f;
  CUDA_TRY(cudaEventElapsedTime(&t, ev0_, ev1_));
  *ms = (double)t / reps;
  if (which == 0) *bytes = A_.spmv_bytes() + sizeof(T) * (double)m_;       // + rho
  else if (which == 1) *bytes = At_.spmv_bytes();
  else if (which == 2) *bytes = P_.spmv_bytes();
  else *bytes = At_.spmv_bytes() + P_.spmv_bytes() - sizeof(T) * (double)n_;
}

template <typename T>
void Engine<T>::get_rho_vec(void* out) { download_vec(out, rho_vec_.p, m_); sync(); }
template <typename T>
void Engine<T>::psd_stats(int64_t* o) {
  o[0] = psd_.tc_projections; o[1] = psd_.tc_fallbacks; o[2] = psd_.tc_.last_steps; o[3] = psd_.tc_.last_checks;
  o[4] = 0; o[5] = 0; o[6] = psd_.last_sweeps; o[7] = psd_.tc_.gemm.k;
}
template <typename T>
void Engine<T>::get_w(void* out) { download_vec(out, W_[cur_].p, (size_t)n_ + m_); sync(); }

template <typename T>
void Engine<T>::infeasibility_test(int which, const void* delta, double* out) {
  CUDA_TRY(cudaSetDevice(device_));
  if (which == 0) {
    upload_vec(dy_, delta, m_);
    primal_infeasible();
  } else if (which == 1) {
    upload_vec(dx_, delta, n_);
    dual_infeasible();
  } else {
    throw EngineError{COSMO_B200_ERR_INVALID, "infeasibility_test: which must be 0 (primal) or 1 (dual)"};
  }
  for (int k = 0; k < 8; ++k) out[k] = inf_rec_[k];
}

template <typename T>
void Engine<T>::psd_lambda_max(const void* v, double* lam) {
  CUDA_TRY(cudaSetDevice(device_));
  upload_vec(vec_m_, v, m_);
  if (!psd_.empty()) psd_.lambda_max(vec_m_.p, stream_, st_.psd_max_sweeps, launches_, lam);
  sync();
}

template <typename T>
void Engine<T>::set_decomposition(const cosmo_b200_decomposition* d, bool traditional) {
  if (nranks_ > 1) throw EngineError{COSMO_B200_ERR_UNSUPPORTED, "set_decomposition: the reverse of a decomposition is single-GPU"};
  CUDA_TRY(cudaSetDevice(device_));
  if (!d) rev_.clear();
  else rev_.set(*d, n_, m_, stream_, traditional);   // either map replaces the other
}

template <typename T>
void Engine<T>::set_forward_map(const cosmo_b200_forward_map* f) {
  if (nranks_ > 1) throw EngineError{COSMO_B200_ERR_UNSUPPORTED, "set_forward_map: a sharded handle holds only a slice of the data"};
  CUDA_TRY(cudaSetDevice(device_));
  if (!f) fwd_.clear();
  else fwd_.set(*f, n_, m_, At_.nnz, stream_);
  have_q0_ = have_b0_ = false;   // their sizes follow the map
}

// reverse_scaling! + reverse_decomposition! (+ psd_completion!) of the iterates the last solve left in HBM
template <typename T>
void Engine<T>::reverse_decomposition(int complete_dual, void* x, void* s, void* mu, int64_t* stats4) {
  if (nranks_ > 1) throw EngineError{COSMO_B200_ERR_UNSUPPORTED, "reverse_decomposition: the reverse of a decomposition is single-GPU"};
  if (!rev_.has_map()) throw EngineError{COSMO_B200_ERR_INVALID, "reverse_decomposition: no decomposition map (cosmo_b200_set_decomposition)"};
  if (!have_solution_)
    throw EngineError{COSMO_B200_ERR_INVALID, "reverse_decomposition: no solve since the engine was created, reset or warm-started"};
  const unsigned dev = caller_arrays({x, s, mu});
  rev_.run<T>(xs_.p, s_.p, mu_.p, scaled_ ? D_.p : nullptr, scaled_ ? E_.p : nullptr, scaled_ ? c_ : 1.0, complete_dual != 0,
              x, s, mu, stats4, stream_, device_);
  if (dev) caller_written();
}

// Checks the caller's array arguments before anything is written: each may be host memory, device memory of this
// handle's device or managed memory (the copies use cudaMemcpyDefault).  When one is device or managed memory, the
// engine stream waits for the work the caller enqueued on its stream.  Returns those arguments as a mask (bit k: the
// k-th pointer).
template <typename T>
unsigned Engine<T>::caller_arrays(std::initializer_list<const void*> ptrs) {
  CUDA_TRY(cudaSetDevice(device_));
  unsigned dev = 0, bit = 1;
  for (const void* p : ptrs) {
    cudaPointerAttributes a{};
    if (p) CUDA_TRY(cudaPointerGetAttributes(&a, p));
    if (p && (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged)) {
      if (a.type == cudaMemoryTypeDevice && a.device != device_)
        throw EngineError{COSMO_B200_ERR_INVALID, "an array lies in the memory of device " + std::to_string(a.device) +
                                                      ", the engine on device " + std::to_string(device_)};
      dev |= bit;
    }
    bit <<= 1;
  }
  if (dev) {
    caller_ev_.create();
    CUDA_TRY(cudaEventRecord(caller_ev_, caller_stream_));
    CUDA_TRY(cudaStreamWaitEvent(stream_, caller_ev_, 0));
  }
  return dev;
}

// After the engine wrote caller device or managed memory: the caller stream waits for the engine stream.
template <typename T>
void Engine<T>::caller_written() {
  caller_ev_.create();
  CUDA_TRY(cudaEventRecord(caller_ev_, stream_));
  CUDA_TRY(cudaStreamWaitEvent(caller_stream_, caller_ev_, 0));
}

// update!(q=, b=) in the model's coordinates, unscaled fp64: through the forward map when one is set, then scaled as the
// host scales (scale_original_qb_kernel), then update_qb's state change.  The b is checked for uncovered rows before
// anything is written.
template <typename T>
void Engine<T>::update_qb_original(const double* q, const double* b) {
  single_gpu("update_qb_original");
  const bool dev_b = (caller_arrays({q, b}) & 2) != 0;
  const bool mapped = fwd_.has_map();
  const size_t n0 = mapped ? (size_t)fwd_.n_orig() : (size_t)n_, m0 = mapped ? (size_t)fwd_.m_orig() : (size_t)m_;
  DevBuf<double> stage;   // a host b is checked on the device before b0_ changes
  const double* bsrc = b;
  if (b && mapped) {
    if (!dev_b && m0) {
      stage.alloc(m0, false);
      stage.upload(b, m0, stream_);
      bsrc = stage.p;
    }
    const long long bad = fwd_.count_uncovered<double>(bsrc, stream_);
    launches_ += 2;
    if (bad)
      throw EngineError{COSMO_B200_ERR_INVALID, "update_qb_original: b is nonzero in " + std::to_string(bad) +
                                                    " rows of a decomposed cone that no clique holds (the sparsity pattern, and with it the decomposition, changes: a new engine is needed)"};
  }
  if (q) {
    if (!q0_.p || q0_.n != n0) q0_.alloc(n0, false);
    if (n0) CUDA_TRY(cudaMemcpyAsync(q0_.p, q, n0 * sizeof(double), cudaMemcpyDefault, stream_));
    have_q0_ = true;
  }
  if (b) {
    if (!b0_.p || b0_.n != m0) b0_.alloc(m0, false);
    if (m0) CUDA_TRY(cudaMemcpyAsync(b0_.p, bsrc, m0 * sizeof(double), cudaMemcpyDefault, stream_));
    have_b0_ = true;
  }
  const T* D = scaled_ ? D_.p : nullptr;
  const T* E = scaled_ ? E_.p : nullptr;
  const long long nq = q ? n_ : 0, mb = b && !mapped ? m_ : 0;
  if (nq + mb) {
    scale_original_qb_kernel<T><<<vgrid(nq + mb), kBlock, 0, stream_>>>(nq, (long long)n0, q0_.p, D, scaled_ ? c_ : 1.0,
                                                                         q_.p, mb, b0_.p, E, b_.p);
    check_launch("scale_original_qb");
  }
  if (b && mapped) {
    fwd_.gather_b<double, T>(b0_.p, b_.p, stream_, E);
    ++launches_;
  }
  if (b) classify_and_set_rho(false);
  sync();
}

template <typename T>
void Engine<T>::original_qb(double* q, double* b) {
  single_gpu("original_qb");
  if ((q && !have_q0_) || (b && !have_b0_))
    throw EngineError{COSMO_B200_ERR_INVALID, "original_qb: no q or b from update_qb_original since the forward map was set"};
  const unsigned dev = caller_arrays({q, b});
  if (q && q0_.n) CUDA_TRY(cudaMemcpyAsync(q, q0_.p, q0_.n * sizeof(double), cudaMemcpyDefault, stream_));
  if (b && b0_.n) CUDA_TRY(cudaMemcpyAsync(b, b0_.p, b0_.n * sizeof(double), cudaMemcpyDefault, stream_));
  if (dev) caller_written();
  sync();
}

// The last solution in the original coordinates: reverse_decomposition's arithmetic with a decomposition map, else the
// same gather through the identity map (x = D x', s = s' / E, mu = (E mu') / c), with y = -mu.
template <typename T>
void Engine<T>::solution(int complete_dual, double* x, double* y, double* s) {
  single_gpu("solution");
  if (!have_solution_)
    throw EngineError{COSMO_B200_ERR_INVALID, "solution: no solve since the engine was created, reset or warm-started"};
  const unsigned dev = caller_arrays({x, y, s});
  rev::Reverse* r = &rev_;
  if (!rev_.has_map()) {
    if (!ident_.has_map()) {
      const int64_t plain[3] = {0, 0, m_};
      cosmo_b200_decomposition d{};
      d.n_orig = n_; d.m_orig = m_; d.n = n_; d.m = m_;
      d.n_plain = m_ ? 1 : 0; d.plain = plain;
      ident_.set(d, n_, m_, stream_);
    }
    r = &ident_;
  }
  r->run<T>(xs_.p, s_.p, mu_.p, scaled_ ? D_.p : nullptr, scaled_ ? E_.p : nullptr, scaled_ ? c_ : 1.0, complete_dual != 0,
            x, s, y, nullptr, stream_, device_, true);
  if (dev) caller_written();
}

// The host's round trip between two solves (reverse_scaling!, then scale_variables! of the result as the next warm
// start) on the resident iterates; like warm_start it ends the last solution.
template <typename T>
void Engine<T>::rescale_iterates() {
  single_gpu("rescale_iterates");
  CUDA_TRY(cudaSetDevice(device_));
  have_solution_ = false;
  rescale_iterates_kernel<T><<<vgrid((long long)n_ + m_), kBlock, 0, stream_>>>(
      n_, m_, scaled_ ? D_.p : nullptr, scaled_ ? E_.p : nullptr, scaled_ ? c_ : 1.0, xs_.p, s_.p, mu_.p);
  check_launch("rescale_iterates");
  sync();
}

}  // namespace cosmo

// ============================================================================
// C ABI
// ============================================================================
struct cosmo_b200_handle {
  cosmo::EngineBase* impl = nullptr;
  std::string err;
};

// The code of the exception in flight, its message into `msg`: call it from a catch block.
static int error_code(std::string& msg) {
  try { throw; }
  catch (const cosmo::EngineError& e) { msg = e.msg; return e.code; }
  catch (const std::bad_alloc&) { msg = "host allocation failed"; return COSMO_B200_ERR_ALLOC; }
  catch (...) { msg = "unknown error"; return COSMO_B200_ERR_INVALID; }
}

#define ABI_GUARD(h, body)                                                   \
  if (!(h) || !(h)->impl) return COSMO_B200_ERR_INVALID;                     \
  try { body; return COSMO_B200_OK; }                                        \
  catch (...) { return error_code((h)->err); }

extern "C" {

int cosmo_b200_abi_version(void) { return COSMO_B200_ABI_VERSION; }

int cosmo_b200_default_settings(cosmo_b200_settings* s) {
  if (!s) return COSMO_B200_ERR_INVALID;
  memset(s, 0, sizeof(*s));
  s->rho = 0.1; s->sigma = 1e-6; s->alpha = 1.6;
  s->eps_abs = 1e-5; s->eps_rel = 1e-5; s->eps_prim_inf = 1e-4; s->eps_dual_inf = 1e-4;
  s->max_iter = 5000; s->check_termination = 25; s->check_infeasibility = 40;
  s->scaling = 10; s->adaptive_rho = 1; s->adaptive_rho_interval = 40; s->kkt_solver = COSMO_B200_KKT_CG;
  s->adaptive_rho_fraction = 0.4; s->setup_time = 0.0; s->MAX_SCALING = 1e4;
  s->obj_true = NAN; s->obj_true_tol = 1e-3;
  s->adaptive_rho_tolerance = 5.0; s->adaptive_rho_max_adaptions = INT64_MAX;
  s->RHO_MIN = 1e-6; s->RHO_MAX = 1e6; s->RHO_TOL = 1e-4; s->RHO_EQ_OVER_RHO_INEQ = 1e3;
  s->COSMO_INFTY = 1e20; s->MIN_SCALING = 1e-4;
  s->time_limit = 0.0; s->tol_constant = 1.0; s->tol_exponent = 1.5;
  s->verbose = 0; s->psd_max_sweeps = 30;
  s->accelerator = COSMO_B200_ACC_EMPTY; s->accelerator_mem = 15; s->accelerator_min_mem = 3;
  s->safeguard = 1; s->safeguard_tol = 2.0;
  return COSMO_B200_OK;
}

int cosmo_b200_create(cosmo_b200_handle** out, const cosmo_b200_problem* prob, const cosmo_b200_settings* settings) {
  if (!out || !prob || !settings) { cosmo::g_create_error = "null argument"; return COSMO_B200_ERR_INVALID; }
  *out = nullptr;
  try {
    cosmo::EngineBase* impl = nullptr;
    if (prob->dtype == COSMO_B200_F64) impl = new cosmo::Engine<double>(*prob, *settings);
    else if (prob->dtype == COSMO_B200_F32) impl = new cosmo::Engine<float>(*prob, *settings);
    else throw cosmo::EngineError{COSMO_B200_ERR_UNSUPPORTED, "dtype must be Float64 or Float32 (BigFloat models fall back to the host loop)"};
    cosmo_b200_handle* h = new cosmo_b200_handle();
    h->impl = impl;
    *out = h;
    return COSMO_B200_OK;
  } catch (...) { return error_code(cosmo::g_create_error); }
}

void cosmo_b200_destroy(cosmo_b200_handle* h) {
  if (!h) return;
  delete h->impl;
  delete h;
}

const char* cosmo_b200_last_error(const cosmo_b200_handle* h) {
  return h ? h->err.c_str() : cosmo::g_create_error.c_str();
}

int cosmo_b200_update_settings(cosmo_b200_handle* h, const cosmo_b200_settings* s) {
  if (!s) return COSMO_B200_ERR_INVALID;
  ABI_GUARD(h, h->impl->update_settings(*s));
}
int cosmo_b200_warm_start(cosmo_b200_handle* h, const void* x, const void* s, const void* mu) { ABI_GUARD(h, h->impl->warm_start(x, s, mu)); }
int cosmo_b200_update_qb(cosmo_b200_handle* h, const void* q, const void* b) { ABI_GUARD(h, h->impl->update_qb(q, b)); }
int cosmo_b200_update_matrices(cosmo_b200_handle* h, const void* Px, int64_t nnzP, const void* Ax, int64_t nnzA, const void* q,
                               const void* b) {
  ABI_GUARD(h, h->impl->update_matrices(Px, nnzP, Ax, nnzA, q, b));
}
int cosmo_b200_update_rho(cosmo_b200_handle* h, const void* rho_vec, double rho) { ABI_GUARD(h, h->impl->update_rho(rho_vec, rho)); }
int cosmo_b200_reset(cosmo_b200_handle* h) { ABI_GUARD(h, h->impl->reset()); }
int cosmo_b200_solve(cosmo_b200_handle* h, cosmo_b200_result* out) { ABI_GUARD(h, h->impl->solve(out)); }
int cosmo_b200_project(cosmo_b200_handle* h, const void* w_s, void* s_out) {
  if (!w_s || !s_out) return COSMO_B200_ERR_INVALID;
  ABI_GUARD(h, h->impl->project(w_s, s_out));
}
int cosmo_b200_kkt_solve(cosmo_b200_handle* h, const void* rhs, void* sol, int64_t* inner) {
  if (!rhs || !sol) return COSMO_B200_ERR_INVALID;
  ABI_GUARD(h, h->impl->kkt_solve(rhs, sol, inner));
}
int cosmo_b200_residuals(cosmo_b200_handle* h, const void* x, const void* s, const void* mu, int32_t ignore_scaling, double out[5]) {
  if (!x || !s || !mu || !out) return COSMO_B200_ERR_INVALID;
  ABI_GUARD(h, h->impl->residuals(x, s, mu, ignore_scaling, out));
}
int cosmo_b200_spmv(cosmo_b200_handle* h, int32_t which, const void* x, void* y) {
  if (!x || !y) return COSMO_B200_ERR_INVALID;
  ABI_GUARD(h, h->impl->spmv(which, x, y));
}
int cosmo_b200_spmv_bench(cosmo_b200_handle* h, int32_t which, int32_t reps, double* ms, double* bytes) {
  if (!ms || !bytes) return COSMO_B200_ERR_INVALID;
  ABI_GUARD(h, h->impl->spmv_bench(which, reps, ms, bytes));
}
int cosmo_b200_get_rho_vec(cosmo_b200_handle* h, void* out) {
  if (!out) return COSMO_B200_ERR_INVALID;
  ABI_GUARD(h, h->impl->get_rho_vec(out));
}
int cosmo_b200_get_w(cosmo_b200_handle* h, void* out) {
  if (!out) return COSMO_B200_ERR_INVALID;
  ABI_GUARD(h, h->impl->get_w(out));
}
int cosmo_b200_psd_stats(cosmo_b200_handle* h, int64_t out[8]) {
  if (!out) return COSMO_B200_ERR_INVALID;
  ABI_GUARD(h, h->impl->psd_stats(out));
}
int cosmo_b200_set_accelerator(cosmo_b200_handle* h, const cosmo_b200_accelerator* acc) {
  ABI_GUARD(h, h->impl->set_accelerator(acc));
}
int cosmo_b200_accelerator_stats(cosmo_b200_handle* h, int64_t out[6]) {
  if (!out) return COSMO_B200_ERR_INVALID;
  ABI_GUARD(h, h->impl->accelerator_stats(out));
}
int cosmo_b200_infeasibility_test(cosmo_b200_handle* h, int32_t which, const void* delta, double out[8]) {
  if (!delta || !out) return COSMO_B200_ERR_INVALID;
  ABI_GUARD(h, h->impl->infeasibility_test(which, delta, out));
}
int cosmo_b200_psd_lambda_max(cosmo_b200_handle* h, const void* v, double* lam) {
  if (!v || !lam) return COSMO_B200_ERR_INVALID;
  ABI_GUARD(h, h->impl->psd_lambda_max(v, lam));
}
int cosmo_b200_get_scaling(cosmo_b200_handle* h, void* D, void* E, double* c) {
  ABI_GUARD(h, h->impl->get_scaling(D, E, c));
}
int cosmo_b200_ldl_stats(cosmo_b200_handle* h, double out[8]) {
  if (!out) return COSMO_B200_ERR_INVALID;
  ABI_GUARD(h, h->impl->ldl_stats(out));
}
int cosmo_b200_ldl_symbolic(const cosmo_b200_problem* p, int64_t* perm, int64_t* parent, int64_t* colcount, int64_t* level) {
  if (!p || !perm || !parent || !colcount || !level) { cosmo::g_create_error = "null argument"; return COSMO_B200_ERR_INVALID; }
  try {
    if (p->m < 0 || p->n < 0 || p->A.nrows != p->m || p->A.ncols != p->n || p->P.nrows != p->n || p->P.ncols != p->n)
      throw cosmo::EngineError{COSMO_B200_ERR_INVALID, "P must be n x n and A m x n"};
    if (p->dtype != COSMO_B200_F64 && p->dtype != COSMO_B200_F32)
      throw cosmo::EngineError{COSMO_B200_ERR_UNSUPPORTED, "dtype must be Float64 or Float32"};
    cosmo::HostCsr a, at, pp, ppt;
    cosmo::csc_to_host_csrs(p->A, p->index_base, a, at);
    cosmo::csc_to_host_csrs(p->P, p->index_base, pp, ppt);
    cosmo::ldl::Symbolic S;
    cosmo::ldl::analyze((int)p->n, (int)p->m, pp.rowptr, pp.col, at.rowptr, at.col, S);
    for (int j = 0; j < S.N; ++j) {
      perm[j] = S.perm[j];
      parent[j] = S.parent[j];
      colcount[j] = S.Lp[j + 1] - S.Lp[j];
      level[j] = S.level[j];
    }
    return COSMO_B200_OK;
  } catch (...) { return error_code(cosmo::g_create_error); }
}
int cosmo_b200_ldl_sn_stats(cosmo_b200_handle* h, int64_t out[8]) {
  if (!out) return COSMO_B200_ERR_INVALID;
  ABI_GUARD(h, h->impl->ldl_sn_stats(out));
}
int cosmo_b200_ldl_sn_symbolic(const cosmo_b200_problem* p, int64_t* perm, int64_t* snode_ptr, int64_t* snode_parent, int64_t stats[8]) {
  if (!p || !perm || !snode_ptr || !snode_parent || !stats) { cosmo::g_create_error = "null argument"; return COSMO_B200_ERR_INVALID; }
  try {
    if (p->m < 0 || p->n < 0 || p->A.nrows != p->m || p->A.ncols != p->n || p->P.nrows != p->n || p->P.ncols != p->n)
      throw cosmo::EngineError{COSMO_B200_ERR_INVALID, "P must be n x n and A m x n"};
    if (p->dtype != COSMO_B200_F64 && p->dtype != COSMO_B200_F32)
      throw cosmo::EngineError{COSMO_B200_ERR_UNSUPPORTED, "dtype must be Float64 or Float32"};
    cosmo::HostCsr a, at, pp, ppt;
    cosmo::csc_to_host_csrs(p->A, p->index_base, a, at);
    cosmo::csc_to_host_csrs(p->P, p->index_base, pp, ppt);
    cosmo::ldl_sn::Symbolic S;
    cosmo::ldl_sn::analyze((int)p->n, (int)p->m, pp.rowptr, pp.col, at.rowptr, at.col, S);
    for (int j = 0; j < S.N; ++j) perm[j] = S.perm[j];
    for (int s = 0; s <= S.ns; ++s) snode_ptr[s] = S.sptr[s];
    for (int s = 0; s < S.ns; ++s) snode_parent[s] = S.sparent[s];
    stats[0] = S.ns; stats[1] = S.max_width; stats[2] = S.stored; stats[3] = S.zeros();
    stats[4] = S.levels; stats[5] = S.simplicial_levels; stats[6] = S.nnz_L; stats[7] = (int64_t)S.update_flops;
    return COSMO_B200_OK;
  } catch (...) { return error_code(cosmo::g_create_error); }
}
int cosmo_b200_custom_cone_compile(const cosmo_b200_custom_cone* type, int32_t dtype, char* log, int64_t log_cap) {
  if (log && log_cap > 0) log[0] = 0;
  try {
    bool compiled = false;
    cosmo::custom::cache().get(cosmo::custom::make_key(type, dtype), &compiled);
    return compiled ? 1 : 0;
  } catch (...) {
    const int rc = error_code(cosmo::g_create_error);
    if (log && log_cap > 0) {
      const size_t k = std::min<size_t>((size_t)log_cap - 1, cosmo::g_create_error.size());
      memcpy(log, cosmo::g_create_error.data(), k);
      log[k] = 0;
    }
    return rc;
  }
}
int cosmo_b200_custom_cone_stats(cosmo_b200_handle* h, int64_t out[4]) {
  if (!out) return COSMO_B200_ERR_INVALID;
  ABI_GUARD(h, h->impl->custom_cone_stats(out));
}
int cosmo_b200_comm_unique_id(void* id128) {
  if (!id128) return COSMO_B200_ERR_INVALID;
  try {
    std::string e;
    if (!cosmo::g_nccl.load(e)) throw cosmo::EngineError{COSMO_B200_ERR_NCCL, e};
    cosmo::NcclUniqueId id;
    if (cosmo::g_nccl.GetUniqueId(&id) != 0) throw cosmo::EngineError{COSMO_B200_ERR_NCCL, "ncclGetUniqueId failed"};
    memcpy(id128, &id, sizeof(id));
    return COSMO_B200_OK;
  } catch (...) { return error_code(cosmo::g_create_error); }
}
int cosmo_b200_comm_init(cosmo_b200_handle* h, int32_t nranks, int32_t rank, const void* id128) {
  if (nranks > 1 && !id128) return COSMO_B200_ERR_INVALID;
  ABI_GUARD(h, h->impl->comm_init(nranks, rank, id128));
}
int cosmo_b200_comm_p2p_export(cosmo_b200_handle* h, void* blob128) {
  if (!blob128) return COSMO_B200_ERR_INVALID;
  ABI_GUARD(h, h->impl->p2p_export(blob128));
}
int cosmo_b200_comm_p2p_attach(cosmo_b200_handle* h, const void* blobs, int32_t nranks) {
  if (!blobs) return COSMO_B200_ERR_INVALID;
  ABI_GUARD(h, h->impl->p2p_attach(blobs, nranks));
}

int cosmo_b200_set_decomposition(cosmo_b200_handle* h, const cosmo_b200_decomposition* d) {
  ABI_GUARD(h, h->impl->set_decomposition(d, false));
}
int cosmo_b200_set_decomposition_noncompact(cosmo_b200_handle* h, const cosmo_b200_decomposition* d) {
  ABI_GUARD(h, h->impl->set_decomposition(d, true));
}
int cosmo_b200_set_forward_map(cosmo_b200_handle* h, const cosmo_b200_forward_map* f) {
  ABI_GUARD(h, h->impl->set_forward_map(f));
}
int cosmo_b200_update_matrices_original(cosmo_b200_handle* h, const void* Px, int64_t nnzP, const void* Ax, int64_t nnzA_orig,
                                        const void* q, const void* b) {
  ABI_GUARD(h, h->impl->update_matrices_original(Px, nnzP, Ax, nnzA_orig, q, b));
}
int cosmo_b200_set_caller_stream(cosmo_b200_handle* h, void* stream) { ABI_GUARD(h, h->impl->set_caller_stream(stream)); }
int cosmo_b200_update_qb_original(cosmo_b200_handle* h, const double* q, const double* b) {
  ABI_GUARD(h, h->impl->update_qb_original(q, b));
}
int cosmo_b200_original_qb(cosmo_b200_handle* h, double* q, double* b) { ABI_GUARD(h, h->impl->original_qb(q, b)); }
int cosmo_b200_solution(cosmo_b200_handle* h, int32_t complete_dual, double* x, double* y, double* s) {
  ABI_GUARD(h, h->impl->solution(complete_dual, x, y, s));
}
int cosmo_b200_rescale_iterates(cosmo_b200_handle* h) { ABI_GUARD(h, h->impl->rescale_iterates()); }
int cosmo_b200_reverse_decomposition(cosmo_b200_handle* h, int32_t complete_dual, void* x, void* s, void* mu, int64_t stats[4]) {
  ABI_GUARD(h, h->impl->reverse_decomposition(complete_dual, x, s, mu, stats));
}

// psd_complete! of a bare column-major N x N matrix (upper triangle read) on the current device
int cosmo_b200_psd_complete(int64_t N, const cosmo_b200_completion* sc, double* Y, int64_t stats[4]) {
  if (!sc || !Y || N < 1 || sc->N != N) {
    cosmo::g_create_error = "psd_complete: null argument, or N is not the schedule's";
    return COSMO_B200_ERR_INVALID;
  }
  cudaStream_t st = nullptr;
  try {
    using namespace cosmo;
    int ndev = 0, dev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) throw EngineError{COSMO_B200_ERR_CUDA, "no CUDA device"};
    CUDA_TRY(cudaGetDevice(&dev));
    rev::check_schedule(*sc, -1, 0);
    CUDA_TRY(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    {
      rev::Cone cone;
      rev::upload_cone(cone, *sc, st);
      DevBuf<double> Yd, W, z;
      DevBuf<int> cnt;
      const size_t nn = (size_t)N * N;
      rev::ensure(Yd, nn, N);
      rev::ensure(W, nn, N);
      z.alloc(std::max<int64_t>(cone.z_total, 1), false);
      cnt.alloc(1);
      Yd.upload(Y, nn, st);
      Event e0, e1;
      e0.create();
      e1.create();
      CUDA_TRY(cudaEventRecord(e0, st));
      rev::permute_in_kernel<<<rev::grid_for((int64_t)nn), rev::kThreads, 0, st>>>(N, Yd.p, cone.new_of.p, W.p);
      CUDA_TRY(cudaGetLastError());
      rev::complete(cone, W.p, z.p, cnt.p, st, dev);
      rev::permute_out_kernel<<<rev::grid_for((int64_t)nn), rev::kThreads, 0, st>>>(N, W.p, cone.new_of.p, Yd.p);
      CUDA_TRY(cudaGetLastError());
      CUDA_TRY(cudaEventRecord(e1, st));
      int fallbacks = 0;
      CUDA_TRY(cudaMemcpyAsync(Y, Yd.p, nn * sizeof(double), cudaMemcpyDeviceToHost, st));
      CUDA_TRY(cudaMemcpyAsync(&fallbacks, cnt.p, sizeof(int), cudaMemcpyDeviceToHost, st));
      CUDA_TRY(cudaStreamSynchronize(st));
      float ms = 0.f;
      CUDA_TRY(cudaEventElapsedTime(&ms, e0, e1));
      if (stats) {
        stats[0] = 1;
        stats[1] = fallbacks;
        stats[2] = (int64_t)(nn * sizeof(double));
        stats[3] = (int64_t)llround(1000.0 * ms);
      }
    }
  } catch (...) {
    if (st) cudaStreamDestroy(st);
    const int rc = error_code(cosmo::g_create_error);
    if (cosmo::g_create_error.rfind("psd_complete", 0) != 0 && cosmo::g_create_error.rfind("completion", 0) != 0)
      cosmo::g_create_error = "psd_complete: " + cosmo::g_create_error;
    return rc;
  }
  cudaStreamDestroy(st);
  return COSMO_B200_OK;
}

// ---- diagnostics of the tensor-core PSD path (tc_gemm.cuh, psd_tc.cuh) ----------------------------------------
// C = A B for symmetric commuting N x N fp64 matrices (column-major, ld = N) through the int8-sliced wgmma product.
int cosmo_b200_tc_gemm_test(int32_t N, int32_t k, int32_t kstep, int32_t gpb, const double* A, const double* B, double* C,
                            int32_t reps, double* ms_per_product, double* frob2) {
  if (N <= 0 || !A || !B || !C) return COSMO_B200_ERR_INVALID;
  (void)gpb;
  cudaStream_t st = nullptr;
  try {
    using namespace cosmo;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) throw EngineError{COSMO_B200_ERR_CUDA, "no CUDA device"};
    CUDA_TRY(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    tc::OzakiGemm<double> g;
    tc::Sliced sa, sb;
    DevBuf<double> A_d, B_d, C_d, coef_d, part_d;
    const size_t nn = (size_t)N * N;
    const double coef[3] = {1.0, 0.0, 0.0};
    g.configure(k, kstep > 0 ? kstep : (k == 8 ? 10 : (k == 7 ? 7 : k + 2)));
    g.set_shape(N, st);
    A_d.alloc(nn, false); B_d.alloc(nn, false); C_d.alloc(nn, false); coef_d.alloc(3, false);
    part_d.alloc((size_t)2 * (g.ntiles + 1), false);
    sa.ensure(g.Np); sb.ensure(g.Np); sa.clear(g.Np, st); sb.clear(g.Np, st);
    A_d.upload(A, nn, st); B_d.upload(B, nn, st); coef_d.upload(coef, 3, st);
    CUDA_TRY(cudaMemsetAsync(C_d.p, 0, nn * 8, st));
    g.slice(A_d.p, sa, st); g.slice(B_d.p, sb, st);
    g.gemm(sa, sb, C_d.p, nullptr, nullptr, 1, coef_d.p, part_d.p, st);
    CUDA_TRY(cudaStreamSynchronize(st));
    if (reps > 0 && ms_per_product) {
      Event e0, e1; e0.create(); e1.create();
      CUDA_TRY(cudaEventRecord(e0, st));
      for (int r = 0; r < reps; ++r) g.gemm(sa, sb, C_d.p, nullptr, nullptr, 1, coef_d.p, part_d.p, st);
      CUDA_TRY(cudaEventRecord(e1, st));
      CUDA_TRY(cudaEventSynchronize(e1));
      float ms = 0.f;
      CUDA_TRY(cudaEventElapsedTime(&ms, e0, e1));
      *ms_per_product = ms / reps;
    }
    CUDA_TRY(cudaMemcpyAsync(C, C_d.p, nn * 8, cudaMemcpyDeviceToHost, st));
    if (frob2) {
      std::vector<double> part(2 * g.ntiles);
      CUDA_TRY(cudaMemcpyAsync(part.data(), part_d.p, part.size() * 8, cudaMemcpyDeviceToHost, st));
      CUDA_TRY(cudaStreamSynchronize(st));
      frob2[0] = frob2[1] = 0.0;
      for (int i = 0; i < g.ntiles; ++i) { frob2[0] += part[2 * i]; frob2[1] += part[2 * i + 1]; }
    }
    CUDA_TRY(cudaStreamSynchronize(st));
  } catch (...) {
    if (st) cudaStreamDestroy(st);
    const int rc = error_code(cosmo::g_create_error);
    cosmo::g_create_error = "tc_gemm_test: " + cosmo::g_create_error;
    return rc;
  }
  cudaStreamDestroy(st);
  return COSMO_B200_OK;
}

}  // extern "C"
