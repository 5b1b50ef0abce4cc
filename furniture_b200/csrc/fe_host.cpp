// fe_host.cpp -- CUDA platform layer of the C-ABI (include/furniture_b200.h): device memory, streams, kernel launches.
//
// The kernels live in fe_kernels.cu, compiled to a cubin that is embedded in this library (.incbin) and loaded through the
// driver API -- one module instance per (device, slice layout).  The slice layout table is a __constant__ object of the
// module (fe_c_lay): each instance has its own copy, written once when the instance is created, so handles with different
// models can be alive on any number of devices and launch concurrently on their own streams.  The driver entry points are
// resolved through cudaGetDriverEntryPoint, so the library has no link-time dependency on libcuda and loads on a box
// without a GPU (the CPU test suite checks its exports there).
#define FE_EMULATE 1 /* host build: the device headers are only used for their plain structs and fe_layout_build */
#define PLAT_IS_CUDA 1
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>
#include <string>
#include <vector>

struct fe_handle;
static void* plat_alloc(size_t bytes) { void* p = nullptr; return cudaMalloc(&p, bytes) == cudaSuccess ? p : nullptr; }
static void plat_free(void* p) { cudaFree(p); }
static void plat_memset0(void* p, size_t n) { cudaMemset(p, 0, n); }
static void plat_upload(void* d, const void* h, size_t n) { cudaMemcpy(d, h, n, cudaMemcpyHostToDevice); }
static void plat_download(void* h, const void* d, size_t n) { cudaMemcpy(h, d, n, cudaMemcpyDeviceToHost); }
static int plat_init(fe_handle* h);
static void plat_fini(fe_handle* h);
static void plat_sync(fe_handle* h);
static int plat_enter(fe_handle* h);
static void plat_leave(fe_handle* h, int prev);
static int plat_run_sim(fe_handle* h, int nsub, int mode, void* stream);
static int plat_run_reset(fe_handle* h, const uint8_t* mask, void* stream);
static int plat_run_step(fe_handle* h, const float* actions, float* reward, uint8_t* done, int32_t* info, void* stream);
static int plat_step_host(fe_handle* h, const float* actions, float* obs, float* reward, uint8_t* done, int32_t* info);
static void plat_copy_d2d(fe_handle* h, void* dst, const void* src, size_t n, void* stream);
static int plat_is_aligned(fe_handle* h, int n, const double* p1, const double* m1, const double* p2, const double* m2, const double* angles,
                           const int32_t* nangles, const double* thr, uint8_t* aligned, double* tq);
static int plat_dense_eval(fe_handle* h, const struct fe_dense_config* dc, const struct fe_dense_recipe* rc, const double* thr, int n_goal, int n_episodes,
                           const int32_t* first, const int32_t* count, int n_records, int nsite, int npart, int act_dim, const double* spos, const double* smat,
                           const double* ppos, const uint8_t* touch, const uint8_t* reset, const uint8_t* connected, const double* ac, double* reward,
                           uint8_t* done, double* info);
static int plat_ctl_eval(fe_handle* h, const struct fe_ctl_config* cc, int n_episodes, const int32_t* first, const int32_t* count, int n_records, const uint8_t* reset,
                         const uint8_t* policy_step, const double* action, const struct FeCtlIn* in, double* torques);

#include "fe_api.inl"

// ---------------------------------------------------------------- embedded cubin + driver entry points
__asm__(".section .rodata\n.balign 16\n.global fe_cubin_start\nfe_cubin_start:\n.incbin \"" FE_CUBIN_FILE "\"\n.global fe_cubin_end\nfe_cubin_end:\n.byte 0\n.previous\n");
extern "C" const unsigned char fe_cubin_start[];

struct DriverApi {
  CUresult (*ModuleLoadData)(CUmodule*, const void*) = nullptr;
  CUresult (*ModuleUnload)(CUmodule) = nullptr;
  CUresult (*ModuleGetFunction)(CUfunction*, CUmodule, const char*) = nullptr;
  CUresult (*ModuleGetGlobal)(CUdeviceptr*, size_t*, CUmodule, const char*) = nullptr;
  CUresult (*MemcpyHtoD)(CUdeviceptr, const void*, size_t) = nullptr;
  CUresult (*FuncSetAttribute)(CUfunction, CUfunction_attribute, int) = nullptr;
  CUresult (*LaunchKernel)(CUfunction, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, CUstream, void**, void**) = nullptr;
  CUresult (*GetErrorString)(CUresult, const char**) = nullptr;
  bool ok = false;
};
static DriverApi g_drv;
static std::mutex g_mu; // guards g_drv and g_modules

static bool drv_load(std::string* err) {
  if (g_drv.ok) return true;
  struct { const char* name; void** slot; } want[] = {
      {"cuModuleLoadData", (void**)&g_drv.ModuleLoadData}, {"cuModuleUnload", (void**)&g_drv.ModuleUnload},
      {"cuModuleGetFunction", (void**)&g_drv.ModuleGetFunction}, {"cuModuleGetGlobal", (void**)&g_drv.ModuleGetGlobal},
      {"cuMemcpyHtoD", (void**)&g_drv.MemcpyHtoD}, {"cuFuncSetAttribute", (void**)&g_drv.FuncSetAttribute},
      {"cuLaunchKernel", (void**)&g_drv.LaunchKernel}, {"cuGetErrorString", (void**)&g_drv.GetErrorString}};
  for (auto& w : want) {
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint(w.name, w.slot, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess || !*w.slot) {
      *err = std::string("driver entry point not available: ") + w.name;
      return false;
    }
  }
  g_drv.ok = true;
  return true;
}
static std::string drv_err(CUresult r) {
  const char* s = nullptr;
  if (g_drv.GetErrorString) g_drv.GetErrorString(r, &s);
  return s ? s : "unknown driver error";
}

// one loaded instance of the kernels: its own copy of the slice layout table
struct FeModule {
  int device;
  FeLayout lay;
  CUmodule mod;
  CUfunction f_sim, f_step, f_ik_step, f_ctl_step, f_reset, f_order, f_aligned, f_dense, f_ctl_eval;
  int users;
};
static std::vector<FeModule*> g_modules;

struct CudaPlat {
  FeModule* km = nullptr;
  size_t smem_sim = 0, smem_env = 0;
  int wpb = 1;
  int* slots = nullptr;  // block slot -> env (or -1)
  float* pred = nullptr; // per env: predicted work of the next step
  int nblocks = 0;
  float* pin_act = nullptr;
  unsigned char* pin_out = nullptr;
  size_t out_bytes = 0;
  cudaStream_t stream = nullptr;       // private stream of fe_env_step_host
  cudaStream_t last_stream = nullptr;  // stream of the last launch issued for this handle
  bool any_launch = false;
  cudaEvent_t order_ev = nullptr;      // orders the private stream behind work issued on other streams
};
#define CUDA_OK(call) do { cudaError_t _e = (call); if (_e != cudaSuccess) return fail(h, -10, std::string(#call) + ": " + cudaGetErrorString(_e)); } while (0)
#define DRV_OK(call) do { CUresult _r = (call); if (_r != CUDA_SUCCESS) return fail(h, -10, std::string(#call) + ": " + drv_err(_r)); } while (0)

// every C-ABI entry makes the handle's device current for the duration of the call and restores the caller's
static int plat_enter(fe_handle* h) {
  int prev = -1;
  cudaGetDevice(&prev);
  if (prev != h->device) cudaSetDevice(h->device);
  return prev;
}
static void plat_leave(fe_handle* h, int prev) {
  if (prev >= 0 && prev != h->device) cudaSetDevice(prev);
}

static int plat_init(fe_handle* h) {
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess) { h->err = std::string("cudaGetDeviceCount: ") + cudaGetErrorString(e); return -10; }
  if (h->device < 0 || h->device >= ndev) { h->err = "fe_create: no such CUDA device"; return -10; }
  FeDevScope dev(h);
  cudaFree(0); // make sure the primary context of the device exists and is current
  CudaPlat* p = new CudaPlat();
  h->plat = p;
  e = cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&p->order_ev, cudaEventDisableTiming);
  if (e != cudaSuccess) { h->err = std::string("stream / event creation: ") + cudaGetErrorString(e); delete p; h->plat = nullptr; return -10; }
  return 0;
}

// module instance for this handle's (device, layout): found or loaded; the caller holds the device current
static int plat_module(fe_handle* h) {
  CudaPlat* p = (CudaPlat*)h->plat;
  if (p->km) return 0;
  std::lock_guard<std::mutex> lock(g_mu);
  std::string err;
  if (!drv_load(&err)) return fail(h, -10, err);
  for (FeModule* m : g_modules)
    if (m->device == h->device && memcmp(&m->lay, &h->lay, sizeof(FeLayout)) == 0) { p->km = m; ++m->users; return 0; }
  FeModule* m = new FeModule();
  m->device = h->device; m->lay = h->lay; m->users = 1;
  CUresult r = g_drv.ModuleLoadData(&m->mod, fe_cubin_start);
  if (r != CUDA_SUCCESS) { delete m; return fail(h, -10, "cuModuleLoadData(embedded sm_90a cubin): " + drv_err(r) + " (this library runs on H100 / sm_90a only)"); }
  struct { const char* name; CUfunction* f; } fn[] = {
      {"fe_sim_kernel", &m->f_sim}, {"fe_env_step_kernel", &m->f_step}, {"fe_env_ik_step_kernel", &m->f_ik_step}, {"fe_env_ctl_step_kernel", &m->f_ctl_step},
      {"fe_env_reset_kernel", &m->f_reset}, {"fe_order_kernel", &m->f_order}, {"fe_is_aligned_kernel", &m->f_aligned}, {"fe_dense_eval_kernel", &m->f_dense},
      {"fe_ctl_eval_kernel", &m->f_ctl_eval}};
  for (auto& f : fn) {
    r = g_drv.ModuleGetFunction(f.f, m->mod, f.name);
    if (r != CUDA_SUCCESS) { g_drv.ModuleUnload(m->mod); delete m; return fail(h, -10, std::string("cuModuleGetFunction ") + f.name + ": " + drv_err(r)); }
  }
  CUdeviceptr sym = 0;
  size_t bytes = 0;
  r = g_drv.ModuleGetGlobal(&sym, &bytes, m->mod, "fe_c_lay");
  if (r == CUDA_SUCCESS && bytes != sizeof(FeLayout)) r = CUDA_ERROR_INVALID_VALUE;
  if (r == CUDA_SUCCESS) r = g_drv.MemcpyHtoD(sym, &h->lay, sizeof(FeLayout));
  // the opt-in shared-memory limit is an attribute of the function: always the hardware maximum (227 KB), for the kernels that run in slices
  for (CUfunction f : {m->f_sim, m->f_step, m->f_ik_step, m->f_ctl_step, m->f_reset})
    if (r == CUDA_SUCCESS) r = g_drv.FuncSetAttribute(f, CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES, 227 * 1024);
  if (r != CUDA_SUCCESS) { g_drv.ModuleUnload(m->mod); delete m; return fail(h, -10, "module set-up (fe_c_lay / shared-memory limit): " + drv_err(r)); }
  g_modules.push_back(m);
  p->km = m;
  return 0;
}

static int plat_prepare(fe_handle* h) {
  CudaPlat* p = (CudaPlat*)h->plat;
  if (int rc = plat_module(h)) return rc;
  if (p->smem_sim) return 0;
  // warps (= envs) per block: as many as fit in 227 KB of shared memory, at most FE_MAX_WPB
  const size_t per_env = (size_t)(h->slice_words + FE_ENV_EXTRA_WORDS) * 4;
  int wpb = (int)((227 * 1024 - 1024) / per_env);
  if (wpb > FE_MAX_WPB) wpb = FE_MAX_WPB;
  if (wpb < 1) return fail(h, -11, "model does not fit in shared memory");
  p->wpb = wpb;
  p->nblocks = (h->N + wpb - 1) / wpb + FE_EXTRA_BLOCKS;
  {
    std::vector<int> init((size_t)p->nblocks * wpb, -1);
    for (int i = 0; i < h->N; ++i) init[i] = i;
    CUDA_OK(cudaMalloc((void**)&p->pred, sizeof(float) * (size_t)h->N));
    CUDA_OK(cudaMemset(p->pred, 0, sizeof(float) * (size_t)h->N));
    CUDA_OK(cudaMalloc((void**)&p->slots, sizeof(int) * init.size()));
    CUDA_OK(cudaMemcpy(p->slots, init.data(), sizeof(int) * init.size(), cudaMemcpyHostToDevice));
  }
  p->smem_env = per_env * wpb;
  const size_t N = h->N;
  p->out_bytes = N * (sizeof(float) * h->hs.obs_dim + sizeof(float) + sizeof(int32_t) * FE_INFO_DIM + 1);
  CUDA_OK(cudaMallocHost((void**)&p->pin_act, sizeof(float) * N * (h->hs.act_dim > 0 ? h->hs.act_dim : 1)));
  CUDA_OK(cudaMallocHost((void**)&p->pin_out, p->out_bytes + 64));
  p->smem_sim = (size_t)h->slice_words * 4 * wpb;
  return 0;
}
static void plat_fini(fe_handle* h) {
  CudaPlat* p = (CudaPlat*)h->plat;
  if (!p) return;
  FeDevScope dev(h);
  cudaDeviceSynchronize();
  if (p->pin_act) cudaFreeHost(p->pin_act);
  if (p->pin_out) cudaFreeHost(p->pin_out);
  if (p->slots) cudaFree(p->slots);
  if (p->pred) cudaFree(p->pred);
  if (p->order_ev) cudaEventDestroy(p->order_ev);
  if (p->stream) cudaStreamDestroy(p->stream);
  if (p->km) {
    std::lock_guard<std::mutex> lock(g_mu);
    if (--p->km->users == 0) {
      for (size_t i = 0; i < g_modules.size(); ++i)
        if (g_modules[i] == p->km) { g_modules.erase(g_modules.begin() + i); break; }
      g_drv.ModuleUnload(p->km->mod);
      delete p->km;
    }
  }
  delete p;
  h->plat = nullptr;
}
static void plat_sync(fe_handle* h) { FeDevScope dev(h); cudaDeviceSynchronize(); }
static void plat_copy_d2d(fe_handle* h, void* dst, const void* src, size_t n, void* stream) {
  FeDevScope dev(h);
  if (dst != src) cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToDevice, (cudaStream_t)stream);
}
static void note_stream(CudaPlat* p, cudaStream_t s) { p->last_stream = s; p->any_launch = true; }

static int launch(fe_handle* h, CUfunction f, unsigned grid, unsigned block, size_t smem, cudaStream_t stream, void** args) {
  DRV_OK(g_drv.LaunchKernel(f, grid, 1, 1, block, 1, 1, (unsigned)smem, (CUstream)stream, args, nullptr));
  return 0;
}
static int launch_step(fe_handle* h, const float* actions, float* reward, uint8_t* done, int32_t* info, cudaStream_t stream) {
  CudaPlat* p = (CudaPlat*)h->plat;
  int slice_words = h->slice_words;
  const int* slots = p->slots;
  // the IK and torque-controller step kernels take their control arguments right after es; all three have the same launch shape
  CUfunction f = p->km->f_step;
  void* control = nullptr;
  if (h->ctl.c) { f = p->km->f_ctl_step; control = &h->ctl; }
  else if (h->ik.c) { f = p->km->f_ik_step; control = &h->ik; }
  void* stock[] = {&h->st, &h->es, &h->dm, &h->ds, &h->cfg, &h->opt, &actions, &reward, &done, &info, &slice_words, &slots};
  void* with_control[] = {&h->st, &h->es, control, &h->dm, &h->ds, &h->cfg, &h->opt, &actions, &reward, &done, &info, &slice_words, &slots};
  if (int rc = launch(h, f, p->nblocks, 32 * p->wpb, p->smem_env, stream, control ? with_control : stock)) return rc;
  int N = h->N, nslots = p->nblocks * p->wpb;
  const int* stats = h->st.stats;
  int* order = h->st.order;
  void* b[] = {&N, &stats, &order, &p->slots, &nslots, &p->wpb, &p->pred};
  if (int rc = launch(h, p->km->f_order, 1, 1024, 0, stream, b)) return rc;
  note_stream(p, stream);
  return 0;
}
static int plat_run_sim(fe_handle* h, int nsub, int mode, void* stream) {
  FeDevScope dev(h);
  if (int rc = plat_prepare(h)) return rc;
  CudaPlat* p = (CudaPlat*)h->plat;
  int slice_words = h->slice_words;
  void* a[] = {&h->st, &h->dm, &h->opt, &nsub, &mode, &h->dbg, &slice_words};
  if (int rc = launch(h, p->km->f_sim, (h->N + p->wpb - 1) / p->wpb, 32 * p->wpb, p->smem_sim, (cudaStream_t)stream, a)) return rc;
  note_stream(p, (cudaStream_t)stream);
  return 0;
}
static int plat_run_reset(fe_handle* h, const uint8_t* mask, void* stream) {
  FeDevScope dev(h);
  if (int rc = plat_prepare(h)) return rc;
  CudaPlat* p = (CudaPlat*)h->plat;
  int slice_words = h->slice_words;
  void* a[] = {&h->st, &h->es, &h->dm, &h->ds, &h->cfg, &h->opt, &mask, &slice_words};
  if (int rc = launch(h, p->km->f_reset, (h->N + p->wpb - 1) / p->wpb, 32 * p->wpb, p->smem_env, (cudaStream_t)stream, a)) return rc;
  note_stream(p, (cudaStream_t)stream);
  return 0;
}
static int plat_run_step(fe_handle* h, const float* actions, float* reward, uint8_t* done, int32_t* info, void* stream) {
  FeDevScope dev(h);
  if (int rc = plat_prepare(h)) return rc;
  return launch_step(h, actions, reward, done, info, (cudaStream_t)stream);
}
static int plat_step_host(fe_handle* h, const float* actions, float* obs, float* reward, uint8_t* done, int32_t* info) {
  FeDevScope dev(h);
  if (int rc = plat_prepare(h)) return rc;
  CudaPlat* p = (CudaPlat*)h->plat;
  const size_t N = h->N, ab = sizeof(float) * N * fe_action_dim(h), ob = sizeof(float) * N * h->hs.obs_dim, rb = sizeof(float) * N, ib = sizeof(int32_t) * N * FE_INFO_DIM;
  memcpy(p->pin_act, actions, ab);
  // The private stream is ordered behind whatever the caller last launched for this handle on another stream
  // (fe_sim_forward, fe_env_reset ...) with an event, not with a device-wide synchronisation.
  if (p->any_launch && p->last_stream != p->stream) {
    CUDA_OK(cudaEventRecord(p->order_ev, p->last_stream));
    CUDA_OK(cudaStreamWaitEvent(p->stream, p->order_ev, 0));
  }
  CUDA_OK(cudaMemcpyAsync(h->dev_act, p->pin_act, ab, cudaMemcpyHostToDevice, p->stream));
  if (int rc = launch_step(h, (const float*)h->dev_act, (float*)h->dev_rew, (uint8_t*)h->dev_done, (int32_t*)h->dev_info, p->stream)) return rc;
  unsigned char* o = p->pin_out;
  CUDA_OK(cudaMemcpyAsync(o, h->es.obs, ob, cudaMemcpyDeviceToHost, p->stream));
  CUDA_OK(cudaMemcpyAsync(o + ob, h->dev_rew, rb, cudaMemcpyDeviceToHost, p->stream));
  CUDA_OK(cudaMemcpyAsync(o + ob + rb, h->dev_info, ib, cudaMemcpyDeviceToHost, p->stream));
  CUDA_OK(cudaMemcpyAsync(o + ob + rb + ib, h->dev_done, N, cudaMemcpyDeviceToHost, p->stream));
  CUDA_OK(cudaStreamSynchronize(p->stream));
  if (obs) memcpy(obs, o, ob);
  if (reward) memcpy(reward, o + ob, rb);
  if (info) memcpy(info, o + ob + rb, ib);
  if (done) memcpy(done, o + ob + rb + ib, N);
  return 0;
}
// device buffers of one host-side evaluation call (fe_is_aligned, fe_dense_eval, fe_ctl_eval), freed when it goes out of scope
struct DevBufs {
  std::vector<void*> bufs;
  bool bad = false; // an allocation or an upload failed
  // a device copy of `bytes` bytes at `src`, or an uninitialised output buffer when src is null
  void* up(const void* src, size_t bytes) {
    void* d = nullptr;
    if (cudaMalloc(&d, bytes ? bytes : 8) != cudaSuccess) { bad = true; return nullptr; }
    bufs.push_back(d);
    if (src && cudaMemcpy(d, src, bytes, cudaMemcpyHostToDevice) != cudaSuccess) bad = true;
    return d;
  }
  ~DevBufs() { for (void* b : bufs) cudaFree(b); }
};

static int plat_is_aligned(fe_handle* h, int n, const double* p1, const double* m1, const double* p2, const double* m2, const double* angles,
                           const int32_t* nangles, const double* thr, uint8_t* aligned, double* tq) {
  FeDevScope dev(h);
  if (int rc = plat_prepare(h)) return rc;
  CudaPlat* p = (CudaPlat*)h->plat;
  // cos/sin of the allowed angles are evaluated on the host in float64 (the same libm the reference's numpy uses)
  std::vector<double> cs(4 * (size_t)n), sn(4 * (size_t)n);
  for (size_t i = 0; i < 4 * (size_t)n; ++i) { double a = angles[i] / 180 * 3.141592653589793; cs[i] = cos(a); sn[i] = sin(a); }
  const size_t N = n;
  DevBufs b;
  void* d_p1 = b.up(p1, 24 * N);
  void* d_m1 = b.up(m1, 72 * N);
  void* d_p2 = b.up(p2, 24 * N);
  void* d_m2 = b.up(m2, 72 * N);
  void* d_cs = b.up(cs.data(), 32 * N);
  void* d_sn = b.up(sn.data(), 32 * N);
  void* d_na = b.up(nangles, 4 * N);
  void* d_thr = b.up(thr, 32 * N);
  void* d_al = b.up(nullptr, N);
  void* d_tq = b.up(nullptr, 32 * N);
  if (b.bad) return fail(h, -2, "fe_is_aligned: device allocation / upload failed");
  void* a[] = {&n, &d_p1, &d_m1, &d_p2, &d_m2, &d_cs, &d_sn, &d_na, &d_thr, &d_al, &d_tq};
  if (int rc = launch(h, p->km->f_aligned, (n + 127) / 128, 128, 0, nullptr, a)) return rc;
  if (cudaMemcpy(aligned, d_al, N, cudaMemcpyDeviceToHost) != cudaSuccess || cudaMemcpy(tq, d_tq, 32 * N, cudaMemcpyDeviceToHost) != cudaSuccess)
    return fail(h, -10, std::string("fe_is_aligned: ") + cudaGetErrorString(cudaGetLastError()));
  return 0;
}
static int plat_dense_eval(fe_handle* h, const fe_dense_config* dc, const fe_dense_recipe* rc, const double* thr, int n_goal, int n_episodes, const int32_t* first,
                           const int32_t* count, int n_records, int nsite, int npart, int act_dim, const double* spos, const double* smat, const double* ppos,
                           const uint8_t* touch, const uint8_t* reset, const uint8_t* connected, const double* ac, double* reward, uint8_t* done, double* info) {
  FeDevScope dev(h);
  if (int rc_ = plat_prepare(h)) return rc_;
  CudaPlat* p = (CudaPlat*)h->plat;
  const size_t R = n_records, E = n_episodes;
  DevBufs b;
  void* d_c = b.up(dc, sizeof(fe_dense_config));
  void* d_rc = b.up(rc, sizeof(fe_dense_recipe));
  void* d_thr = b.up(thr, 32);
  void* d_first = b.up(first, 4 * E);
  void* d_count = b.up(count, 4 * E);
  void* d_spos = b.up(spos, 24 * R * nsite);
  void* d_smat = b.up(smat, 72 * R * nsite);
  void* d_ppos = b.up(ppos, 24 * R * npart);
  void* d_touch = b.up(touch, R * npart);
  void* d_reset = b.up(reset, R);
  void* d_conn = b.up(connected, R);
  void* d_ac = b.up(ac, 8 * R * act_dim);
  void* d_rew = b.up(nullptr, 8 * R);
  void* d_done = b.up(nullptr, R);
  void* d_info = b.up(nullptr, 8 * R * FE_DENSE_INFO);
  if (b.bad) return fail(h, -2, "fe_dense_eval: device allocation / upload failed");
  void* a[] = {&d_c, &d_rc, &d_thr, &n_goal, &n_episodes, &d_first, &d_count, &nsite, &npart, &act_dim, &d_spos, &d_smat, &d_ppos, &d_touch, &d_reset, &d_conn, &d_ac,
               &d_rew, &d_done, &d_info};
  if (int rc_ = launch(h, p->km->f_dense, (n_episodes + 31) / 32, 32, 0, nullptr, a)) return rc_;
  if (cudaMemcpy(reward, d_rew, 8 * R, cudaMemcpyDeviceToHost) != cudaSuccess || cudaMemcpy(done, d_done, R, cudaMemcpyDeviceToHost) != cudaSuccess ||
      cudaMemcpy(info, d_info, 8 * R * FE_DENSE_INFO, cudaMemcpyDeviceToHost) != cudaSuccess)
    return fail(h, -10, std::string("fe_dense_eval: ") + cudaGetErrorString(cudaGetLastError()));
  return 0;
}
static int plat_ctl_eval(fe_handle* h, const fe_ctl_config* cc, int n_episodes, const int32_t* first, const int32_t* count, int n_records, const uint8_t* reset,
                         const uint8_t* policy_step, const double* action, const FeCtlIn* in, double* torques) {
  FeDevScope dev(h);
  if (int rc_ = plat_prepare(h)) return rc_;
  CudaPlat* p = (CudaPlat*)h->plat;
  const size_t R = n_records, E = n_episodes;
  DevBufs b;
  void* d_c = b.up(cc, sizeof(fe_ctl_config));
  void* d_first = b.up(first, 4 * E);
  void* d_count = b.up(count, 4 * E);
  void* d_reset = b.up(reset, R);
  void* d_pol = b.up(policy_step, R);
  void* d_act = b.up(action, 56 * R);
  void* d_in = b.up(in, sizeof(FeCtlIn) * R);
  void* d_tau = b.up(nullptr, 56 * R);
  if (b.bad) return fail(h, -2, "fe_ctl_eval: device allocation / upload failed");
  void* a[] = {&d_c, &n_episodes, &d_first, &d_count, &d_reset, &d_pol, &d_act, &d_in, &d_tau};
  if (int rc_ = launch(h, p->km->f_ctl_eval, (n_episodes + 31) / 32, 32, 0, nullptr, a)) return rc_;
  if (cudaMemcpy(torques, d_tau, 56 * R, cudaMemcpyDeviceToHost) != cudaSuccess) return fail(h, -10, std::string("fe_ctl_eval: ") + cudaGetErrorString(cudaGetLastError()));
  return 0;
}
