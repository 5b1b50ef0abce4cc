// fe_warp.h -- one-warp-per-environment execution model.
//
// Every physics routine is written as a sequence of *lane regions*: inside LANES_BEGIN/LANES_END each of the 32
// lanes runs the body with its own `lane`; lanes talk to each other only through the warp's shared-memory slice and
// only across a region boundary (LANES_END is a __syncwarp()).  Reductions / ballots are done between regions on a
// scratch array.  On sm_90a this compiles to straight SIMT code (the lane loop has one trip).  The same source also
// builds with a host compiler (FE_EMULATE) where a region is a 32-trip loop -- used ONLY by the CPU test harness
// (tests/emu) so kernel logic can be exercised without a GPU; the product never loads that build.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__) && !defined(FE_EMULATE)
#define FE_DEVICE_BUILD 1
#define FE_HD __device__ __forceinline__
#define FE_FN __device__ __noinline__
#define FE_HDN __device__ __noinline__
#define FE_BOTH __host__ __device__ __forceinline__
#define FE_MEMBER __device__ __forceinline__ /* member functions of device-side helper structs */
#define LANES_BEGIN { const int lane = (int)(threadIdx.x & 31u); (void)lane; {
#define LANES_END } } __syncwarp();
// register-only region: touches lane-private values only, so no barrier is needed after it
#define REGS_BEGIN { const int lane = (int)(threadIdx.x & 31u); (void)lane; {
#define REGS_END } }
#define FE_LDG(p) __ldg(p)
#define FE_SYNC __syncwarp()
#define FE_BLOCK_SYNC __syncthreads()
#else
#define FE_DEVICE_BUILD 0
#define FE_HD static inline
#define FE_FN static
#define FE_HDN static
#define FE_BOTH static inline
#define FE_MEMBER inline
#define LANES_BEGIN for (int lane = 0; lane < 32; ++lane) { {
#define LANES_END } }
#define REGS_BEGIN LANES_BEGIN
#define REGS_END LANES_END
#define FE_LDG(p) (*(p))
#define FE_SYNC ((void)0)
#define FE_BLOCK_SYNC ((void)0)
#endif

// Cycle counters of the per-call statistics: FE_TICK_START starts the clock in a function, FE_TICK(ctr, slot, ...) adds the
// cycles since the previous tick (clock64 / 16, by lane 0) to ctr[slot] for every slot listed and restarts the clock.  The
// emulated build has no clock: its counters stay 0.
#if FE_DEVICE_BUILD
#define FE_TICK_START long long t0_ = clock64();
#define FE_TICK(ctr, ...) { const long long t1_ = clock64(); \
    if ((threadIdx.x & 31u) == 0) { const int d_ = (int)((t1_ - t0_) >> 4), s_[] = {__VA_ARGS__}; for (int i_ : s_) (ctr)[i_] += d_; } t0_ = t1_; }
#else
#define FE_TICK_START
#define FE_TICK(ctr, ...)
#endif

// sum of scr[0..31] with a fixed butterfly order (identical result on every lane and in the emulation build)
FE_HD float fe_sum32(const float* scr) {
#if FE_DEVICE_BUILD
  float v = scr[threadIdx.x & 31u];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncwarp();
  return v;
#else
  float t[32];
  for (int i = 0; i < 32; ++i) t[i] = scr[i];
  for (int o = 16; o > 0; o >>= 1) {
    float u[32];
    for (int i = 0; i < 32; ++i) u[i] = t[i] + t[i ^ o];
    for (int i = 0; i < 32; ++i) t[i] = u[i];
  }
  return t[0];
#endif
}
// bit i set iff flag[i] != 0
FE_HD unsigned fe_ballot32(const int* flag) {
#if FE_DEVICE_BUILD
  unsigned r = __ballot_sync(0xffffffffu, flag[threadIdx.x & 31u] != 0);
  __syncwarp();
  return r;
#else
  unsigned r = 0;
  for (int i = 0; i < 32; ++i) r |= (flag[i] != 0 ? 1u : 0u) << i;
  return r;
#endif
}


// ---- lane-private values that live across regions (registers on the device, one slot per lane in the emulation),
// and the collectives applied to them BETWEEN regions
#if FE_DEVICE_BUILD
#define FE_PRIV(T, name) T name
#define FE_PRIVA(T, name, n) T name[n]
#define PV(name) name
#define PV_ALL(name) name /* the private value as a collective operand */
#define FE_GSUM8(name) do { name += __shfl_xor_sync(0xffffffffu, name, 1); name += __shfl_xor_sync(0xffffffffu, name, 2); name += __shfl_xor_sync(0xffffffffu, name, 4); } while (0)
#define FE_GSUM8_ARR(name, n) do { _Pragma("unroll") for (int k_ = 0; k_ < (n); ++k_) FE_GSUM8(name[k_]); } while (0)
#define FE_ANY(name) (__any_sync(0xffffffffu, (name) != 0) != 0)
// sums over the lane's 4-lane unit, or over its 8-lane pair of units where `wide` is set (per-lane flag, equal within a group)
#define FE_GSUMV(name, wide) do { name += __shfl_xor_sync(0xffffffffu, name, 1); name += __shfl_xor_sync(0xffffffffu, name, 2); \
    const float t_gs_ = __shfl_xor_sync(0xffffffffu, name, 4); if (wide) name += t_gs_; } while (0)
#define FE_GSUMV_ARRN(name, n, used, wide) do { _Pragma("unroll") for (int k_ = 0; k_ < (used); ++k_) FE_GSUMV(name[k_], wide); } while (0)
#define FE_WSUM(name) do { _Pragma("unroll") for (int o_ = 16; o_ > 0; o_ >>= 1) name += __shfl_xor_sync(0xffffffffu, name, o_); } while (0)
#define FE_SHFL(dst, src, idx) do { dst = __shfl_sync(0xffffffffu, src, (idx)); } while (0)
#define FE_SHFLA(dst, arr, elem, idx) do { dst = __shfl_sync(0xffffffffu, arr[elem], (idx)); } while (0)
#define FE_UNI(name) (name) /* a private value known to be equal on all lanes (after a collective) */
// lane-indexed shuffle (every lane names its own source lane), ballot of a private predicate, and for every lane the lowest
// lane that holds the same key
#define FE_SHFLV(dst, src, idx) do { dst = __shfl_sync(0xffffffffu, src, (idx)); } while (0)
#define FE_BALLOTP(name) __ballot_sync(0xffffffffu, (name) != 0)
#define FE_MATCH_LEADER(dst, key) do { dst = __ffs(__match_any_sync(0xffffffffu, (key))) - 1; } while (0)
#else
#define FE_PRIV(T, name) T name[32]
#define FE_PRIVA(T, name, n) T name[32][n]
#define PV(name) name[lane]
#define PV_ALL(name) name
static inline void fe_emu_gsum8(float* a, int stride) {
  for (int o = 1; o < 8; o <<= 1) {
    float t[32];
    for (int i = 0; i < 32; ++i) t[i] = a[i * stride] + a[(i ^ o) * stride];
    for (int i = 0; i < 32; ++i) a[i * stride] = t[i];
  }
}
#define FE_GSUM8(name) fe_emu_gsum8(name, 1)
static inline void fe_emu_gsumv(float* a, int stride, const int* wide) {
  for (int o = 1; o < 8; o <<= 1) {
    float t[32];
    for (int i = 0; i < 32; ++i) t[i] = (o < 4 || wide[i]) ? a[i * stride] + a[(i ^ o) * stride] : a[i * stride];
    for (int i = 0; i < 32; ++i) a[i * stride] = t[i];
  }
}
#define FE_GSUMV_ARRN(name, n, used, wide) do { for (int k_ = 0; k_ < (used); ++k_) fe_emu_gsumv(&name[0][k_], (n), wide); } while (0)
#define FE_GSUM8_ARR(name, n) do { for (int k_ = 0; k_ < (n); ++k_) fe_emu_gsum8(&name[0][k_], (n)); } while (0)
static inline bool fe_emu_any(const int* a) { for (int i = 0; i < 32; ++i) if (a[i]) return true; return false; }
#define FE_ANY(name) fe_emu_any(name)
static inline void fe_emu_wsum(float* a) {
  for (int o = 16; o > 0; o >>= 1) {
    float t[32];
    for (int i = 0; i < 32; ++i) t[i] = a[i] + a[i ^ o];
    for (int i = 0; i < 32; ++i) a[i] = t[i];
  }
}
#define FE_WSUM(name) fe_emu_wsum(name)
#define FE_SHFL(dst, src, idx) do { const float t_shfl_ = src[(idx)]; for (int i_ = 0; i_ < 32; ++i_) dst[i_] = t_shfl_; } while (0)
#define FE_SHFLA(dst, arr, elem, idx) do { const float t_shfl_ = arr[(idx)][(elem)]; for (int i_ = 0; i_ < 32; ++i_) dst[i_] = t_shfl_; } while (0)
#define FE_UNI(name) (name[0])
#define FE_SHFLV(dst, src, idx) do { float t_sv_[32]; for (int i_ = 0; i_ < 32; ++i_) t_sv_[i_] = src[idx[i_] & 31]; for (int i_ = 0; i_ < 32; ++i_) dst[i_] = t_sv_[i_]; } while (0)
static inline unsigned fe_emu_ballotp(const int* a) { unsigned r = 0; for (int i = 0; i < 32; ++i) r |= (a[i] != 0 ? 1u : 0u) << i; return r; }
#define FE_BALLOTP(name) fe_emu_ballotp(name)
#define FE_MATCH_LEADER(dst, key) do { for (int i_ = 0; i_ < 32; ++i_) { int l_ = i_; for (int j_ = 0; j_ < i_; ++j_) if (key[j_] == key[i_]) { l_ = j_; break; } dst[i_] = l_; } } while (0)
#endif

// ---------------------------------------------------------------- small vector math (fp32)
FE_HD void v3set(float* r, float a, float b, float c) { r[0] = a; r[1] = b; r[2] = c; }
FE_HD void v3cpy(float* r, const float* a) { r[0] = a[0]; r[1] = a[1]; r[2] = a[2]; }
FE_HD void v3add(float* r, const float* a, const float* b) { r[0] = a[0] + b[0]; r[1] = a[1] + b[1]; r[2] = a[2] + b[2]; }
FE_HD void v3sub(float* r, const float* a, const float* b) { r[0] = a[0] - b[0]; r[1] = a[1] - b[1]; r[2] = a[2] - b[2]; }
FE_HD void v3madd(float* r, const float* a, const float* b, float s) { r[0] = a[0] + s * b[0]; r[1] = a[1] + s * b[1]; r[2] = a[2] + s * b[2]; }
FE_HD float v3dot(const float* a, const float* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
FE_HD void v3cross(float* r, const float* a, const float* b) {
  float x = a[1] * b[2] - a[2] * b[1], y = a[2] * b[0] - a[0] * b[2], z = a[0] * b[1] - a[1] * b[0];
  r[0] = x; r[1] = y; r[2] = z;
}
FE_HD float v3norm(const float* a) { return sqrtf(v3dot(a, a)); }
FE_HD float v3normalize(float* a) {
  float n = v3norm(a);
  if (n < 1e-20f) { a[0] = 1.f; a[1] = 0.f; a[2] = 0.f; return 0.f; }
  float s = 1.0f / n;
  a[0] *= s; a[1] *= s; a[2] *= s;
  return n;
}
// r = R a (R row-major 3x3) ; rt = R^T a
FE_HD void m3mulv(float* r, const float* R, const float* a) {
  float x = R[0] * a[0] + R[1] * a[1] + R[2] * a[2], y = R[3] * a[0] + R[4] * a[1] + R[5] * a[2], z = R[6] * a[0] + R[7] * a[1] + R[8] * a[2];
  r[0] = x; r[1] = y; r[2] = z;
}
FE_HD void m3tmulv(float* r, const float* R, const float* a) {
  float x = R[0] * a[0] + R[3] * a[1] + R[6] * a[2], y = R[1] * a[0] + R[4] * a[1] + R[7] * a[2], z = R[2] * a[0] + R[5] * a[1] + R[8] * a[2];
  r[0] = x; r[1] = y; r[2] = z;
}
FE_HD void m3mul(float* C, const float* A, const float* B) {
  float t[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) t[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
  for (int k = 0; k < 9; ++k) C[k] = t[k];
}
FE_HD void qmul(float* r, const float* a, const float* b) {
  float w = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  float x = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  float y = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1];
  float z = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
  r[0] = w; r[1] = x; r[2] = y; r[3] = z;
}
FE_HD void qnormalize(float* q) {
  float n = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  if (n < 1e-20f) { q[0] = 1.f; q[1] = q[2] = q[3] = 0.f; return; }
  float s = 1.0f / n;
  q[0] *= s; q[1] *= s; q[2] *= s; q[3] *= s;
}
FE_HD void q2mat(float* R, const float* q) {
  float w = q[0], x = q[1], y = q[2], z = q[3];
  R[0] = w * w + x * x - y * y - z * z; R[1] = 2.f * (x * y - w * z); R[2] = 2.f * (x * z + w * y);
  R[3] = 2.f * (x * y + w * z); R[4] = w * w - x * x + y * y - z * z; R[5] = 2.f * (y * z - w * x);
  R[6] = 2.f * (x * z - w * y); R[7] = 2.f * (y * z + w * x); R[8] = w * w - x * x - y * y + z * z;
}
// symmetric 3x3 stored xx yy zz xy xz yz, r = I a
FE_HD void sym3mulv(float* r, const float* I, const float* a) {
  float x = I[0] * a[0] + I[3] * a[1] + I[4] * a[2], y = I[3] * a[0] + I[1] * a[1] + I[5] * a[2], z = I[4] * a[0] + I[5] * a[1] + I[2] * a[2];
  r[0] = x; r[1] = y; r[2] = z;
}
// rotate a symmetric tensor: out = R I R^T
FE_HD void sym3rot(float* out, const float* R, const float* I) {
  float A[9] = {I[0], I[3], I[4], I[3], I[1], I[5], I[4], I[5], I[2]}, T[9], Rt[9] = {R[0], R[3], R[6], R[1], R[4], R[7], R[2], R[5], R[8]};
  m3mul(T, R, A);
  m3mul(A, T, Rt);
  out[0] = A[0]; out[1] = A[4]; out[2] = A[8]; out[3] = A[1]; out[4] = A[2]; out[5] = A[5];
}
// compact spatial inertia about a reference point P: I = {m, h[3] = m (c - P), Io[6]}; motion V = [w; vP]; F = [n_P; f]
FE_HD void inert_mulv(float* F, const float* I, const float* V) {
  float t[3], u[3];
  sym3mulv(t, I + 4, V);
  v3cross(u, I + 1, V + 3);
  F[0] = t[0] + u[0]; F[1] = t[1] + u[1]; F[2] = t[2] + u[2];
  v3cross(u, I + 1, V);
  F[3] = I[0] * V[3] - u[0]; F[4] = I[0] * V[4] - u[1]; F[5] = I[0] * V[5] - u[2];
}
FE_HD void crossm(float* r, const float* V, const float* S) { /* V x_m S */
  float a[3], b[3], c[3];
  v3cross(a, V, S); v3cross(b, V, S + 3); v3cross(c, V + 3, S);
  r[0] = a[0]; r[1] = a[1]; r[2] = a[2]; r[3] = b[0] + c[0]; r[4] = b[1] + c[1]; r[5] = b[2] + c[2];
}
FE_HD void crossf(float* r, const float* V, const float* F) { /* V x* F */
  float a[3], b[3], c[3];
  v3cross(a, V, F); v3cross(b, V + 3, F + 3); v3cross(c, V, F + 3);
  r[0] = a[0] + b[0]; r[1] = a[1] + b[1]; r[2] = a[2] + b[2]; r[3] = c[0]; r[4] = c[1]; r[5] = c[2];
}
FE_HD float dot6(const float* a, const float* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2] + a[3] * b[3] + a[4] * b[4] + a[5] * b[5]; }
