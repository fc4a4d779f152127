// A test double of libcudart.so.12 — TEST INFRASTRUCTURE, never linked or shipped with the product.
//
// Purpose: the engine (llmlb_b200/csrc/engine.cu) is half host code — request queue, iteration-level scheduler, page
// allocator, preemption, timeouts, event delivery, the C ABI's locking — and until now none of it could run where
// there is no GPU, so none of it had ever seen a sanitizer.  Preloading this library under the UNMODIFIED product
// libllmlb_b200.so makes every CUDA runtime call a host-side no-op: "device" memory is zero-filled host memory
// (anonymous shared memory, so that the IPC-handle calls work across processes like CUDA IPC does between ranks), copies
// are memcpy, kernel launches and graph launches do nothing, events complete at once.  No arithmetic happens — every
// sampled token id is whatever the zero-filled buffers hold (0) — so this says NOTHING about the kernels or about
// parity; it exercises counts, ordering, resource accounting and thread safety of the host side, at a step rate no
// GPU would reach.  The product still refuses to start without a real device: nothing here is reachable unless a test
// sets LD_PRELOAD (tests/test_engine_host_logic_cpu.py).
//
// Build: g++ -shared -fPIC -I/usr/local/cuda/include fake_cudart.cpp -Wl,-soname,libcudart.so.12
//            -Wl,--version-script=fake_cudart.map -o libcudart.so.12
#include <cuda_runtime_api.h>

#ifndef _GNU_SOURCE
#define _GNU_SOURCE
#endif
#include <fcntl.h>
#include <sys/mman.h>
#include <unistd.h>

#include <atomic>
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>

namespace {
struct Alloc { int fd = -1; size_t size = 0; bool dirty = false; };   // dirty: something was copied / set into it
std::mutex g_mu;
std::map<void*, Alloc> g_allocs;
std::map<void*, size_t> g_opened;
std::map<const void*, size_t> g_smem_optin;          // cudaFuncAttributeMaxDynamicSharedMemorySize per kernel function
std::map<const void*, std::string> g_kernels;      // host stub -> mangled device name (__cudaRegisterFunction)
std::atomic<unsigned long long> g_seq{0};
std::atomic<size_t> g_allocated{0};
std::atomic<uint64_t> g_launches{0};
std::atomic<uint64_t> g_tmaps{0};
struct Ev { double t_ms; };
double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
thread_local struct { dim3 grid, block; size_t smem; void* stream; } g_cfg;
// Stream capture (thread-local mode, as the engine uses it): between Begin and End the capturing thread may only enqueue
// work; synchronous calls are refused like the driver refuses them (cudaErrorStreamCaptureUnsupported) and poison the capture.
thread_local bool g_capturing = false, g_capture_poisoned = false;
inline bool illegal_in_capture(const char* what) {
  if (!g_capturing) return false;
  g_capture_poisoned = true;
  fprintf(stderr, "fake cudart: %s during stream capture\n", what);
  return true;
}
// cuTensorMapEncodeTiled stand-in.  The descriptor stays opaque (zeroed), but the ARGUMENTS are checked against the rules
// the driver documents for the call, so that a geometry whose tensor map the real driver would refuse fails here too:
// rank 1..5, 16-byte aligned base, dims in [1, 2^32], strides multiples of 16 below 2^40, box dims in [1, 256], element
// strides in [1, 8], inner box extent a multiple of 16 bytes and within the swizzle span (32 / 64 / 128 bytes).
int fake_encode_tiled(void* map, int data_type, unsigned rank, void* base, const unsigned long long* dims, const unsigned long long* strides,
                      const unsigned* box, const unsigned* elem_strides, int interleave, int swizzle, int, int) {
  static const int kElemBytes[] = {1, 2, 4, 4, 8, 8, 2, 4, 8, 2, 4, 4, 4};   // CUtensorMapDataType order: u8,u16,u32,i32,u64,i64,f16,f32,f64,bf16,...
  const int eb = (data_type >= 0 && data_type < int(sizeof kElemBytes / sizeof *kElemBytes)) ? kElemBytes[data_type] : 0;
  bool ok = map && eb && rank >= 1 && rank <= 5 && base && (reinterpret_cast<uintptr_t>(base) & 15) == 0 && dims && box && elem_strides && interleave == 0;
  for (unsigned i = 0; ok && i < rank; ++i) {
    ok = dims[i] >= 1 && dims[i] <= (1ull << 32) && box[i] >= 1 && box[i] <= 256 && elem_strides[i] >= 1 && elem_strides[i] <= 8;
    if (ok && i + 1 < rank) ok = strides && strides[i] % 16 == 0 && strides[i] < (1ull << 40) && strides[i] > 0;
  }
  if (ok) {
    const unsigned long long inner = (unsigned long long)box[0] * unsigned(eb);
    const unsigned long long span = swizzle == 1 ? 32 : swizzle == 2 ? 64 : swizzle >= 3 ? 128 : ~0ull;   // CU_TENSOR_MAP_SWIZZLE_{32,64,128}B(+ATOM variants)
    ok = inner % 16 == 0 && inner <= span && swizzle >= 0 && swizzle <= 6;
  }
  if (!ok) {
    fprintf(stderr, "fake cudart: cuTensorMapEncodeTiled would be refused (type %d rank %u base %p box0 %u swizzle %d)\n", data_type, rank, base,
            box ? box[0] : 0u, swizzle);
    return 1;   // CUDA_ERROR_INVALID_VALUE
  }
  memset(map, 0, 128);
  ++g_tmaps;
  return 0;
}
}  // namespace

extern "C" {
static void mark_dirty(void* d);
static bool smem_allowed(const void* fn, size_t smem);
static bool config_allowed(dim3 g, dim3 b);
cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
cudaError_t cudaSetDevice(int) { return cudaSuccess; }
cudaError_t cudaDeviceSynchronize(void) { return illegal_in_capture("cudaDeviceSynchronize") ? cudaErrorStreamCaptureUnsupported : cudaSuccess; }
// launches made with <<<...>>> report their error through cudaGetLastError (returned once, then cleared)
thread_local cudaError_t g_last_error = cudaSuccess;
cudaError_t cudaGetLastError(void) { const cudaError_t e = g_last_error; g_last_error = cudaSuccess; return e; }
const char* cudaGetErrorString(cudaError_t) { return "fake cudart"; }
// "Device" allocations are anonymous shared memory (memfd) so that another PROCESS can map them through the IPC-handle
// calls, the way tensor-parallel ranks map each other's exchange regions: zero-filled like calloc, nothing named in
// /dev/shm, gone with the process however it dies.
cudaError_t cudaMalloc(void** p, size_t n) {
  if (illegal_in_capture("cudaMalloc")) return cudaErrorStreamCaptureUnsupported;
  if (!n) n = 1;
  const int fd = memfd_create("fakecuda", 0);
  void* m = MAP_FAILED;
  if (fd >= 0 && ftruncate(fd, off_t(n)) == 0) m = mmap(nullptr, n, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
  if (m == MAP_FAILED) { if (fd >= 0) close(fd); return cudaErrorMemoryAllocation; }
  { std::lock_guard<std::mutex> lk(g_mu); g_allocs[m] = Alloc{fd, n}; }
  *p = m;
  g_allocated += n;
  return cudaSuccess;
}
cudaError_t cudaFree(void* p) {
  if (!p) return cudaSuccess;
  Alloc a;
  {
    std::lock_guard<std::mutex> lk(g_mu);
    auto it = g_allocs.find(p);
    if (it == g_allocs.end()) return cudaErrorInvalidValue;
    a = it->second;
    g_allocs.erase(it);
  }
  munmap(p, a.size);
  close(a.fd);
  g_allocated -= a.size;
  return cudaSuccess;
}
cudaError_t cudaHostAlloc(void** p, size_t n, unsigned) { *p = calloc(1, n ? n : 1); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
cudaError_t cudaFreeHost(void* p) { free(p); return cudaSuccess; }
cudaError_t cudaMemGetInfo(size_t* fr, size_t* total) {
  *total = size_t(183) << 30;
  *fr = *total - (g_allocated.load() < *total ? g_allocated.load() : 0);
  return cudaSuccess;
}
cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { if (illegal_in_capture("cudaMemcpy")) return cudaErrorStreamCaptureUnsupported; if (d && s && n) { mark_dirty(d); memmove(d, s, n); } return cudaSuccess; }
cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t) { if (d && s && n) { mark_dirty(d); memmove(d, s, n); } return cudaSuccess; }
cudaError_t cudaMemcpy2D(void* d, size_t dp, const void* s, size_t sp, size_t w, size_t h, cudaMemcpyKind) {
  mark_dirty(d);
  for (size_t r = 0; r < h; ++r) memmove(static_cast<char*>(d) + r * dp, static_cast<const char*>(s) + r * sp, w);
  return cudaSuccess;
}
// the symbol argument is the host shadow of the __device__ / __constant__ variable: same size, harmless to write
cudaError_t cudaMemcpyToSymbol(const void* sym, const void* s, size_t n, size_t off, cudaMemcpyKind) {
  if (sym && s && n) memmove(static_cast<char*>(const_cast<void*>(sym)) + off, s, n);
  return cudaSuccess;
}
// Zeroing a whole allocation that nothing has written yet is skipped (it is zero pages already): an engine with 8B- or
// 70B-shaped weights then costs address space, not memory — nothing ever touches the weights here.
static bool untouched_whole_alloc(void* d, size_t n) {
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_allocs.find(d);
  return it != g_allocs.end() && it->second.size == n && !it->second.dirty;
}
static void mark_dirty(void* d) {            // d points into a device allocation (or into host memory: then nothing to do)
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_allocs.upper_bound(d);
  if (it == g_allocs.begin()) return;
  --it;
  if (static_cast<char*>(d) < static_cast<char*>(it->first) + it->second.size) it->second.dirty = true;
}
static void fake_memset(void* d, int v, size_t n) {
  if (!d || !n || (v == 0 && untouched_whole_alloc(d, n))) return;
  mark_dirty(d);
  memset(d, v, n);
}
cudaError_t cudaMemset(void* d, int v, size_t n) { if (illegal_in_capture("cudaMemset")) return cudaErrorStreamCaptureUnsupported; fake_memset(d, v, n); return cudaSuccess; }
cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t) { fake_memset(d, v, n); return cudaSuccess; }
cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = static_cast<cudaStream_t>(malloc(8)); return cudaSuccess; }
cudaError_t cudaStreamDestroy(cudaStream_t s) { free(s); return cudaSuccess; }
cudaError_t cudaStreamSynchronize(cudaStream_t) { return illegal_in_capture("cudaStreamSynchronize") ? cudaErrorStreamCaptureUnsupported : cudaSuccess; }
cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = reinterpret_cast<cudaEvent_t>(new Ev{now_ms()}); return cudaSuccess; }
cudaError_t cudaEventDestroy(cudaEvent_t e) { delete reinterpret_cast<Ev*>(e); return cudaSuccess; }
cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t) { reinterpret_cast<Ev*>(e)->t_ms = now_ms(); return cudaSuccess; }
cudaError_t cudaEventSynchronize(cudaEvent_t) { return illegal_in_capture("cudaEventSynchronize") ? cudaErrorStreamCaptureUnsupported : cudaSuccess; }
cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b) {
  const double d = reinterpret_cast<Ev*>(b)->t_ms - reinterpret_cast<Ev*>(a)->t_ms;
  *ms = float(d > 0 ? d : 0.001);
  return cudaSuccess;
}
cudaError_t cudaStreamBeginCapture(cudaStream_t, cudaStreamCaptureMode) {
  if (g_capturing) return cudaErrorIllegalState;
  g_capturing = true;
  g_capture_poisoned = false;
  return cudaSuccess;
}
cudaError_t cudaStreamEndCapture(cudaStream_t, cudaGraph_t* g) {
  if (!g_capturing) return cudaErrorIllegalState;
  g_capturing = false;
  if (g_capture_poisoned) { *g = nullptr; return cudaErrorStreamCaptureInvalidated; }
  *g = static_cast<cudaGraph_t>(malloc(8));
  return cudaSuccess;
}
cudaError_t cudaGraphInstantiate(cudaGraphExec_t* x, cudaGraph_t, unsigned long long) { *x = static_cast<cudaGraphExec_t>(malloc(8)); return cudaSuccess; }
// One decode step = one graph launch.  FAKE_CUDART_STEP_US gives it a duration (so that deadlines and queue timeouts can
// expire while a request is running), FAKE_CUDART_FAIL_AFTER=n makes the n-th graph launch — and every launch after it —
// fail the way a device fault would (the engine must fail every request in flight, and say so on later submits).
cudaError_t cudaGraphLaunch(cudaGraphExec_t, cudaStream_t) {
  static const long step_us = getenv("FAKE_CUDART_STEP_US") ? atol(getenv("FAKE_CUDART_STEP_US")) : 0;
  static const long fail_after = getenv("FAKE_CUDART_FAIL_AFTER") ? atol(getenv("FAKE_CUDART_FAIL_AFTER")) : -1;
  static std::atomic<long> graph_launches{0};
  const long n = ++graph_launches;
  ++g_launches;
  if (fail_after >= 0 && n >= fail_after) return cudaErrorLaunchFailure;
  if (step_us > 0) usleep(useconds_t(step_us));
  return cudaSuccess;
}
cudaError_t cudaGraphDestroy(cudaGraph_t g) { free(g); return cudaSuccess; }
cudaError_t cudaGraphExecDestroy(cudaGraphExec_t x) { free(x); return cudaSuccess; }
// FAKE_CUDART_LAUNCH_LOG=<file>: one line per kernel launch — mangled kernel name, grid, block, dynamic shared memory,
// cluster dims and whether it was launched as a programmatic dependent (PDL) — the engine's LAUNCH PLAN for any geometry,
// readable without a GPU (tests/test_launch_plan_cpu.py checks co-residency and resource limits on it).  Launches of the
// projection GEMMs (gemm_tc_kernel / gemm_tc2_kernel, whose 10th parameter is split_k) append that K-split count, so that
// tests/test_kernel_coverage_cpu.py can tell a K-split launch from a plain one.  Launches of the K-split decode GEMV
// (gemv_ks_kernel, whose 9th parameter is TW, the warps of a team) append TW, which sets the kernel's team count.  The
// residual fold (rmsnorm_parts_kernel / rmsnorm_parts_cluster_kernel) appends n_parts, whether a gain was given (0 / 1)
// and hidden; rope_append_kernel appends n_heads and n_kv; rmsnorm_kernel and embed_kernel append hidden; sample_kernel
// appends vocab; both decode attention kernels append n_heads, n_kv and the sequence count (grid z of the cluster kernel,
// grid y of the tensor-core kernel).
static void log_launch(const void* fn, dim3 g, dim3 b, size_t smem, dim3 cluster, int pdl, void** args = nullptr) {
  static FILE* f = getenv("FAKE_CUDART_LAUNCH_LOG") ? fopen(getenv("FAKE_CUDART_LAUNCH_LOG"), "a") : nullptr;
  if (!f) return;
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_kernels.find(fn);
  const char* name = it == g_kernels.end() ? "?" : it->second.c_str();
  auto u32 = [&](int i) { return *static_cast<const uint32_t*>(args[i]); };
  fprintf(f, "%s %u %u %u %u %u %u %zu %u %u %u %d", name, g.x, g.y, g.z, b.x, b.y, b.z, smem, cluster.x, cluster.y, cluster.z, pdl);
  if (args && (strstr(name, "gemm_tc_kernel") || strstr(name, "gemm_tc2_kernel"))) fprintf(f, " %u", u32(9));
  if (args && strstr(name, "gemv_ks_kernel")) fprintf(f, " %u", u32(8));
  if (args && strstr(name, "rmsnorm_parts"))     // (x, parts, n_parts, part_stride, gain, y, hidden, ...)
    fprintf(f, " %u %d %u", u32(2), *static_cast<void* const*>(args[4]) != nullptr, u32(6));
  if (args && strstr(name, "18rope_append_kernel")) fprintf(f, " %u %u", u32(6), u32(7));
  if (args && (strstr(name, "14rmsnorm_kernel") || strstr(name, "12embed_kernel"))) fprintf(f, " %u", u32(3));
  if (args && strstr(name, "13sample_kernel")) fprintf(f, " %u", u32(1));     // (logits, vocab, ...)
  // (qkv, k_pages, v_pages, block_tables, bt_stride, bt_rows, seq_lens, rope, out, n_heads, n_kv, ...)
  if (args && strstr(name, "23decode_attention_kernel")) fprintf(f, " %u %u %u", u32(9), u32(10), g.z);
  if (args && strstr(name, "27decode_attention_mma_kernel")) fprintf(f, " %u %u %u", u32(9), u32(10), g.y);
  fputc('\n', f);
  fflush(f);
}
cudaError_t cudaLaunchKernel(const void* fn, dim3 g, dim3 b, void** args, size_t smem, cudaStream_t) {
  if (!config_allowed(g, b)) return g_last_error = cudaErrorInvalidConfiguration;
  if (!smem_allowed(fn, smem)) return g_last_error = cudaErrorInvalidValue;
  ++g_launches;
  log_launch(fn, g, b, smem, dim3(1, 1, 1), 0, args);
  return cudaSuccess;
}
cudaError_t cudaLaunchKernelExC(const cudaLaunchConfig_t* c, const void* fn, void** args) {
  if (!config_allowed(c->gridDim, c->blockDim)) return g_last_error = cudaErrorInvalidConfiguration;
  if (!smem_allowed(fn, c->dynamicSmemBytes)) return g_last_error = cudaErrorInvalidValue;
  ++g_launches;
  dim3 cluster(1, 1, 1);
  int pdl = 0;
  for (unsigned i = 0; i < c->numAttrs; ++i) {
    if (c->attrs[i].id == cudaLaunchAttributeClusterDimension) cluster = dim3(c->attrs[i].val.clusterDim.x, c->attrs[i].val.clusterDim.y, c->attrs[i].val.clusterDim.z);
    if (c->attrs[i].id == cudaLaunchAttributeProgrammaticStreamSerialization) pdl = c->attrs[i].val.programmaticStreamSerializationAllowed;
  }
  log_launch(fn, c->gridDim, c->blockDim, c->dynamicSmemBytes, cluster, pdl, args);
  return cudaSuccess;
}
// More than 48 KiB of dynamic shared memory needs an opt-in per kernel FUNCTION (each template instantiation is its own):
// the opt-in is recorded here and every launch is checked against it, like the driver does (cudaErrorInvalidValue).
cudaError_t cudaFuncSetAttribute(const void* fn, cudaFuncAttribute attr, int value) {
  if (attr == cudaFuncAttributeMaxDynamicSharedMemorySize) {
    if (value > 227 * 1024) return cudaErrorInvalidValue;
    std::lock_guard<std::mutex> lk(g_mu);
    g_smem_optin[fn] = size_t(value);
  }
  return cudaSuccess;
}
// launch configuration limits of the device (compute capability 10.0): refused with cudaErrorInvalidConfiguration
static bool config_allowed(dim3 g, dim3 b) {
  const unsigned long long threads = (unsigned long long)b.x * b.y * b.z;
  const bool ok = g.x >= 1 && g.y >= 1 && g.z >= 1 && g.x <= 2147483647u && g.y <= 65535u && g.z <= 65535u &&
                  b.x >= 1 && b.y >= 1 && b.z >= 1 && b.x <= 1024 && b.y <= 1024 && b.z <= 64 && threads <= 1024;
  if (!ok) fprintf(stderr, "fake cudart: invalid launch configuration grid %ux%ux%u block %ux%ux%u\n", g.x, g.y, g.z, b.x, b.y, b.z);
  return ok;
}
static bool smem_allowed(const void* fn, size_t smem) {
  if (smem <= 48 * 1024) return true;
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_smem_optin.find(fn);
  const bool ok = it != g_smem_optin.end() && smem <= it->second;
  if (!ok) {
    auto k = g_kernels.find(fn);
    fprintf(stderr, "fake cudart: launch of %s with %zu bytes of dynamic shared memory without a sufficient opt-in (%zu)\n",
            k == g_kernels.end() ? "?" : k->second.c_str(), smem, it == g_smem_optin.end() ? size_t(0) : it->second);
  }
  return ok;
}
cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessorWithFlags(int* n, const void*, int, size_t, unsigned) { *n = 1; return cudaSuccess; }
cudaError_t cudaGetDriverEntryPoint(const char* sym, void** fn, unsigned long long, cudaDriverEntryPointQueryResult* st) {
  const bool known = sym && !strcmp(sym, "cuTensorMapEncodeTiled");
  *fn = known ? reinterpret_cast<void*>(&fake_encode_tiled) : nullptr;
  if (st) *st = known ? cudaDriverEntryPointSuccess : cudaDriverEntryPointSymbolNotFound;
  return known ? cudaSuccess : cudaErrorSymbolNotFound;
}
// the 64-byte handle carries (size, owner pid, owner fd); a peer opens the owner's descriptor through /proc
cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t* h, void* p) {
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_allocs.find(p);
  if (it == g_allocs.end()) return cudaErrorInvalidValue;
  memset(h, 0, sizeof *h);
  const uint64_t v[3] = {it->second.size, uint64_t(getpid()), uint64_t(it->second.fd)};
  memcpy(h, v, sizeof v);
  return cudaSuccess;
}
cudaError_t cudaIpcOpenMemHandle(void** p, cudaIpcMemHandle_t h, unsigned) {
  uint64_t v[3];
  memcpy(v, &h, sizeof v);
  char path[64];
  snprintf(path, sizeof path, "/proc/%llu/fd/%llu", (unsigned long long)v[1], (unsigned long long)v[2]);
  const int fd = open(path, O_RDWR);
  if (fd < 0) return cudaErrorInvalidValue;
  void* m = mmap(nullptr, size_t(v[0]), PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
  close(fd);
  if (m == MAP_FAILED) return cudaErrorMemoryAllocation;
  { std::lock_guard<std::mutex> lk(g_mu); g_opened[m] = size_t(v[0]); }
  *p = m;
  return cudaSuccess;
}
cudaError_t cudaIpcCloseMemHandle(void* p) {
  size_t n = 0;
  { std::lock_guard<std::mutex> lk(g_mu); auto it = g_opened.find(p); if (it == g_opened.end()) return cudaErrorInvalidValue; n = it->second; g_opened.erase(it); }
  munmap(p, n);
  return cudaSuccess;
}

// what nvcc's host stubs call
void** __cudaRegisterFatBinary(void*) { static void* dummy[4]; return dummy; }
void __cudaRegisterFatBinaryEnd(void**) {}
void __cudaUnregisterFatBinary(void**) {}
void __cudaRegisterFunction(void**, const char* host_fn, char*, const char* device_name, int, uint3*, uint3*, dim3*, dim3*, int*) {
  std::lock_guard<std::mutex> lk(g_mu);
  g_kernels[host_fn] = device_name ? device_name : "?";
}
void __cudaRegisterVar(void**, char*, char*, const char*, int, size_t, int, int) {}
unsigned __cudaPushCallConfiguration(dim3 grid, dim3 block, size_t smem, struct CUstream_st* stream) {
  g_cfg.grid = grid; g_cfg.block = block; g_cfg.smem = smem; g_cfg.stream = stream;
  return 0;
}
cudaError_t __cudaPopCallConfiguration(dim3* grid, dim3* block, size_t* smem, void* stream) {
  *grid = g_cfg.grid; *block = g_cfg.block; *smem = g_cfg.smem; *static_cast<void**>(stream) = g_cfg.stream;
  return cudaSuccess;
}
// for the tests: how many launches the engine issued
unsigned long long fake_cudart_launches(void) { return g_launches.load(); }
unsigned long long fake_cudart_tensor_maps(void) { return g_tmaps.load(); }
}  // extern "C"
