// tests/cudaemu/emu/emu_runtime.cpp — TEST INFRASTRUCTURE: block-by-block execution of an emulated launch.
//
// One set of threads per launch; every thread walks the blocks of the grid in order.  __syncthreads() is a barrier over
// the threads of the block that have not returned from the kernel yet (what the hardware does), a second barrier
// separates consecutive blocks (shared memory is reused).
#include "cuda_runtime.h"

#include <cxxabi.h>
#include <dlfcn.h>

#include <condition_variable>
#include <map>
#include <mutex>
#include <string>

thread_local uint3_emu threadIdx, blockIdx;
thread_local dim3 blockDim, gridDim;

namespace b200emu {

uint8_t *dyn_smem = nullptr;

struct LiveBarrier {
  std::mutex m;
  std::condition_variable cv;
  unsigned expected = 0, arrived = 0;
  unsigned long generation = 0;
  void reset (unsigned n) { expected = n; arrived = 0; }
  void wait ()
  {
    std::unique_lock<std::mutex> l (m);
    const unsigned long g = generation;
    if (++arrived >= expected) { arrived = 0; generation++; cv.notify_all (); return; }
    cv.wait (l, [&] { return generation != g; });
  }
  void leave ()                  // a thread returned from the kernel: it no longer takes part in __syncthreads
  {
    std::unique_lock<std::mutex> l (m);
    if (expected) expected--;
    if (expected && arrived >= expected) { arrived = 0; generation++; cv.notify_all (); }
  }
};

static LiveBarrier g_sync;
static LiveBarrier g_warp[64];                 // one per warp of the block
static unsigned g_wa[64][32][4], g_wb[64][32][2];
static pthread_barrier_t g_block;

void barrier () { g_sync.wait (); }

static unsigned g_wx[64][32];

unsigned lane_id ()
{
  return (threadIdx.x + blockDim.x * (threadIdx.y + blockDim.y * threadIdx.z)) & 31;
}

void warp_gather (unsigned v, unsigned out[32])
{
  const unsigned tid = threadIdx.x + blockDim.x * (threadIdx.y + blockDim.y * threadIdx.z);
  const unsigned w = tid >> 5, lane = tid & 31;
  g_wx[w][lane] = v;
  g_warp[w].wait ();
  for (int i = 0; i < 32; i++) out[i] = g_wx[w][i];
  g_warp[w].wait ();
}

static void warp_mma (int d[4], unsigned a0, unsigned a1, unsigned a2, unsigned a3, unsigned b0, unsigned b1, const int c[4],
    bool a_signed);

void warp_mma_u8s8 (int d[4], unsigned a0, unsigned a1, unsigned a2, unsigned a3, unsigned b0, unsigned b1, const int c[4])
{
  warp_mma (d, a0, a1, a2, a3, b0, b1, c, false);
}

void warp_mma_s8u8 (int d[4], unsigned a0, unsigned a1, unsigned a2, unsigned a3, unsigned b0, unsigned b1, const int c[4])
{
  warp_mma (d, a0, a1, a2, a3, b0, b1, c, true);
}

static void warp_mma (int d[4], unsigned a0, unsigned a1, unsigned a2, unsigned a3, unsigned b0, unsigned b1, const int c[4],
    bool a_signed)
{
  const unsigned tid = threadIdx.x + blockDim.x * (threadIdx.y + blockDim.y * threadIdx.z);
  const unsigned w = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  g_wa[w][lane][0] = a0; g_wa[w][lane][1] = a1; g_wa[w][lane][2] = a2; g_wa[w][lane][3] = a3;
  g_wb[w][lane][0] = b0; g_wb[w][lane][1] = b1;
  g_warp[w].wait ();
  auto A = [&] (unsigned row, unsigned k) -> int {                 // u8
    const unsigned src = (row & 7) * 4 + ((k & 15) >> 2), reg = (row >> 3) + 2 * (k >> 4);
    const unsigned v = (g_wa[w][src][reg] >> (8 * (k & 3))) & 0xff;
    return a_signed ? (int) (int8_t) v : (int) v;
  };
  auto B = [&] (unsigned k, unsigned n) -> int {                   // s8
    const unsigned src = n * 4 + ((k & 15) >> 2), reg = k >> 4;
    const unsigned v = (g_wb[w][src][reg] >> (8 * (k & 3))) & 0xff;
    return a_signed ? (int) v : (int) (int8_t) v;                  // the operand that is not the taps holds u8 pixels
  };
  const unsigned rows[4] = {g, g, g + 8, g + 8}, cols[4] = {2 * t, 2 * t + 1, 2 * t, 2 * t + 1};
  for (int i = 0; i < 4; i++) {
    int acc = c[i];
    for (unsigned k = 0; k < 32; k++) acc += A (rows[i], k) * B (k, cols[i]);
    d[i] = acc;
  }
  g_warp[w].wait ();
}

struct Job {
  const std::function<void ()> *body;
  dim3 grid, block;
  unsigned tid, nt;
};

static void *thread_main (void *arg)
{
  Job *j = (Job *) arg;
  gridDim = j->grid; blockDim = j->block;
  threadIdx.x = j->tid % j->block.x;
  threadIdx.y = (j->tid / j->block.x) % j->block.y;
  threadIdx.z = j->tid / (j->block.x * j->block.y);
  for (unsigned bz = 0; bz < j->grid.z; bz++)
    for (unsigned by = 0; by < j->grid.y; by++)
      for (unsigned bx = 0; bx < j->grid.x; bx++) {
        blockIdx = uint3_emu {bx, by, bz};
        (*j->body) ();
        g_sync.leave ();
        if (pthread_barrier_wait (&g_block) == PTHREAD_BARRIER_SERIAL_THREAD)
          g_sync.reset (j->nt);                                    // every thread is between blocks here
        pthread_barrier_wait (&g_block);
      }
  return nullptr;
}

static std::string g_log;                      // kernels launched in record-only mode, one per line
static int g_record_only = 0;                  // 0: run launches; 1: log the kernel; 2: the kernel and its launch configuration

// the instantiation `fn` points at, without namespace, return type and parameters ("vcs_generic_kernel<false>"); the
// launch site's spelling where the symbol is not exported (a function pointer's variable name, e.g. "fn")
static std::string kernel_label (const char *name, const void *fn)
{
  Dl_info info;
  if (!dladdr (fn, &info) || !info.dli_sname || info.dli_saddr != fn) return name;
  int status = -1;
  char *d = abi::__cxa_demangle (info.dli_sname, nullptr, nullptr, &status);
  if (status != 0 || !d) { free (d); return name; }
  const std::string s (d);
  free (d);
  size_t start = 0, end = s.size ();
  int depth = 0;
  for (size_t i = 0; i < s.size (); i++) {
    if (s[i] == '<') depth++;
    else if (s[i] == '>') depth--;
    else if (depth == 0 && s[i] == '(') { end = i; break; }
    else if (depth == 0 && (s[i] == ' ' || s.compare (i, 2, "::") == 0)) start = i + (s[i] == ' ' ? 1 : 2);
  }
  return s.substr (start, end - start);
}

void launch (dim3 grid, dim3 block, size_t smem_bytes, const std::function<void ()> & body, const char *name, const void *fn)
{
  if (g_record_only) {
    g_log += kernel_label (name, fn);
    if (g_record_only >= 2)
      g_log += " grid=" + std::to_string (grid.x) + "," + std::to_string (grid.y) + "," + std::to_string (grid.z) + " block=" +
               std::to_string (block.x) + "," + std::to_string (block.y) + "," + std::to_string (block.z) + " smem=" +
               std::to_string (smem_bytes);
    g_log += '\n';
    return;
  }
  const unsigned nt = block.x * block.y * block.z;
  // exactly the requested bytes (rounded to 16): an address sanitizer build then catches a kernel that runs past them
  uint8_t *smem = (uint8_t *) aligned_alloc (16, std::max<size_t> (16, (smem_bytes + 15) & ~(size_t) 15));
  dyn_smem = smem;
  std::vector<pthread_t> th (nt);
  std::vector<Job> jobs (nt);
  pthread_attr_t attr;
  pthread_attr_init (&attr);
  pthread_attr_setstacksize (&attr, 256 * 1024);
  pthread_barrier_init (&g_block, nullptr, nt);
  g_sync.reset (nt);
  for (unsigned w = 0; w < 64; w++) g_warp[w].reset (32);
  for (unsigned t = 0; t < nt; t++) {
    jobs[t] = Job {&body, grid, block, t, nt};
    pthread_create (&th[t], &attr, thread_main, &jobs[t]);
  }
  for (unsigned t = 0; t < nt; t++) pthread_join (th[t], nullptr);
  pthread_barrier_destroy (&g_block);
  pthread_attr_destroy (&attr);
  dyn_smem = nullptr;
  free (smem);
}

// ---- allocations, copies, streams and events ------------------------------------------------------------------------
// Handles and allocations are named by creation order since the last log clear (s0, e0, a0, ...; "?" for one created
// before it), so a level-3 log holds no addresses.
static std::map<uintptr_t, std::pair<size_t, std::string>> g_allocs;    // base -> (bytes, name)
static std::map<void *, std::string> g_handles;                        // stream / event -> name
static int g_n_alloc = 0, g_n_stream = 0, g_n_event = 0;
static int g_fail_create = 0;                  // > 0: the n-th stream or event creation from now fails

static void note (const std::string & line)
{
  if (g_record_only >= 3) g_log += line + '\n';
}

static std::string handle_name (void *h)
{
  if (!h) return "0";                          // the legacy default stream
  auto it = g_handles.find (h);
  return it == g_handles.end () ? "?" : it->second;
}

// "a<k>+<offset>" for a pointer into a device allocation, "host" for any other
static std::string where (const void *p)
{
  const uintptr_t a = (uintptr_t) p;
  auto it = g_allocs.upper_bound (a);
  if (it == g_allocs.begin ()) return "host";
  --it;
  if (a >= it->first + std::max<size_t> (it->second.first, 1)) return "host";
  return it->second.second + "+" + std::to_string (a - it->first);
}

static bool create_fails ()
{
  return g_fail_create > 0 && --g_fail_create == 0;
}

static void forget_names ()
{
  for (auto & a : g_allocs) a.second.second = "?";
  for (auto & h : g_handles) h.second = "?";
  g_n_alloc = g_n_stream = g_n_event = 0;
}

}  // namespace b200emu

using namespace b200emu;

cudaError_t cudaMalloc (void **p, size_t n)
{
  *p = malloc (n ? n : 1);
  if (!*p) return cudaErrorMemoryAllocation;
  const std::string name = "a" + std::to_string (g_n_alloc++);
  g_allocs[(uintptr_t) *p] = {n, name};
  note ("cudaMalloc " + name + " bytes=" + std::to_string (n));
  return cudaSuccess;
}

cudaError_t cudaFree (void *p)
{
  if (!p) { note ("cudaFree null"); return cudaSuccess; }
  auto it = g_allocs.find ((uintptr_t) p);
  note ("cudaFree " + (it == g_allocs.end () ? std::string ("host") : it->second.second));
  if (it != g_allocs.end ()) g_allocs.erase (it);
  free (p);
  return cudaSuccess;
}

cudaError_t cudaMemsetAsync (void *d, int v, size_t n, cudaStream_t s)
{
  note ("cudaMemsetAsync " + where (d) + " value=" + std::to_string (v) + " bytes=" + std::to_string (n) + " stream=" + handle_name (s));
  memset (d, v, n);
  return cudaSuccess;
}

cudaError_t cudaMemcpyAsync (void *d, const void *s, size_t n, cudaMemcpyKind k, cudaStream_t st)
{
  const char *dir = k == cudaMemcpyHostToDevice ? "H2D" : (k == cudaMemcpyDeviceToHost ? "D2H" : "D2D");
  std::string line = std::string ("cudaMemcpyAsync ") + dir + " bytes=" + std::to_string (n) + " stream=" + handle_name (st);
  if (k != cudaMemcpyHostToDevice) line += " src=" + where (s);
  if (k != cudaMemcpyDeviceToHost) line += " dst=" + where (d);
  note (line);
  memcpy (d, s, n);
  return cudaSuccess;
}

cudaError_t cudaDeviceSynchronize () { note ("cudaDeviceSynchronize"); return cudaSuccess; }

cudaError_t cudaStreamCreateWithFlags (cudaStream_t *s, unsigned)
{
  if (create_fails ()) { note ("cudaStreamCreate failed"); return cudaErrorUnknown; }
  *s = new char;
  g_handles[*s] = "s" + std::to_string (g_n_stream++);
  note ("cudaStreamCreate " + g_handles[*s]);
  return cudaSuccess;
}

cudaError_t cudaEventCreateWithFlags (cudaEvent_t *e, unsigned)
{
  if (create_fails ()) { note ("cudaEventCreate failed"); return cudaErrorUnknown; }
  *e = new char;
  g_handles[*e] = "e" + std::to_string (g_n_event++);
  note ("cudaEventCreate " + g_handles[*e]);
  return cudaSuccess;
}

static cudaError_t destroy_handle (const char *what, void *h)
{
  note (std::string (what) + " " + handle_name (h));
  g_handles.erase (h);
  delete (char *) h;
  return cudaSuccess;
}

cudaError_t cudaStreamDestroy (cudaStream_t s) { return destroy_handle ("cudaStreamDestroy", s); }
cudaError_t cudaEventDestroy (cudaEvent_t e) { return destroy_handle ("cudaEventDestroy", e); }
cudaError_t cudaStreamSynchronize (cudaStream_t s) { note ("cudaStreamSynchronize " + handle_name (s)); return cudaSuccess; }
cudaError_t cudaEventSynchronize (cudaEvent_t e) { note ("cudaEventSynchronize " + handle_name (e)); return cudaSuccess; }
cudaError_t cudaEventRecord (cudaEvent_t e, cudaStream_t s)
{
  note ("cudaEventRecord " + handle_name (e) + " stream=" + handle_name (s));
  return cudaSuccess;
}
cudaError_t cudaStreamWaitEvent (cudaStream_t s, cudaEvent_t e, unsigned)
{
  note ("cudaStreamWaitEvent stream=" + handle_name (s) + " " + handle_name (e));
  return cudaSuccess;
}

extern "C" {

// the kernels launched since the last clear, one name per line (valid until the next launch or clear)
const char *b200emu_launch_log () { return b200emu::g_log.c_str (); }
void b200emu_clear_launch_log () { b200emu::g_log.clear (); b200emu::forget_names (); }
// 1: launches are logged by kernel and no block runs (route tests); 2: the same, each line followed by
// " grid=x,y,z block=x,y,z smem=bytes"; 3: level 2 and, in between, the allocations, copies, memsets and stream / event
// calls; 0 (the default): launches run and nothing is logged
void b200emu_set_record_only (int level) { b200emu::g_record_only = level; }
// test hook: the n-th stream or event creation from now fails with an error (0: none fails)
void b200emu_fail_create (int n) { b200emu::g_fail_create = n; }

}
