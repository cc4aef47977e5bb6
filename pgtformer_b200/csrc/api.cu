// Status plumbing, launch accounting and device queries for libpgt_b200.
#include <atomic>
#include <cstdio>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "tmap.cuh"

namespace pgt {
static thread_local char g_last_error[512] = "";
static std::atomic<long long> g_launches{0};

void set_cuda_error(cudaError_t e, const char* where) {
  snprintf(g_last_error, sizeof(g_last_error), "%s: %s (%s)", where, cudaGetErrorName(e), cudaGetErrorString(e));
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
int num_sms() {
  static std::atomic<int> per_dev[64];                 // per device: a process may drive several GPUs
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  int n = per_dev[dev].load(std::memory_order_relaxed);
  if (n == 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    per_dev[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}

// ---- tensor-map cache (tmap.cuh)
static std::atomic<long long> g_tmap_hits{0}, g_tmap_misses{0};
std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash>& tmap_cache() {
  static std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> c;
  return c;
}
std::mutex& tmap_cache_mutex() {
  static std::mutex m;
  return m;
}
void tmap_cache_count(bool hit) { (hit ? g_tmap_hits : g_tmap_misses).fetch_add(1, std::memory_order_relaxed); }
void tmap_cache_stats(long long* hits, long long* misses) { *hits = g_tmap_hits.load(); *misses = g_tmap_misses.load(); }

// ---- optional per-launch profiler: CUDA events on the launching stream around every launch of a class
struct ProfRec { cudaEvent_t e0, e1; int cls; double work; char desc[96]; };
static bool g_prof_on = false;
static std::vector<ProfRec> g_prof;
bool prof_enabled() { return g_prof_on; }
void prof_before(int cls, double work, cudaStream_t st, const char* desc) {
  ProfRec r; r.cls = cls; r.work = work;
  snprintf(r.desc, sizeof(r.desc), "%s", desc ? desc : "");
  cudaEventCreate(&r.e0); cudaEventCreate(&r.e1);
  cudaEventRecord(r.e0, st);
  g_prof.push_back(r);
}
void prof_after(cudaStream_t st) { cudaEventRecord(g_prof.back().e1, st); }
}  // namespace pgt

extern "C" int pgt_profile_begin(void) {
  pgt::g_prof.clear();
  pgt::g_prof_on = true;
  return PGT_OK;
}
extern "C" int pgt_profile_end(double* work, double* ms, int64_t* launches);
static FILE* g_prof_csv = nullptr;
extern "C" int pgt_profile_end_csv(const char* path, double* work, double* ms, int64_t* launches) {
  g_prof_csv = fopen(path, "w");
  if (g_prof_csv) fprintf(g_prof_csv, "class,desc,work,ms\n");
  int rc = pgt_profile_end(work, ms, launches);
  if (g_prof_csv) { fclose(g_prof_csv); g_prof_csv = nullptr; }
  return rc;
}
extern "C" int pgt_profile_end(double* work, double* ms, int64_t* launches) {
  pgt::g_prof_on = false;
  for (int i = 0; i < PGT_PROF_CLASSES; ++i) { work[i] = 0; ms[i] = 0; launches[i] = 0; }
  for (auto& r : pgt::g_prof) {
    float t = 0.f;
    if (cudaEventSynchronize(r.e1) == cudaSuccess && cudaEventElapsedTime(&t, r.e0, r.e1) == cudaSuccess &&
        r.cls >= 0 && r.cls < PGT_PROF_CLASSES) {
      work[r.cls] += r.work; ms[r.cls] += t; launches[r.cls] += 1;
      if (g_prof_csv) fprintf(g_prof_csv, "%d,%s,%.6e,%.6f\n", r.cls, r.desc, r.work, t);
    }
    cudaEventDestroy(r.e0); cudaEventDestroy(r.e1);
  }
  pgt::g_prof.clear();
  return PGT_OK;
}

extern "C" const char* pgt_strerror(int status) {
  switch (status) {
    case PGT_OK: return "ok";
    case PGT_ERR_INVALID: return "invalid argument (shape / alignment / null pointer)";
    case PGT_ERR_CUDA: return "CUDA runtime error (see pgt_last_cuda_error)";
    case PGT_ERR_UNSUPPORTED: return "configuration not covered by the sm_90a kernels";
    case PGT_ERR_DRIVER: return "cuTensorMapEncodeTiled unavailable or failed";
    default: return "unknown status";
  }
}
extern "C" const char* pgt_last_cuda_error(void) { return pgt::g_last_error; }
extern "C" int pgt_version(void) { return 200; }
extern "C" void pgt_tmap_cache_stats(int64_t* hits, int64_t* misses) {
  long long h = 0, m = 0;
  pgt::tmap_cache_stats(&h, &m);
  if (hits) *hits = h;
  if (misses) *misses = m;
}
extern "C" int64_t pgt_launch_count(void) { return pgt::g_launches.load(); }
extern "C" void pgt_reset_launch_count(void) { pgt::g_launches.store(0); }
