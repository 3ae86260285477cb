// Handle management, error reporting and bookkeeping for libb2rl's C ABI
// (include/b2rl.h).
#include "common.cuh"

#include <stdarg.h>
#include <string.h>
#include <new>

namespace b2rl {
static thread_local char g_err[512] = "";
std::atomic<int64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
}  // namespace b2rl

using namespace b2rl;

extern "C" const char* b2rl_last_error(void) { return g_err; }
extern "C" int b2rl_version(void) { return 100; }
extern "C" int64_t b2rl_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

static void free_all(b2rl_replay* h) {
  dedup_free(h);
  for (int f = 0; f < B2RL_MAX_FIELDS; ++f) {
    if (h->host_field[f]) cudaFreeHost(h->host_field[f]);
    else if (h->field[f]) cudaFree(h->field[f]);
  }
  if (h->tree.leaf) cudaFree(h->tree.leaf);
  if (h->tree.sum) cudaFree(h->tree.sum);
  if (h->tree.minv) cudaFree(h->tree.minv);
  if (h->tag) cudaFree(h->tag);
  if (h->scratch_val) cudaFree(h->scratch_val);
  if (h->rng_dev) cudaFree(h->rng_dev);
  if (h->n_valid_dev) cudaFree(h->n_valid_dev);
  if (h->build_ticket) cudaFree(h->build_ticket);
  if (h->pipe_prios) cudaFree(h->pipe_prios);
  if (h->ev_reserved) cudaEventDestroy(h->ev_reserved);
  if (h->ev_copied) cudaEventDestroy(h->ev_copied);
  if (h->ingest_stream) cudaStreamDestroy(h->ingest_stream);
}

extern "C" int b2rl_replay_create(const b2rl_replay_desc* d, b2rl_replay** out) {
  return b2rl_replay_create_placed(d, nullptr, out);
}

extern "C" int b2rl_replay_create_placed(const b2rl_replay_desc* d, const int32_t* on_host, b2rl_replay** out) {
  B2RL_REQUIRE(d != nullptr && out != nullptr, "null argument");
  B2RL_REQUIRE(d->capacity >= 1 && d->capacity <= (1LL << 31), "capacity must be in [1, 2^31]");
  B2RL_REQUIRE(d->n_fields >= 0 && d->n_fields <= B2RL_MAX_FIELDS, "n_fields out of range");
  for (int f = 0; f < d->n_fields; ++f) B2RL_REQUIRE(d->field_bytes[f] >= 1, "field_bytes must be >= 1");
  for (int f = 0; on_host != nullptr && f < d->n_fields; ++f)
    B2RL_REQUIRE(!on_host[f] || d->field_bytes[f] % 16 == 0,
                 "a field placed on the host must have rows of a whole number of 16-byte units");
  int ndev = 0;
  B2RL_CUDA(cudaGetDeviceCount(&ndev));
  B2RL_REQUIRE(d->device >= 0 && d->device < ndev, "no such CUDA device");
  DeviceGuard g(d->device);
  b2rl_replay* h = new (std::nothrow) b2rl_replay();
  if (!h) { set_error("out of host memory"); return B2RL_ERR_NOMEM; }
  h->device = d->device;
  h->capacity = d->capacity;
  h->levels = 1;            // at least two leaves, so that there is always a stored root level above them
  h->cap2 = 2;
  while (h->cap2 < d->capacity) { h->cap2 <<= 1; h->levels++; }
  TreeView& t = h->tree;
  t.cap2 = h->cap2;
  t.levels = h->levels;
  t.G = (h->levels + 3) / 4;
  t.top_bits = h->levels - 4 * (t.G - 1);
  int64_t total = 0;
  for (int k = 1; k <= t.G; ++k) {
    t.off[k] = total;
    const int64_t nk = (k == t.G) ? 1 : (h->cap2 >> (4 * k));
    total += (nk + 15) & ~(int64_t)15;     // every stored level starts on a 128-byte line
  }
  h->n_fields = d->n_fields;
  cudaError_t e = cudaSuccess;
  auto alloc = [&](void** p, size_t bytes) {
    if (e == cudaSuccess) e = cudaMalloc(p, bytes);
  };
  for (int f = 0; f < d->n_fields; ++f) {
    h->field_bytes[f] = d->field_bytes[f];
    // +16 B so a 16-byte bulk/vector access on the last row never leaves the allocation
    const size_t bytes = (size_t)d->capacity * (size_t)d->field_bytes[f] + 16;
    if (on_host == nullptr || !on_host[f]) {
      alloc((void**)&h->field[f], bytes);
      continue;
    }
    if (e != cudaSuccess) continue;
    h->on_host[f] = h->any_on_host = true;
    const cudaError_t eh = cudaHostAlloc((void**)&h->host_field[f], bytes, cudaHostAllocMapped | cudaHostAllocPortable);
    if (eh != cudaSuccess) {
      h->host_field[f] = nullptr;
      set_error("cudaHostAlloc of %.3f GB (%zu bytes) of pinned host memory for field %d failed: %s", bytes * 1e-9,
                bytes, f, cudaGetErrorString(eh));
      free_all(h);
      delete h;
      cudaGetLastError();
      return B2RL_ERR_NOMEM;
    }
    e = cudaHostGetDevicePointer((void**)&h->field[f], h->host_field[f], 0);
  }
  alloc((void**)&t.leaf, sizeof(float) * (size_t)h->cap2);
  alloc((void**)&t.sum, sizeof(double) * (size_t)total);
  alloc((void**)&t.minv, sizeof(float) * (size_t)total);
  alloc((void**)&h->tag, sizeof(uint32_t) * (size_t)h->cap2);
  alloc((void**)&h->scratch_val, sizeof(float) * (size_t)h->capacity);
  alloc((void**)&h->rng_dev, sizeof(uint64_t) * 3);   // {seed, counter, last-block ticket}
  alloc((void**)&h->n_valid_dev, sizeof(float));
  alloc((void**)&h->build_ticket, sizeof(unsigned int));
  if (e != cudaSuccess) {
    set_error("cudaMalloc failed while creating a %lld-slot replay: %s", (long long)d->capacity,
              cudaGetErrorString(e));
    free_all(h);
    delete h;
    cudaGetLastError();
    return B2RL_ERR_NOMEM;
  }
  B2RL_CUDA(cudaMemset(h->build_ticket, 0, sizeof(unsigned int)));
  // empty tree: sums 0, mins +inf, tags 0
  {
    int rc = b2rl_tree_build(h, nullptr, 0, nullptr);   // empty tree: sums 0, mins +inf
    if (rc != B2RL_OK) { free_all(h); delete h; return rc; }
  }
  B2RL_CUDA(cudaMemset(h->tag, 0, sizeof(uint32_t) * (size_t)h->cap2));
  {
    const uint64_t init[3] = {1234ULL, 0ULL, 0ULL};
    B2RL_CUDA(cudaMemcpy(h->rng_dev, init, sizeof(init), cudaMemcpyHostToDevice));
  }
  B2RL_CUDA(cudaDeviceSynchronize());
  *out = h;
  return B2RL_OK;
}

extern "C" int b2rl_replay_destroy(b2rl_replay* h) {
  if (!h) return B2RL_OK;
  DeviceGuard g(h->device);
  cudaDeviceSynchronize();
  free_all(h);
  delete h;
  return B2RL_OK;
}

extern "C" int b2rl_replay_size(const b2rl_replay* h, int64_t* size, int64_t* capacity, int64_t* head) {
  B2RL_REQUIRE(h != nullptr, "null handle");
  if (size) *size = h->size;
  if (capacity) *capacity = h->capacity;
  if (head) *head = h->head;
  return B2RL_OK;
}

extern "C" int b2rl_replay_field_ptr(const b2rl_replay* h, int32_t field, void** ptr_dev) {
  B2RL_REQUIRE(h != nullptr && ptr_dev != nullptr, "null argument");
  B2RL_REQUIRE(field >= 0 && field < h->n_fields, "no such field");
  *ptr_dev = h->on_host[field] ? h->host_field[field] : h->field[field];
  return B2RL_OK;
}

extern "C" int b2rl_replay_field_placement(const b2rl_replay* h, int32_t field, int32_t* on_host) {
  B2RL_REQUIRE(h != nullptr && on_host != nullptr, "null argument");
  B2RL_REQUIRE(field >= 0 && field < h->n_fields, "no such field");
  *on_host = h->on_host[field] ? 1 : 0;
  return B2RL_OK;
}
