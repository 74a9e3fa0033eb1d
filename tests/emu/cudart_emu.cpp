// Minimal CUDA runtime stand-in for running the HOST side of tl/nvl (team creation, launch queue, zero-copy board, score
// selection, asymmetric staging in the core, CUDA graphs, the IPC cache...) without a GPU: "device" memory is host memory with a
// registry behind cudaPointerGetAttributes, a stream is a worker thread draining a queue of closures, an event completes when the
// closure recorded behind the preceding work runs.  Kernels are the host-emulated ones (nvl_emu_launch.cpp) enqueued on the same
// queues.  Only what libucc_tl_nvl / libucc_mc_cuda call is implemented.
//   Capture: while a stream captures, kernels (with their argument block), cudaMemcpyAsync and cudaMemsetAsync on it are recorded
//   instead of run; a graph launch replays the recording, in issue order, on the target stream.  An event recorded in a capturing
//   stream marks a point of that capture, and a stream that waits for it joins the capture.  A capturing stream cannot wait for an
//   event recorded outside it, and synchronizing or querying a capturing stream, or the device while anything captures, invalidates
//   the capture, as with a global-mode capture on a GPU.
//   IPC: a handle names an allocation (base + allocation id).  Opening it returns the allocation itself; closing its last opening
//   marks the range dead, and the emulated launchers (nvl_emu_launch.cpp) refuse kernels whose pointer tables reach into a dead
//   range (emu_range_dead).  Members of one process share heaps by pointer and publish raw pointers, so only a driver that plays
//   several processes (tests/test_nvl_ipc_cache.py) opens handles.
#include <cuda_runtime_api.h>
#include <atomic>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <functional>
#include <map>
#include <mutex>
#include <set>
#include <thread>
#include <vector>
#include <sched.h>

namespace {
struct EmuStream {
    std::mutex m; std::condition_variable cv; std::deque<std::function<void()>> q; bool stop = false; bool busy = false; std::thread th;
    EmuStream() { th = std::thread([this] { run(); }); }
    void run()
    {
        for (;;) {
            std::function<void()> f;
            { std::unique_lock<std::mutex> l(m); cv.wait(l, [this] { return stop || !q.empty(); }); if (q.empty()) return; f = std::move(q.front()); q.pop_front(); busy = true; }
            f();
            { std::lock_guard<std::mutex> l(m); busy = false; }
            cv.notify_all();
        }
    }
    void push(std::function<void()> f) { { std::lock_guard<std::mutex> l(m); q.push_back(std::move(f)); } cv.notify_all(); }
    void sync() { std::unique_lock<std::mutex> l(m); cv.wait(l, [this] { return q.empty() && !busy; }); }
    ~EmuStream() { { std::lock_guard<std::mutex> l(m); stop = true; } cv.notify_all(); if (th.joinable()) th.join(); }
};
struct EmuEvent { std::atomic<uint64_t> recorded{0}, completed{0}; };
struct EmuAlloc { size_t size; int type; uint64_t id; };   // type: cudaMemoryType; id: tells a reused base from the freed one
struct EmuGraph { std::vector<std::function<void()>> nodes; };
struct EmuCapture { EmuGraph *g; bool invalidated = false; };

// all under g_lock
std::mutex g_lock;
std::map<uintptr_t, EmuAlloc> g_allocs;                  // base -> allocation
uint64_t g_alloc_ids;
std::vector<EmuStream *> g_streams;
EmuStream *g_default;
std::map<EmuStream *, EmuCapture *> g_capture;           // streams that capture (origin and joined)
std::set<EmuEvent *> g_captured_events;                  // last recorded in a capturing stream
std::map<uintptr_t, std::pair<size_t, long>> g_ipc;      // opened allocation base -> (size, open count)
std::map<uintptr_t, size_t> g_dead;                      // ranges whose last IPC mapping was closed
long g_ipc_opens, g_ipc_closes;
thread_local cudaError_t t_last = cudaSuccess;

// (takes g_lock for the default stream: resolve a stream before taking the lock)
EmuStream *S(cudaStream_t s)
{
    if (s) return reinterpret_cast<EmuStream *>(s);
    std::lock_guard<std::mutex> l(g_lock);
    if (!g_default) { g_default = new EmuStream(); g_streams.push_back(g_default); }
    return g_default;
}
cudaError_t fail(cudaError_t e) { t_last = e; return e; }
void *reg_alloc(size_t n, int type)
{
    void *p = nullptr;
    if (posix_memalign(&p, 512, n ? n : 1)) return nullptr;
    std::lock_guard<std::mutex> l(g_lock);
    g_allocs[(uintptr_t)p] = {n, type, ++g_alloc_ids};
    g_dead.erase((uintptr_t)p);
    return p;
}
// the allocation around p, or null; under g_lock
const std::pair<const uintptr_t, EmuAlloc> *alloc_of(const void *p)
{
    auto it = g_allocs.upper_bound((uintptr_t)p);
    if (it == g_allocs.begin()) return nullptr;
    --it;
    return (uintptr_t)p < it->first + (it->second.size ? it->second.size : 1) ? &*it : nullptr;
}
EmuCapture *capture_of(EmuStream *e) { std::lock_guard<std::mutex> l(g_lock); auto it = g_capture.find(e); return it == g_capture.end() ? nullptr : it->second; }
cudaError_t invalidate(EmuCapture *c) { c->invalidated = true; return fail(cudaErrorStreamCaptureUnsupported); }
// runs f behind the work already queued on s, or records it into the graph s captures
void enqueue(cudaStream_t s, std::function<void()> f)
{
    EmuStream *e = S(s);
    {
        std::lock_guard<std::mutex> l(g_lock);
        auto it = g_capture.find(e);
        if (it != g_capture.end()) { it->second->g->nodes.push_back(std::move(f)); return; }
    }
    e->push(std::move(f));
}
}  // namespace

// used by nvl_emu_launch.cpp: run `f` behind the work already queued on `s` (or record it, when `s` captures)
extern "C" void emu_stream_enqueue(cudaStream_t s, std::function<void()> *f) { enqueue(s, *f); }
// 1 when [p, p + n) overlaps a range whose last IPC mapping was closed
extern "C" int emu_range_dead(const void *p, size_t n)
{
    std::lock_guard<std::mutex> l(g_lock);
    uintptr_t a = (uintptr_t)p;
    auto it = g_dead.upper_bound(a);
    if (it != g_dead.begin()) { auto d = std::prev(it); if (a < d->first + d->second) return 1; }
    return it != g_dead.end() && it->first < a + (n ? n : 1);
}
// IPC statistics of the tests: what = 0 opens, 1 closes, 2 allocations mapped right now
extern "C" long emu_ipc_count(int what)
{ std::lock_guard<std::mutex> l(g_lock); return what == 0 ? g_ipc_opens : what == 1 ? g_ipc_closes : (long)g_ipc.size(); }

extern "C" {
cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return cudaSuccess; }
cudaError_t cudaGetDevice(int *d) { *d = 0; return cudaSuccess; }
cudaError_t cudaSetDevice(int) { return cudaSuccess; }
cudaError_t cudaGetLastError(void) { cudaError_t e = t_last; t_last = cudaSuccess; return e; }
cudaError_t cudaPeekAtLastError(void) { return t_last; }
const char *cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : (e == cudaErrorNotReady ? "not ready" : "emulated CUDA error"); }
static int emu_stream_value_stub(void *, unsigned long long, unsigned, unsigned) { return 999; /* CUDA_ERROR_UNKNOWN: never called, tl/nvl only checks that the entry points exist before it enables the zero-copy board */ }
static int emu_mem_get_address_range(unsigned long long *base, size_t *len, unsigned long long ptr)   /* cuMemGetAddressRange: the allocation around ptr */
{
    std::lock_guard<std::mutex> l(g_lock);
    auto *a = alloc_of((const void *)(uintptr_t)ptr);
    if (!a) return 1;   /* CUDA_ERROR_INVALID_VALUE */
    *base = a->first; *len = a->second.size;
    return 0;
}
cudaError_t cudaGetDriverEntryPoint(const char *name, void **fn, unsigned long long, cudaDriverEntryPointQueryResult *qr)
{
    if (!strcmp(name, "cuStreamWaitValue32") || !strcmp(name, "cuStreamWriteValue32")) *fn = (void *)emu_stream_value_stub;
    else if (!strcmp(name, "cuMemGetAddressRange")) *fn = (void *)emu_mem_get_address_range;
    else { *fn = nullptr; if (qr) *qr = cudaDriverEntryPointSymbolNotFound; return fail(cudaErrorNotSupported); }   /* no VMM / multicast: heaps are shared by pointer */
    if (qr) *qr = cudaDriverEntryPointSuccess;
    return cudaSuccess;
}
cudaError_t cudaGetDeviceProperties_v2(cudaDeviceProp *p, int)
{ memset(p, 0, sizeof(*p)); snprintf(p->name, sizeof(p->name), "host-emulated device"); p->multiProcessorCount = 2; p->major = 9; p->minor = 0; p->totalGlobalMem = 1ull << 34; return cudaSuccess; }
cudaError_t cudaDeviceGetAttribute(int *v, cudaDeviceAttr, int) { *v = 0; return cudaSuccess; }
cudaError_t cudaDeviceEnablePeerAccess(int, unsigned) { return cudaSuccess; }
cudaError_t cudaDeviceCanAccessPeer(int *can, int, int) { *can = 1; return cudaSuccess; }

cudaError_t cudaMalloc(void **p, size_t n) { *p = reg_alloc(n, cudaMemoryTypeDevice); return *p ? cudaSuccess : fail(cudaErrorMemoryAllocation); }
cudaError_t cudaMallocManaged(void **p, size_t n, unsigned) { *p = reg_alloc(n, cudaMemoryTypeManaged); return *p ? cudaSuccess : fail(cudaErrorMemoryAllocation); }
cudaError_t cudaHostAlloc(void **p, size_t n, unsigned) { *p = reg_alloc(n, cudaMemoryTypeHost); return *p ? cudaSuccess : fail(cudaErrorMemoryAllocation); }
cudaError_t cudaMallocHost(void **p, size_t n) { return cudaHostAlloc(p, n, 0); }
cudaError_t cudaHostGetDevicePointer(void **d, void *h, unsigned) { *d = h; return cudaSuccess; }
cudaError_t cudaFree(void *p) { if (!p) return cudaSuccess; { std::lock_guard<std::mutex> l(g_lock); g_allocs.erase((uintptr_t)p); g_dead.erase((uintptr_t)p); } free(p); return cudaSuccess; }
cudaError_t cudaFreeHost(void *p) { return cudaFree(p); }
cudaError_t cudaPointerGetAttributes(cudaPointerAttributes *a, const void *ptr)
{
    memset(a, 0, sizeof(*a));
    a->type = cudaMemoryTypeUnregistered; a->hostPointer = const_cast<void *>(ptr);
    std::lock_guard<std::mutex> l(g_lock);
    if (auto *x = alloc_of(ptr)) { a->type = (cudaMemoryType)x->second.type; a->device = 0; a->devicePointer = const_cast<void *>(ptr); }
    return cudaSuccess;
}
cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) { memmove(d, s, n); return cudaSuccess; }
cudaError_t cudaMemset(void *d, int v, size_t n) { memset(d, v, n); return cudaSuccess; }
cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t st) { enqueue(st, [=] { memmove(d, s, n); }); return cudaSuccess; }
cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t st) { enqueue(st, [=] { memset(d, v, n); }); return cudaSuccess; }
cudaError_t cudaDeviceSynchronize(void)
{
    std::vector<EmuStream *> all;
    {
        std::lock_guard<std::mutex> l(g_lock);
        if (!g_capture.empty()) { for (auto &c : g_capture) c.second->invalidated = true; return fail(cudaErrorStreamCaptureUnsupported); }
        all = g_streams;
    }
    for (auto *s : all) s->sync();
    return cudaSuccess;
}

/* leak checks of the tests: objects currently alive (what = 0 streams, 1 events, 2 device / pinned allocations) */
long emu_live_objects(int what);
cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { auto *e = new EmuStream(); { std::lock_guard<std::mutex> l(g_lock); g_streams.push_back(e); } *s = reinterpret_cast<cudaStream_t>(e); return cudaSuccess; }
cudaError_t cudaStreamCreate(cudaStream_t *s) { return cudaStreamCreateWithFlags(s, 0); }
cudaError_t cudaStreamDestroy(cudaStream_t s)
{ auto *e = reinterpret_cast<EmuStream *>(s); if (!e) return cudaSuccess; e->sync(); { std::lock_guard<std::mutex> l(g_lock); for (auto &x : g_streams) if (x == e) { x = g_streams.back(); g_streams.pop_back(); break; } } delete e; return cudaSuccess; }
cudaError_t cudaStreamSynchronize(cudaStream_t s) { auto *e = S(s); if (auto *c = capture_of(e)) return invalidate(c); e->sync(); return cudaSuccess; }
cudaError_t cudaStreamQuery(cudaStream_t s)
{
    auto *e = S(s);
    if (auto *c = capture_of(e)) return invalidate(c);
    std::lock_guard<std::mutex> l(e->m);
    return e->q.empty() && !e->busy ? cudaSuccess : cudaErrorNotReady;
}
cudaError_t cudaStreamIsCapturing(cudaStream_t s, cudaStreamCaptureStatus *st)
{ auto *c = capture_of(S(s)); *st = !c ? cudaStreamCaptureStatusNone : c->invalidated ? cudaStreamCaptureStatusInvalidated : cudaStreamCaptureStatusActive; return cudaSuccess; }
cudaError_t cudaStreamBeginCapture(cudaStream_t s, cudaStreamCaptureMode)
{
    auto *e = S(s);
    std::lock_guard<std::mutex> l(g_lock);
    if (g_capture.count(e)) return fail(cudaErrorIllegalState);
    g_capture[e] = new EmuCapture{new EmuGraph()};
    return cudaSuccess;
}
// ends the capture of its origin stream s; streams that joined it stop capturing too
cudaError_t cudaStreamEndCapture(cudaStream_t s, cudaGraph_t *graph)
{
    auto *e = S(s);
    std::lock_guard<std::mutex> l(g_lock);
    auto it = g_capture.find(e);
    if (it == g_capture.end()) return fail(cudaErrorIllegalState);
    EmuCapture *c = it->second;
    for (auto j = g_capture.begin(); j != g_capture.end();) { if (j->second == c) j = g_capture.erase(j); else ++j; }
    bool bad = c->invalidated;
    if (bad) { delete c->g; *graph = nullptr; } else *graph = reinterpret_cast<cudaGraph_t>(c->g);
    delete c;
    return bad ? fail(cudaErrorStreamCaptureInvalidated) : cudaSuccess;
}
cudaError_t cudaGraphInstantiate(cudaGraphExec_t *exec, cudaGraph_t graph, unsigned long long)
{ if (!graph) return fail(cudaErrorInvalidValue); *exec = reinterpret_cast<cudaGraphExec_t>(new EmuGraph(*reinterpret_cast<EmuGraph *>(graph))); return cudaSuccess; }
cudaError_t cudaGraphLaunch(cudaGraphExec_t exec, cudaStream_t s) { for (auto &f : reinterpret_cast<EmuGraph *>(exec)->nodes) enqueue(s, f); return cudaSuccess; }
cudaError_t cudaGraphExecDestroy(cudaGraphExec_t exec) { delete reinterpret_cast<EmuGraph *>(exec); return cudaSuccess; }
cudaError_t cudaGraphDestroy(cudaGraph_t g) { delete reinterpret_cast<EmuGraph *>(g); return cudaSuccess; }

static std::atomic<long> g_live_events{0};
cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned) { *e = reinterpret_cast<cudaEvent_t>(new EmuEvent()); g_live_events++; return cudaSuccess; }
cudaError_t cudaEventCreate(cudaEvent_t *e) { return cudaEventCreateWithFlags(e, 0); }
cudaError_t cudaEventDestroy(cudaEvent_t e) { delete reinterpret_cast<EmuEvent *>(e); g_live_events--; return cudaSuccess; }   // (callers destroy only completed events)
long emu_live_objects(int what)
{ std::lock_guard<std::mutex> l(g_lock); return what == 0 ? (long)g_streams.size() : what == 1 ? g_live_events.load() : (long)g_allocs.size(); }
// (in issue order a replay needs no node for an event record or wait inside a capture)
cudaError_t cudaEventRecord(cudaEvent_t ev, cudaStream_t s)
{
    auto *e = reinterpret_cast<EmuEvent *>(ev);
    auto *st = S(s);
    {
        std::lock_guard<std::mutex> l(g_lock);
        if (g_capture.count(st)) { g_captured_events.insert(e); return cudaSuccess; }
        g_captured_events.erase(e);
    }
    uint64_t seq = ++e->recorded;
    st->push([e, seq] { uint64_t c = e->completed.load(); while (c < seq && !e->completed.compare_exchange_weak(c, seq)) {} });
    return cudaSuccess;
}
cudaError_t cudaEventQuery(cudaEvent_t ev)
{
    auto *e = reinterpret_cast<EmuEvent *>(ev);
    { std::lock_guard<std::mutex> l(g_lock); if (g_captured_events.count(e)) return fail(cudaErrorStreamCaptureUnsupported); }
    return e->completed.load() >= e->recorded.load() ? cudaSuccess : fail(cudaErrorNotReady);
}
cudaError_t cudaEventSynchronize(cudaEvent_t ev) { auto *e = reinterpret_cast<EmuEvent *>(ev); while (e->completed.load() < e->recorded.load()) sched_yield(); return cudaSuccess; }
cudaError_t cudaStreamWaitEvent(cudaStream_t s, cudaEvent_t ev, unsigned)
{
    auto *e = reinterpret_cast<EmuEvent *>(ev);
    auto *st = S(s);
    {
        std::lock_guard<std::mutex> l(g_lock);
        auto it = g_capture.find(st);
        if (g_captured_events.count(e)) {
            if (it != g_capture.end()) return cudaSuccess;
            if (g_capture.empty()) return fail(cudaErrorStreamCaptureIsolation);
            g_capture[st] = g_capture.begin()->second;   // joins the capture (the tests keep one capture open when streams join)
            return cudaSuccess;
        }
        if (it != g_capture.end()) { it->second->invalidated = true; return fail(cudaErrorStreamCaptureIsolation); }
    }
    uint64_t seq = e->recorded.load();
    st->push([e, seq] { while (e->completed.load() < seq) sched_yield(); });
    return cudaSuccess;
}
cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t, cudaEvent_t) { *ms = 0.f; return cudaSuccess; }

cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t *h, void *p)
{
    std::lock_guard<std::mutex> l(g_lock);
    auto it = g_allocs.find((uintptr_t)p);
    if (it == g_allocs.end() || it->second.type != cudaMemoryTypeDevice) return fail(cudaErrorInvalidValue);
    memset(h, 0, sizeof(*h));
    uint64_t v[2] = {(uint64_t)(uintptr_t)p, it->second.id};
    memcpy(h->reserved, v, sizeof(v));
    return cudaSuccess;
}
cudaError_t cudaIpcOpenMemHandle(void **p, cudaIpcMemHandle_t h, unsigned)
{
    uint64_t v[2];
    memcpy(v, h.reserved, sizeof(v));
    std::lock_guard<std::mutex> l(g_lock);
    auto a = g_allocs.find((uintptr_t)v[0]);
    if (a == g_allocs.end() || a->second.id != v[1]) return fail(cudaErrorInvalidResourceHandle);   /* freed since the export */
    auto &o = g_ipc[a->first];
    o.first = a->second.size; o.second++;
    g_dead.erase(a->first);
    g_ipc_opens++;
    *p = (void *)a->first;
    return cudaSuccess;
}
cudaError_t cudaIpcCloseMemHandle(void *p)
{
    std::lock_guard<std::mutex> l(g_lock);
    auto it = g_ipc.find((uintptr_t)p);
    if (it == g_ipc.end()) return fail(cudaErrorInvalidValue);
    g_ipc_closes++;
    if (--it->second.second == 0) { g_dead[it->first] = it->second.first; g_ipc.erase(it); }
    return cudaSuccess;
}
}
