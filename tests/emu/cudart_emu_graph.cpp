// The emulated CUDA runtime of cudart_emu.cpp plus stream capture, CUDA graphs, CUDA IPC and cuMemGetAddressRange: the runtime of
// the graph tests (tests/emu/build_hostemu_graph.sh).  The entry points that change are compiled from cudart_emu.cpp under other
// names and wrapped here.
//   Capture: while a stream captures, kernels (with their argument block), cudaMemcpyAsync and cudaMemsetAsync on it are recorded
//   instead of run; a graph launch replays the recording, in issue order, on the target stream.  An event recorded in a capturing
//   stream marks a point of that capture, and a stream that waits for it joins the capture.  A capturing stream cannot wait for an
//   event recorded outside it, and synchronizing or querying a capturing stream, or the device while anything captures, invalidates
//   the capture, as with a global-mode capture on a GPU.
//   IPC: a handle names an allocation (base + allocation id).  Opening it returns the allocation itself; closing its last opening
//   marks the range dead, and the graph build of the emulated launchers (nvl_emu_launch_graph.cpp) refuses kernels whose pointer
//   tables reach into a dead range (emu_range_dead).
#define cudaMalloc cudaMalloc_base
#define cudaFree cudaFree_base
#define cudaMemcpyAsync cudaMemcpyAsync_base
#define cudaMemsetAsync cudaMemsetAsync_base
#define cudaDeviceSynchronize cudaDeviceSynchronize_base
#define cudaStreamSynchronize cudaStreamSynchronize_base
#define cudaStreamQuery cudaStreamQuery_base
#define cudaStreamIsCapturing cudaStreamIsCapturing_base
#define cudaEventRecord cudaEventRecord_base
#define cudaEventQuery cudaEventQuery_base
#define cudaStreamWaitEvent cudaStreamWaitEvent_base
#define cudaIpcGetMemHandle cudaIpcGetMemHandle_base
#define cudaIpcOpenMemHandle cudaIpcOpenMemHandle_base
#define cudaIpcCloseMemHandle cudaIpcCloseMemHandle_base
#define cudaGetDriverEntryPoint cudaGetDriverEntryPoint_base
#define emu_stream_enqueue emu_stream_enqueue_base
#include "cudart_emu.cpp"
#undef cudaMalloc
#undef cudaFree
#undef cudaMemcpyAsync
#undef cudaMemsetAsync
#undef cudaDeviceSynchronize
#undef cudaStreamSynchronize
#undef cudaStreamQuery
#undef cudaStreamIsCapturing
#undef cudaEventRecord
#undef cudaEventQuery
#undef cudaStreamWaitEvent
#undef cudaIpcGetMemHandle
#undef cudaIpcOpenMemHandle
#undef cudaIpcCloseMemHandle
#undef cudaGetDriverEntryPoint
#undef emu_stream_enqueue
#include <set>

namespace {
struct EmuGraph { std::vector<std::function<void()>> nodes; };
struct EmuCapture { EmuGraph *g; bool invalidated = false; };

// all under g_lock
std::map<EmuStream *, EmuCapture *> g_capture;           // streams that capture (origin and joined)
std::set<EmuEvent *> g_captured_events;                  // last recorded in a capturing stream
std::map<uintptr_t, uint64_t> g_alloc_id;                // device allocation base -> allocation id
uint64_t g_alloc_ids;
std::map<uintptr_t, std::pair<size_t, long>> g_ipc;      // opened allocation base -> (size, open count)
std::map<uintptr_t, size_t> g_dead;                      // ranges whose last IPC mapping was closed
long g_ipc_opens, g_ipc_closes;

EmuCapture *capture_of(EmuStream *e) { std::lock_guard<std::mutex> l(g_lock); auto it = g_capture.find(e); return it == g_capture.end() ? nullptr : it->second; }
// 1: s captures, and f was recorded into its graph
bool record(cudaStream_t s, const std::function<void()> &f)
{
    std::lock_guard<std::mutex> l(g_lock);
    auto it = g_capture.find(S(s));
    if (it == g_capture.end()) return false;
    it->second->g->nodes.push_back(f);
    return true;
}
cudaError_t invalidate(EmuCapture *c) { c->invalidated = true; return fail(cudaErrorStreamCaptureUnsupported); }
}  // namespace

extern "C" void emu_stream_enqueue(cudaStream_t s, std::function<void()> *f) { if (!record(s, *f)) emu_stream_enqueue_base(s, f); }
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
cudaError_t cudaMalloc(void **p, size_t n)
{
    cudaError_t e = cudaMalloc_base(p, n);
    if (e == cudaSuccess) { std::lock_guard<std::mutex> l(g_lock); g_alloc_id[(uintptr_t)*p] = ++g_alloc_ids; g_dead.erase((uintptr_t)*p); }
    return e;
}
cudaError_t cudaFree(void *p) { { std::lock_guard<std::mutex> l(g_lock); g_alloc_id.erase((uintptr_t)p); g_dead.erase((uintptr_t)p); } return cudaFree_base(p); }
cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind k, cudaStream_t st)
{ return record(st, [=] { memmove(d, s, n); }) ? cudaSuccess : cudaMemcpyAsync_base(d, s, n, k, st); }
cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t st)
{ return record(st, [=] { memset(d, v, n); }) ? cudaSuccess : cudaMemsetAsync_base(d, v, n, st); }
cudaError_t cudaDeviceSynchronize(void)
{
    {
        std::lock_guard<std::mutex> l(g_lock);
        if (!g_capture.empty()) { for (auto &c : g_capture) c.second->invalidated = true; return fail(cudaErrorStreamCaptureUnsupported); }
    }
    return cudaDeviceSynchronize_base();
}
cudaError_t cudaStreamSynchronize(cudaStream_t s) { if (auto *c = capture_of(S(s))) return invalidate(c); return cudaStreamSynchronize_base(s); }
cudaError_t cudaStreamQuery(cudaStream_t s) { if (auto *c = capture_of(S(s))) return invalidate(c); return cudaStreamQuery_base(s); }
cudaError_t cudaStreamIsCapturing(cudaStream_t s, cudaStreamCaptureStatus *st)
{ auto *c = capture_of(S(s)); *st = !c ? cudaStreamCaptureStatusNone : c->invalidated ? cudaStreamCaptureStatusInvalidated : cudaStreamCaptureStatusActive; return cudaSuccess; }
cudaError_t cudaStreamBeginCapture(cudaStream_t s, cudaStreamCaptureMode)
{
    std::lock_guard<std::mutex> l(g_lock);
    auto *e = S(s);
    if (g_capture.count(e)) return fail(cudaErrorIllegalState);
    g_capture[e] = new EmuCapture{new EmuGraph()};
    return cudaSuccess;
}
// ends the capture of its origin stream s; streams that joined it stop capturing too
cudaError_t cudaStreamEndCapture(cudaStream_t s, cudaGraph_t *graph)
{
    std::lock_guard<std::mutex> l(g_lock);
    auto it = g_capture.find(S(s));
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
cudaError_t cudaGraphLaunch(cudaGraphExec_t exec, cudaStream_t s)
{ for (auto &f : reinterpret_cast<EmuGraph *>(exec)->nodes) { auto g = f; emu_stream_enqueue(s, &g); } return cudaSuccess; }
cudaError_t cudaGraphExecDestroy(cudaGraphExec_t exec) { delete reinterpret_cast<EmuGraph *>(exec); return cudaSuccess; }
cudaError_t cudaGraphDestroy(cudaGraph_t g) { delete reinterpret_cast<EmuGraph *>(g); return cudaSuccess; }
// (in issue order a replay needs no node for an event record or wait inside a capture)
cudaError_t cudaEventRecord(cudaEvent_t ev, cudaStream_t s)
{
    auto *e = reinterpret_cast<EmuEvent *>(ev);
    {
        std::lock_guard<std::mutex> l(g_lock);
        if (g_capture.count(S(s))) { g_captured_events.insert(e); return cudaSuccess; }
        g_captured_events.erase(e);
    }
    return cudaEventRecord_base(ev, s);
}
cudaError_t cudaEventQuery(cudaEvent_t ev)
{
    { std::lock_guard<std::mutex> l(g_lock); if (g_captured_events.count(reinterpret_cast<EmuEvent *>(ev))) return fail(cudaErrorStreamCaptureUnsupported); }
    return cudaEventQuery_base(ev);
}
cudaError_t cudaStreamWaitEvent(cudaStream_t s, cudaEvent_t ev, unsigned flags)
{
    {
        std::lock_guard<std::mutex> l(g_lock);
        auto *st = S(s);
        auto it = g_capture.find(st);
        if (g_captured_events.count(reinterpret_cast<EmuEvent *>(ev))) {
            if (it != g_capture.end()) return cudaSuccess;
            if (g_capture.empty()) return fail(cudaErrorStreamCaptureIsolation);
            g_capture[st] = g_capture.begin()->second;   // joins the capture (the tests keep one capture open when streams join)
            return cudaSuccess;
        }
        if (it != g_capture.end()) { it->second->invalidated = true; return fail(cudaErrorStreamCaptureIsolation); }
    }
    return cudaStreamWaitEvent_base(s, ev, flags);
}

cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t *h, void *p)
{
    std::lock_guard<std::mutex> l(g_lock);
    auto it = g_alloc_id.find((uintptr_t)p);
    if (it == g_alloc_id.end()) return fail(cudaErrorInvalidValue);
    memset(h, 0, sizeof(*h));
    uint64_t v[2] = {(uint64_t)(uintptr_t)p, it->second};
    memcpy(h->reserved, v, sizeof(v));
    return cudaSuccess;
}
cudaError_t cudaIpcOpenMemHandle(void **p, cudaIpcMemHandle_t h, unsigned)
{
    uint64_t v[2];
    memcpy(v, h.reserved, sizeof(v));
    std::lock_guard<std::mutex> l(g_lock);
    auto id = g_alloc_id.find((uintptr_t)v[0]);
    if (id == g_alloc_id.end() || id->second != v[1]) return fail(cudaErrorInvalidResourceHandle);   /* freed since the export */
    auto &o = g_ipc[(uintptr_t)v[0]];
    o.first = g_allocs[(uintptr_t)v[0]].first; o.second++;
    g_dead.erase((uintptr_t)v[0]);
    g_ipc_opens++;
    *p = (void *)(uintptr_t)v[0];
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

static int emu_mem_get_address_range(unsigned long long *base, size_t *len, unsigned long long ptr)   /* cuMemGetAddressRange: the allocation around ptr */
{
    std::lock_guard<std::mutex> l(g_lock);
    auto it = g_allocs.upper_bound((uintptr_t)ptr);
    if (it == g_allocs.begin()) return 1;   /* CUDA_ERROR_INVALID_VALUE */
    --it;
    if ((uintptr_t)ptr >= it->first + (it->second.first ? it->second.first : 1)) return 1;
    *base = it->first; *len = it->second.first;
    return 0;
}
cudaError_t cudaGetDriverEntryPoint(const char *name, void **fn, unsigned long long flags, cudaDriverEntryPointQueryResult *qr)
{
    if (!strcmp(name, "cuMemGetAddressRange")) { *fn = (void *)emu_mem_get_address_range; if (qr) *qr = cudaDriverEntryPointSuccess; return cudaSuccess; }
    return cudaGetDriverEntryPoint_base(name, fn, flags, qr);
}
}
