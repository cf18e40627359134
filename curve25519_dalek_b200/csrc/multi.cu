// multi.cu -- one MSM spanning several GPUs of one node from a SINGLE process (SURVEY 8b/8e): the seam a Rust
// caller of curve25519-dalek/src/backend.rs:79-97 would bind when it wants all GPUs behind one call.
//
// The pair range is cut into contiguous shards, one per device.  One host thread per device enqueues that shard's
// MSM (msm.cu pipeline, host input streamed in chunks) on the device's own context; each shard's record of window
// accumulators (W x 160 B + status word, ~2.7 KB) is written straight into the gather buffer on the first device
// with a peer copy over NVLink; the first device waits for the peers' events, adds the accumulators per window and
// runs the Horner pass (pippenger.rs:159).  No host bounce: the only read-back is the 192-byte result.  (With one
// process per GPU the same exchange is an NCCL all-gather on the engine's stream: curve25519_dalek_b200/sharding.py.)
#include <algorithm>
#include <new>
#include <thread>
#include <vector>

#include "../../include/dalek_b200.h"
#include "engine.h"

struct dalek_b200_multi {
    std::vector<dalek_b200_ctx *> ctx;
    std::vector<cudaEvent_t> done;         // shard r's record has landed in the gather buffer
    void *d_gather = nullptr;              // on ctx[0]'s device: ndev records
    size_t gather_cap = 0;
    std::string last_error;
};

extern "C" {

int dalek_b200_init_multi(const int *devices, int ndev, dalek_b200_multi **out)
{
    if (!out) return DALEK_E_INVALID_ARG;
    *out = nullptr;
    if (!devices || ndev < 1 || ndev > 64) return DALEK_E_INVALID_ARG;
    for (int i = 0; i < ndev; i++)
        for (int j = 0; j < i; j++) if (devices[i] == devices[j]) return DALEK_E_INVALID_ARG;
    dalek_b200_multi *m = new (std::nothrow) dalek_b200_multi();
    if (!m) return DALEK_E_NOMEM;
    for (int i = 0; i < ndev; i++) {
        dalek_b200_ctx *c = nullptr;
        int rc = dalek_b200_init(devices[i], &c);
        if (rc) { dalek_b200_destroy_multi(m); return rc; }
        m->ctx.push_back(c);
        cudaEvent_t e;
        if (cudaSetDevice(devices[i]) != cudaSuccess || cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) {
            dalek_b200_destroy_multi(m); return DALEK_E_CUDA;
        }
        m->done.push_back(e);
        if (i > 0) {                      // direct peer writes into the first device's gather buffer (NVLink)
            int can = 0;
            if (cudaDeviceCanAccessPeer(&can, devices[i], devices[0]) == cudaSuccess && can) {
                cudaError_t e2 = cudaDeviceEnablePeerAccess(devices[0], 0);
                if (e2 != cudaSuccess && e2 != cudaErrorPeerAccessAlreadyEnabled) { dalek_b200_destroy_multi(m); return DALEK_E_CUDA; }
                cudaGetLastError();
            }
        }
    }
    *out = m;
    return DALEK_OK;
}

void dalek_b200_destroy_multi(dalek_b200_multi *m)
{
    if (!m) return;
    for (size_t i = 0; i < m->ctx.size(); i++) {
        if (i < m->done.size()) { cudaSetDevice(m->ctx[i]->device); cudaEventDestroy(m->done[i]); }
    }
    if (m->d_gather && !m->ctx.empty()) { cudaSetDevice(m->ctx[0]->device); cudaFree(m->d_gather); }
    for (dalek_b200_ctx *c : m->ctx) dalek_b200_destroy(c);
    delete m;
}

int dalek_b200_multi_device_count(const dalek_b200_multi *m) { return m ? (int)m->ctx.size() : 0; }

dalek_b200_ctx *dalek_b200_multi_ctx(dalek_b200_multi *m, int i)
{
    return (m && i >= 0 && i < (int)m->ctx.size()) ? m->ctx[i] : nullptr;
}

const char *dalek_b200_multi_last_error(const dalek_b200_multi *m) { return m ? m->last_error.c_str() : "null handle"; }

int dalek_b200_edwards_vartime_msm_multi(dalek_b200_multi *m, const uint8_t *scalars, const void *points, int point_fmt,
                                         size_t n, uint8_t out_compressed[32], uint64_t out_limbs[20])
{
    if (!m || m->ctx.empty() || (n && (!scalars || !points)) ||
        (point_fmt != DALEK_POINTS_COMPRESSED && point_fmt != DALEK_POINTS_EXTENDED))
        return DALEK_E_INVALID_ARG;
    // small inputs are not worth the exchange: the first device alone
    int ndev = (int)m->ctx.size();
    if (n < ((size_t)ndev << 14)) ndev = 1;
    dalek_b200_ctx *c0 = m->ctx[0];
    if (ndev == 1) return dalek_b200_edwards_vartime_msm(c0, scalars, points, point_fmt, n, out_compressed, out_limbs);
    const size_t n_shard = (n + ndev - 1) / ndev;
    const size_t rec = dalek_b200_msm_partial_bytes(c0, n_shard);
    if (cudaSetDevice(c0->device) != cudaSuccess) return DALEK_E_CUDA;
    if (m->gather_cap < rec * ndev) {
        if (m->d_gather) cudaFree(m->d_gather);
        m->d_gather = nullptr; m->gather_cap = 0;
        if (cudaMalloc(&m->d_gather, rec * ndev) != cudaSuccess) { m->last_error = "cudaMalloc of the gather buffer failed"; return DALEK_E_NOMEM; }
        m->gather_cap = rec * ndev;
    }
    const size_t pin = msm_point_bytes(point_fmt);
    std::vector<int> rcs(ndev, 0);
    auto shard = [&](int r) {
        dalek_b200_ctx *c = m->ctx[r];
        const size_t base = n / ndev, rem = n % ndev;                 // contiguous shards, sizes differ by at most one
        const size_t lo = (size_t)r * base + std::min<size_t>(r, rem), cnt = base + ((size_t)r < rem ? 1 : 0);
        int rc = msm_partial_enqueue_record(c, scalars + 32 * lo, (const char *)points + pin * lo, false, point_fmt, cnt, n_shard,
                                            (char *)m->d_gather + rec * r, c0->device);
        if (!rc && cudaEventRecord(m->done[r], c->stream) != cudaSuccess) rc = DALEK_E_CUDA;
        c->async_open = false;                                         // the device span of this call is taken on ctx[0]
        rcs[r] = rc;
    };
    {
        std::vector<std::thread> th;
        for (int r = 1; r < ndev; r++) th.emplace_back(shard, r);
        shard(0);
        for (auto &t : th) t.join();
    }
    for (int r = 0; r < ndev; r++)
        if (rcs[r]) { m->last_error = std::string("shard ") + std::to_string(r) + ": " + m->ctx[r]->last_error; return rcs[r]; }
    if (cudaSetDevice(c0->device) != cudaSuccess) return DALEK_E_CUDA;
    for (int r = 1; r < ndev; r++)
        if (cudaStreamWaitEvent(c0->stream, m->done[r], 0) != cudaSuccess) return DALEK_E_CUDA;
    c0->async_open = true;                                             // ev_call0 was recorded by shard 0's enqueue
    int rc = msm_combine_records(c0, m->d_gather, true, rec, ndev, n_shard, out_compressed, out_limbs);
    if (rc < 0) m->last_error = c0->last_error;
    return rc;
}

}  // extern "C"
