// Band receiver (include/nrsc5_b200.h: nrsc5b_band_*): one handle that channelises a live wideband capture, scans every
// channel once per window, attaches an engine stream to every station the policy finds present, and routes each
// attached channel's samples from the window buffer into its stream.  Built only from the channeliser's streaming push,
// the scanner and the engine's feed seam (chan_feed.h); the one kernel of its own is k_band_route.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <deque>
#include <type_traits>
#include <vector>

#include "../../include/nrsc5_b200.h"
#include "chan_feed.h"
#include "chan_scan.h"

namespace {

constexpr int ROUTE_THREADS = 256;
constexpr long long SLACK = 32;                    // columns past W: one input sample emits at most 4 outputs (32 / D)
constexpr size_t ENGINE_INPUT = 4u << 20;          // cs16 bytes per engine stream: 4.4 MB FM windows (512 symbols) go in pieces
constexpr size_t ENGINE_LOG = 2u << 20;            // record bytes per engine stream between two drains

}  // namespace

struct RouteArgs {
    const int16_t *win;       // the window buffer [nch][2 cols]
    long long win_stride;     // int16 values per row
    long long col0;           // first sample of the rows to route
    long long n;              // samples per session
    int16_t *base;            // the engine's input buffers
    const long long *tab;     // [sessions][2]: channel row, destination (int16 values from base)
};

// V words (complex samples) per access: the run's head up to V-word alignment of the destination, V-word vectors, tail
template <int V>
__device__ __forceinline__ void copy_run(const uint32_t *__restrict__ src, uint32_t *__restrict__ dst, long long n)
{
    using Vec = typename std::conditional<V == 4, uint4, typename std::conditional<V == 2, uint2, uint32_t>::type>::type;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x, step = (long long)gridDim.x * blockDim.x;
    long long head = (long long)((V - (int)(((uintptr_t)dst >> 2) & (V - 1))) & (V - 1));
    if (head > n) head = n;
    const long long nv = (n - head) / V, tail0 = head + nv * V;
    if (t < head) dst[t] = src[t];
    if (t < n - tail0) dst[tail0 + t] = src[tail0 + t];
    const Vec *s = reinterpret_cast<const Vec *>(src + head);
    Vec *d = reinterpret_cast<Vec *>(dst + head);
    for (long long i = t; i < nv; i += step) d[i] = __ldg(s + i);
}

// grid (x: pieces of the run, y: sessions): session y's rows [col0, col0 + n) -> its engine stream
__global__ void __launch_bounds__(ROUTE_THREADS) k_band_route(RouteArgs a)
{
    const long long ch = a.tab[2 * blockIdx.y], at = a.tab[2 * blockIdx.y + 1];
    const uint32_t *src = reinterpret_cast<const uint32_t *>(a.win + ch * a.win_stride) + a.col0;
    uint32_t *dst = reinterpret_cast<uint32_t *>(a.base + at);
    const int sa = (int)(((uintptr_t)src >> 2) & 3), da = (int)(((uintptr_t)dst >> 2) & 3);
    if (sa == da) copy_run<4>(src, dst, a.n);
    else if (((sa ^ da) & 1) == 0) copy_run<2>(src, dst, a.n);
    else copy_run<1>(src, dst, a.n);
}

namespace {

// CUDA event pairs around one stage, read once the work has finished (after a synchronise)
struct StageTimer {
    std::vector<cudaEvent_t> pool;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> open;
    cudaEvent_t cur = nullptr;
    double ms = 0;
    cudaEvent_t get()
    {
        if (pool.empty()) {
            cudaEvent_t ev = nullptr;
            cudaEventCreate(&ev);
            return ev;
        }
        cudaEvent_t ev = pool.back();
        pool.pop_back();
        return ev;
    }
    void begin()
    {
        cur = get();
        cudaEventRecord(cur, nullptr);
    }
    void end()
    {
        cudaEvent_t b = get();
        cudaEventRecord(b, nullptr);
        open.push_back({cur, b});
    }
    void settle()
    {
        for (auto &p : open) {
            float t = 0;
            if (cudaEventSynchronize(p.second) == cudaSuccess && cudaEventElapsedTime(&t, p.first, p.second) == cudaSuccess) ms += t;
            pool.push_back(p.first);
            pool.push_back(p.second);
        }
        open.clear();
    }
    ~StageTimer()
    {
        for (auto &p : open) pool.push_back(p.first), pool.push_back(p.second);
        for (cudaEvent_t e : pool) cudaEventDestroy(e);
    }
};

enum { T_CHAN, T_SCAN, T_ROUTE, T_ENGINE };

struct Session {
    nrsc5b_band_session_t pub;
    std::vector<uint8_t> rec;   // records not taken yet
};

struct Window {
    long long index;
    std::vector<nrsc5b_scan_t> rows;
    std::vector<uint32_t> flags;
};

int plan_limit(int mode, int decim) { return mode == NRSC5B_MODE_AM ? 74 : decim == 32 ? 117 : decim == 16 ? 59 : 29; }

}  // namespace

struct nrsc5b_band {
    nrsc5b_band_config_t cfg;
    std::vector<int> offsets;
    int nch = 0;
    long long S = 0, W = 0, cols = 0;          // symbol, window and row length in samples
    int r = 0, tol = 0;                        // suppression: offset distance and timing tolerance (P / 2)
    nrsc5b_channelizer_t *chan = nullptr;
    nrsc5b_scanner_t *scan = nullptr;
    nrsc5b_engine_t *eng = nullptr;
    int16_t *d_win = nullptr;
    long long fill = 0, window = 0;            // samples in the window buffer, index of the window it holds
    bool ended = false;
    std::vector<int> open;                     // per channel: its open session, -1
    std::vector<int> absent;                   // per channel with an open session: consecutive windows not present
    std::vector<int> owner;                    // per engine stream: the session on it, -1
    std::vector<Session> sessions;
    std::deque<Window> windows;
    std::vector<uint8_t> drain_buf;
    long long *h_tab = nullptr, *d_tab = nullptr;
    cudaEvent_t tab_done = nullptr;
    StageTimer timer[4];
    unsigned long long route_bytes = 0;
};

static int bad_config(const nrsc5b_band_config_t *c, std::vector<int> *offs)
{
    if (!c) return 1;
    if (c->device < 0 || (c->mode != NRSC5B_MODE_FM && c->mode != NRSC5B_MODE_AM)) return 1;
    if (c->mode == NRSC5B_MODE_FM ? (c->decim != 8 && c->decim != 16 && c->decim != 32) : c->decim != 32) return 1;
    if (c->window_symbols < 32 || c->window_symbols > 512 || c->hold_windows < 1 || c->max_stations < 1 || c->max_stations > 4096)
        return 1;
    int lim = plan_limit(c->mode, c->decim);
    if (c->rate_hz) {
        int L = 0, M = 0, mo = 0;
        if (nrsc5b_chan_resampler_tables(c->mode, c->decim, c->rate_hz, &L, &M, &mo, nullptr) != NRSC5B_OK) return 1;
        if (mo > 0 && mo < lim) lim = mo;
    }
    offs->clear();
    if (!c->offsets) {
        if (c->nch != 0) return 1;
        for (int m = -lim; m <= lim; m++) offs->push_back(m);
        return 0;
    }
    if (c->nch <= 0 || c->nch > 4096) return 1;
    offs->assign(c->offsets, c->offsets + c->nch);
    std::vector<int> sorted(*offs);
    std::sort(sorted.begin(), sorted.end());
    for (int i = 0; i < c->nch; i++)
        if (sorted[i] < -lim || sorted[i] > lim || (i && sorted[i] == sorted[i - 1])) return 1;
    return 0;
}

extern "C" void nrsc5b_band_destroy(nrsc5b_band_t *b)
{
    if (!b) return;
    cudaSetDevice(b->cfg.device);
    cudaStreamSynchronize(nullptr);
    if (b->eng) nrsc5b_destroy(b->eng);
    if (b->scan) nrsc5b_scan_destroy(b->scan);
    if (b->chan) nrsc5b_chan_destroy(b->chan);
    cudaFree(b->d_win);
    cudaFree(b->d_tab);
    if (b->h_tab) cudaFreeHost(b->h_tab);
    if (b->tab_done) cudaEventDestroy(b->tab_done);
    delete b;
}

extern "C" int nrsc5b_band_create(nrsc5b_band_t **out, const nrsc5b_band_config_t *cfg)
{
    std::vector<int> offs;
    if (!out || bad_config(cfg, &offs)) return NRSC5B_EINVAL;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || cfg->device >= ndev) {
        fprintf(stderr, "nrsc5_b200: no usable CUDA device (the band receiver has no CPU path)\n");
        return NRSC5B_ENODEV;
    }
    if (cudaSetDevice(cfg->device) != cudaSuccess) return NRSC5B_ENODEV;
    nrsc5b_band *b = new nrsc5b_band();
    b->cfg = *cfg;
    b->cfg.offsets = nullptr;                  // the handle keeps its own copy
    b->offsets = offs;
    b->nch = (int)offs.size();
    const bool am = cfg->mode == NRSC5B_MODE_AM;
    b->S = am ? 270 : 2160;
    b->r = am ? 2 : 1;
    b->tol = am ? 7 : 56;
    b->W = (long long)cfg->window_symbols * b->S;
    b->cols = (b->W + SLACK + 3) & ~3LL;
    const int *po = b->offsets.data();
    int rc;
    if (cfg->rate_hz)
        rc = cfg->input_cs16 ? nrsc5b_chan_create_rate_cs16(&b->chan, cfg->device, cfg->mode, cfg->decim, cfg->rate_hz, po, b->nch)
                             : nrsc5b_chan_create_rate(&b->chan, cfg->device, cfg->mode, cfg->decim, cfg->rate_hz, po, b->nch);
    else if (am)
        rc = cfg->input_cs16 ? nrsc5b_chan_create_am_cs16(&b->chan, cfg->device, po, b->nch) : nrsc5b_chan_create_am(&b->chan, cfg->device, po, b->nch);
    else
        rc = cfg->input_cs16 ? nrsc5b_chan_create_fm_cs16(&b->chan, cfg->device, cfg->decim, po, b->nch)
                             : nrsc5b_chan_create_fm(&b->chan, cfg->device, cfg->decim, po, b->nch);
    if (!rc) rc = nrsc5b_scan_create(&b->scan, cfg->device, cfg->mode, b->nch);
    if (!rc) {
        nrsc5b_config_t ec{};
        ec.device = cfg->device;
        ec.nstreams = cfg->max_stations;
        ec.mode = cfg->mode;
        ec.input_capacity = ENGINE_INPUT;
        ec.log_capacity = ENGINE_LOG;
        ec.emit_soft = 0;
        ec.input_cs16 = 1;
        rc = nrsc5b_create(&b->eng, &ec);
        if (!rc && cfg->l2) rc = nrsc5b_enable_l2(b->eng, 1);
    }
    if (!rc) {
        const size_t S = (size_t)cfg->max_stations;
        bool ok = cudaMalloc(&b->d_win, (size_t)b->nch * b->cols * 4) == cudaSuccess &&
                  cudaMalloc(&b->d_tab, S * 2 * sizeof(long long)) == cudaSuccess &&
                  cudaHostAlloc(reinterpret_cast<void **>(&b->h_tab), S * 2 * sizeof(long long), cudaHostAllocDefault) == cudaSuccess &&
                  cudaEventCreateWithFlags(&b->tab_done, cudaEventDisableTiming) == cudaSuccess;
        if (!ok) rc = NRSC5B_ENOMEM;
    }
    if (rc) {
        nrsc5b_band_destroy(b);
        return rc;
    }
    b->open.assign(b->nch, -1);
    b->absent.assign(b->nch, 0);
    b->owner.assign(cfg->max_stations, -1);
    b->drain_buf.resize(ENGINE_LOG + 64);
    *out = b;
    return NRSC5B_OK;
}

// every open session's stream: run the engine, then move its records to the session (REC_L2's frame_off rebased to the
// session's buffer, so that a nrsc5b_band_records output reads like one nrsc5b_drain)
static int process_and_drain(nrsc5b_band *b)
{
    b->timer[T_ENGINE].begin();
    int rc = nrsc5b_process(b->eng);
    b->timer[T_ENGINE].end();
    if (rc) return rc;
    for (int s = 0; s < b->cfg.max_stations; s++) {
        if (b->owner[s] < 0) continue;
        Session &se = b->sessions[b->owner[s]];
        size_t need = 0;
        const long n = nrsc5b_drain(b->eng, s, b->drain_buf.data(), b->drain_buf.size(), &need);
        if (n < 0) return (int)n;
        if (nrsc5b_take_overflow(b->eng, s)) return NRSC5B_EOVERFLOW;
        const size_t base = se.rec.size();
        se.rec.insert(se.rec.end(), b->drain_buf.begin(), b->drain_buf.begin() + n);
        for (size_t off = base; off + 8 <= se.rec.size();) {
            uint32_t ty, len;
            memcpy(&ty, &se.rec[off], 4);
            memcpy(&len, &se.rec[off + 4], 4);
            if (ty == NRSC5B_REC_L2 && len >= 4) {
                uint32_t fo;
                memcpy(&fo, &se.rec[off + 8], 4);
                fo += (uint32_t)base;
                memcpy(&se.rec[off + 8], &fo, 4);
            }
            off += 8 + ((len + 3) & ~3u);
        }
    }
    b->timer[T_ENGINE].settle();
    return NRSC5B_OK;
}

// window columns [col0, col0 + n) of every open session's channel -> the end of its engine stream.  When a stream has
// no room even after trimming, the engine runs and the route tries again, in halves if need be: no sample is dropped.
static int route(nrsc5b_band *b, long long col0, long long n)
{
    std::vector<int> slots, chans;
    for (int s = 0; s < b->cfg.max_stations; s++)
        if (b->owner[s] >= 0) {
            slots.push_back(s);
            chans.push_back(b->sessions[b->owner[s]].pub.channel);
        }
    const int ns = (int)slots.size();
    if (!ns) return NRSC5B_OK;
    std::vector<long long> dst(ns);
    int dev, mode, cs16, nch;
    nbchan_info(b->chan, &dev, &mode, &cs16, &nch);
    while (n > 0) {
        long long piece = n;
        bool processed = false;
        FeedTarget t;
        for (;;) {
            const int rc = nbfeed_reserve(b->eng, dev, mode, slots.data(), ns, piece, &t, dst.data());
            if (rc == NRSC5B_OK) break;
            if (rc != NRSC5B_EFULL) return rc;
            if (!processed) {
                const int pc = process_and_drain(b);
                if (pc) return pc;
                processed = true;
            } else if (piece > 1) {
                piece = (piece + 1) / 2;
            } else {
                return NRSC5B_EFULL;
            }
        }
        if (cudaEventSynchronize(b->tab_done) != cudaSuccess) return NRSC5B_ECUDA;   // the table's last copy has run
        for (int i = 0; i < ns; i++) {
            b->h_tab[2 * i] = chans[i];
            b->h_tab[2 * i + 1] = dst[i];
        }
        if (cudaMemcpyAsync(b->d_tab, b->h_tab, (size_t)ns * 2 * sizeof(long long), cudaMemcpyHostToDevice, t.stream) != cudaSuccess ||
            cudaEventRecord(b->tab_done, t.stream) != cudaSuccess)
            return NRSC5B_ECUDA;
        RouteArgs a;
        a.win = b->d_win;
        a.win_stride = 2 * b->cols;
        a.col0 = col0;
        a.n = piece;
        a.base = t.base;
        a.tab = b->d_tab;
        long long gx = (piece + 4 * ROUTE_THREADS - 1) / (4 * ROUTE_THREADS);
        if (gx > 1024) gx = 1024;
        b->timer[T_ROUTE].begin();
        k_band_route<<<dim3((unsigned)gx, (unsigned)ns), ROUTE_THREADS, 0, t.stream>>>(a);
        b->timer[T_ROUTE].end();
        if (cudaGetLastError() != cudaSuccess) return NRSC5B_ECUDA;
        b->route_bytes += 8ull * (unsigned long long)piece * (unsigned long long)ns;   // read and written
        const int rc = nbfeed_commit(b->eng, slots.data(), ns, piece);
        if (rc) return rc;
        col0 += piece;
        n -= piece;
    }
    return NRSC5B_OK;
}

// closes the sessions on `slots` at channel sample n1: their streams have been processed and drained
static int close_sessions(nrsc5b_band *b, const std::vector<int> &slots, long long n1)
{
    for (int s : slots) {
        Session &se = b->sessions[b->owner[s]];
        se.pub.n1 = n1;
        se.pub.slot = -1;
        b->open[se.pub.channel] = -1;
        b->owner[s] = -1;
        const int rc = nrsc5b_reset(b->eng, s);
        if (rc) return rc;
    }
    return NRSC5B_OK;
}

static bool leakage(const nrsc5b_band *b, const std::vector<nrsc5b_scan_t> &rows, int k)
{
    for (int j = 0; j < b->nch; j++) {
        if (j == k || !rows[j].detected || std::abs(b->offsets[j] - b->offsets[k]) > b->r) continue;
        const bool stronger = rows[j].score > rows[k].score || (rows[j].score == rows[k].score && b->offsets[j] < b->offsets[k]);
        long long dt = std::llabs((long long)rows[j].timing - rows[k].timing) % b->S;
        if (b->S - dt < dt) dt = b->S - dt;
        if (stronger && dt <= b->tol) return true;
    }
    return false;
}

// the full window in the buffer: its verdict, the policy, the route, the engine
static int complete_window(nrsc5b_band *b)
{
    Window w;
    w.index = b->window;
    w.rows.resize(b->nch);
    w.flags.assign(b->nch, 0);
    b->timer[T_SCAN].begin();
    int rc = nrsc5b_scan_push_device(b->scan, b->d_win, 2 * b->cols, b->W, nullptr);
    if (!rc) rc = nrsc5b_scan_result(b->scan, w.rows.data(), nullptr);
    if (!rc) rc = nrsc5b_scan_reset(b->scan);
    b->timer[T_SCAN].end();
    if (rc) return rc;
    b->timer[T_CHAN].settle();
    b->timer[T_SCAN].settle();
    std::vector<char> present(b->nch, 0);
    for (int k = 0; k < b->nch; k++) {
        if (!w.rows[k].detected) continue;
        w.flags[k] |= NRSC5B_BAND_DETECTED;
        if (leakage(b, w.rows, k)) w.flags[k] |= NRSC5B_BAND_LEAKAGE;
        else present[k] = 1;
    }
    // detach: hold_windows windows in a row without the station; the session ends where its last routed window ends
    std::vector<int> closing;
    for (int k = 0; k < b->nch; k++) {
        if (b->open[k] < 0) continue;
        b->absent[k] = present[k] ? 0 : b->absent[k] + 1;
        if (b->absent[k] >= b->cfg.hold_windows) closing.push_back(b->sessions[b->open[k]].pub.slot);
    }
    if (!closing.empty()) {
        if ((rc = process_and_drain(b)) || (rc = close_sessions(b, closing, b->window * b->W))) return rc;
    }
    // attach, in channel order, to the lowest free stream; the session starts with this window
    for (int k = 0; k < b->nch; k++) {
        if (!present[k] || b->open[k] >= 0) continue;
        int s = 0;
        while (s < b->cfg.max_stations && b->owner[s] >= 0) s++;
        if (s == b->cfg.max_stations) {
            w.flags[k] |= NRSC5B_BAND_NO_SLOT;
            continue;
        }
        Session se;
        memset(&se.pub, 0, sizeof(se.pub));
        se.pub.id = (int)b->sessions.size();
        se.pub.channel = k;
        se.pub.offset = b->offsets[k];
        se.pub.slot = s;
        se.pub.n0 = b->window * b->W;
        se.pub.n1 = -1;
        se.pub.window = b->window;
        se.pub.verdict = w.rows[k];
        b->owner[s] = se.pub.id;
        b->open[k] = se.pub.id;
        b->absent[k] = 0;
        b->sessions.push_back(std::move(se));
    }
    for (int k = 0; k < b->nch; k++)
        if (b->open[k] >= 0) w.flags[k] |= NRSC5B_BAND_ATTACHED;
    if ((rc = route(b, 0, b->W)) || (rc = process_and_drain(b))) return rc;
    b->timer[T_ROUTE].settle();
    b->windows.push_back(std::move(w));
    // outputs past W (a rate stage's last sample may emit several) start the next window
    const long long extra = b->fill - b->W;
    if (extra > 0 && cudaMemcpy2DAsync(b->d_win, (size_t)b->cols * 4, b->d_win + 2 * b->W, (size_t)b->cols * 4, (size_t)extra * 4, b->nch,
                                       cudaMemcpyDeviceToDevice, nullptr) != cudaSuccess)
        return NRSC5B_ECUDA;
    b->fill = extra;
    b->window++;
    return NRSC5B_OK;
}

extern "C" int nrsc5b_band_push(nrsc5b_band_t *b, const void *capture, size_t nvalues)
{
    if (!b || b->ended || (nvalues & 1) || (nvalues && !capture)) return NRSC5B_EINVAL;
    if (!nvalues) return NRSC5B_OK;
    if (cudaSetDevice(b->cfg.device) != cudaSuccess) return NRSC5B_ENODEV;
    const long long total = (long long)(nvalues / 2);
    const size_t bps = b->cfg.input_cs16 ? 4 : 2;
    for (long long done = 0; done < total;) {
        // the longest piece that does not pass the window's end (outputs grow with the piece); at least one sample
        const long long room = b->W - b->fill;
        long long lo = 0, hi = total - done;
        while (lo < hi) {
            const long long mid = lo + (hi - lo + 1) / 2;
            if (nbchan_outputs_after(b->chan, mid) <= room) lo = mid;
            else hi = mid - 1;
        }
        if (lo == 0) lo = 1;
        if (b->fill + nbchan_outputs_after(b->chan, lo) > b->cols) return NRSC5B_ECUDA;   // cannot happen: SLACK bounds it
        const void *src = reinterpret_cast<const uint8_t *>(capture) + bps * done;
        long long nout = 0;
        int16_t *at = b->d_win + 2 * b->fill;
        b->timer[T_CHAN].begin();
        int rc = b->cfg.input_cs16
                     ? nrsc5b_chan_push_cs16(b->chan, reinterpret_cast<const int16_t *>(src), 2 * (size_t)lo, at, 2 * b->cols, nullptr, &nout)
                     : nrsc5b_chan_push(b->chan, reinterpret_cast<const uint8_t *>(src), 2 * (size_t)lo, at, 2 * b->cols, nullptr, &nout);
        b->timer[T_CHAN].end();
        if (rc) return rc;
        b->fill += nout;
        done += lo;
        if (b->fill >= b->W && (rc = complete_window(b))) return rc;
    }
    // the channeliser reads page-locked and device input by an asynchronous copy: wait for it, so that the caller may
    // reuse its buffer as soon as the call returns (and read the channelise stage's events while at it)
    if (cudaStreamSynchronize(nullptr) != cudaSuccess) return NRSC5B_ECUDA;
    b->timer[T_CHAN].settle();
    return NRSC5B_OK;
}

extern "C" int nrsc5b_band_flush(nrsc5b_band_t *b)
{
    if (!b) return NRSC5B_EINVAL;
    if (b->ended) return NRSC5B_OK;
    if (cudaSetDevice(b->cfg.device) != cudaSuccess) return NRSC5B_ENODEV;
    int rc;
    if ((rc = route(b, 0, b->fill)) || (rc = process_and_drain(b))) return rc;
    std::vector<int> all;
    for (int s = 0; s < b->cfg.max_stations; s++)
        if (b->owner[s] >= 0) all.push_back(s);
    if ((rc = close_sessions(b, all, b->window * b->W + b->fill))) return rc;
    b->timer[T_CHAN].settle();
    b->timer[T_ROUTE].settle();
    b->ended = true;
    return NRSC5B_OK;
}

extern "C" int nrsc5b_band_windows(nrsc5b_band_t *b, int64_t *index, nrsc5b_scan_t *rows, uint32_t *flags, int cap, int *pending)
{
    if (!b || cap < 0) return NRSC5B_EINVAL;
    if (pending) *pending = (int)b->windows.size();
    int n = 0;
    for (; n < cap && !b->windows.empty(); n++) {
        const Window &w = b->windows.front();
        if (index) index[n] = w.index;
        if (rows) memcpy(rows + (size_t)n * b->nch, w.rows.data(), (size_t)b->nch * sizeof(nrsc5b_scan_t));
        if (flags) memcpy(flags + (size_t)n * b->nch, w.flags.data(), (size_t)b->nch * sizeof(uint32_t));
        b->windows.pop_front();
    }
    return n;
}

extern "C" int nrsc5b_band_sessions(nrsc5b_band_t *b, nrsc5b_band_session_t *out, int cap, int *n)
{
    if (!b || cap < 0 || (cap && !out)) return NRSC5B_EINVAL;
    const int total = (int)b->sessions.size();
    if (n) *n = total;
    const int w = cap < total ? cap : total;
    for (int i = 0; i < w; i++) out[i] = b->sessions[i].pub;
    return w;
}

extern "C" long nrsc5b_band_records(nrsc5b_band_t *b, int id, uint8_t *out, size_t cap, size_t *needed)
{
    if (!b || id < 0 || id >= (int)b->sessions.size()) return NRSC5B_EINVAL;
    Session &se = b->sessions[id];
    const size_t avail = se.rec.size();
    if (needed) *needed = avail;
    if (avail == 0 || !out || cap < avail) return avail == 0 ? 0 : NRSC5B_EFULL;
    memcpy(out, se.rec.data(), avail);
    se.rec.clear();
    if (se.pub.n1 >= 0) std::vector<uint8_t>().swap(se.rec);   // a closed session gets no more: free its buffer
    return (long)avail;
}

extern "C" int nrsc5b_band_channels(nrsc5b_band_t *b, int *offsets, int *nch)
{
    if (!b) return NRSC5B_EINVAL;
    if (nch) *nch = b->nch;
    if (offsets) memcpy(offsets, b->offsets.data(), (size_t)b->nch * sizeof(int));
    return NRSC5B_OK;
}

extern "C" int nrsc5b_band_times(nrsc5b_band_t *b, double *ms4, unsigned long long *route_bytes)
{
    if (!b) return NRSC5B_EINVAL;
    if (cudaSetDevice(b->cfg.device) != cudaSuccess || cudaStreamSynchronize(nullptr) != cudaSuccess) return NRSC5B_ECUDA;
    for (int i = 0; i < 4; i++) {
        b->timer[i].settle();
        if (ms4) ms4[i] = b->timer[i].ms;
    }
    if (route_bytes) *route_bytes = b->route_bytes;
    return NRSC5B_OK;
}
