// wprep.cu - weight preparation shared by the tensor-core convolution kernels.
//   conv weights [Co][Ci][kh*kw] (Conv2d: mode 0 gathers x, output channel n = co;  DGRAD / ConvTranspose2d:
//   mode 1 gathers dy, output channel n = ci) -> wp[2][N][Kp]: the K order of the consuming kernel, each value
//   split into its tf32 rounding (copy 0) and the remainder (copy 1).
//   A block stages the weights of a few output channels in shared memory with coalesced reads (mode 0: one
//   contiguous run; mode 1: one run of nb*KK floats per gathered channel) and writes full rows of wp.
#include "ccb_common.cuh"

#ifndef CCB_CPU_SIM
#include <vector>
namespace ccb {

__device__ __forceinline__ bool wprep_decode(const WPrepDesc& a, int k, int& slot, int& c) {
    slot = k / a.p0;                                  // k = slot * cpad + c
    c = k - slot * a.p0;
    return slot < a.ntaps && c < a.Cc;
}

__device__ __forceinline__ void wprep_block(const WPrepDesc& a, int nb, int block, float* sw) {
    const int n0 = block * nb;
    const int nn = min(nb, a.N - n0);
    const int row = a.Cc * a.KK;                          // staged floats per output channel
    if (a.mode == 0) {
        const float* src = a.w + (long long)n0 * row;     // [nn][Cc][KK] is one contiguous run
        for (int i = threadIdx.x; i < nn * row; i += 256) sw[i] = __ldg(src + i);
    } else {
        const int seg = nn * a.KK;                        // per gathered channel: [nn][KK] contiguous
        for (int i = threadIdx.x; i < a.Cc * seg; i += 256) {
            const int c = i / seg, r = i - c * seg;
            sw[i] = __ldg(a.w + ((long long)c * a.Ci + n0) * a.KK + r);
        }
    }
    __syncthreads();
    const long long plane = (long long)a.N * a.Kp;
    // a thread owns k positions and walks the staged output channels: the (slot, channel) decode - integer divisions -
    // runs once per k, not once per element, and consecutive threads write consecutive k (coalesced)
    for (int k = threadIdx.x; k < a.Kp; k += 256) {
        int slot, c;
        const bool valid = wprep_decode(a, k, slot, c);
        const int tap = valid ? a.tap_index[slot] : 0;
        const int base = valid ? ((a.mode == 0) ? c * a.KK + tap : c * nn * a.KK + tap) : 0;
        const int step = (a.mode == 0) ? a.Cc * a.KK : a.KK;
        for (int nl = 0; nl < nn; ++nl) {
            const float v = valid ? sw[base + nl * step] : 0.f;
            uint32_t hb;
            asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hb) : "f"(v));
            const float h = __uint_as_float(hb);
            const long long o = (long long)(n0 + nl) * a.Kp + k;
            a.wp[o] = h;
            uint32_t lb;                                   // the remainder rounded to tf32 as well: the hardware reads it exactly
            asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lb) : "f"(v - h));
            a.wp[plane + o] = __uint_as_float(lb);
        }
    }
}

__global__ void __launch_bounds__(256) wprep_staged_kernel(const WPrepDesc a, int nb) {
    CCB_PDL_WAIT();
    extern __shared__ float sw[];
    wprep_block(a, nb, blockIdx.x, sw);
}

// Every prepared copy of a weight cache in ONE launch: block -> (entry, block inside the entry) through a table.
struct WCacheEntry {
    WPrepDesc d;
    int nb, first_block;
};
__global__ void __launch_bounds__(256) wprep_all_kernel(const WCacheEntry* __restrict__ entries, const int* __restrict__ block_entry) {
    CCB_PDL_WAIT();
    extern __shared__ float sw[];
    __shared__ WPrepDesc sd;
    __shared__ int s_nb, s_first;
    const int e = block_entry[blockIdx.x];
    {
        const int* src = (const int*)&entries[e].d;
        int* dst = (int*)&sd;
        for (int i = threadIdx.x; i < (int)(sizeof(WPrepDesc) / 4); i += 256) dst[i] = src[i];
        if (threadIdx.x == 0) { s_nb = entries[e].nb; s_first = entries[e].first_block; }
    }
    __syncthreads();
    wprep_block(sd, s_nb, blockIdx.x - s_first, sw);
}

static int wprep_nb(const WPrepDesc& d) {
    const long long row_bytes = (long long)d.Cc * d.KK * 4;
    int nb = (int)((64 * 1024) / (row_bytes > 0 ? row_bytes : 1));
    if (nb > 8) nb = 8;
    if (nb < 1) nb = 1;
    // keep enough blocks in flight
    while (nb > 1 && cdiv(d.N, nb) < NUM_SMS) nb >>= 1;
    return nb;
}

int launch_wprep(const WPrepDesc& d, cudaStream_t st) {
    const long long row_bytes = (long long)d.Cc * d.KK * 4;
    CCB_REQUIRE(row_bytes <= 96 * 1024, CCB_ERR_UNSUPPORTED, "wprep: %d x %d weights per output channel do not fit shared memory", d.Cc, d.KK);
    const int nb = wprep_nb(d);
    const int smem = (int)(nb * row_bytes);
    static bool attr_set = false;
    if (!attr_set) {
        cudaFuncSetAttribute(wprep_staged_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
        attr_set = true;
    }
    CCB_LAUNCH(wprep_staged_kernel, dim3((unsigned)cdiv(d.N, nb)), dim3(256), smem, st, d, nb);
    return check_launch("wprep");
}

// ---------------------------------------------------------------------------------------------------------------
// Weight cache (opt-in, one per trainer): the prepared copies only change when the weights do, i.e. once per optimiser
// step - not once per convolution call.  While RECORDING, every prepared layout a conv launch asks for is noted
// (and still produced on the spot); after commit the launches get a pointer into the caller's persistent buffer and
// ccb_wcache_refresh() re-prepares every copy in one launch (the trainer runs it right after Adam).
// ---------------------------------------------------------------------------------------------------------------
struct WCache {
    std::vector<WCacheEntry> entries;
    std::vector<long long> offs;
    std::vector<int> block_entry;
    int state = 0;                 // 0 recording, 1 committed
    float* buf = nullptr;
    long long buf_floats = 0;
    WCacheEntry* d_entries = nullptr;
    int* d_block_entry = nullptr;
    int max_smem = 0;
    long long hits = 0, misses = 0;
};
thread_local WCache* g_cur_wcache = nullptr;

static bool wprep_same(const WPrepDesc& a, const WPrepDesc& b) {
    return a.w == b.w && a.N == b.N && a.Cc == b.Cc && a.KK == b.KK && a.Ci == b.Ci && a.mode == b.mode && a.Kp == b.Kp &&
           a.ntaps == b.ntaps && a.layout == b.layout && a.p0 == b.p0 && a.p1 == b.p1 && a.p2 == b.p2 &&
           memcmp(a.tap_index, b.tap_index, sizeof(a.tap_index)) == 0;
}

// The prepared copy of d.w in d's layout: out of the active weight cache when it holds one, else produced now in d.wp.
int wprep_get(const WPrepDesc& d, cudaStream_t st, const float** out) {
    WCache* c = g_cur_wcache;
    if (c) {
        for (size_t i = 0; i < c->entries.size(); ++i)
            if (wprep_same(c->entries[i].d, d)) {
                if (c->state == 1) { ++c->hits; *out = c->buf + c->offs[i]; return CCB_OK; }
                c = nullptr;       // recorded already, cache not committed yet
                break;
            }
        if (c && c->state == 0) {
            WCacheEntry e;
            memset(&e, 0, sizeof(e));
            e.d = d; e.d.wp = nullptr; e.nb = wprep_nb(d);
            c->entries.push_back(e);
        } else if (c) {
            ++c->misses;
        }
    }
    *out = d.wp;
    return launch_wprep(d, st);
}

}  // namespace ccb

using namespace ccb;

extern "C" void* ccb_wcache_create(void) { return new WCache(); }
extern "C" void ccb_wcache_destroy(void* h) { delete (WCache*)h; }
extern "C" long long ccb_wcache_plan_floats(void* h) {
    WCache* c = (WCache*)h;
    long long tot = 0;
    c->offs.clear();
    for (auto& e : c->entries) {
        c->offs.push_back(tot);
        tot += (2ll * e.d.N * e.d.Kp + 63) / 64 * 64;          // 256-byte aligned copies
    }
    return tot;
}
extern "C" long long ccb_wcache_table_bytes(void* h) {
    WCache* c = (WCache*)h;
    long long blocks = 0;
    for (auto& e : c->entries) blocks += cdiv(e.d.N, e.nb);
    return (long long)c->entries.size() * sizeof(WCacheEntry) + blocks * 4 + 256;
}
extern "C" int ccb_wcache_commit(void* h, float* buf, long long buf_floats, void* table, long long table_bytes, ccb_stream_t stream) {
    WCache* c = (WCache*)h;
    CCB_REQUIRE(c && buf && table, CCB_ERR_ARG, "wcache_commit: bad argument");
    CCB_REQUIRE(buf_floats >= ccb_wcache_plan_floats(h) && table_bytes >= ccb_wcache_table_bytes(h), CCB_ERR_ARG, "wcache_commit: buffers too small");
    c->block_entry.clear();
    c->max_smem = 0;
    for (size_t i = 0; i < c->entries.size(); ++i) {
        WCacheEntry& e = c->entries[i];
        e.d.wp = buf + c->offs[i];
        e.first_block = (int)c->block_entry.size();
        for (int b = 0; b < cdiv(e.d.N, e.nb); ++b) c->block_entry.push_back((int)i);
        const int smem = (int)((long long)e.nb * e.d.Cc * e.d.KK * 4);
        if (smem > c->max_smem) c->max_smem = smem;
    }
    const size_t eb = (c->entries.size() * sizeof(WCacheEntry) + 255) / 256 * 256;
    c->d_entries = (WCacheEntry*)table;
    c->d_block_entry = (int*)((char*)table + eb);
    cudaMemcpyAsync(c->d_entries, c->entries.data(), c->entries.size() * sizeof(WCacheEntry), cudaMemcpyHostToDevice, (cudaStream_t)stream);
    cudaMemcpyAsync(c->d_block_entry, c->block_entry.data(), c->block_entry.size() * 4, cudaMemcpyHostToDevice, (cudaStream_t)stream);
    cudaStreamSynchronize((cudaStream_t)stream);                // the host vectors may be reallocated later
    c->buf = buf; c->buf_floats = buf_floats; c->state = 1;
    return check_launch("wcache_commit");
}
extern "C" int ccb_wcache_refresh(void* h, ccb_stream_t stream) {
    WCache* c = (WCache*)h;
    CCB_REQUIRE(c && c->state == 1, CCB_ERR_ARG, "wcache_refresh: cache not committed");
    if (c->block_entry.empty()) return CCB_OK;
    cudaFuncSetAttribute(wprep_all_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
    CCB_LAUNCH(wprep_all_kernel, dim3((unsigned)c->block_entry.size()), dim3(256), c->max_smem, stream, (const WCacheEntry*)c->d_entries,
               (const int*)c->d_block_entry);
    return check_launch("wcache_refresh");
}
extern "C" void ccb_wcache_stats(void* h, long long* out4) {
    WCache* c = (WCache*)h;
    out4[0] = (long long)c->entries.size(); out4[1] = c->hits; out4[2] = c->misses; out4[3] = c->state;
}
#else
extern "C" void* ccb_wcache_create(void) { return nullptr; }
extern "C" void ccb_wcache_destroy(void*) {}
extern "C" long long ccb_wcache_plan_floats(void*) { return 0; }
extern "C" long long ccb_wcache_table_bytes(void*) { return 0; }
extern "C" int ccb_wcache_commit(void*, float*, long long, void*, long long, ccb_stream_t) { return CCB_ERR_UNSUPPORTED; }
extern "C" int ccb_wcache_refresh(void*, ccb_stream_t) { return CCB_ERR_UNSUPPORTED; }
extern "C" void ccb_wcache_stats(void*, long long* out4) { out4[0] = out4[1] = out4[2] = out4[3] = 0; }
#endif
