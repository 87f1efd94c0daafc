/* rec_store_bench.cu -- how fast can the lane kernel's recorder write its rings, by store pattern.
 *
 * Footprint of bench.py's record mode (configs[1]): 65 536 writers in 64-thread blocks, one per lane, each owning
 * a 16 KB ring of 16 B event records (record_cap 1 024), a 2 KB ring of 16 B Sink samples and a 1 KB ring of
 * 8 B service times (sample_cap = service_cap = 128).  Every writer starts at a seeded random 128 B line of
 * its ring and wraps.  By default each pattern writes what one bench step writes (3.96e10 events:
 * 634 GB of records, 126 GB of samples + service times).
 *
 * Records are staged as in the lane kernel: every loop iteration each lane puts 3..6 records (a chain) into
 * shared-memory staging and a lane holding a full group of 8 (one 128 B line) has it written out:
 *   P0     the owner lane writes its line itself, 8 x st.global.cs.v4 from its [row][lane] staging column
 *          (each warp store instruction sends up to 32 16 B pieces to 32 lines);
 *   P1a    warp-cooperative: the owners are found by ballot; each store instruction writes 4 whole lines,
 *          lanes 8k..8k+7 the 8 rows of owner k (a quarter-warp reads one staging column: 8-way bank conflict);
 *   P1b    as P1a with lane l on owner l % 4, row l / 4 (a quarter-warp reads 2 rows of 4 owners);
 *   P2     Hopper bulk copy: the owner lane issues one cp.async.bulk.global.shared::cta of its 128 B from a
 *          contiguous per-lane [lane][row] staging slice (P2w: 256 B groups of 16 records, 32 rows);
 * and, for the Sink-sample / service-time streams (data from registers, no staging): each writer owns a 2 KB
 * sample ring and a 1 KB service ring and fills them in the ratio of the bytes they get (a chunk of a third of
 * the volume goes to the service ring: chunks 0, 1 of every three to the samples, chunk 2 to the service times):
 *   P3s    each lane writes one 32 B sector per iteration, as two 16 B halves;
 *   P3w    each lane writes one 64 B chunk per iteration, as four 16 B stores;
 *   P3q    warp-cooperative 64 B chunks: a writer has a chunk ready in about 3 of 16 iterations (the lane kernel's
 *          rate: about one Sink sample and one service start per two loop iterations), the ready writers
 *          (owners) are found by ballot, and each store instruction writes 8 owners' chunks, 4 lanes x 16 B each;
 *   P3l    as P3q with whole 128 B lines, 4 owners per store instruction, 8 lanes x 16 B each (as P1b), a chunk
 *          ready in about 3 of 32 iterations;
 *   P4     ceiling: a fully coalesced sequential write of the record volume over the same 1 GB.
 * Every pattern writes the same bytes to the same places (P0/P1/P2 record rings are checksummed against each
 * other).  GB/s = bytes written / device time (CUDA events), best and median of --reps runs, the patterns
 * interleaved run by run.  P2 and P2w need more shared memory than the lane kernel has to spare (padding), so
 * their figures bound what a bulk-copy flush could reach, not what fits.
 *
 *   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o rec_store_bench rec_store_bench.cu
 *   ./rec_store_bench [--events 3.96e10] [--reps 5] [--seed 1]       (tools/rec_store_bench.py builds and runs it) */
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { \
    fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); exit(1); } } while (0)

constexpr int THREADS = 64;
constexpr uint32_t REC_CAP = 1024, SMP_CAP = 128, SVC_CAP = 64;  /* 16 B slots: 16 KB record, 2 KB sample and 1 KB
                                                                    service rings */
constexpr uint32_t FULL = 0xffffffffu;

__device__ __forceinline__ uint32_t mix(uint32_t x)
{
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16; return x;
}
__device__ __forceinline__ void st_cs(void *p, const uint4 a)
{
    asm volatile("st.global.cs.v4.b32 [%0], {%1,%2,%3,%4};" :: "l"(p), "r"(a.x), "r"(a.y), "r"(a.z), "r"(a.w) : "memory");
}
/* the i-th record of writer w: the same value whichever pattern writes it */
__device__ __forceinline__ uint4 rec_value(uint32_t w, uint32_t i) { return make_uint4(w, i, mix(w * 4099u + i), ~i); }
/* records of the chain a writer runs at iteration it: 3..6 */
__device__ __forceinline__ uint32_t chain_len(uint32_t w, uint32_t it) { return 3u + (mix(w ^ (it * 0x9e3779b9u)) & 3u); }

enum { P0 = 0, P1A, P1B, P2, P2W };

/* P0 / P1a / P1b / P2 / P2w: `groups` whole groups per writer, staged chain by chain, flushed as they fill */
template <int PAT>
__global__ void __launch_bounds__(THREADS) k_records(uint4 *__restrict__ rec, const uint32_t *__restrict__ start_line,
                                                     uint32_t groups)
{
    constexpr uint32_t FL = (PAT == P2W) ? 16u : 8u;                 /* records per flush                    */
    constexpr uint32_t ST = 2u * FL;                                  /* staged rows                          */
    constexpr bool LANE_MAJOR = (PAT == P2 || PAT == P2W);            /* [lane][row] (+1 row padding) for bulk */
    constexpr uint32_t LSTRIDE = ST + 1u;
    __shared__ __align__(128) uint4 sh[LANE_MAJOR ? THREADS * LSTRIDE : ST * THREADS];
    const uint32_t tid = threadIdx.x, lane = tid & 31u, wbase = tid & ~31u;
    const uint32_t w = blockIdx.x * THREADS + tid;
    uint4 *ring = rec + (size_t)w * REC_CAP;
    uint32_t pos = start_line[w] * 8u;                                /* ring slot of record st_fl            */
    const uint32_t total = groups * FL;
    uint32_t st_wr = 0, st_fl = 0;
    auto slot = [&](uint32_t row) -> uint4 & { return LANE_MAJOR ? sh[tid * LSTRIDE + row] : sh[row * THREADS + tid]; };
    for (uint32_t it = 0; __any_sync(FULL, st_fl < total); ++it) {
        if (LANE_MAJOR) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
        const uint32_t n = min(chain_len(w, it), total - st_wr);
        for (uint32_t j = 0; j < n; ++j) slot((st_wr + j) % ST) = rec_value(w, st_wr + j);
        st_wr += n;
        const bool full = (st_wr - st_fl) >= FL;
        if (PAT == P0) {
            if (full) {
                const uint32_t r0 = st_fl % ST;
#pragma unroll
                for (uint32_t g = 0; g < FL; ++g) st_cs(ring + pos + g, sh[(r0 + g) * THREADS + tid]);
            }
        } else if (PAT == P1A || PAT == P1B) {
            __syncwarp();
            uint32_t m = __ballot_sync(FULL, full);
            const uint32_t k = (PAT == P1A) ? lane >> 3 : lane & 3u;    /* which of the round's 4 owners     */
            const uint32_t row = (PAT == P1A) ? lane & 7u : lane >> 2;  /* which record of its group          */
            const uint32_t my_row0 = st_fl % ST;
            while (m) {
                /* the k-th lowest owner still in m (or none) */
                uint32_t mm = m, owner = 32u;
#pragma unroll
                for (uint32_t q = 0; q < 4; ++q) {
                    const uint32_t o = mm ? (uint32_t)__ffs(mm) - 1u : 32u;
                    if (q == k) owner = o;
                    mm &= mm - 1u;
                }
                const uint32_t src = owner < 32u ? owner : lane;
                const uint32_t o_pos = __shfl_sync(FULL, pos, src);
                const uint32_t o_row0 = __shfl_sync(FULL, my_row0, src);
                if (owner < 32u) {
                    const uint32_t ow = blockIdx.x * THREADS + wbase + owner;
                    st_cs(rec + (size_t)ow * REC_CAP + o_pos + row, sh[(o_row0 + row) * THREADS + wbase + owner]);
                }
                m = mm;
            }
            __syncwarp();
        } else {
            if (full) {
                const uint32_t s = (uint32_t)__cvta_generic_to_shared(&sh[tid * LSTRIDE + st_fl % ST]);
                asm volatile("fence.proxy.async.shared::cta;\n\t"
                             "cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;\n\t"
                             "cp.async.bulk.commit_group;" :: "l"(ring + pos), "r"(s), "n"(FL * 16) : "memory");
            }
        }
        if (full) { st_fl += FL; pos = (pos + FL) % REC_CAP; }
    }
    if (LANE_MAJOR) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

/* P3s / P3w: `chunks` chunks of B bytes per writer into its 2 KB sample and 1 KB service ring, scattered, data from
 * registers */
template <uint32_t B>
__global__ void __launch_bounds__(THREADS) k_sectors(uint4 *__restrict__ smp, uint4 *__restrict__ svc,
                                                     const uint32_t *__restrict__ start_line, uint32_t chunks)
{
    const uint32_t w = blockIdx.x * THREADS + threadIdx.x;
    uint4 *const ring_s = smp + (size_t)w * SMP_CAP, *const ring_v = svc + (size_t)w * SVC_CAP;
    constexpr uint32_t E = B / 16u;
    uint32_t pos_s = (start_line[w] * 8u) % SMP_CAP, pos_v = (start_line[w] * 8u) % SVC_CAP;
    for (uint32_t c = 0; c < chunks; ++c) {
        const bool v = (c % 3u == 2u);
        uint4 *const p = v ? ring_v + pos_v : ring_s + pos_s;
#pragma unroll
        for (uint32_t j = 0; j < E; ++j) st_cs(p + j, rec_value(w, c * E + j));
        if (v) pos_v = (pos_v + E) % SVC_CAP; else pos_s = (pos_s + E) % SMP_CAP;
    }
}

/* P3q / P3l: `chunks` chunks of B bytes per writer into the same rings, written by the warp: the owners of a round
 * are found by ballot, lane l moves 16 B piece l / C of the chunk of the (l % C)-th owner, C = 512 / B owners per
 * store instruction; only the owner's ring position crosses lanes */
template <uint32_t B>
__global__ void __launch_bounds__(THREADS) k_coop(uint4 *__restrict__ smp, uint4 *__restrict__ svc,
                                                  const uint32_t *__restrict__ start_line, uint32_t chunks)
{
    constexpr uint32_t E = B / 16u, C = 32u / E;
    const uint32_t tid = threadIdx.x, lane = tid & 31u, wbase = blockIdx.x * THREADS + (tid & ~31u);
    const uint32_t w = blockIdx.x * THREADS + tid;
    uint32_t pos_s = (start_line[w] * 8u) % SMP_CAP, pos_v = (start_line[w] * 8u) % SVC_CAP;
    uint32_t c = 0;                                              /* chunks written so far */
    const uint32_t k = lane % C, piece = lane / C;
    for (uint32_t it = 0; __any_sync(FULL, c < chunks); ++it) {
        const bool ready = c < chunks && (mix(w ^ (it * 0x9e3779b9u)) & 31u) < (B == 64u ? 6u : 3u);
        const bool v = (c % 3u == 2u);
        const uint32_t my = v ? (1u << 31) | pos_v : pos_s;     /* ring select + slot */
        uint32_t owners = __ballot_sync(FULL, ready);
        while (owners) {
            const uint32_t owner = min(__fns(owners, 0u, (int)k + 1), 32u);
            uint32_t rest = owners;
#pragma unroll
            for (uint32_t q = 0; q < C; ++q) rest &= rest - 1u;
            const uint32_t src = owner < 32u ? owner : lane;
            const uint32_t o_my = __shfl_sync(FULL, my, src), o_c = __shfl_sync(FULL, c, src);
            if (owner < 32u) {
                const uint32_t ow = wbase + owner;
                uint4 *base = (o_my >> 31) ? svc + (size_t)ow * SVC_CAP : smp + (size_t)ow * SMP_CAP;
                st_cs(base + (o_my & 0x7fffffffu) + piece, rec_value(ow, o_c * E + piece));
            }
            owners = rest;
        }
        if (ready) {
            if (v) pos_v = (pos_v + E) % SVC_CAP; else pos_s = (pos_s + E) % SMP_CAP;
            c++;
        }
    }
}

/* P4: the record volume as one fully coalesced sequential sweep over the 1 GB of record rings */
__global__ void __launch_bounds__(THREADS) k_sequential(uint4 *__restrict__ rec, size_t slot_mask, size_t n_writes)
{
    const size_t stride = (size_t)gridDim.x * THREADS;
    for (size_t i = (size_t)blockIdx.x * THREADS + threadIdx.x; i < n_writes; i += stride)
        st_cs(rec + (i & slot_mask), make_uint4((uint32_t)i, (uint32_t)(i >> 32), 0u, ~(uint32_t)i));
}

__global__ void k_checksum(const uint4 *__restrict__ rec, size_t n, unsigned long long *out)
{
    unsigned long long s = 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint4 v = rec[i];
        s += (unsigned long long)mix(v.x ^ mix(v.y ^ mix(v.z ^ mix(v.w ^ (uint32_t)i))));
    }
    atomicAdd(out, s);
}

int main(int argc, char **argv)
{
    double events = 3.96e10;          /* one bench step: 65 536 replicas x 1e4 sim-s of M/M/1 (rate 8, mean 0.1)  */
    int reps = 5;
    uint32_t seed = 1;
    for (int i = 1; i + 1 < argc; i += 2) {
        if (!strcmp(argv[i], "--events")) events = atof(argv[i + 1]);
        else if (!strcmp(argv[i], "--reps")) reps = atoi(argv[i + 1]);
        else if (!strcmp(argv[i], "--seed")) seed = (uint32_t)atoi(argv[i + 1]);
        else { fprintf(stderr, "usage: %s [--events E] [--reps R] [--seed S]\n", argv[0]); return 2; }
    }
    const uint32_t W = 65536, blocks = W / THREADS;
    /* per event 16 B of record; per request (7.55 events) one 16 B Sink sample and one 8 B service time */
    const double requests = events / 7.55;
    const uint32_t groups = (uint32_t)(events / W / 8.0 + 0.5);               /* 128 B record groups per writer */
    const uint32_t sectors = (uint32_t)(requests * 24.0 / W / 32.0 + 0.5);    /* sample + service bytes, in 32 B */

    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    printf("# device: %s, %d SMs, %.0f MHz max SM clock, L2 %d MB\n", prop.name, prop.multiProcessorCount,
           prop.clockRate / 1e3, prop.l2CacheSize >> 20);
    printf("# %u writers x (16 KB + 2 KB + 1 KB) rings, seeded random start lines (seed %u); %.3g events: %u record groups "
           "and %u sample/service sectors per writer\n", W, seed, events, groups, sectors);

    uint4 *rec = nullptr, *smp = nullptr, *svc = nullptr;
    uint32_t *start = nullptr;
    unsigned long long *sum = nullptr;
    CK(cudaMalloc(&rec, (size_t)W * REC_CAP * 16));
    CK(cudaMalloc(&smp, (size_t)W * SMP_CAP * 16));
    CK(cudaMalloc(&svc, (size_t)W * SVC_CAP * 16));
    CK(cudaMalloc(&start, W * 4));
    CK(cudaMalloc(&sum, 8));
    std::vector<uint32_t> h(W);
    uint64_t s = 0x9e3779b97f4a7c15ull * (seed + 1);
    for (auto &x : h) { s ^= s << 13; s ^= s >> 7; s ^= s << 17; x = (uint32_t)(s % (REC_CAP / 8)); }
    CK(cudaMemcpy(start, h.data(), W * 4, cudaMemcpyHostToDevice));

    struct Pat { const char *name, *what; double bytes; bool checksum; };
    const double rec_bytes = (double)W * groups * 128.0, sec_bytes = (double)W * sectors * 32.0;
    std::vector<Pat> pats = {
        {"P0", "owner lane, 8 x st.global.cs.v4 per 128 B line", rec_bytes, true},
        {"P1a", "warp-cooperative, 4 lines per store, lanes 8k..8k+7 on one line", rec_bytes, true},
        {"P1b", "warp-cooperative, 4 lines per store, lane l on line l%4", rec_bytes, true},
        {"P2", "owner lane, cp.async.bulk 128 B from [lane][row] staging (+1 KB smem)", rec_bytes, true},
        {"P2w", "owner lane, cp.async.bulk 256 B from [lane][row] staging (+17 KB smem)", (double)W * (groups / 2) * 256.0, true},
        {"P3s", "scattered 32 B sectors, two 16 B halves (sample/service pattern)", sec_bytes, false},
        {"P3w", "scattered 64 B chunks, four 16 B stores", (double)W * (sectors / 2) * 64.0, false},
        {"P3q", "warp-cooperative 64 B chunks, 8 chunks per store, 4 lanes x 16 B each", (double)W * (sectors / 2) * 64.0, false},
        {"P3l", "warp-cooperative 128 B lines, 4 lines per store, 8 lanes x 16 B each", (double)W * (sectors / 4) * 128.0, false},
        {"P4", "fully coalesced sequential write (ceiling)", rec_bytes, false},
    };
    auto launch = [&](int p) {
        switch (p) {
        case 0: k_records<P0><<<blocks, THREADS>>>(rec, start, groups); break;
        case 1: k_records<P1A><<<blocks, THREADS>>>(rec, start, groups); break;
        case 2: k_records<P1B><<<blocks, THREADS>>>(rec, start, groups); break;
        case 3: k_records<P2><<<blocks, THREADS>>>(rec, start, groups); break;
        case 4: k_records<P2W><<<blocks, THREADS>>>(rec, start, groups / 2); break;
        case 5: k_sectors<32><<<blocks, THREADS>>>(smp, svc, start, sectors); break;
        case 6: k_sectors<64><<<blocks, THREADS>>>(smp, svc, start, sectors / 2); break;
        case 7: k_coop<64><<<blocks, THREADS>>>(smp, svc, start, sectors / 2); break;
        case 8: k_coop<128><<<blocks, THREADS>>>(smp, svc, start, sectors / 4); break;
        case 9: k_sequential<<<blocks, THREADS>>>(rec, (size_t)W * REC_CAP - 1, (size_t)W * groups * 8); break;
        }
        CK(cudaGetLastError());
    };
    const int np = (int)pats.size();
    std::vector<std::vector<float>> ms(np);
    std::vector<unsigned long long> sums(np, 0);
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    for (int p = 0; p < np; ++p) {                       /* warm-up, and the record rings' checksum per pattern */
        launch(p);
        CK(cudaDeviceSynchronize());
        if (pats[p].checksum) {
            CK(cudaMemset(sum, 0, 8));
            k_checksum<<<1024, 256>>>(rec, (size_t)W * REC_CAP, sum);
            CK(cudaMemcpy(&sums[p], sum, 8, cudaMemcpyDeviceToHost));
        }
    }
    for (int r = 0; r < reps; ++r)
        for (int p = 0; p < np; ++p) {
            CK(cudaEventRecord(e0));
            launch(p);
            CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1));
            float t;
            CK(cudaEventElapsedTime(&t, e0, e1));
            ms[p].push_back(t);
        }
    printf("%-4s %9s %9s %9s %9s %7s  %s\n", "pat", "GB", "best_ms", "best_GB/s", "med_GB/s", "vs_P0", "what");
    double p0 = 0.0;
    for (int p = 0; p < np; ++p) {
        std::vector<float> v = ms[p];
        std::sort(v.begin(), v.end());
        const double best = pats[p].bytes / (v.front() * 1e-3) / 1e9, med = pats[p].bytes / (v[v.size() / 2] * 1e-3) / 1e9;
        if (p == 0) p0 = best;
        printf("%-4s %9.1f %9.2f %9.1f %9.1f %7.2f  %s\n", pats[p].name, pats[p].bytes / 1e9, v.front(), best, med,
               best / p0, pats[p].what);
    }
    bool same = true;
    for (int p = 1; p < 4; ++p) same &= sums[p] == sums[0];
    printf("# record rings identical across P0/P1a/P1b/P2: %s\n", same ? "yes" : "NO");
    CK(cudaFree(rec)); CK(cudaFree(smp)); CK(cudaFree(svc)); CK(cudaFree(start)); CK(cudaFree(sum));
    return same ? 0 : 1;
}
