// Sweep-and-prune broad phase on the device.  Replaces collect_collision_pairs / sweep_and_prune
// (src/collision/broad_phase.rs:343-487).
//
// The reference keeps the intervals in a persistent Vec, insertion-sorts it by aabb.min.x every step (a STABLE sort:
// it swaps only on strict '>'; broad_phase.rs:383,479-487) and sweeps i<j with a break on min.x[j] > max.x[i].
// The emitted pairs are ordered by (rank of i, rank of j) in that sorted array.  Device plan, bit-exact with it:
//   1. key = order-preserving integer image of min.x with -0.0 canonicalised to +0.0 (they compare equal in the
//      reference), value = position in the persistent order;
//   2. hand-written stable LSD radix sort, 8-bit digits: per-tile digit histogram -> single-block exclusive scan ->
//      stable scatter ranked with warp match/ballot (4 passes for f32 keys, 8 for f64);
//   3. gather the interval columns into sorted SoA arrays (coalesced for the sweep);
//   4. per interval i: upper bound of max.x[i] in the sorted min.x = the reference's `break` position;
//   5. candidate search through a (y, z) cell grid under the x-sorted ranks (broadphase_cells.cuh): count pass, exclusive scan,
//      emit pass into a (rank i, rank j) buffer, per-interval segment sort by j, materialisation of the ABI columns.  Intervals
//      with a huge x-window (a ground slab) are swept brute force by sweep_wide_kernel, one block per 4 096 candidates.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "avn_math.cuh"
#include "context.hpp"

#include "device_prims.cuh"

namespace avn {
namespace {

template <class S> struct KeyOf;
template <> struct KeyOf<float> { using type = uint32_t; static constexpr int passes = 4; };
template <> struct KeyOf<double> { using type = uint64_t; static constexpr int passes = 8; };

__device__ __forceinline__ uint32_t sortable(float f) {
    uint32_t b = __float_as_uint(f);
    if (b == 0x80000000u) b = 0;  // -0.0 == +0.0 for the reference's comparison
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ uint64_t sortable(double f) {
    uint64_t b = (uint64_t)__double_as_longlong(f);
    if (b == 0x8000000000000000ull) b = 0;
    return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
}

// Also raises *nonfinite when any component of an AABB is NaN or infinite: the reference drops such intervals in update_aabb_intervals
// (broad_phase.rs:243-245); here the host then compacts the columns and runs again (Broadphase::drop_nonfinite), the common case pays one
// flag per step.
template <class S>
__global__ void make_keys(const S* __restrict__ aabb_min, const S* __restrict__ aabb_max, int n, typename KeyOf<S>::type* __restrict__ keys,
                          uint32_t* __restrict__ vals, unsigned long long* __restrict__ nonfinite) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const S a = aabb_min[3 * i], b = aabb_min[3 * i + 1], c = aabb_min[3 * i + 2], d = aabb_max[3 * i], e = aabb_max[3 * i + 1], f = aabb_max[3 * i + 2];
        // x - x is 0 for finite x and NaN for NaN / +-inf
        const S z = (a - a) + (b - b) + (c - c) + (d - d) + (e - e) + (f - f);
        if (!(z == S(0))) *nonfinite = 1ull;
        keys[i] = sortable(a);
        vals[i] = uint32_t(i);
    }
}

// sorted SoA for the sweep
template <class S>
struct Sweep {
    int n;
    const S* minx; const S* maxx;          // [n]
    const Vec4<S>* yz;                     // [n] {min.y, max.y, min.z, max.z}
    const uint4* meta;                     // [n] {collider, body, memberships, filters}
    const uint8_t* flags;                  // [n]
    const int* end;                        // [n] first j with min.x[j] > max.x[i]
    const uint8_t* is_wide;                // [n] 1: handled by sweep_wide_kernel (more than SW_WIDE candidates)
    const uint64_t* existing; uint64_t existing_mask;   // open-addressing hash set of PairKey (0 = empty; keys stored +1)
    const uint64_t* jdis; uint64_t jdis_mask;
};

template <class S>
__global__ void gather_sorted(const uint32_t* __restrict__ order, int n, const S* __restrict__ mn, const S* __restrict__ mx,
                              const uint32_t* __restrict__ collider, const uint32_t* __restrict__ body, const uint32_t* __restrict__ memberships,
                              const uint32_t* __restrict__ filters, const uint8_t* __restrict__ flags, S* __restrict__ minx, S* __restrict__ maxx,
                              Vec4<S>* __restrict__ yz, uint4* __restrict__ meta, uint8_t* __restrict__ sflags) {
    int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    uint32_t p = order[r];
    minx[r] = mn[3 * p];
    maxx[r] = mx[3 * p];
    yz[r] = mk4<S>(mn[3 * p + 1], mx[3 * p + 1], mn[3 * p + 2], mx[3 * p + 2]);
    meta[r] = make_uint4(collider[p], body[p], memberships ? memberships[p] : 1u, filters ? filters[p] : 0xFFFFFFFFu);
    sflags[r] = flags ? flags[p] : uint8_t(AVN_AABB_GENERATE_CONSTRAINTS);
}

// end[i] = first j > i with min.x[j] > max.x[i]  (the `break` of broad_phase.rs:390-392)
// Intervals with more than SW_WIDE x-candidates whose (y, z) footprint also covers more than 32 cells (a ground slab under the
// whole scene) go to a list that sweep_wide_kernel sweeps brute force, one block per SW_SUB candidates.
constexpr int SW_WIDE = 4096;
constexpr int SW_WIDE_CAP = 1 << 14;   // intervals beyond the cap stay in the tiled sweep (correct, only slower)
template <class S> struct CellGrid;
template <class S> __device__ __forceinline__ long long query_cell_count(const CellGrid<S>& g, Vec4<S> yi);
template <class S>
__global__ void sweep_bounds(const S* __restrict__ minx, const S* __restrict__ maxx, const Vec4<S>* __restrict__ yz, const CellGrid<S>* __restrict__ grid,
                             int n, int* __restrict__ end, int* __restrict__ wide_list, int* __restrict__ wide_count, uint8_t* __restrict__ is_wide,
                             const uint8_t* __restrict__ sflags) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (sflags[i] & AVN_AABB_HALO) {  // a halo interval never starts a sweep: empty window
        end[i] = i + 1;
        is_wide[i] = 0;
        return;
    }
    S m = maxx[i];
    int lo = i + 1, hi = n;
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (minx[mid] > m) hi = mid; else lo = mid + 1;
    }
    end[i] = lo;
    uint8_t wide = 0;
    // wide = a large x-window AND a (y, z) footprint well beyond the 3x3 cells of a small interval: one 16-lane group would have to
    // walk a large part of the window through many cell lists, so the interval is swept brute force by whole blocks instead
    if (lo - i - 1 > SW_WIDE && query_cell_count(*grid, yz[i]) > 32) {
        int slot = atomicAdd(wide_count, 1);
        if (slot < SW_WIDE_CAP) { wide_list[slot] = i; wide = 1; }
    }
    is_wide[i] = wide;
}

__device__ __forceinline__ uint64_t pair_key(uint32_t a, uint32_t b) {  // data_structures/pair_key.rs:15-21
    return a < b ? (uint64_t(a) << 32) | b : (uint64_t(b) << 32) | a;
}

// the non-geometric filters of broad_phase.rs:405-428 for a candidate (i, j) that overlaps on all three axes
template <class S>
__device__ __forceinline__ bool pair_filters(const Sweep<S>& s, uint4 mi, uint32_t fi, int j, uint32_t& pair_flags, uint4& mj) {
    mj = s.meta[j];
    uint32_t fj = s.flags[j];
    bool interacts = (mi.z & mj.w) != 0 && (mj.z & mi.w) != 0;  // CollisionLayers::interacts_with, layers.rs:423-426
    if ((fi & fj & AVN_AABB_IS_INACTIVE) || !interacts || mi.y == mj.y) return false;
    if ((fj & AVN_AABB_NOT_J) || ((fi & AVN_AABB_SPLIT_I) && (fj & AVN_AABB_HALO))) return false;  // x-slab partition (include/avian_b200.h)
    if (s.existing && hash_contains(s.existing, s.existing_mask, pair_key(mi.x, mj.x))) return false;
    if (s.jdis && hash_contains(s.jdis, s.jdis_mask, pair_key(mi.y, mj.y))) return false;
    uint32_t u = fi | fj;
    pair_flags = ((u & AVN_AABB_CONTACT_EVENTS) ? AVN_PAIR_CONTACT_EVENTS : 0u) | ((u & AVN_AABB_MODIFY_CONTACTS) ? AVN_PAIR_MODIFY_CONTACTS : 0u) |
                 ((u & AVN_AABB_GENERATE_CONSTRAINTS) ? AVN_PAIR_GENERATE_CONSTRAINTS : 0u) | ((u & AVN_AABB_CUSTOM_FILTER) ? AVN_PAIR_NEEDS_HOOK : 0u);
    return true;
}

constexpr int SW_THREADS = 256, SW_WARPS = SW_THREADS / 32;

// Wide intervals: the candidate range of interval i is cut into sub-ranges of SW_SUB candidates, one block each
// (blockIdx.x = sub-range, blockIdx.y strides the wide list).  Count pass: sub_counts[w * nsub + s]; wide_finish turns them
// into per-sub-range offsets and counts[i]; the emit pass starts each block at offsets[i] + sub_off.  Inside a block the 256
// lanes take 256 consecutive candidates per round and the 8 warp ballots are combined through shared memory, so the j order
// is kept.
constexpr int SW_SUB = 4096;
template <class S, bool EMIT>
__global__ void __launch_bounds__(SW_THREADS) sweep_wide_kernel(const __grid_constant__ Sweep<S> s, const int* __restrict__ wide_list,
                                                                const int* __restrict__ wide_count, uint32_t* __restrict__ sub_counts, int nsub,
                                                                const uint64_t* __restrict__ offsets, uint2* __restrict__ pairs, uint64_t capacity) {
    __shared__ uint32_t s_warp_cnt[SW_WARPS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nw = min(*wide_count, SW_WIDE_CAP);
    for (int w = blockIdx.y; w < nw; w += gridDim.y) {
        const int i = wide_list[w], e = s.end[i];
        if (EMIT && offsets[i + 1] == offsets[i]) continue;   // block-uniform: the count pass found nothing for this interval
        const int sub = blockIdx.x;
        const int jb = i + 1 + sub * SW_SUB, je = min(e, jb + SW_SUB);
        if (jb >= e) { if (!EMIT && threadIdx.x == 0) sub_counts[w * nsub + sub] = 0; continue; }
        const Vec4<S> yi = s.yz[i];
        const uint4 mi = s.meta[i];
        const uint32_t fi = s.flags[i];
        uint64_t running = EMIT ? offsets[i] + sub_counts[w * nsub + sub] : 0ull;   // (emit pass: sub_counts holds exclusive offsets)
        uint32_t total = 0;
        for (int j0 = jb; j0 < je; j0 += SW_THREADS) {
            const int j = j0 + threadIdx.x;
            bool ok = j < je;
            if (ok) {
                const Vec4<S> yj = s.yz[j];
                ok = !(yi.x > yj.y || yi.y < yj.x) && !(yi.z > yj.w || yi.w < yj.z);
            }
            uint32_t pf = 0;
            uint4 mj = make_uint4(0, 0, 0, 0);
            if (ok) ok = pair_filters(s, mi, fi, j, pf, mj);
            const uint32_t bal = __ballot_sync(0xffffffffu, ok);
            if (lane == 0) s_warp_cnt[warp] = __popc(bal);
            __syncthreads();
            uint32_t before = 0, round_total = 0;
#pragma unroll
            for (int k = 0; k < SW_WARPS; ++k) {
                const uint32_t c = s_warp_cnt[k];
                if (k < warp) before += c;
                round_total += c;
            }
            if (EMIT && ok) {
                const uint64_t at = running + before + __popc(bal & ((1u << lane) - 1u));
                if (at < capacity) pairs[at] = make_uint2(uint32_t(i), uint32_t(j));
            }
            running += round_total;
            total += round_total;
            __syncthreads();
        }
        if (!EMIT && threadIdx.x == 0) sub_counts[w * nsub + sub] = total;
    }
}
// per wide interval: exclusive scan of its sub-range counts (in place) and its total into counts[i]
__global__ void wide_finish(const int* __restrict__ wide_list, const int* __restrict__ wide_count, uint32_t* __restrict__ sub_counts, int nsub,
                            uint32_t* __restrict__ counts) {
    const int nw = min(*wide_count, SW_WIDE_CAP);
    for (int w = blockIdx.x * blockDim.x + threadIdx.x; w < nw; w += gridDim.x * blockDim.x) {
        uint32_t run = 0;
        for (int k = 0; k < nsub; ++k) {
            uint32_t c = sub_counts[w * nsub + k];
            sub_counts[w * nsub + k] = run;
            run += c;
        }
        counts[wide_list[w]] = run;
    }
}

}  // namespace
}  // namespace avn
#include "broadphase_cells.cuh"
namespace avn {
namespace {

template <class S>
class Broadphase final : public BroadphaseBase {
    using K = typename KeyOf<S>::type;

   public:
    Broadphase(cudaStream_t stream, ErrorSink* err, int device) : stream_(stream), err_(err) {
        cudaDeviceProp prop;
        if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) sm_count_ = prop.multiProcessorCount;
        cudaEventCreate(&ev0_);
        cudaEventCreate(&ev1_);
        cudaHostAlloc(&h_total_, 2 * sizeof(uint64_t), cudaHostAllocDefault);   // [0] pair count, [1] non-finite flag
        const char* g = getenv("AVN_BP_GRAPH");
        use_graph_ = !(g && !strcmp(g, "0"));
    }
    ~Broadphase() override {
        cudaEventDestroy(ev0_);
        cudaEventDestroy(ev1_);
        if (h_total_) cudaFreeHost(h_total_);
        if (graph_exec_) cudaGraphExecDestroy(graph_exec_);
    }
    AvnStatus upload(AvnAabbColumns* a) override;
    AvnStatus run() override;
    AvnStatus download(AvnPairList* out) override;
    AvnStatus device_pairs(DevicePairs* out) override;
    AvnStatus download_order(uint64_t* out_pair_count) override;
    void set_existing_device(const uint64_t* table, uint64_t mask) override { ext_existing_ = table; ext_existing_mask_ = mask; }
    void timings(AvnTimings* t) const override { *t = tm_; }

   private:
    template <class T> AvnStatus up(DevBuf& buf, const void* host, size_t count, const T** dev) {
        *dev = nullptr;
        if (!host || count == 0) return AVN_OK;
        AVN_CUDA(buf.ensure(count * sizeof(T)));
        AVN_CUDA(cudaMemcpyAsync(buf.p, host, count * sizeof(T), cudaMemcpyHostToDevice, stream_));
        *dev = buf.as<T>();
        return AVN_OK;
    }
    AvnStatus build_set(DevBuf& keys_buf, DevBuf& table_buf, const uint64_t* host_keys, uint64_t count, const uint64_t** table, uint64_t* mask);
    static constexpr int WIDE_ROWS = 64;
    uint32_t graph_replays_ = 0;
    Sweep<S> sweep_desc() const {
        Sweep<S> sw;
        sw.n = n_; sw.minx = s_minx_.as<S>(); sw.maxx = s_maxx_.as<S>(); sw.yz = s_yz_.as<Vec4<S>>(); sw.meta = s_meta_.as<uint4>();
        sw.flags = s_flags_.as<uint8_t>(); sw.end = s_end_.as<int>(); sw.is_wide = wide_flag_.as<uint8_t>();
        sw.existing = d_existing_; sw.existing_mask = existing_mask_; sw.jdis = d_jdis_; sw.jdis_mask = jdis_mask_;
        return sw;
    }
    CellSweep<S> cell_desc() const {
        CellSweep<S> cs;
        cs.grid = grid_.as<CellGrid<S>>(); cs.cranks = cv0_.as<uint32_t>(); cs.cstart = cbounds_.as<int>(); cs.cend = cbounds_.as<int>() + 0x10000;
        cs.capacity = pair_capacity_;
        return cs;
    }
    AvnStatus ensure_buffers(int n);
    void enqueue_front(int n);          // every launch from make_keys to the pair-count readback: no allocation, no synchronisation
    AvnStatus drop_nonfinite();
    AvnStatus settle();                 // waits for the run; reruns it for dropped non-finite intervals / a grown pair capacity
    AvnStatus finish_download();        // persistent order + timings to the host
    const uint64_t* ext_existing_ = nullptr; uint64_t ext_existing_mask_ = 0;   // the contact store's pair set (device)

    // The front part of a run is a fixed sequence of ~25 small launches: captured once into a CUDA graph and replayed as long
    // as the interval count and every buffer address stay the same (buffers are grow-only, so a steady scene replays forever).
    struct GraphKey {
        int n = -1;
        const void* p[24] = {};
        uint64_t m[2] = {};
        bool operator==(const GraphKey& o) const { return n == o.n && !memcmp(p, o.p, sizeof p) && !memcmp(m, o.m, sizeof m); }
    };
    GraphKey graph_key() const;
    bool use_graph_ = true;
    cudaGraphExec_t graph_exec_ = nullptr;
    GraphKey graph_key_{};
    uint32_t front_launches_ = 0;
    DevBuf nf_flag_;
    // update_aabb_intervals' retain (broad_phase.rs:243-245): set when non-finite intervals were dropped from this upload
    bool dropped_ = false;
    std::vector<uint32_t> keep_;        // compacted row -> row of the caller's columns
    std::vector<unsigned char> c_min_, c_max_;
    std::vector<uint32_t> c_col_, c_body_, c_memb_, c_filt_;
    std::vector<uint8_t> c_flags_;

    cudaStream_t stream_;
    ErrorSink* err_;
    int sm_count_ = 132;
    cudaEvent_t ev0_, ev1_;
    uint64_t* h_total_ = nullptr;
    AvnTimings tm_{};
    uint32_t launches_ = 0, upload_launches_ = 0;
    bool uploaded_ = false, ran_ = false;
    int n_ = 0;
    uint64_t pair_capacity_ = 0;
    AvnAabbColumns host_{};
    AvnAabbColumns* caller_ = nullptr;   // retained_count is written back at download
    const S* d_min_ = nullptr; const S* d_max_ = nullptr;
    const uint32_t* d_collider_ = nullptr; const uint32_t* d_body_ = nullptr; const uint32_t* d_memb_ = nullptr; const uint32_t* d_filt_ = nullptr;
    const uint8_t* d_flags_ = nullptr;
    const uint64_t* d_existing_ = nullptr; uint64_t existing_mask_ = 0;
    const uint64_t* d_jdis_ = nullptr; uint64_t jdis_mask_ = 0;
    DevBuf b_min_, b_max_, b_col_, b_body_, b_memb_, b_filt_, b_flags_, b_exk_, b_ext_, b_jdk_, b_jdt_;
    DevBuf k0_, k1_, v0_, v1_, hist_;
    DevBuf s_minx_, s_maxx_, s_yz_, s_meta_, s_flags_, s_end_, counts_, offsets_, block_sums_, wide_, wide_sub_, wide_flag_, grid_, ck0_, ck1_, cv0_, cv1_, cbounds_, pairs_, stats_, stats2_;
    DevBuf o_c1_, o_c2_, o_b1_, o_b2_, o_fl_;
    uint32_t* d_order_ = nullptr;
};

template <class S>
AvnStatus Broadphase<S>::build_set(DevBuf& keys_buf, DevBuf& table_buf, const uint64_t* host_keys, uint64_t count, const uint64_t** table, uint64_t* mask) {
    *table = nullptr;
    *mask = 0;
    if (!host_keys || count == 0) return AVN_OK;
    uint64_t cap = 64;
    while (cap < count * 2) cap <<= 1;
    const uint64_t* dkeys;
    AvnStatus st = up<uint64_t>(keys_buf, host_keys, count, &dkeys);
    if (st != AVN_OK) return st;
    AVN_CUDA(table_buf.ensure(cap * sizeof(uint64_t)));
    AVN_CUDA(cudaMemsetAsync(table_buf.p, 0, cap * sizeof(uint64_t), stream_));
    hash_insert<<<unsigned((count + 255) / 256), 256, 0, stream_>>>(dkeys, count, table_buf.as<uint64_t>(), cap - 1);
    ++launches_;
    *table = table_buf.as<uint64_t>();
    *mask = cap - 1;
    return AVN_OK;
}

template <class S>
AvnStatus Broadphase<S>::upload(AvnAabbColumns* a) {
    if (!a) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "aabbs is required");
    if (a->count && (!a->collider || !a->body || !a->aabb_min || !a->aabb_max))
        return err_->fail(AVN_ERR_INVALID_ARGUMENT, "aabbs: collider, body, aabb_min and aabb_max are required");
    a->retained_count = a->count;
    if (a->count > 0x7fffffffu - RS_TILE) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "aabbs: too many intervals");
    uploaded_ = ran_ = false;
    launches_ = 0;
    upload_launches_ = 0;
    dropped_ = false;
    n_ = int(a->count);
    host_ = *a;
    caller_ = a;
    const size_t n = a->count;
    AvnStatus st;
#define UPB(buf, host, cnt, T, dst) if ((st = up<T>(buf, host, cnt, &dst)) != AVN_OK) return st
    UPB(b_min_, a->aabb_min, 3 * n, S, d_min_);
    UPB(b_max_, a->aabb_max, 3 * n, S, d_max_);
    UPB(b_col_, a->collider, n, uint32_t, d_collider_);
    UPB(b_body_, a->body, n, uint32_t, d_body_);
    UPB(b_memb_, a->memberships, n, uint32_t, d_memb_);
    UPB(b_filt_, a->filters, n, uint32_t, d_filt_);
    UPB(b_flags_, a->flags, n, uint8_t, d_flags_);
#undef UPB
    if ((st = build_set(b_exk_, b_ext_, a->existing_pairs, a->existing_pair_count, &d_existing_, &existing_mask_)) != AVN_OK) return st;
    if (!d_existing_ && ext_existing_) { d_existing_ = ext_existing_; existing_mask_ = ext_existing_mask_; }   // ContactGraph::pair_set lives on the device
    if ((st = build_set(b_jdk_, b_jdt_, a->joint_disabled_body_pairs, a->joint_disabled_pair_count, &d_jdis_, &jdis_mask_)) != AVN_OK) return st;
    upload_launches_ = launches_;
    uploaded_ = true;
    return AVN_OK;
}

template <class S>
AvnStatus Broadphase<S>::ensure_buffers(int n) {
    const int nblocks = (n + RS_TILE - 1) / RS_TILE;
    AVN_CUDA(k0_.ensure(size_t(n) * sizeof(K))); AVN_CUDA(k1_.ensure(size_t(n) * sizeof(K)));
    AVN_CUDA(v0_.ensure(size_t(n) * 4)); AVN_CUDA(v1_.ensure(size_t(n) * 4));
    AVN_CUDA(hist_.ensure(size_t(256) * nblocks * 4));
    AVN_CUDA(s_minx_.ensure(size_t(n) * sizeof(S))); AVN_CUDA(s_maxx_.ensure(size_t(n) * sizeof(S)));
    AVN_CUDA(s_yz_.ensure(size_t(n) * sizeof(Vec4<S>))); AVN_CUDA(s_meta_.ensure(size_t(n) * sizeof(uint4)));
    AVN_CUDA(s_flags_.ensure(size_t(n))); AVN_CUDA(s_end_.ensure(size_t(n) * 4));
    AVN_CUDA(counts_.ensure(size_t(n) * 4)); AVN_CUDA(offsets_.ensure((size_t(n) + 1) * 8));
    AVN_CUDA(grid_.ensure(sizeof(CellGrid<S>)));
    AVN_CUDA(ck0_.ensure(size_t(n) * 4)); AVN_CUDA(ck1_.ensure(size_t(n) * 4)); AVN_CUDA(cv0_.ensure(size_t(n) * 4)); AVN_CUDA(cv1_.ensure(size_t(n) * 4));
    AVN_CUDA(cbounds_.ensure(size_t(2) * 0x10000 * 4));
    AVN_CUDA(stats_.ensure(size_t(YZ_BLOCKS) * sizeof(YzPartial<S>)));
    AVN_CUDA(stats2_.ensure(size_t(2) * YZ_BLOCKS * sizeof(S)));
    AVN_CUDA(wide_.ensure((size_t(SW_WIDE_CAP) + 1) * 4));
    AVN_CUDA(wide_flag_.ensure(size_t(n)));
    const int nsub = (n + SW_SUB - 1) / SW_SUB;
    AVN_CUDA(wide_sub_.ensure(size_t(nsub) * size_t(std::min(n, SW_WIDE_CAP)) * 4));
    AVN_CUDA(block_sums_.ensure(size_t((n + 1023) / 1024) * 8));
    AVN_CUDA(nf_flag_.ensure(8));
    pair_capacity_ = std::max<uint64_t>(pair_capacity_, uint64_t(4) * uint64_t(n) + 1024);
    AVN_CUDA(o_c1_.ensure(pair_capacity_ * 4)); AVN_CUDA(o_c2_.ensure(pair_capacity_ * 4)); AVN_CUDA(o_b1_.ensure(pair_capacity_ * 4)); AVN_CUDA(o_b2_.ensure(pair_capacity_ * 4));
    AVN_CUDA(o_fl_.ensure(pair_capacity_));
    AVN_CUDA(pairs_.ensure(pair_capacity_ * sizeof(uint2)));
    return AVN_OK;
}

template <class S>
typename Broadphase<S>::GraphKey Broadphase<S>::graph_key() const {
    GraphKey k;
    k.n = n_;
    const void* ptrs[] = {d_min_, d_max_, d_collider_, d_body_, d_memb_, d_filt_, d_flags_, d_existing_, d_jdis_, k0_.p, k1_.p, v0_.p, v1_.p, hist_.p,
                          s_minx_.p, s_maxx_.p, s_yz_.p, s_meta_.p, s_flags_.p, s_end_.p, counts_.p, offsets_.p, grid_.p, ck0_.p};
    static_assert(sizeof ptrs == sizeof k.p, "graph key size");
    memcpy(k.p, ptrs, sizeof ptrs);
    // the remaining buffers are allocated together with the ones above (same n): their addresses change only when those do
    k.m[0] = existing_mask_ ^ (uint64_t(uintptr_t(cv0_.p)) << 1) ^ (uint64_t(uintptr_t(wide_sub_.p)) << 2);
    k.m[0] ^= (pair_capacity_ * 0x9e3779b97f4a7c15ull) ^ (uint64_t(uintptr_t(pairs_.p)) << 3) ^ (uint64_t(uintptr_t(o_c1_.p)) << 4) ^ (uint64_t(uintptr_t(o_fl_.p)) << 5);
    k.m[1] = jdis_mask_ ^ (uint64_t(uintptr_t(cbounds_.p)) << 1) ^ (uint64_t(uintptr_t(block_sums_.p)) << 2) ^ (uint64_t(uintptr_t(wide_flag_.p)) << 3);
    return k;
}

template <class S>
void Broadphase<S>::enqueue_front(int n) {
    const int nblocks = (n + RS_TILE - 1) / RS_TILE;
    uint32_t launches = 0;
    K* ka = k0_.as<K>(); K* kb = k1_.as<K>();
    uint32_t* va = v0_.as<uint32_t>(); uint32_t* vb = v1_.as<uint32_t>();
    cudaMemsetAsync(nf_flag_.p, 0, 8, stream_);
    make_keys<S><<<(n + 255) / 256, 256, 0, stream_>>>(d_min_, d_max_, n, ka, va, nf_flag_.as<unsigned long long>());
    ++launches;
    for (int pass = 0; pass < KeyOf<S>::passes; ++pass) {
        const int shift = 8 * pass;
        rs_histogram<K><<<nblocks, RS_THREADS, 0, stream_>>>(ka, n, shift, hist_.as<uint32_t>(), nblocks);
        if (nblocks <= RS_FUSE_MAX_BLOCKS) {
            rs_scatter<K, true><<<nblocks, RS_THREADS, 0, stream_>>>(ka, va, n, shift, hist_.as<uint32_t>(), nblocks, kb, vb);
        } else {
            rs_scan<<<1, 1024, 0, stream_>>>(hist_.as<uint32_t>(), 256 * nblocks);
            rs_scatter<K, false><<<nblocks, RS_THREADS, 0, stream_>>>(ka, va, n, shift, hist_.as<uint32_t>(), nblocks, kb, vb);
        }
        launches += nblocks <= RS_FUSE_MAX_BLOCKS ? 2 : 3;
        std::swap(ka, kb);
        std::swap(va, vb);
    }
    d_order_ = va;  // even number of passes: back in buffer 0
    gather_sorted<S><<<(n + 255) / 256, 256, 0, stream_>>>(d_order_, n, d_min_, d_max_, d_collider_, d_body_, d_memb_, d_filt_, d_flags_,
                                                           s_minx_.as<S>(), s_maxx_.as<S>(), s_yz_.as<Vec4<S>>(), s_meta_.as<uint4>(),
                                                           s_flags_.as<uint8_t>());
    // (y, z) cell grid under the x-sorted ranks: stats -> cell ids -> stable 2-pass radix sort of the ranks by cell id -> cell bounds
    CellGrid<S>* d_grid = grid_.as<CellGrid<S>>();
    int* cstart = cbounds_.as<int>();
    int* cend = cbounds_.as<int>() + 0x10000;
    yz_stats<S><<<YZ_BLOCKS, 256, 0, stream_>>>(s_yz_.as<Vec4<S>>(), n, stats_.as<YzPartial<S>>());
    yz_fold<S><<<1, 32, 0, stream_>>>(stats_.as<YzPartial<S>>(), YZ_BLOCKS, n, d_grid);
    yz_small_max<S><<<YZ_BLOCKS, 256, 0, stream_>>>(s_yz_.as<Vec4<S>>(), n, d_grid, stats2_.as<S>());
    yz_grid<S><<<1, 32, 0, stream_>>>(stats_.as<YzPartial<S>>(), stats2_.as<S>(), YZ_BLOCKS, n, d_grid);
    int* wide_count = wide_.as<int>();
    int* wide_list = wide_.as<int>() + 1;
    cudaMemsetAsync(wide_count, 0, 4, stream_);
    sweep_bounds<S><<<(n + 255) / 256, 256, 0, stream_>>>(s_minx_.as<S>(), s_maxx_.as<S>(), s_yz_.as<Vec4<S>>(), d_grid, n, s_end_.as<int>(), wide_list, wide_count,
                                                          wide_flag_.as<uint8_t>(), s_flags_.as<uint8_t>());
    const Sweep<S> sw = sweep_desc();
    cell_keys<S><<<(n + 255) / 256, 256, 0, stream_>>>(s_yz_.as<Vec4<S>>(), n, d_grid, ck0_.as<uint32_t>(), cv0_.as<uint32_t>());
    {
        uint32_t* cka = ck0_.as<uint32_t>(); uint32_t* ckb = ck1_.as<uint32_t>();
        uint32_t* cva = cv0_.as<uint32_t>(); uint32_t* cvb = cv1_.as<uint32_t>();
        for (int pass = 0; pass < 2; ++pass) {
            rs_histogram<uint32_t><<<nblocks, RS_THREADS, 0, stream_>>>(cka, n, 8 * pass, hist_.as<uint32_t>(), nblocks);
            if (nblocks <= RS_FUSE_MAX_BLOCKS) {
                rs_scatter<uint32_t, true><<<nblocks, RS_THREADS, 0, stream_>>>(cka, cva, n, 8 * pass, hist_.as<uint32_t>(), nblocks, ckb, cvb);
            } else {
                rs_scan<<<1, 1024, 0, stream_>>>(hist_.as<uint32_t>(), 256 * nblocks);
                rs_scatter<uint32_t, false><<<nblocks, RS_THREADS, 0, stream_>>>(cka, cva, n, 8 * pass, hist_.as<uint32_t>(), nblocks, ckb, cvb);
            }
            std::swap(cka, ckb);
            std::swap(cva, cvb);
        }
    }
    cudaMemsetAsync(cstart, 0x7f, size_t(0x10000) * 4, stream_);
    cudaMemsetAsync(cend, 0, size_t(0x10000) * 4, stream_);
    cell_bounds<<<(n + 255) / 256, 256, 0, stream_>>>(ck0_.as<uint32_t>(), n, cstart, cend);
    const CellSweep<S> cs = cell_desc();
    const int grid = std::min((n + (256 / CG_GROUP) - 1) / (256 / CG_GROUP), sm_count_ * 32);
    sweep_cells_kernel<S, false><<<grid, 256, 0, stream_>>>(sw, cs, counts_.as<uint32_t>(), nullptr, nullptr);
    // intervals with a huge x-window: brute force, one block per SW_SUB candidates; the grid's y dimension strides the wide list
    const int nsub = (n + SW_SUB - 1) / SW_SUB;
    sweep_wide_kernel<S, false><<<dim3(nsub, WIDE_ROWS), SW_THREADS, 0, stream_>>>(sw, wide_list, wide_count, wide_sub_.as<uint32_t>(), nsub, nullptr, nullptr, 0);
    wide_finish<<<1, 256, 0, stream_>>>(wide_list, wide_count, wide_sub_.as<uint32_t>(), nsub, counts_.as<uint32_t>());
    launches += nblocks <= RS_FUSE_MAX_BLOCKS ? 15 : 17;
    const int sblocks = (n + 1023) / 1024;
    scan_block_sums<<<sblocks, 1024, 0, stream_>>>(counts_.as<uint32_t>(), n, block_sums_.as<uint64_t>());
    scan_block_offsets<<<1, 1024, 0, stream_>>>(block_sums_.as<uint64_t>(), sblocks, offsets_.as<uint64_t>() + n);
    scan_apply<<<sblocks, 1024, 0, stream_>>>(counts_.as<uint32_t>(), n, block_sums_.as<uint64_t>(), offsets_.as<uint64_t>());
    launches += 3;
    // emit pass straight after the count pass, into buffers of pair_capacity_ entries (grown by download() when the count says so): the count
    // never visits the host in between, so a run is ONE graph launch with no synchronisation
    {
        uint2* pairs = pairs_.as<uint2>();
        sweep_cells_kernel<S, true><<<grid, 256, 0, stream_>>>(sw, cs, nullptr, offsets_.as<uint64_t>(), pairs);
        sweep_wide_kernel<S, true><<<dim3(nsub, WIDE_ROWS), SW_THREADS, 0, stream_>>>(sw, wide_list, wide_count, wide_sub_.as<uint32_t>(), nsub,
                                                                                      offsets_.as<uint64_t>(), pairs, pair_capacity_);
        segment_sort<<<(n + 255) / 256, 256, 0, stream_>>>(offsets_.as<uint64_t>(), wide_flag_.as<uint8_t>(), n, pairs, pair_capacity_);
        const unsigned mblocks = unsigned(std::min<uint64_t>((pair_capacity_ + 255) / 256, uint64_t(sm_count_) * 16));
        materialize_pairs<S><<<mblocks, 256, 0, stream_>>>(sw, pairs, offsets_.as<uint64_t>() + n, pair_capacity_, o_c1_.as<uint32_t>(), o_c2_.as<uint32_t>(),
                                                           o_b1_.as<uint32_t>(), o_b2_.as<uint32_t>(), o_fl_.as<uint8_t>());
        launches += 4;
    }
    // count + non-finite flag for download(): one 16-byte readback, not waited for here
    cudaMemcpyAsync(h_total_, offsets_.as<uint64_t>() + n, sizeof(uint64_t), cudaMemcpyDeviceToHost, stream_);
    cudaMemcpyAsync(h_total_ + 1, nf_flag_.p, sizeof(uint64_t), cudaMemcpyDeviceToHost, stream_);
    front_launches_ = launches;
}

template <class S>
AvnStatus Broadphase<S>::run() {
    if (!uploaded_) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_broadphase_run before avn_broadphase_upload");
    const int n = n_;
    launches_ = upload_launches_;   // launches of THIS run (+ the hash-set builds of its upload), not of every run since the upload
    cudaEventRecord(ev0_, stream_);
    h_total_[0] = 0;
    h_total_[1] = 0;
    if (n > 0) {
        AvnStatus st = ensure_buffers(n);
        if (st != AVN_OK) return st;
        if (use_graph_) {
            const GraphKey key = graph_key();
            if (!graph_exec_ || !(key == graph_key_)) {
                if (graph_exec_) { cudaGraphExecDestroy(graph_exec_); graph_exec_ = nullptr; }
                cudaGraph_t g = nullptr;
                AVN_CUDA(cudaStreamBeginCapture(stream_, cudaStreamCaptureModeThreadLocal));
                enqueue_front(n);
                cudaError_t ce = cudaStreamEndCapture(stream_, &g);
                if (ce == cudaSuccess) ce = cudaGraphInstantiate(&graph_exec_, g, 0);
                if (g) cudaGraphDestroy(g);
                if (ce != cudaSuccess) {   // capture refused: plain launches from now on (same kernels)
                    (void)cudaGetLastError();
                    graph_exec_ = nullptr;
                    use_graph_ = false;
                } else {
                    graph_key_ = key;
                }
            }
        }
        if (use_graph_ && graph_exec_) {
            AVN_CUDA(cudaGraphLaunch(graph_exec_, stream_));
            graph_replays_ += 1;
        } else {
            enqueue_front(n);
        }
        launches_ += front_launches_;
    }
    cudaEventRecord(ev1_, stream_);
    AVN_CUDA(cudaGetLastError());
    ran_ = true;
    return AVN_OK;
}

// update_aabb_intervals' `retain` (broad_phase.rs:236-246): intervals whose AABB is not finite leave the interval list.  The flag raised by
// make_keys brings us here (rare): compact the caller's columns on the host, upload the survivors and run again.  order_out then lists the
// surviving intervals only (retained_count of them, as rows of the CALLER's columns).
template <class S>
AvnStatus Broadphase<S>::drop_nonfinite() {
    const size_t n = host_.count;
    const S* mn = static_cast<const S*>(host_.aabb_min);
    const S* mx = static_cast<const S*>(host_.aabb_max);
    keep_.clear();
    keep_.reserve(n);
    for (size_t i = 0; i < n; ++i) {
        bool finite = true;
        for (int k = 0; k < 3; ++k) finite = finite && std::isfinite(mn[3 * i + k]) && std::isfinite(mx[3 * i + k]);
        if (finite) keep_.push_back(uint32_t(i));
    }
    const size_t m = keep_.size();
    c_min_.resize(3 * m * sizeof(S)); c_max_.resize(3 * m * sizeof(S));
    c_col_.resize(m); c_body_.resize(m);
    if (host_.memberships) c_memb_.resize(m);
    if (host_.filters) c_filt_.resize(m);
    if (host_.flags) c_flags_.resize(m);
    S* cmn = reinterpret_cast<S*>(c_min_.data());
    S* cmx = reinterpret_cast<S*>(c_max_.data());
    for (size_t r = 0; r < m; ++r) {
        const size_t i = keep_[r];
        for (int k = 0; k < 3; ++k) { cmn[3 * r + k] = mn[3 * i + k]; cmx[3 * r + k] = mx[3 * i + k]; }
        c_col_[r] = host_.collider[i];
        c_body_[r] = host_.body[i];
        if (host_.memberships) c_memb_[r] = host_.memberships[i];
        if (host_.filters) c_filt_[r] = host_.filters[i];
        if (host_.flags) c_flags_[r] = host_.flags[i];
    }
    AvnStatus st;
#define UPB(buf, host, cnt, T, dst) if ((st = up<T>(buf, host, cnt, &dst)) != AVN_OK) return st
    UPB(b_min_, cmn, 3 * m, S, d_min_);
    UPB(b_max_, cmx, 3 * m, S, d_max_);
    UPB(b_col_, c_col_.data(), m, uint32_t, d_collider_);
    UPB(b_body_, c_body_.data(), m, uint32_t, d_body_);
    UPB(b_memb_, host_.memberships ? c_memb_.data() : nullptr, m, uint32_t, d_memb_);
    UPB(b_filt_, host_.filters ? c_filt_.data() : nullptr, m, uint32_t, d_filt_);
    UPB(b_flags_, host_.flags ? c_flags_.data() : nullptr, m, uint8_t, d_flags_);
#undef UPB
    AVN_CUDA(cudaStreamSynchronize(stream_));   // the compacted columns are pageable host vectors
    n_ = int(m);
    dropped_ = true;
    return run();
}

template <class S>
AvnStatus Broadphase<S>::settle() {
    if (!ran_) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "avn_broadphase_download before avn_broadphase_run");
    // the run left its pair count and the non-finite flag in pinned memory; this is where the host first looks at them
    AVN_CUDA(cudaStreamSynchronize(stream_));
    for (int attempt = 0; attempt < 3; ++attempt) {
        if (h_total_[1] != 0) {                       // a NaN / infinite AABB: drop those intervals and run again (drop_nonfinite reruns)
            AvnStatus st = drop_nonfinite();
            if (st != AVN_OK) return st;
            AVN_CUDA(cudaStreamSynchronize(stream_));
            continue;
        }
        if (h_total_[0] > pair_capacity_) {           // more pairs than the emit buffers held: grow them and run again
            pair_capacity_ = h_total_[0] + h_total_[0] / 4 + 1024;
            AvnStatus st = run();
            if (st != AVN_OK) return st;
            AVN_CUDA(cudaStreamSynchronize(stream_));
            continue;
        }
        break;
    }
    return AVN_OK;
}

template <class S>
AvnStatus Broadphase<S>::finish_download() {
    if (host_.order_out && n_ > 0) AVN_CUDA(cudaMemcpyAsync(host_.order_out, d_order_, size_t(n_) * 4, cudaMemcpyDeviceToHost, stream_));
    AVN_CUDA(cudaStreamSynchronize(stream_));
    if (dropped_ && host_.order_out)
        for (int r = 0; r < n_; ++r) host_.order_out[r] = keep_[host_.order_out[r]];   // compacted rows -> rows of the caller's columns
    if (caller_) caller_->retained_count = uint32_t(n_);
    float ms = 0;
    tm_ = AvnTimings{};
    if (cudaEventElapsedTime(&ms, ev0_, ev1_) == cudaSuccess) { tm_.broad_phase_ms = ms; tm_.total_ms = ms; }
    tm_.kernel_launches = launches_;
    return AVN_OK;
}

template <class S>
AvnStatus Broadphase<S>::download(AvnPairList* out) {
    if (!out) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "out_pairs is required");
    AvnStatus st = settle();
    if (st != AVN_OK) return st;
    const uint64_t total = *h_total_;
    out->count = total;
    const uint64_t ncopy = std::min<uint64_t>(total, out->capacity);
    if (ncopy) {
        if (!out->collider1 || !out->collider2 || !out->body1 || !out->body2 || !out->flags)
            return err_->fail(AVN_ERR_INVALID_ARGUMENT, "out_pairs arrays are required when capacity > 0");
        AVN_CUDA(cudaMemcpyAsync(out->collider1, o_c1_.p, ncopy * 4, cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaMemcpyAsync(out->collider2, o_c2_.p, ncopy * 4, cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaMemcpyAsync(out->body1, o_b1_.p, ncopy * 4, cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaMemcpyAsync(out->body2, o_b2_.p, ncopy * 4, cudaMemcpyDeviceToHost, stream_));
        AVN_CUDA(cudaMemcpyAsync(out->flags, o_fl_.p, ncopy, cudaMemcpyDeviceToHost, stream_));
    }
    if ((st = finish_download()) != AVN_OK) return st;
    if (total > out->capacity) return err_->fail(AVN_ERR_CAPACITY, "pair list capacity %llu < %llu pairs found", (unsigned long long)out->capacity,
                                                 (unsigned long long)total);
    return AVN_OK;
}

template <class S>
AvnStatus Broadphase<S>::download_order(uint64_t* out_pair_count) {
    AvnStatus st = settle();
    if (st != AVN_OK) return st;
    if (out_pair_count) *out_pair_count = *h_total_;
    return finish_download();
}

template <class S>
AvnStatus Broadphase<S>::device_pairs(DevicePairs* out) {
    if (!out) return err_->fail(AVN_ERR_INVALID_ARGUMENT, "out is required");
    AvnStatus st = settle();
    if (st != AVN_OK) return st;
    *out = DevicePairs{};
    out->count = *h_total_;
    out->c1 = o_c1_.as<uint32_t>(); out->c2 = o_c2_.as<uint32_t>(); out->b1 = o_b1_.as<uint32_t>(); out->b2 = o_b2_.as<uint32_t>(); out->flags = o_fl_.as<uint8_t>();
    return AVN_OK;
}

}  // namespace

BroadphaseBase* make_broadphase(uint32_t scalar_bits, cudaStream_t stream, ErrorSink* err, int device) {
    if (scalar_bits == 32) return new Broadphase<float>(stream, err, device);
    if (scalar_bits == 64) return new Broadphase<double>(stream, err, device);
    return nullptr;
}

}  // namespace avn
