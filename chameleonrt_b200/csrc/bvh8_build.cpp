// bvh8_build.cpp — host-side builder for the compressed 8-wide BVH (format: bvh8.h).
//
// Pipeline: (1) binned-SAH BVH2 with one triangle per leaf, built in parallel over subtrees
// on a std::thread task pool; (2) optimal SAH collapse of the binary tree into 8-wide nodes
// with <= 3 triangles per leaf (dynamic programme of Ylitie et al. 2017, §4); (3) emission:
// octant-ordered child slots, 8-bit quantised child boxes that are conservative in the
// arithmetic the traversal kernel uses, inner children and leaf triangles made contiguous.
//
// The reference has no builder (Embree / OptiX do it, SURVEY.md §2.3); nothing here is
// derived from reference code.
#include "bvh8.h"
#include "host_parallel.h"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <limits>
#include <mutex>
#include <thread>

namespace crt {
namespace {

struct Box {
    float lo[3], hi[3];
    void reset()
    {
        for (int a = 0; a < 3; ++a) {
            lo[a] = std::numeric_limits<float>::max();
            hi[a] = -std::numeric_limits<float>::max();
        }
    }
    void grow(const Box &b)
    {
        for (int a = 0; a < 3; ++a) {
            lo[a] = std::min(lo[a], b.lo[a]);
            hi[a] = std::max(hi[a], b.hi[a]);
        }
    }
    void grow_pt(const float *p)
    {
        for (int a = 0; a < 3; ++a) {
            lo[a] = std::min(lo[a], p[a]);
            hi[a] = std::max(hi[a], p[a]);
        }
    }
    float half_area() const
    {
        const float dx = hi[0] - lo[0], dy = hi[1] - lo[1], dz = hi[2] - lo[2];
        return dx * dy + dy * dz + dz * dx;
    }
};

struct B2Node {
    Box box;
    uint32_t left;   // inner: index of left child (right = left + 1); leaf: triangle index
    uint32_t count;  // 0 = inner, 1 = leaf
};

// 4-wide float / int vectors (GCC/Clang vector extensions: SSE on x86-64, NEON on aarch64). Lane 3 is
// padding everywhere below. vmin/vmax pick their operand exactly like std::min/std::max.
typedef float f4 __attribute__((vector_size(16)));
typedef int i4 __attribute__((vector_size(16)));
inline f4 vmin(f4 a, f4 b) { return b < a ? b : a; }
inline f4 vmax(f4 a, f4 b) { return a < b ? b : a; }
inline f4 splat(float x) { return f4{x, x, x, x}; }
constexpr float kFltMax = std::numeric_limits<float>::max();

struct VBox {
    f4 lo, hi;
    void reset()
    {
        lo = splat(kFltMax);
        hi = splat(-kFltMax);
    }
    void grow(const VBox &o)
    {
        lo = vmin(lo, o.lo);
        hi = vmax(hi, o.hi);
    }
    void grow_pt(f4 p)
    {
        lo = vmin(lo, p);
        hi = vmax(hi, p);
    }
    Box box() const
    {
        Box b;
        for (int a = 0; a < 3; ++a) {
            b.lo[a] = lo[a];
            b.hi[a] = hi[a];
        }
        return b;
    }
    float half_area() const
    {
        const float dx = hi[0] - lo[0], dy = hi[1] - lo[1], dz = hi[2] - lo[2];
        return dx * dy + dy * dz + dz * dx;
    }
};

// One primitive of the BVH2 build: 32 bytes, kept physically in tree order (partitioned in place, or
// through a scratch buffer for big ranges), so every pass over a node's range is a sequential stream.
struct Prim {
    // box; the padding lanes carry the triangle index as the mantissas of two floats in [1, 2)
    // (low 23 bits in lo[3], the rest in hi[3]): the lanes ride through the vector arithmetic below,
    // and a raw index there would be a denormal operand (a microcode assist per operation)
    f4 lo, hi;
    static float pack23(uint32_t m)
    {
        const uint32_t u = 0x3F800000u | (m & 0x7FFFFFu);
        float f;
        std::memcpy(&f, &u, 4);
        return f;
    }
    static uint32_t unpack23(float f)
    {
        uint32_t u;
        std::memcpy(&u, &f, 4);
        return u & 0x7FFFFFu;
    }
    void set_id(uint32_t i)
    {
        lo[3] = pack23(i);
        hi[3] = pack23(i >> 23);
    }
    uint32_t id() const { return unpack23(lo[3]) | (unpack23(hi[3]) << 23); }
    f4 centroid() const { return splat(0.5f) * (lo + hi); }
};

struct Task {
    uint32_t node, first, count;
    VBox box, cbox;  // bounds of the range's boxes and of its centroids (known from the parent's split)
};

constexpr int kBins = 16;
constexpr uint32_t kParallelThreshold = 1u << 15;  // both halves at least this big: share the right half
constexpr uint32_t kBigTask = 1u << 19;            // ranges this big are binned / partitioned by several threads
constexpr uint32_t kBlock = 1u << 14;              // block of a big range (fixed: results do not depend on threads)

struct Bins {
    VBox box[3][kBins];
    uint32_t cnt[3][kBins];
    void reset()
    {
        for (int a = 0; a < 3; ++a) {
            for (int b = 0; b < kBins; ++b) {
                box[a][b].reset();
                cnt[a][b] = 0;
            }
        }
    }
    void merge(const Bins &o)
    {
        for (int a = 0; a < 3; ++a) {
            for (int b = 0; b < kBins; ++b) {
                box[a][b].grow(o.box[a][b]);
                cnt[a][b] += o.cnt[a][b];
            }
        }
    }
};

struct BinFrame {
    f4 cmin, scale;
    bool valid[3];
    explicit BinFrame(const VBox &cbox)
    {
        cmin = cbox.lo;
        scale = splat(0.f);
        for (int a = 0; a < 3; ++a) {
            const float ext = cbox.hi[a] - cbox.lo[a];
            valid[a] = ext > 0.f;
            scale[a] = valid[a] ? kBins / ext : 0.f;
        }
        cmin[3] = 0.f;
    }
    // bin of the centroid on every axis: clamp((int)((c - cmin) * scale), 0, kBins - 1), NaN to bin 0. A centroid or a
    // centroid bound at +-inf (an infinite vertex, or lo + hi overflowing) makes x = inf * 0 or inf - inf; the clamp
    // takes the bound as its first operand, so that a NaN fails both compares and becomes the bound.
    i4 bins(const Prim &p) const
    {
        f4 x = (p.centroid() - cmin) * scale;
        x = vmin(splat((float)(kBins - 1)), vmax(splat(0.f), x));
        return __builtin_convertvector(x, i4);
    }
};

struct Bvh2Builder {
    std::vector<Prim> prims, scratch;
    std::vector<B2Node> nodes;
    std::atomic<uint32_t> next_node{1};
    int threads = 1;
    std::atomic<int> big_running{0};  // big ranges being split right now: they share the helper threads

    std::mutex mtx;
    std::condition_variable cv;
    std::deque<Task> shared;
    int outstanding = 0;  // tasks queued or running (guarded by mtx)

    void push_shared(const Task &t)
    {
        {
            std::lock_guard<std::mutex> lk(mtx);
            shared.push_back(t);
            ++outstanding;
        }
        cv.notify_one();
    }

    void bin_range(uint32_t first, uint32_t count, const BinFrame &fr, Bins &bins) const
    {
        bins.reset();
        const Prim *p = prims.data() + first;
        for (uint32_t i = 0; i < count; ++i) {
            const i4 b = fr.bins(p[i]);
            for (int a = 0; a < 3; ++a) {
                VBox &bb = bins.box[a][b[a]];
                bb.lo = vmin(bb.lo, p[i].lo);
                bb.hi = vmax(bb.hi, p[i].hi);
                bins.cnt[a][b[a]]++;
            }
        }
    }

    // Binned SAH over the three axes; returns false if no split separates the primitives.
    static bool choose_split(const Bins &bins, const BinFrame &fr, int &best_axis, int &best_bin)
    {
        float best_cost = std::numeric_limits<float>::max();
        best_axis = -1;
        best_bin = 0;
        for (int a = 0; a < 3; ++a) {
            if (!fr.valid[a]) {
                continue;
            }
            float right_area[kBins];
            uint32_t right_cnt[kBins];
            VBox acc;
            acc.reset();
            uint32_t cnt = 0;
            for (int b = kBins - 1; b > 0; --b) {
                acc.grow(bins.box[a][b]);
                cnt += bins.cnt[a][b];
                right_area[b] = cnt ? acc.half_area() : 0.f;
                right_cnt[b] = cnt;
            }
            acc.reset();
            cnt = 0;
            for (int b = 0; b < kBins - 1; ++b) {
                acc.grow(bins.box[a][b]);
                cnt += bins.cnt[a][b];
                if (cnt == 0 || right_cnt[b + 1] == 0) {
                    continue;
                }
                const float cost = acc.half_area() * cnt + right_area[b + 1] * right_cnt[b + 1];
                // (a bin whose prims are all NaN on an axis keeps its reset bounds, FLT_MAX..-FLT_MAX, so a cost can be
                // -inf or NaN; such a split would peel the range one prim at a time. Finite boxes give costs >= 0.)
                if (cost >= 0.f && cost < best_cost) {
                    best_cost = cost;
                    best_axis = a;
                    best_bin = b;
                }
            }
        }
        return best_axis >= 0;
    }

    void range_bounds(uint32_t first, uint32_t count, VBox &box, VBox &cbox) const
    {
        box.reset();
        cbox.reset();
        for (uint32_t i = first; i < first + count; ++i) {
            box.lo = vmin(box.lo, prims[i].lo);
            box.hi = vmax(box.hi, prims[i].hi);
            cbox.grow_pt(prims[i].centroid());
        }
    }

    // Splits the task's range; fills the two child tasks (ranges and bounds).
    void split(const Task &t, Task &tl, Task &tr)
    {
        const uint32_t first = t.first, count = t.count;
        const BinFrame fr(t.cbox);
        Bins bins;
        const bool big = count >= kBigTask;
        const uint32_t nblocks = big ? (count + kBlock - 1) / kBlock : 0;
        std::vector<Bins> block_bins;
        int nthreads = 1;
        if (big) {
            const int running = big_running.fetch_add(1) + 1;
            nthreads = std::max(1, threads / running);
            block_bins.resize(nblocks);
            parallel_blocks(nblocks, nthreads, [&](uint32_t b) {
                const uint32_t bf = first + b * kBlock;
                bin_range(bf, std::min(kBlock, first + count - bf), fr, block_bins[b]);
            });
            bins.reset();
            for (uint32_t b = 0; b < nblocks; ++b) {
                bins.merge(block_bins[b]);
            }
        } else {
            bin_range(first, count, fr, bins);
        }
        int axis, bin;
        uint32_t mid = first + count / 2;
        bool have_bounds = false;
        if (choose_split(bins, fr, axis, bin)) {
            uint32_t nleft = 0;
            for (int b = 0; b <= bin; ++b) {
                nleft += bins.cnt[axis][b];
            }
            tl.cbox.reset();
            tr.cbox.reset();
            if (big) {
                // stable partition through the scratch buffer, block by block: the left / right
                // offsets of a block follow from its own bin counts
                std::vector<uint32_t> loff(nblocks), roff(nblocks);
                std::vector<VBox> lcb(nblocks), rcb(nblocks);
                uint32_t l = 0, r = 0;
                for (uint32_t b = 0; b < nblocks; ++b) {
                    loff[b] = l;
                    roff[b] = r;
                    uint32_t bl = 0, bc = 0;
                    for (int k = 0; k < kBins; ++k) {
                        bc += block_bins[b].cnt[axis][k];
                        bl += k <= bin ? block_bins[b].cnt[axis][k] : 0;
                    }
                    l += bl;
                    r += bc - bl;
                }
                parallel_blocks(nblocks, nthreads, [&](uint32_t b) {
                    const uint32_t bf = first + b * kBlock, be = std::min(bf + kBlock, first + count);
                    Prim *dl = scratch.data() + first + loff[b], *dr = scratch.data() + first + nleft + roff[b];
                    VBox cl, cr;
                    cl.reset();
                    cr.reset();
                    for (uint32_t i = bf; i < be; ++i) {
                        const Prim &p = prims[i];
                        if (fr.bins(p)[axis] <= bin) {
                            *dl++ = p;
                            cl.grow_pt(p.centroid());
                        } else {
                            *dr++ = p;
                            cr.grow_pt(p.centroid());
                        }
                    }
                    lcb[b] = cl;
                    rcb[b] = cr;
                });
                parallel_blocks(nblocks, nthreads, [&](uint32_t b) {
                    const uint32_t bf = first + b * kBlock, be = std::min(bf + kBlock, first + count);
                    std::memcpy(prims.data() + bf, scratch.data() + bf, (size_t)(be - bf) * sizeof(Prim));
                });
                for (uint32_t b = 0; b < nblocks; ++b) {
                    tl.cbox.grow(lcb[b]);
                    tr.cbox.grow(rcb[b]);
                }
                mid = first + nleft;
            } else {
                // in-place two-pointer partition (the order std::partition produces), collecting the
                // centroid bounds of both sides on the way
                Prim *lo = prims.data() + first, *hi = prims.data() + first + count;
                for (;;) {
                    while (lo < hi && fr.bins(*lo)[axis] <= bin) {
                        tl.cbox.grow_pt(lo->centroid());
                        ++lo;
                    }
                    while (lo < hi && !(fr.bins(hi[-1])[axis] <= bin)) {
                        tr.cbox.grow_pt(hi[-1].centroid());
                        --hi;
                    }
                    if (lo >= hi) {
                        break;
                    }
                    std::swap(*lo, hi[-1]);
                }
                mid = (uint32_t)(lo - prims.data());
            }
            // box bounds of the halves are the unions of their bins
            tl.box.reset();
            tr.box.reset();
            for (int b = 0; b < kBins; ++b) {
                if (bins.cnt[axis][b]) {
                    (b <= bin ? tl : tr).box.grow(bins.box[axis][b]);
                }
            }
            have_bounds = true;
        }
        if (big) {
            big_running.fetch_sub(1);
        }
        tl.first = first;
        tl.count = mid - first;
        tr.first = mid;
        tr.count = first + count - mid;
        if (!have_bounds) {  // coincident centroids: split the range in the middle
            range_bounds(tl.first, tl.count, tl.box, tl.cbox);
            range_bounds(tr.first, tr.count, tr.box, tr.cbox);
        }
    }

    void process(const Task &root_task)
    {
        std::vector<Task> local;
        local.push_back(root_task);
        while (!local.empty()) {
            const Task t = local.back();
            local.pop_back();
            B2Node &n = nodes[t.node];
            n.box = t.box.box();
            if (t.count == 1) {
                n.left = prims[t.first].id();
                n.count = 1;
                continue;
            }
            Task tl, tr;
            split(t, tl, tr);
            const uint32_t left = next_node.fetch_add(2);
            n.left = left;
            n.count = 0;
            tl.node = left;
            tr.node = left + 1;
            if (tl.count >= kParallelThreshold && tr.count >= kParallelThreshold) {
                push_shared(tr);
                local.push_back(tl);
            } else {
                local.push_back(tr);
                local.push_back(tl);
            }
        }
    }

    void worker()
    {
        for (;;) {
            Task t;
            {
                std::unique_lock<std::mutex> lk(mtx);
                cv.wait(lk, [&] { return !shared.empty() || outstanding == 0; });
                if (shared.empty()) {
                    return;
                }
                t = shared.front();
                shared.pop_front();
            }
            process(t);
            bool done;
            {
                std::lock_guard<std::mutex> lk(mtx);
                --outstanding;
                done = outstanding == 0;
            }
            if (done) {
                cv.notify_all();
            }
        }
    }

    // verts: 9 floats per triangle
    void build(const float *verts, uint32_t n, int nthreads)
    {
        threads = std::max(1, nthreads);
        prims.resize(n);
        if (n >= kBigTask) {
            scratch.resize(n);
        }
        const uint32_t nblocks = (n + kBlock - 1) / kBlock;
        std::vector<VBox> bb(nblocks), bc(nblocks);
        parallel_blocks(nblocks, threads, [&](uint32_t b) {
            bb[b].reset();
            bc[b].reset();
            const uint32_t e = std::min(n, (b + 1) * kBlock);
            for (uint32_t i = b * kBlock; i < e; ++i) {
                const float *v = verts + 9 * (size_t)i;
                VBox x;
                x.reset();
                for (int k = 0; k < 3; ++k) {
                    x.grow_pt(f4{v[3 * k], v[3 * k + 1], v[3 * k + 2], 0.f});
                }
                Prim &p = prims[i];
                p.lo = x.lo;
                p.hi = x.hi;
                bb[b].grow(x);
                bc[b].grow_pt(p.centroid());
                p.set_id(i);
            }
        });
        Task root;
        root.node = 0;
        root.first = 0;
        root.count = n;
        root.box.reset();
        root.cbox.reset();
        for (uint32_t b = 0; b < nblocks; ++b) {
            root.box.grow(bb[b]);
            root.cbox.grow(bc[b]);
        }
        nodes.resize(2 * (size_t)n - 1);
        push_shared(root);
        std::vector<std::thread> pool;
        for (int i = 1; i < threads; ++i) {
            pool.emplace_back([this] { worker(); });
        }
        worker();
        for (auto &th : pool) {
            th.join();
        }
        nodes.resize(next_node.load());
        std::vector<Prim>().swap(prims);
        std::vector<Prim>().swap(scratch);
    }
};

// ---------------------------------------------------------------------------------------
// Collapse BVH2 -> BVH8 (Ylitie et al. 2017 §4.1-4.2)
// ---------------------------------------------------------------------------------------
constexpr float kPrimCost = 0.3f;
constexpr float kNodeCost = 1.0f;
enum : uint8_t { kLeaf = 0, kInternal = 1, kDistribute = 2 };

struct Decision {
    uint8_t type : 2;
    uint8_t dist_left : 3;
    uint8_t dist_right : 3;
};

struct Collapser {
    const std::vector<B2Node> &n2;
    std::vector<float> cost;         // 7 per node
    std::vector<Decision> decision;  // 7 per node
    std::vector<uint32_t> tri_count;

    explicit Collapser(const std::vector<B2Node> &nodes) : n2(nodes)
    {
        cost.resize(nodes.size() * 7);
        decision.resize(nodes.size() * 7);
        tri_count.resize(nodes.size());
    }

    // The dynamic programme only looks at a node's two children, so disjoint subtrees are independent:
    // the tree is cut at a frontier of subtree roots, the subtrees are solved in parallel, then the few
    // nodes above the frontier are solved from the finished subtree roots.
    void run_parallel(uint32_t root, int threads)
    {
        std::vector<uint32_t> frontier{root};
        const size_t want = (size_t)std::max(1, threads) * 8;
        std::vector<uint8_t> is_frontier;
        if (threads > 1 && n2.size() > (1u << 16)) {
            // level-wise expansion; leaves stay in the frontier (they are trivial subtrees)
            while (frontier.size() < want) {
                std::vector<uint32_t> next;
                bool expanded = false;
                for (uint32_t n : frontier) {
                    if (n2[n].count) {
                        next.push_back(n);
                    } else {
                        next.push_back(n2[n].left);
                        next.push_back(n2[n].left + 1);
                        expanded = true;
                    }
                }
                frontier.swap(next);
                if (!expanded) {
                    break;
                }
            }
            is_frontier.assign(n2.size(), 0);
            for (uint32_t n : frontier) {
                is_frontier[n] = 1;
            }
            parallel_blocks((uint32_t)frontier.size(), threads, [&](uint32_t i) { run(frontier[i], nullptr); });
            run(root, is_frontier.data());
        } else {
            run(root, nullptr);
        }
    }

    // post-order over an explicit stack (SAH trees can be deep); nodes flagged in `solved` are taken as
    // already computed and not descended into
    void run(uint32_t root, const uint8_t *solved)
    {
        if (solved && solved[root]) {
            return;
        }
        std::vector<std::pair<uint32_t, bool>> stack;
        stack.emplace_back(root, false);
        while (!stack.empty()) {
            auto [n, expanded] = stack.back();
            stack.pop_back();
            if (solved && solved[n]) {
                continue;
            }
            const B2Node &node = n2[n];
            if (node.count) {
                tri_count[n] = 1;
                const float c = node.box.half_area() * kPrimCost;
                for (int i = 0; i < 7; ++i) {
                    cost[7 * (size_t)n + i] = c;
                    decision[7 * (size_t)n + i] = Decision{kLeaf, 0, 0};
                }
                continue;
            }
            if (!expanded) {
                stack.emplace_back(n, true);
                stack.emplace_back(node.left, false);
                stack.emplace_back(node.left + 1, false);
                continue;
            }
            const uint32_t l = node.left, r = node.left + 1;
            const uint32_t cnt = tri_count[l] + tri_count[r];
            tri_count[n] = cnt;
            const float area = node.box.half_area();
            const float *cl = &cost[7 * (size_t)l], *cr = &cost[7 * (size_t)r];
            float *cn = &cost[7 * (size_t)n];
            Decision *dn = &decision[7 * (size_t)n];
            // i = 0: a single root — either a leaf (<= 3 triangles) or an internal node whose
            // 8 slots are distributed between the two subtrees
            {
                const float cost_leaf = cnt <= 3 ? area * (float)cnt * kPrimCost : std::numeric_limits<float>::infinity();
                float best = std::numeric_limits<float>::infinity();
                int bl = 0, br = 0;
                for (int k = 0; k < 7; ++k) {
                    const float c = cl[k] + cr[6 - k];
                    if (c < best) {
                        best = c;
                        bl = k;
                        br = 6 - k;
                    }
                }
                const float cost_internal = best + area * kNodeCost;
                if (cost_leaf < cost_internal) {
                    cn[0] = cost_leaf;
                    dn[0] = Decision{kLeaf, 0, 0};
                } else {
                    cn[0] = cost_internal;
                    dn[0] = Decision{kInternal, (uint8_t)bl, (uint8_t)br};
                }
            }
            // i = 1..6: a forest of up to i+1 roots
            for (int i = 1; i < 7; ++i) {
                cn[i] = cn[i - 1];
                dn[i] = dn[i - 1];
                for (int k = 0; k < i; ++k) {
                    const float c = cl[k] + cr[i - k - 1];
                    if (c < cn[i]) {
                        cn[i] = c;
                        dn[i] = Decision{kDistribute, (uint8_t)k, (uint8_t)(i - k - 1)};
                    }
                }
            }
        }
    }

    // Children (BVH2 node ids) of the forest (n, i)
    void get_children(uint32_t n, int i, uint32_t *children, int &num) const
    {
        const B2Node &node = n2[n];
        if (node.count) {
            children[num++] = n;
            return;
        }
        const Decision d = decision[7 * (size_t)n + i];
        const uint32_t l = node.left, r = node.left + 1;
        if (decision[7 * (size_t)l + d.dist_left].type == kDistribute) {
            get_children(l, d.dist_left, children, num);
        } else {
            children[num++] = l;
        }
        if (decision[7 * (size_t)r + d.dist_right].type == kDistribute) {
            get_children(r, d.dist_right, children, num);
        } else {
            children[num++] = r;
        }
    }
};

// Triangle indices under BVH2 node n (a collapsed leaf: <= 3 triangles), left to right; returns the count.
uint32_t collect_tris(const std::vector<B2Node> &n2, uint32_t n, uint32_t *out)
{
    uint32_t stack[8];
    int sp = 0;
    uint32_t k = 0;
    stack[sp++] = n;
    while (sp) {
        const uint32_t c = stack[--sp];
        if (n2[c].count) {
            out[k++] = n2[c].left;
        } else {
            stack[sp++] = n2[c].left + 1;
            stack[sp++] = n2[c].left;
        }
    }
    return k;
}

inline float pow2_from_biased(uint8_t e)
{
    const uint32_t bits = (uint32_t)e << 23;
    float f;
    std::memcpy(&f, &bits, 4);
    return f;
}

// What the serial layout pass decides for one BVH8 node; the parallel pass fills the node from it.
struct NodePlan {
    uint32_t b2node;
    uint32_t children[8];  // BVH2 node ids
    int8_t slot_child[8];  // slot -> index into children, -1 = empty
    uint8_t num_children;
    uint32_t child_base, tri_base;
};

inline bool is_leaf_child(const std::vector<B2Node> &n2, const Collapser &col, uint32_t cn)
{
    return n2[cn].count || col.decision[7 * (size_t)cn].type == kLeaf;
}

// Slot assignment: slot s should hold the child met first by rays of octant s (bit 2/1/0 set =
// negative x/y/z direction); greedy minimum of dot(centroid offset, d_s).
void assign_slots(const std::vector<B2Node> &n2, NodePlan &pl)
{
    const Box &box = n2[pl.b2node].box;
    const int num_children = pl.num_children;
    float cx = 0.5f * (box.lo[0] + box.hi[0]), cy = 0.5f * (box.lo[1] + box.hi[1]), cz = 0.5f * (box.lo[2] + box.hi[2]);
    float cst[8][8];
    for (int c = 0; c < num_children; ++c) {
        const Box &b = n2[pl.children[c]].box;
        const float ox = 0.5f * (b.lo[0] + b.hi[0]) - cx, oy = 0.5f * (b.lo[1] + b.hi[1]) - cy,
                    oz = 0.5f * (b.lo[2] + b.hi[2]) - cz;
        for (int s = 0; s < 8; ++s) {
            const float dx = (s & 4) ? -1.f : 1.f, dy = (s & 2) ? -1.f : 1.f, dz = (s & 1) ? -1.f : 1.f;
            cst[c][s] = ox * dx + oy * dy + oz * dz;
        }
    }
    for (int s = 0; s < 8; ++s) {
        pl.slot_child[s] = -1;
    }
    bool child_done[8] = {false};
    for (int it = 0; it < num_children; ++it) {
        float best = std::numeric_limits<float>::max();
        int bc = -1, bs = -1;
        for (int c = 0; c < num_children; ++c) {
            if (child_done[c]) {
                continue;
            }
            for (int s = 0; s < 8; ++s) {
                if (pl.slot_child[s] >= 0) {
                    continue;
                }
                if (cst[c][s] < best || bc < 0) {  // (the first candidate is taken whatever its cost, as on the device)
                    best = cst[c][s];
                    bc = c;
                    bs = s;
                }
            }
        }
        child_done[bc] = true;
        pl.slot_child[bs] = (int8_t)bc;
    }
}

// Writes one BVH8 node (quantisation frame, child boxes, meta bytes) and its leaves' triangle order.
void fill_node(const std::vector<B2Node> &n2, const Collapser &col, const NodePlan &pl, Bvh8Node &out, uint32_t *tri_order)
{
    const Box &box = n2[pl.b2node].box;
    std::memset(&out, 0, sizeof(out));
    float max_ext = 0.f;
    for (int a = 0; a < 3; ++a) {
        out.p[a] = box.lo[a];
        max_ext = std::max(max_ext, box.hi[a] - box.lo[a]);
    }
    float step[3];
    for (int a = 0; a < 3; ++a) {
        // flat axes get a thin but non-zero grid so that every child box has thickness
        float ext = std::max(box.hi[a] - box.lo[a], max_ext * (1.f / 65536.f));
        ext = std::max(ext, 1e-30f);
        int e = (int)std::ceil(std::log2((double)ext / 255.0));
        e = std::min(std::max(e, -100), 100);
        // make sure the far plane of the node is representable: lo + 255*2^e >= hi
        while (e < 100 && (double)box.lo[a] + 255.0 * std::ldexp(1.0, e) < (double)box.hi[a]) {
            ++e;
        }
        out.e[a] = (uint8_t)(e + 127);
        step[a] = pow2_from_biased(out.e[a]);
    }
    out.child_base = pl.child_base;
    out.tri_base = pl.tri_base;

    uint8_t *qlo[3] = {out.qlo_x, out.qlo_y, out.qlo_z};
    uint8_t *qhi[3] = {out.qhi_x, out.qhi_y, out.qhi_z};
    uint32_t tri_off = 0;
    for (int s = 0; s < 8; ++s) {
        const int c = pl.slot_child[s];
        if (c < 0) {
            out.meta[s] = 0;
            continue;
        }
        const uint32_t cn = pl.children[c];
        const Box &b = n2[cn].box;
        for (int a = 0; a < 3; ++a) {
            const double p = out.p[a], st = step[a];
            int lo = (int)std::floor(((double)b.lo[a] - p) / st);
            int hi = (int)std::ceil(((double)b.hi[a] - p) / st);
            lo = std::min(std::max(lo, 0), 255);
            hi = std::min(std::max(hi, 0), 255);
            // conservative in double arithmetic (p + q*step is exact in double)
            while (lo > 0 && p + lo * st > (double)b.lo[a]) {
                --lo;
            }
            while (hi < 255 && p + hi * st < (double)b.hi[a]) {
                ++hi;
            }
            if (hi <= lo) {  // give flat boxes one grid cell of thickness
                if (hi < 255) {
                    hi = lo + 1;
                } else {
                    lo = hi - 1;
                }
            }
            qlo[a][s] = (uint8_t)lo;
            qhi[a][s] = (uint8_t)hi;
        }
        if (is_leaf_child(n2, col, cn)) {
            const uint32_t k = collect_tris(n2, cn, tri_order + pl.tri_base + tri_off);
            const uint8_t unary = k == 1 ? 0b001 : (k == 2 ? 0b011 : 0b111);
            out.meta[s] = (uint8_t)((unary << 5) | tri_off);
            tri_off += k;
        } else {
            out.meta[s] = (uint8_t)((0b001 << 5) | (24 + s));
            out.imask |= (uint8_t)(1u << s);
        }
    }
}

}  // namespace

void build_bvh8(const float *verts, size_t num_tris, int threads, Bvh8 &out)
{
    const auto t0 = std::chrono::steady_clock::now();
    out.nodes.clear();
    out.tri_order.clear();
    out.level_begin.clear();
    out.max_depth = 0;
    if (threads <= 0) {
        threads = std::max(1u, std::thread::hardware_concurrency());
    }
    for (int a = 0; a < 3; ++a) {
        out.scene_lo[a] = 0.f;
        out.scene_hi[a] = 0.f;
    }
    if (num_tris == 0) {
        Bvh8Node root;
        std::memset(&root, 0, sizeof(root));
        root.e[0] = root.e[1] = root.e[2] = 127;
        out.nodes.push_back(root);
        return;
    }
    const bool timing = std::getenv("CRT_BVH8_TIMING") != nullptr;
    auto lap = [&, last = t0](const char *what) mutable {
        const auto now = std::chrono::steady_clock::now();
        if (timing) {
            std::fprintf(stderr, "[bvh8] %-10s %.3f s\n", what, std::chrono::duration<double>(now - last).count());
        }
        last = now;
    };
    Bvh2Builder b2;
    b2.build(verts, (uint32_t)num_tris, threads);
    const std::vector<B2Node> &n2 = b2.nodes;
    for (int a = 0; a < 3; ++a) {
        out.scene_lo[a] = n2[0].box.lo[a];
        out.scene_hi[a] = n2[0].box.hi[a];
    }

    lap("bvh2");
    Collapser col(n2);
    col.run_parallel(0, threads);
    lap("collapse");

    // Layout pass, breadth-first, one level at a time: in parallel over the level's nodes, which BVH2
    // nodes become the children of each BVH8 node and which slot each takes; then serially, where the
    // node's children and triangles start. Siblings are contiguous (child_base + rank among the inner
    // children in slot order), triangles of a node likewise; the order is plain BFS.
    std::vector<NodePlan> plans;
    plans.reserve(num_tris / 6 + 16);  // ~1 node per 10 triangles in practice; grows if needed
    plans.emplace_back();
    plans[0].b2node = 0;
    uint32_t tri_total = 0;
    out.sah_cost = 0.0;
    const double root_area = std::max(1e-30f, n2[0].box.half_area());
    size_t level_begin = 0, level_end = 1;
    while (level_begin < level_end) {
        ++out.max_depth;
        out.level_begin.push_back((uint32_t)level_begin);
        const uint32_t kPlanBlock = 256;
        const uint32_t nb = (uint32_t)((level_end - level_begin + kPlanBlock - 1) / kPlanBlock);
        parallel_blocks(nb, threads, [&](uint32_t b) {
            const size_t e = std::min(level_end, level_begin + (size_t)(b + 1) * kPlanBlock);
            for (size_t i = level_begin + (size_t)b * kPlanBlock; i < e; ++i) {
                NodePlan &pl = plans[i];
                int num = 0;
                if (is_leaf_child(n2, col, pl.b2node)) {
                    // only possible for the scene root (<= 3 triangles): one leaf child
                    pl.children[num++] = pl.b2node;
                } else {
                    col.get_children(pl.b2node, 0, pl.children, num);
                }
                pl.num_children = (uint8_t)num;
                assign_slots(n2, pl);
            }
        });
        for (size_t cur = level_begin; cur < level_end; ++cur) {
            // (plans may reallocate below: index, do not hold references across emplace_back)
            plans[cur].child_base = (uint32_t)plans.size();
            plans[cur].tri_base = tri_total;
            out.sah_cost += n2[plans[cur].b2node].box.half_area() / root_area * kNodeCost;
            for (int s = 0; s < 8; ++s) {
                const int c = plans[cur].slot_child[s];
                if (c < 0) {
                    continue;
                }
                const uint32_t cn = plans[cur].children[c];
                if (is_leaf_child(n2, col, cn)) {
                    tri_total += col.tri_count[cn];
                } else {
                    plans.emplace_back();
                    plans.back().b2node = cn;
                }
            }
        }
        level_begin = level_end;
        level_end = plans.size();
    }
    out.level_begin.push_back((uint32_t)plans.size());
    lap("layout");
    // Fill pass (parallel): quantised child boxes, meta bytes and triangle order of every node.
    out.nodes.resize(plans.size());
    out.tri_order.resize(tri_total);
    {
        const uint32_t kFillBlock = 1024;
        const uint32_t nb = ((uint32_t)plans.size() + kFillBlock - 1) / kFillBlock;
        parallel_blocks(nb, threads, [&](uint32_t b) {
            const size_t e = std::min(plans.size(), (size_t)(b + 1) * kFillBlock);
            for (size_t i = (size_t)b * kFillBlock; i < e; ++i) {
                fill_node(n2, col, plans[i], out.nodes[i], out.tri_order.data());
            }
        });
    }
    lap("emit");
    out.build_seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

}  // namespace crt
