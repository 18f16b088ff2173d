// sorted_traversal.cpp — RESEARCH CODE, not product and not part of the test suite.
// CPU experiment behind DESIGN.md §2 "measured headroom": replaces the product's CWBVH-style traversal order
// (children of a node visited in ray-octant order, whole node groups on the stack) by stack entries that carry
// each child's own entry distance, and counts node visits / triangle tests on the bench scene's ray population.
// Built by scripts/experiments/run_sorted_traversal.py on top of chameleonrt_b200/csrc/hostcheck.cpp (the
// test-only host instantiation of the product's builder + traversal), which it includes textually.
//   mode 1: octant order as the product, but every child is its own stack entry and is culled at pop when its
//           entry distance exceeds the current hit; leaf slots beyond the current hit are skipped
//   mode 0: children pushed far-to-near (true distance order), culled at pop
//   mode 2: mode 0 with the leaf triangle groups deferred as distance-keyed entries too
//   mode 3: mode 1 with the truly nearest hit child moved to the top of the stack (one min-selection, no sort)
#include <cstdio>
#include <functional>
#include "../../chameleonrt_b200/csrc/hostcheck.cpp"

// ---------------- experiment: distance-sorted traversal with per-child entry distances on the stack
namespace {
struct Ent { uint32_t node; float tmin; };
inline void child_boxes(const float4 *nodes, const crt::TravState &s, uint32_t node_index, float *tmin8, bool *hit8,
                        uint32_t &imask, uint32_t &child_base, uint32_t &tri_base, uint8_t *meta8, float *area8 = nullptr,
                        float *tmax8 = nullptr)
{
    using namespace crt;
    const Ray &ray = s.ray;
    const float4 *np = nodes + (size_t)node_index * 5;
    const float4 n0 = np[0], n1 = np[1], n2 = np[2], n3 = np[3], n4 = np[4];
    const uint32_t e_imask = f2u(n0.w);
    const float adx = u2f((e_imask & 0xffu) << 23) * s.idx * 32768.f;
    const float ady = u2f(((e_imask >> 8) & 0xffu) << 23) * s.idy * 32768.f;
    const float adz = u2f(((e_imask >> 16) & 0xffu) << 23) * s.idz * 32768.f;
    const float ob0x = (n0.x - ray.ox) * s.idx, ob0y = (n0.y - ray.oy) * s.idy, ob0z = (n0.z - ray.oz) * s.idz;
    const float obx = ob0x - adx, oby = ob0y - ady, obz = ob0z - adz;
    const float sx = 4e-7f * fabsf(ob0x) + 2.4e-7f * fabsf(adx);
    const float sy = 4e-7f * fabsf(ob0y) + 2.4e-7f * fabsf(ady);
    const float sz = 4e-7f * fabsf(ob0z) + 2.4e-7f * fabsf(adz);
    imask = e_imask >> 24;
    child_base = f2u(n1.x);
    tri_base = f2u(n1.y);
    for (int half = 0; half < 2; ++half) {
        const uint32_t meta4 = f2u(half == 0 ? n1.z : n1.w);
        const uint32_t qlox = f2u(half == 0 ? n2.x : n2.y), qloy = f2u(half == 0 ? n2.z : n2.w);
        const uint32_t qloz = f2u(half == 0 ? n3.x : n3.y), qhix = f2u(half == 0 ? n3.z : n3.w);
        const uint32_t qhiy = f2u(half == 0 ? n4.x : n4.y), qhiz = f2u(half == 0 ? n4.z : n4.w);
        const uint32_t xmin = ray.dx < 0.f ? qhix : qlox, xmax = ray.dx < 0.f ? qlox : qhix;
        const uint32_t ymin = ray.dy < 0.f ? qhiy : qloy, ymax = ray.dy < 0.f ? qloy : qhiy;
        const uint32_t zmin = ray.dz < 0.f ? qhiz : qloz, zmax = ray.dz < 0.f ? qloz : qhiz;
        for (int j = 0; j < 4; ++j) {
            const int slot = half * 4 + j;
            meta8[slot] = (meta4 >> (8 * j)) & 0xff;
            const float tminx = fma_(byte_unit(xmin, j, s.one), adx, obx - sx);
            const float tminy = fma_(byte_unit(ymin, j, s.one), ady, oby - sy);
            const float tminz = fma_(byte_unit(zmin, j, s.one), adz, obz - sz);
            const float tmaxx = fma_(byte_unit(xmax, j, s.one), adx, obx + sx);
            const float tmaxy = fma_(byte_unit(ymax, j, s.one), ady, oby + sy);
            const float tmaxz = fma_(byte_unit(zmax, j, s.one), adz, obz + sz);
            const float tmin = fmaxf(fmaxf(tminx, tminy), fmaxf(tminz, ray.tnear));
            const float tmax = fminf(fminf(tmaxx, tmaxy), fminf(tmaxz, s.tfar));
            tmin8[slot] = tmin;
            hit8[slot] = meta8[slot] != 0 && tmin <= tmax;
            if (tmax8) {
                tmax8[slot] = tmax;
            }
            if (area8) {
                const float ex = u2f((e_imask & 0xffu) << 23), ey = u2f(((e_imask >> 8) & 0xffu) << 23),
                            ez = u2f(((e_imask >> 16) & 0xffu) << 23);
                const float dx = ex * (float)(((qhix >> (8 * j)) & 0xff) - ((qlox >> (8 * j)) & 0xff));
                const float dy = ey * (float)(((qhiy >> (8 * j)) & 0xff) - ((qloy >> (8 * j)) & 0xff));
                const float dz = ez * (float)(((qhiz >> (8 * j)) & 0xff) - ((qloz >> (8 * j)) & 0xff));
                area8[slot] = dx * dy + dy * dz + dz * dx;
            }
        }
    }
}
}  // namespace

// mode 0: stack entries carry the child's entry distance, nearest child first, culled at pop
// mode 1: like the product (octant order) but with cull-at-pop by entry distance
extern "C" void crt_hostcheck_trace_exp(void *p, const float *rays, uint64_t n, int any_hit, int mode, float *hits, uint32_t *counters)
{
    using namespace crt;
    HostCheck *h = static_cast<HostCheck *>(p);
    const float4 *nodes = reinterpret_cast<const float4 *>(h->node_f4.data());
    const float4 *tris = reinterpret_cast<const float4 *>(h->tri_records.data());
    for (uint64_t i = 0; i < n; ++i) {
        Ray r;
        std::memcpy(&r, rays + 8 * i, 32);
        TravState s;
        trav_init(s, r);
        Ent stack[256];
        int sp = 0;
        stack[sp++] = Ent{0, r.tnear};
        uint32_t nvis = 0, ntri = 0, maxsp = 0, nempty = 0;
        bool done = false;
        while (sp && !done) {
            const Ent e = stack[--sp];
            if (mode < 10 && e.tmin > s.tfar) {
                continue;
            }
            if (e.node & 0x80000000u) {
                const uint32_t k = (e.node >> 29) & 3u, first = e.node & 0x1fffffffu;
                uint2 tg;
                tg.x = first;
                tg.y = (1u << k) - 1u;
                while (tg.y) {
                    ++ntri;
                    if (test_next_triangle(tris, s, tg) && any_hit) {
                        done = true;
                        break;
                    }
                }
                continue;
            }
            ++nvis;
            float tmin8[8], area8[8], tmax8[8];
            bool hit8[8];
            uint8_t meta8[8];
            uint32_t imask, child_base, tri_base;
            child_boxes(nodes, s, e.node, tmin8, hit8, imask, child_base, tri_base, meta8, area8, tmax8);
            if (mode >= 10) {
                // any-hit ordering experiments: the stack key is a priority, not a distance (nothing is culled:
                // an any-hit ray's interval never shrinks). Highest key is visited first.
                for (int slot = 0; slot < 8; ++slot) {
                    if (hit8[slot] && (imask & (1u << slot))) {
                        const float key = mode == 10 ? tmin8[slot]                          // farthest entry first
                                          : mode == 11 ? area8[slot]                          // largest child first
                                          : mode == 12 ? (tmax8[slot] - tmin8[slot])          // longest ray segment inside first
                                                       : (tmax8[slot] - tmin8[slot]) * area8[slot];
                        tmin8[slot] = -key;  // reuse the sort below: entries sorted far-to-near by "tmin"
                    }
                }
            }
            {
                bool any_child = false;
                for (int slot = 0; slot < 8; ++slot) {
                    any_child = any_child || hit8[slot];
                }
                nempty += any_child ? 0u : 1u;
            }
            // leaves first (as the product does: triangles of a node are tested when the node is visited)
            Ent inner[16];
            int ni = 0;
            for (int slot = 0; slot < 8; ++slot) {
                if (!hit8[slot]) {
                    continue;
                }
                if (imask & (1u << slot)) {
                    const uint32_t rel = (uint32_t)popc(imask & ((1u << slot) - 1u));
                    inner[ni++] = Ent{child_base + rel, tmin8[slot]};
                } else {
                    const uint32_t off = meta8[slot] & 0x1f, un = meta8[slot] >> 5;
                    const uint32_t k = un == 1 ? 1 : (un == 3 ? 2 : 3);
                    if (mode == 2) {
                        inner[ni++] = Ent{0x80000000u | (k << 29) | (tri_base + off), tmin8[slot]};
                        continue;
                    }
                    if (mode < 10 && tmin8[slot] > s.tfar) {
                        continue;
                    }
                    uint2 tg;
                    tg.x = tri_base;
                    tg.y = ((1u << k) - 1u) << off;
                    while (tg.y) {
                        ++ntri;
                        if (test_next_triangle(tris, s, tg) && any_hit) {
                            done = true;
                            break;
                        }
                    }
                    if (done) {
                        break;
                    }
                }
            }
            if (mode == 0 || mode == 2 || mode == 4 || mode >= 10) {
                // far first onto the stack
                for (int a = 0; a < ni; ++a) {
                    for (int b = a + 1; b < ni; ++b) {
                        if (inner[b].tmin > inner[a].tmin) {
                            Ent t = inner[a];
                            inner[a] = inner[b];
                            inner[b] = t;
                        }
                    }
                }
                for (int a = 0; a < ni; ++a) {
                    stack[sp++] = inner[a];
                }
            } else {
                // octant order as the product: slot s visited in order of (s ^ octant) descending priority
                // product visits highest bit of (slot ^ oct_inv) first; emulate by sorting on that key
                const uint32_t oi = s.oct_inv4 & 0x7u;
                // recover slots: recompute from node index relation is lossy; approximate by entry order of key
                // (inner[] was filled in slot order, so slot of inner[a] is the a-th set inner bit among hit ones)
                int slots[8], q = 0;
                for (int slot = 0; slot < 8; ++slot) {
                    if (hit8[slot] && (imask & (1u << slot))) {
                        slots[q++] = slot;
                    }
                }
                for (int a = 0; a < ni; ++a) {
                    for (int b = a + 1; b < ni; ++b) {
                        if (((uint32_t)slots[b] ^ oi) < ((uint32_t)slots[a] ^ oi)) {
                            Ent t = inner[a]; inner[a] = inner[b]; inner[b] = t;
                            int ts = slots[a]; slots[a] = slots[b]; slots[b] = ts;
                        }
                    }
                }
                if (mode == 3 && ni > 1) {
                    // octant order, except that the truly nearest child is moved to the top of the stack
                    int best_a = 0;
                    for (int a = 1; a < ni; ++a) {
                        if (inner[a].tmin < inner[best_a].tmin) {
                            best_a = a;
                        }
                    }
                    const Ent t = inner[best_a];
                    for (int a = best_a; a + 1 < ni; ++a) {
                        inner[a] = inner[a + 1];
                    }
                    inner[ni - 1] = t;
                }
                for (int a = 0; a < ni; ++a) {
                    stack[sp++] = inner[a];  // lowest key pushed first -> highest key popped first
                }
            }
            if ((uint32_t)sp > maxsp) {
                maxsp = sp;
            }
        }
        float *o = hits + 4 * i;
        o[0] = s.hit.t;
        o[1] = s.hit.u;
        o[2] = s.hit.v;
        std::memcpy(&o[3], &s.hit.flat, 4);
        counters[3 * i] = nvis;
        counters[3 * i + 1] = ntri;
        counters[3 * i + 2] = mode == 4 ? nempty : maxsp;
    }
}

// ---------------- debugging aid: follow the path from the root to the leaf that holds a given triangle (by
// flattened primitive id) and report, level by level, whether the ray's box test accepts the child on that path
extern "C" void crt_hostcheck_explain(void *p, const float *ray8, uint32_t flat_id)
{
    using namespace crt;
    HostCheck *h = static_cast<HostCheck *>(p);
    const float4 *nodes = reinterpret_cast<const float4 *>(h->node_f4.data());
    uint32_t leaf_index = 0xffffffffu;
    for (size_t i = 0; i < h->shade.size(); ++i) {
        if (h->shade[i].flat_id == flat_id) {
            leaf_index = (uint32_t)i;
        }
    }
    std::printf("triangle flat %u is leaf-order index %u\n", flat_id, leaf_index);
    Ray r;
    std::memcpy(&r, ray8, 32);
    TravState s;
    trav_init(s, r);
    // depth-first search for the node path
    struct Frame { uint32_t node; int slot; };
    std::vector<uint32_t> path;
    std::vector<int> slots;
    std::function<bool(uint32_t)> find = [&](uint32_t node) -> bool {
        float tmin8[8], tmax8[8], area8[8];
        bool hit8[8];
        uint8_t meta8[8];
        uint32_t imask, child_base, tri_base;
        child_boxes(nodes, s, node, tmin8, hit8, imask, child_base, tri_base, meta8, area8, tmax8);
        for (int slot = 0; slot < 8; ++slot) {
            if (meta8[slot] == 0) continue;
            bool contains = false;
            if (imask & (1u << slot)) {
                const uint32_t rel = (uint32_t)popc(imask & ((1u << slot) - 1u));
                contains = find(child_base + rel);
            } else {
                const uint32_t off = meta8[slot] & 0x1f, un = meta8[slot] >> 5;
                const uint32_t k = un == 1 ? 1 : (un == 3 ? 2 : 3);
                contains = leaf_index >= tri_base + off && leaf_index < tri_base + off + k;
            }
            if (contains) {
                std::printf("  node %u slot %d (%s): box test %s  tmin %.9g tmax %.9g\n", node, slot, (imask & (1u << slot)) ? "inner" : "leaf",
                            hit8[slot] ? "HIT" : "MISS", tmin8[slot], tmax8[slot]);
                return true;
            }
        }
        return false;
    };
    find(0);
}
