// tests/cpp/test_triangle_pairs.cpp -- Bvh<T>::triangle_pairs and triangle_pairs_with of the C++ host mirror include/bvh_b200.hpp on
// two fixed tetrahedra, through the C ABI on the GPU.  A = conv{(0,0,0), (2,0,0), (0,2,0), (0,0,2)}; B = A + (2, 0, 0) touches A at the
// single point (2, 0, 0), a vertex of three faces of each; C = A + (3, 0, 0) misses A.  Every two faces of one tetrahedron share an
// edge.  Exit code 0 = all passed.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <set>
#include <utility>
#include <vector>

#include "bvh_b200.hpp"

#define REQUIRE(cond)                                                              \
    do {                                                                           \
        if (!(cond)) { std::fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); std::exit(1); } \
    } while (0)

template <class T> struct Tri {
    T v[9];
    size_t node_index = 0;
    bvh::Aabb<T> aabb() const {
        bvh::Aabb<T> a;
        for (int k = 0; k < 3; ++k) {
            a.min[k] = std::fmin(std::fmin(v[k], v[3 + k]), v[6 + k]);
            a.max[k] = std::fmax(std::fmax(v[k], v[3 + k]), v[6 + k]);
        }
        return a;
    }
    void set_bh_node_index(size_t i) { node_index = i; }
    size_t bh_node_index() const { return node_index; }
};

// The four faces (0 1 2), (0 1 3), (0 2 3), (1 2 3) of the tetrahedron A shifted by dx along x.
template <class T> static void tetra(T dx, std::vector<Tri<T>>& out) {
    const T v[4][3] = {{dx, 0, 0}, {dx + 2, 0, 0}, {dx, 2, 0}, {dx, 0, 2}};
    const int faces[4][3] = {{0, 1, 2}, {0, 1, 3}, {0, 2, 3}, {1, 2, 3}};
    for (auto& f : faces) {
        Tri<T> t;
        for (int j = 0; j < 3; ++j)
            for (int k = 0; k < 3; ++k) t.v[3 * j + k] = v[f[j]][k];
        out.push_back(t);
    }
}

// the CSR as a set of (row, hit), checking that no pair appears twice
static std::set<std::pair<uint32_t, uint32_t>> pairs(const std::vector<uint32_t>& off, const std::vector<uint32_t>& hits) {
    std::set<std::pair<uint32_t, uint32_t>> out;
    for (size_t s = 0; s + 1 < off.size(); ++s)
        for (uint32_t i = off[s]; i < off[s + 1]; ++i) REQUIRE(out.insert({(uint32_t)s, hits[i]}).second);
    REQUIRE(off.back() == hits.size());
    return out;
}

template <class T> static bvh::Bvh<T> with_triangles(std::vector<Tri<T>>& tris) {
    bvh::Bvh<T> b = bvh::Bvh<T>::build(tris);
    std::vector<T> abc;
    for (auto& t : tris) abc.insert(abc.end(), t.v, t.v + 9);
    b.set_triangles(abc);
    return b;
}

template <class T> static void run() {
    std::vector<Tri<T>> ab, a, b, c;
    tetra<T>(0, ab); tetra<T>(2, ab);
    tetra<T>(0, a); tetra<T>(2, b); tetra<T>(3, c);
    std::vector<uint32_t> off, hits;
    {
        bvh::Bvh<T> unset = bvh::Bvh<T>::build(a);
        bool refused = false;
        try { unset.triangle_pairs(true, off, hits); } catch (const bvh::Error& e) { refused = e.status == BVHGPU_ERR_INVALID; }
        REQUIRE(refused);                                                  // needs set_triangles first
    }
    // both tetrahedra in one tree: with skip_shared every contact is at a shared vertex, so nothing is left; without it the 6 face
    // pairs of each tetrahedron and the 3 x 3 faces around (2, 0, 0), each once
    bvh::Bvh<T> both = with_triangles(ab);
    both.triangle_pairs(true, off, hits);
    REQUIRE(off.size() == 9 && hits.empty());
    both.triangle_pairs(false, off, hits);
    std::set<std::pair<uint32_t, uint32_t>> got = pairs(off, hits), want;
    for (auto p : got) REQUIRE(want.insert({std::min(p.first, p.second), std::max(p.first, p.second)}).second);
    std::set<std::pair<uint32_t, uint32_t>> expect;
    for (uint32_t s = 0; s < 4; ++s)
        for (uint32_t t = s + 1; t < 4; ++t) { expect.insert({s, t}); expect.insert({s + 4, t + 4}); }
    for (uint32_t s : {0u, 1u, 3u})
        for (uint32_t t : {4u, 5u, 6u}) expect.insert({s, t});
    REQUIRE(want == expect);
    // between trees: A against B touches at the faces around (2, 0, 0); A against C does not touch
    bvh::Bvh<T> ta = with_triangles(a), tb = with_triangles(b), tc = with_triangles(c);
    ta.triangle_pairs_with(tb, off, hits);
    got = pairs(off, hits);
    expect.clear();
    for (uint32_t s : {0u, 1u, 3u})
        for (uint32_t t : {0u, 1u, 2u}) expect.insert({s, t});
    REQUIRE(off.size() == 5 && got == expect);
    ta.triangle_pairs_with(tc, off, hits);
    REQUIRE(off.size() == 5 && hits.empty() && off[4] == 0);
    // a tree against itself: every face meets itself and the three others
    ta.triangle_pairs_with(ta, off, hits);
    REQUIRE(pairs(off, hits).size() == 16);
}

int main() {
    run<float>();
    run<double>();
    std::printf("all triangle pair tests passed\n");
    return 0;
}
