// tests/cpp/test_crossings.cpp -- Bvh<T>::count_hits, contains and signed_distance of the C++ host mirror include/bvh_b200.hpp on a
// fixed cube (12 triangles, outward winding), through the C ABI on the GPU: crossings of rays through and past it, the centre inside
// and points offset by 2 outside under both rules, signed distances, and the refusals.  Exit code 0 = all passed.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <limits>
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

// The unit cube [-1, 1]^3 as 12 triangles, counter-clockwise seen from outside.
template <class T> static std::vector<Tri<T>> cube() {
    const int quads[6][4][3] = {{{-1, -1, -1}, {-1, 1, -1}, {1, 1, -1}, {1, -1, -1}}, {{-1, -1, 1}, {1, -1, 1}, {1, 1, 1}, {-1, 1, 1}},
                                {{-1, -1, -1}, {1, -1, -1}, {1, -1, 1}, {-1, -1, 1}}, {{-1, 1, -1}, {-1, 1, 1}, {1, 1, 1}, {1, 1, -1}},
                                {{-1, -1, -1}, {-1, -1, 1}, {-1, 1, 1}, {-1, 1, -1}}, {{1, -1, -1}, {1, 1, -1}, {1, 1, 1}, {1, -1, 1}}};
    std::vector<Tri<T>> out;
    for (auto& q : quads)
        for (int h = 0; h < 2; ++h) {
            const int idx[3] = {0, 1 + h, 2 + h};
            Tri<T> t;
            for (int j = 0; j < 3; ++j)
                for (int k = 0; k < 3; ++k) t.v[3 * j + k] = T(q[idx[j]][k]);
            out.push_back(t);
        }
    return out;
}

template <class T> static void run() {
    const T inf = std::numeric_limits<T>::infinity();
    std::vector<Tri<T>> tris = cube<T>();
    bvh::Bvh<T> b = bvh::Bvh<T>::build(tris);
    std::vector<T> abc;
    for (auto& t : tris) abc.insert(abc.end(), t.v, t.v + 9);
    std::vector<uint32_t> f, k;
    std::vector<uint8_t> in;
    std::vector<T> pts{T(0), T(0), T(0), T(2), T(0), T(0), T(0), T(-2), T(0), T(0.1), T(0.2), T(2.3), T(0.5), T(-0.25), T(0.125)};
    bool refused = false;
    try { b.contains(pts, BVHGPU_FILL_EVEN_ODD, in); } catch (const bvh::Error& e) { refused = e.status == BVHGPU_ERR_INVALID; }
    REQUIRE(refused);                                                     // needs set_triangles first
    b.set_triangles(abc);
    // a ray through the cube enters a front face and leaves through a back face; from inside only the back face; past it nothing
    std::vector<bvh::Ray<T>> rays{bvh::Ray<T>({T(-5), T(0.1), T(0.3)}, {T(1), T(0.01), T(0.02)}),
                                  bvh::Ray<T>({T(0.2), T(0.1), T(0.3)}, {T(0.3), T(1), T(0.1)}),
                                  bvh::Ray<T>({T(-5), T(3), T(0)}, {T(1), T(0), T(0)})};
    b.count_hits(rays, {}, f, k);
    REQUIRE(f[0] == 1 && k[0] == 1 && f[1] == 0 && k[1] == 1 && f[2] == 0 && k[2] == 0);
    b.count_hits(rays, {T(5), inf, inf}, f, k);                           // the exit at x = 1 lies beyond 5 along the first ray: ~6
    REQUIRE(f[0] == 1 && k[0] == 0 && k[1] == 1);
    b.count_hits(rays, {T(0), -T(0), std::nan("")}, f, k);
    for (size_t i = 0; i < 3; ++i) REQUIRE(f[i] == 0 && k[i] == 0);
    // the centre and a point inside are inside, points offset by 2 are outside, under both rules
    for (int rule : {BVHGPU_FILL_EVEN_ODD, BVHGPU_FILL_NONZERO}) {
        b.contains(pts, rule, in);
        REQUIRE(in.size() == 5 && in[0] == 1 && in[1] == 0 && in[2] == 0 && in[3] == 0 && in[4] == 1);
    }
    std::vector<uint32_t> s;
    std::vector<T> d, q;
    b.signed_distance(pts, BVHGPU_FILL_EVEN_ODD, s, d, &q);
    const T want[5] = {T(-1), T(1), T(1), T(1.3), T(-0.5)};
    for (int i = 0; i < 5; ++i) REQUIRE(s[i] != UINT32_MAX && std::fabs(d[i] - want[i]) < T(1e-5));
    REQUIRE(std::fabs(q[3] - T(1)) < T(1e-5) && std::fabs(q[4]) < T(1e-5) && std::fabs(q[5]) < T(1e-5));   // (2, 0, 0) -> (1, 0, 0)
    refused = false;
    try { b.contains(pts, 7, in); } catch (const bvh::Error& e) { refused = e.status == BVHGPU_ERR_INVALID; }
    REQUIRE(refused);
    refused = false;
    try { b.count_hits(rays, {T(1)}, f, k); } catch (const bvh::Error& e) { refused = e.status == BVHGPU_ERR_INVALID; }
    REQUIRE(refused);
}

int main() {
    run<float>();
    run<double>();
    std::printf("all crossing tests passed\n");
    return 0;
}
