// tests/cpp/test_multi_hit.cpp -- Bvh<T>::multi_hit of the C++ host mirror include/bvh_b200.hpp on fixed scenes, through the C ABI on
// the GPU: the first k boxes and triangles along a line of boxes, with per-ray limits, no limits, uv, padding and the refusals.
// Exit code 0 = all passed.
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

template <class T> struct UnitBox {
    T pos[3];
    size_t node_index = 0;
    UnitBox(T x, T y, T z) : pos{x, y, z} {}
    bvh::Aabb<T> aabb() const {
        bvh::Aabb<T> a;
        for (int k = 0; k < 3; ++k) { a.min[k] = pos[k] + T(-0.5); a.max[k] = pos[k] + T(0.5); }
        return a;
    }
    void set_bh_node_index(size_t i) { node_index = i; }
    size_t bh_node_index() const { return node_index; }
};

template <class T> static bool refused(const bvh::Bvh<T>& b, const std::vector<bvh::Ray<T>>& rays, uint32_t k, const std::vector<T>& tmax, bool tri) {
    std::vector<uint32_t> s;
    std::vector<T> d;
    try { b.multi_hit(rays, k, tmax, tri, s, d); } catch (const bvh::Error& e) { return e.status == BVHGPU_ERR_INVALID; }
    return false;
}

template <class T> static void run() {
    const T inf = std::numeric_limits<T>::infinity();
    const uint32_t none = UINT32_MAX;
    // boxes centred at x = 10, 20, ..., 100 on the x axis (shapes 0 .. 9); one box off the axis (shape 10)
    std::vector<UnitBox<T>> boxes;
    for (int i = 1; i <= 10; ++i) boxes.emplace_back(T(10 * i), T(0), T(0));
    boxes.emplace_back(T(50), T(30), T(0));
    bvh::Bvh<T> b = bvh::Bvh<T>::build(boxes);
    // rays from the origin along +x (boxes entered at 9.5, 19.5, ..., 99.5), from (50, 1, 0) along +y (only the off-axis box, at
    // 28.5), and along -x (nothing)
    std::vector<bvh::Ray<T>> rays{bvh::Ray<T>({T(0), T(0), T(0)}, {T(1), T(0), T(0)}), bvh::Ray<T>({T(50), T(1), T(0)}, {T(0), T(1), T(0)}),
                                  bvh::Ray<T>({T(0), T(0), T(0)}, {T(-1), T(0), T(0)})};
    std::vector<uint32_t> s;
    std::vector<T> d, uv;
    b.multi_hit(rays, 3, {}, false, s, d, &uv);
    REQUIRE(s.size() == 9 && d.size() == 9 && uv.size() == 18);
    REQUIRE(s[0] == 0 && s[1] == 1 && s[2] == 2 && d[0] == T(9.5) && d[1] == T(19.5) && d[2] == T(29.5));
    REQUIRE(s[3] == 10 && d[3] == T(28.5) && s[4] == none && d[4] == inf && s[5] == none);
    REQUIRE(s[6] == none && s[7] == none && s[8] == none && d[8] == inf);
    for (T x : uv) REQUIRE(x == T(0));                                   // AABB mode: zeros
    b.multi_hit(rays, 64, {T(40), T(28.5), inf}, false, s, d);            // the limit is strict: the entry itself is not < tmax
    REQUIRE(s[0] == 0 && s[3] == 3 && s[4] == none && d[3] == T(39.5) && s[64] == none && s[128] == none);
    b.multi_hit(rays, 12, {}, false, s, d);                               // every box on the +x ray, in order
    for (int j = 0; j < 10; ++j) REQUIRE(s[j] == uint32_t(j) && d[j] == T(10 * j + 9.5));
    REQUIRE(s[10] == none && s[11] == none);
    b.multi_hit(rays, 2, {std::nan(""), -T(0), T(-1)}, false, s, d);
    for (uint32_t x : s) REQUIRE(x == none);
    // k = 1 is closest_hit
    std::vector<uint32_t> cs;
    std::vector<T> cd;
    b.closest_hit(rays, false, cs, cd);
    b.multi_hit(rays, 1, {}, false, s, d);
    for (size_t i = 0; i < rays.size(); ++i) REQUIRE(s[i] == cs[i] && (d[i] == cd[i] || (std::isinf(d[i]) && std::isinf(cd[i]))));
    // triangles: one facing -x in the plane x = 10 i of every box on the axis, a tiny one in the off-axis box
    REQUIRE(refused(b, rays, 2, {}, true));                               // triangle mode needs set_triangles first
    std::vector<T> tris;
    for (int i = 1; i <= 10; ++i) {
        const T x = T(10 * i);
        const T t[9] = {x, T(-0.5), T(-0.5), x, T(-0.5), T(0.5), x, T(0.5), T(0)};
        tris.insert(tris.end(), t, t + 9);
    }
    const T t10[9] = {T(50), T(30), T(0), T(50.1), T(30), T(0), T(50), T(30.1), T(0)};
    tris.insert(tris.end(), t10, t10 + 9);
    b.set_triangles(tris);
    b.multi_hit(rays, 4, {}, true, s, d, &uv);
    REQUIRE(s[0] == 0 && s[1] == 1 && s[2] == 2 && s[3] == 3 && d[0] == T(10) && d[3] == T(40));
    REQUIRE(uv[0] == T(0.25) && uv[1] == T(0.5));                         // the hit point (10, 0, 0) = a + 0.25 ab + 0.5 ac
    for (int j = 4; j < 12; ++j) REQUIRE(s[j] == none && d[j] == inf && uv[2 * j] == T(0) && uv[2 * j + 1] == T(0));
    b.multi_hit(rays, 4, {T(30), inf, inf}, true, s, d);                  // the triangle at exactly 30 is not < 30
    REQUIRE(s[0] == 0 && s[1] == 1 && s[2] == none);
    // refusals
    REQUIRE(refused(b, rays, 0, {}, false));
    REQUIRE(refused(b, rays, 65, {}, false));
    REQUIRE(refused(b, rays, 2, {T(1)}, false));                          // one limit per ray, or none
    // an empty tree: rows of padding
    std::vector<UnitBox<T>> empty;
    bvh::Bvh<T> e = bvh::Bvh<T>::build(empty);
    e.multi_hit(rays, 2, {}, false, s, d);
    for (size_t j = 0; j < s.size(); ++j) REQUIRE(s[j] == none && d[j] == inf);
}

int main() {
    run<float>();
    run<double>();
    std::printf("all multi-hit tests passed\n");
    return 0;
}
