// tests/cpp/test_any_hit.cpp -- Bvh<T>::any_hit of the C++ host mirror include/bvh_b200.hpp on fixed scenes, through the C ABI on
// the GPU: occlusion by unit boxes and by triangles along a line of boxes, with per-ray limits, no limits, and the refusals.
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

template <class T> static void run() {
    const T inf = std::numeric_limits<T>::infinity();
    const uint32_t none = UINT32_MAX;
    // boxes centred at x = 10, 20, ..., 100 on the x axis; one box off the axis
    std::vector<UnitBox<T>> boxes;
    for (int i = 1; i <= 10; ++i) boxes.emplace_back(T(10 * i), T(0), T(0));
    boxes.emplace_back(T(50), T(30), T(0));
    bvh::Bvh<T> b = bvh::Bvh<T>::build(boxes);
    // rays from the origin along +x (the first box is entered at 9.5), from (50, 1, 0) along +y (only the off-axis box, entered at 28.5),
    // and along -x (nothing)
    std::vector<bvh::Ray<T>> rays{bvh::Ray<T>({T(0), T(0), T(0)}, {T(1), T(0), T(0)}), bvh::Ray<T>({T(50), T(1), T(0)}, {T(0), T(1), T(0)}),
                                  bvh::Ray<T>({T(0), T(0), T(0)}, {T(-1), T(0), T(0)})};
    std::vector<uint32_t> s;
    b.any_hit(rays, {}, false, s);                                      // no limit: every ray that enters a box
    REQUIRE(s.size() == 3 && s[0] != none && s[0] < 10 && s[1] == 10 && s[2] == none);
    b.any_hit(rays, {T(9.5), T(28.5), inf}, false, s);                  // the entry itself is not < tmax
    REQUIRE(s[0] == none && s[1] == none && s[2] == none);
    b.any_hit(rays, {std::nextafter(T(9.5), inf), T(29), inf}, false, s);
    REQUIRE(s[0] == 0 && s[1] == 10 && s[2] == none);                   // only box 0 lies before tmax on the +x ray
    b.any_hit(rays, {T(95), T(0), -T(0)}, false, s);
    REQUIRE(s[0] != none && s[0] < 9 && s[1] == none && s[2] == none);
    b.any_hit(rays, {std::nan(""), -T(1), inf}, false, s);
    REQUIRE(s[0] == none && s[1] == none && s[2] == none);
    // the closest hit agrees: a hit with tmax = next float above its distance, none with tmax = its distance
    std::vector<uint32_t> cs;
    std::vector<T> cd;
    b.closest_hit(rays, false, cs, cd);
    std::vector<T> above, at;
    for (T d : cd) { above.push_back(std::nextafter(d, inf)); at.push_back(d); }
    b.any_hit(rays, above, false, s);
    for (size_t i = 0; i < rays.size(); ++i) REQUIRE((s[i] != none) == (cs[i] != none));
    b.any_hit(rays, at, false, s);
    for (size_t i = 0; i < rays.size(); ++i) REQUIRE(s[i] == none);
    // triangles: one facing -x in the plane x = 10 i of every box on the axis (at y = +-0.5), a tiny one in the off-axis box
    bool refused = false;
    try { b.any_hit(rays, {}, true, s); } catch (const bvh::Error& e) { refused = e.status == BVHGPU_ERR_INVALID; }
    REQUIRE(refused);                                                   // triangle mode needs set_triangles first
    std::vector<T> tris;
    for (int i = 1; i <= 10; ++i) {
        const T x = T(10 * i);
        const T t[9] = {x, T(-0.5), T(-0.5), x, T(-0.5), T(0.5), x, T(0.5), T(0)};
        tris.insert(tris.end(), t, t + 9);
    }
    const T t10[9] = {T(50), T(30), T(0), T(50.1), T(30), T(0), T(50), T(30.1), T(0)};
    tris.insert(tris.end(), t10, t10 + 9);
    b.set_triangles(tris);
    b.any_hit(rays, {}, true, s);
    REQUIRE(s[0] != none && s[0] < 10 && s[1] == none && s[2] == none);   // ray 1 runs in the plane of the off-axis triangle: det = 0
    b.any_hit(rays, {T(10), inf, inf}, true, s);                         // the first triangle lies at exactly 10: not < 10
    REQUIRE(s[0] == none);
    b.any_hit(rays, {T(10.5), inf, inf}, true, s);
    REQUIRE(s[0] == 0);
    refused = false;
    try { b.any_hit(rays, {T(1)}, false, s); } catch (const bvh::Error& e) { refused = e.status == BVHGPU_ERR_INVALID; }
    REQUIRE(refused);                                                   // one limit per ray, or none
    // an empty tree: no hit
    std::vector<UnitBox<T>> empty;
    bvh::Bvh<T> e = bvh::Bvh<T>::build(empty);
    e.any_hit(rays, {}, false, s);
    REQUIRE(s[0] == none && s[1] == none && s[2] == none);
}

int main() {
    run<float>();
    run<double>();
    std::printf("all any-hit tests passed\n");
    return 0;
}
