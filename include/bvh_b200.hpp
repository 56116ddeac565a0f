// include/bvh_b200.hpp -- C++17 host-side mirror of the reference crate's interface for the hot path,
// header-only, on top of the C ABI (bvh_b200.h).  Same names, argument meaning and error behaviour as
// svenstaro/bvh 0.12.0 (file:line relative to the reference checkout):
//
//   bvh::Aabb<T>            src/aabb/aabb_impl.rs:10-16   (empty/join/grow/size/center/surface_area/largest_axis)
//   bvh::Ray<T>             src/ray/ray_impl.rs:17-80     (Ray(origin, direction) normalises; intersects_aabb)
//   Bounded / BHShape       src/aabb/aabb_impl.rs:28-56, src/bounding_hierarchy.rs:53-65: any type with
//                           `Aabb<T> aabb() const`, `void set_bh_node_index(size_t)`, `size_t bh_node_index() const`
//   bvh::Bvh<T>::build / build_par    src/bvh/bvh_impl.rs:40-96, src/bounding_hierarchy.rs:158-177
//   Bvh<T>::nodes()                   `pub nodes` (src/bvh/bvh_impl.rs:27-33), materialised from the device
//   Bvh<T>::flatten()                 src/flat_bvh.rs:312-319
//   Bvh<T>::traverse / traverse_iterator / FlatBvh<T>::traverse     src/bvh/bvh_impl.rs:104-134, src/flat_bvh.rs:396-431
//   Bvh<T>::traverse_batch            the batched form (CSR), the reason the GPU path exists
//
// Where the reference panics, this mirror throws bvh::Error.  The build / flatten / traverse work runs on the
// GPU through libbvh_b200.so; the small Aabb / Ray helpers below are the value types callers need to
// implement `aabb()` for their shapes (they are not a CPU fallback for the path).
#pragma once
#include <cmath>
#include <algorithm>
#include <cstdint>
#include <limits>
#include <memory>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <vector>
#include <utility>

#include "bvh_b200.h"

namespace bvh {

struct Error : std::runtime_error {
    int status;
    Error(int s, const std::string& m) : std::runtime_error("bvh_b200: " + m), status(s) {}
};
inline void check(int status) {
    if (status != BVHGPU_OK) throw Error(status, bvhgpu_last_error());
}

template <class T> struct Aabb {                       // src/aabb/aabb_impl.rs:10-16
    T min[3], max[3];
    static Aabb empty() {                              // :119-124
        const T inf = std::numeric_limits<T>::infinity();
        return Aabb{{inf, inf, inf}, {-inf, -inf, -inf}};
    }
    static Aabb with_bounds(const T (&mn)[3], const T (&mx)[3]) { return Aabb{{mn[0], mn[1], mn[2]}, {mx[0], mx[1], mx[2]}}; }
    Aabb join(const Aabb& o) const {                   // :303-308
        Aabb r;
        for (int k = 0; k < 3; ++k) { r.min[k] = min[k] <= o.min[k] ? min[k] : o.min[k]; r.max[k] = max[k] >= o.max[k] ? max[k] : o.max[k]; }
        return r;
    }
    Aabb grow(const T (&p)[3]) const {                 // :375-380
        Aabb r;
        for (int k = 0; k < 3; ++k) { r.min[k] = min[k] <= p[k] ? min[k] : p[k]; r.max[k] = max[k] >= p[k] ? max[k] : p[k]; }
        return r;
    }
    void size(T (&s)[3]) const { for (int k = 0; k < 3; ++k) s[k] = max[k] - min[k]; }                 // :459-461
    void center(T (&c)[3]) const { for (int k = 0; k < 3; ++k) c[k] = min[k] * T(0.5) + max[k] * T(0.5); }   // :501-504
    T surface_area() const { T s[3]; size(s); return T(2) * ((s[0] * s[0] + s[1] * s[1]) + s[2] * s[2]); }   // :551-554
    int largest_axis() const { T s[3]; size(s); int a = 0; if (s[1] > s[a]) a = 1; if (s[2] > s[a]) a = 2; return a; }   // :594-596
    bool operator==(const Aabb& o) const { for (int k = 0; k < 3; ++k) if (min[k] != o.min[k] || max[k] != o.max[k]) return false; return true; }
};

template <class T> struct Ray {                        // src/ray/ray_impl.rs:17-29
    T origin[3], direction[3], inv_direction[3];
    Ray() = default;
    Ray(const T (&o)[3], const T (&d)[3]) {            // Ray::new, :70-80
        const T n = std::sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]);
        for (int k = 0; k < 3; ++k) { origin[k] = o[k]; direction[k] = d[k] / n; inv_direction[k] = T(1) / direction[k]; }
    }
    bool intersects_aabb(const Aabb<T>& b) const {     // src/ray/intersect_default.rs:16-37
        T l[3], r[3];
        for (int k = 0; k < 3; ++k) { l[k] = (b.min[k] - origin[k]) * inv_direction[k]; r[k] = (b.max[k] - origin[k]) * inv_direction[k]; }
        for (int k = 0; k < 3; ++k) if (std::isnan(l[k]) || std::isnan(r[k])) return false;
        T tmin = l[0] <= r[0] ? l[0] : r[0], tmax = l[0] >= r[0] ? l[0] : r[0];
        for (int k = 1; k < 3; ++k) {
            const T lo = l[k] <= r[k] ? l[k] : r[k], hi = l[k] >= r[k] ? l[k] : r[k];
            tmin = tmin >= lo ? tmin : lo;
            tmax = tmax <= hi ? tmax : hi;
        }
        return tmax >= (tmin > T(0) ? tmin : T(0));
    }
};

namespace detail {
template <class T> struct Abi;
template <> struct Abi<float> {
    using aabb = bvh_aabb3f; using ray = bvh_ray3f; using node = bvh_node3f; using flat = bvh_flat3f; using tree = bvhgpu_tree3f;
    static int build(bvhgpu_ctx* c, const aabb* a, size_t n, int m, tree** o) { return bvhgpu_build_f32x3(c, a, n, m, o); }
    static void free_tree(tree* t) { bvhgpu_tree_free_f32x3(t); }
    static int nodes(tree* t, node* o, uint32_t* i) { return bvhgpu_tree_nodes_f32x3(t, o, i); }
    static int flatten(tree* t, flat* o, size_t cap, size_t* len) { return bvhgpu_flatten_f32x3(t, o, cap, len); }
    static int traverse(tree* t, int m, const ray* r, size_t n, uint32_t* off, uint32_t* h, size_t cap, size_t* tot) { return bvhgpu_traverse_f32x3(t, m, r, n, off, h, cap, tot); }
    static int fetch(tree* t, uint32_t* h, size_t cap) { return bvhgpu_traverse_fetch_f32x3(t, h, cap); }
    static int refit(tree* t, const aabb* a, size_t n) { return bvhgpu_refit_f32x3(t, a, n); }
    static int optimize(tree* t, const aabb* a, size_t n, double g, size_t* r) { return bvhgpu_optimize_f32x3(t, a, n, g, r); }
    static int candidates(tree* t, const float* p, size_t n, uint32_t* off, uint32_t* c, size_t cap, size_t* tot) { return bvhgpu_nearest_candidates_f32x3(t, p, n, off, c, cap, tot); }
    static int update(tree* t, const uint32_t* c, const aabb* a, size_t m, double g, size_t* r) { return bvhgpu_update_f32x3(t, c, a, m, g, r); }
    static int set_triangles(tree* t, const float* abc, size_t n) { return bvhgpu_tree_set_triangles_f32x3(t, abc, n); }
    static int closest(tree* t, const ray* r, size_t n, int tri, uint32_t* s, float* d, float* uv) { return bvhgpu_closest_hit_f32x3(t, r, n, tri, s, d, uv); }
    static int any(tree* t, const ray* r, size_t n, const float* tm, int tri, uint32_t* s) { return bvhgpu_any_hit_f32x3(t, r, n, tm, tri, s); }
    static int multi(tree* t, const ray* r, size_t n, uint32_t k, const float* tm, int tri, uint32_t* s, float* d, float* uv) { return bvhgpu_multi_hit_f32x3(t, r, n, k, tm, tri, s, d, uv); }
    static int count_hits(tree* t, const ray* r, size_t n, const float* tm, uint32_t* f, uint32_t* b) { return bvhgpu_count_hits_f32x3(t, r, n, tm, f, b); }
    static int contains(tree* t, const float* p, size_t n, int rule, uint8_t* in) { return bvhgpu_contains_points_f32x3(t, p, n, rule, in); }
    static int signed_distance(tree* t, const float* p, size_t n, int rule, uint32_t* s, float* d, float* q) { return bvhgpu_signed_distance_f32x3(t, p, n, rule, s, d, q); }
    static int add(tree* t, const aabb* a, size_t k, double g, size_t* r) { return bvhgpu_add_shapes_f32x3(t, a, k, g, r); }
    static int remove(tree* t, const uint32_t* i, size_t k) { return bvhgpu_remove_shapes_f32x3(t, i, k); }
    static int overlap(tree* t, uint32_t* off, uint32_t* h, size_t cap, size_t* tot) { return bvhgpu_overlap_pairs_f32x3(t, off, h, cap, tot); }
    static int overlap_trees(tree* a, tree* b, uint32_t* off, uint32_t* h, size_t cap, size_t* tot) { return bvhgpu_overlap_trees_f32x3(a, b, off, h, cap, tot); }
    static int tri_pairs(tree* t, int skip, uint32_t* off, uint32_t* h, size_t cap, size_t* tot) { return bvhgpu_triangle_pairs_f32x3(t, skip, off, h, cap, tot); }
    static int tri_pairs_trees(tree* a, tree* b, uint32_t* off, uint32_t* h, size_t cap, size_t* tot) { return bvhgpu_triangle_pairs_trees_f32x3(a, b, off, h, cap, tot); }
};
template <> struct Abi<double> {
    using aabb = bvh_aabb3d; using ray = bvh_ray3d; using node = bvh_node3d; using flat = bvh_flat3d; using tree = bvhgpu_tree3d;
    static int build(bvhgpu_ctx* c, const aabb* a, size_t n, int m, tree** o) { return bvhgpu_build_f64x3(c, a, n, m, o); }
    static void free_tree(tree* t) { bvhgpu_tree_free_f64x3(t); }
    static int nodes(tree* t, node* o, uint32_t* i) { return bvhgpu_tree_nodes_f64x3(t, o, i); }
    static int flatten(tree* t, flat* o, size_t cap, size_t* len) { return bvhgpu_flatten_f64x3(t, o, cap, len); }
    static int traverse(tree* t, int m, const ray* r, size_t n, uint32_t* off, uint32_t* h, size_t cap, size_t* tot) { return bvhgpu_traverse_f64x3(t, m, r, n, off, h, cap, tot); }
    static int fetch(tree* t, uint32_t* h, size_t cap) { return bvhgpu_traverse_fetch_f64x3(t, h, cap); }
    static int refit(tree* t, const aabb* a, size_t n) { return bvhgpu_refit_f64x3(t, a, n); }
    static int optimize(tree* t, const aabb* a, size_t n, double g, size_t* r) { return bvhgpu_optimize_f64x3(t, a, n, g, r); }
    static int candidates(tree* t, const double* p, size_t n, uint32_t* off, uint32_t* c, size_t cap, size_t* tot) { return bvhgpu_nearest_candidates_f64x3(t, p, n, off, c, cap, tot); }
    static int update(tree* t, const uint32_t* c, const aabb* a, size_t m, double g, size_t* r) { return bvhgpu_update_f64x3(t, c, a, m, g, r); }
    static int set_triangles(tree* t, const double* abc, size_t n) { return bvhgpu_tree_set_triangles_f64x3(t, abc, n); }
    static int closest(tree* t, const ray* r, size_t n, int tri, uint32_t* s, double* d, double* uv) { return bvhgpu_closest_hit_f64x3(t, r, n, tri, s, d, uv); }
    static int any(tree* t, const ray* r, size_t n, const double* tm, int tri, uint32_t* s) { return bvhgpu_any_hit_f64x3(t, r, n, tm, tri, s); }
    static int multi(tree* t, const ray* r, size_t n, uint32_t k, const double* tm, int tri, uint32_t* s, double* d, double* uv) { return bvhgpu_multi_hit_f64x3(t, r, n, k, tm, tri, s, d, uv); }
    static int count_hits(tree* t, const ray* r, size_t n, const double* tm, uint32_t* f, uint32_t* b) { return bvhgpu_count_hits_f64x3(t, r, n, tm, f, b); }
    static int contains(tree* t, const double* p, size_t n, int rule, uint8_t* in) { return bvhgpu_contains_points_f64x3(t, p, n, rule, in); }
    static int signed_distance(tree* t, const double* p, size_t n, int rule, uint32_t* s, double* d, double* q) { return bvhgpu_signed_distance_f64x3(t, p, n, rule, s, d, q); }
    static int add(tree* t, const aabb* a, size_t k, double g, size_t* r) { return bvhgpu_add_shapes_f64x3(t, a, k, g, r); }
    static int remove(tree* t, const uint32_t* i, size_t k) { return bvhgpu_remove_shapes_f64x3(t, i, k); }
    static int overlap(tree* t, uint32_t* off, uint32_t* h, size_t cap, size_t* tot) { return bvhgpu_overlap_pairs_f64x3(t, off, h, cap, tot); }
    static int overlap_trees(tree* a, tree* b, uint32_t* off, uint32_t* h, size_t cap, size_t* tot) { return bvhgpu_overlap_trees_f64x3(a, b, off, h, cap, tot); }
    static int tri_pairs(tree* t, int skip, uint32_t* off, uint32_t* h, size_t cap, size_t* tot) { return bvhgpu_triangle_pairs_f64x3(t, skip, off, h, cap, tot); }
    static int tri_pairs_trees(tree* a, tree* b, uint32_t* off, uint32_t* h, size_t cap, size_t* tot) { return bvhgpu_triangle_pairs_trees_f64x3(a, b, off, h, cap, tot); }
};
struct Ctx {
    bvhgpu_ctx* h = nullptr;
    explicit Ctx(int device) { check(bvhgpu_create(device, &h)); }
    ~Ctx() { bvhgpu_destroy(h); }
};
inline std::shared_ptr<Ctx> default_ctx(int device = 0) {
    static std::shared_ptr<Ctx> ctx;
    if (!ctx) ctx = std::make_shared<Ctx>(device);
    return ctx;
}
}  // namespace detail

// BvhNode<T,3> (src/bvh/bvh_node.rs:21-47)
template <class T> struct BvhNode {
    bool leaf;
    size_t parent_index;
    size_t shape_index;                         // Leaf
    size_t child_l_index, child_r_index;        // Node
    Aabb<T> child_l_aabb, child_r_aabb;
};
// FlatNode<T,3> (src/flat_bvh.rs:17-46)
template <class T> struct FlatNode {
    Aabb<T> aabb;
    uint32_t entry_index, exit_index, shape_index;
    bool is_leaf() const { return entry_index == UINT32_MAX; }
};

template <class T> class Bvh;

// FlatBvh<T,3> = Vec<FlatNode> (src/flat_bvh.rs:153): the node array plus a handle on the device tree it came from.
template <class T> class FlatBvh {
  public:
    std::vector<FlatNode<T>> nodes;
    size_t size() const { return nodes.size(); }
    bool empty() const { return nodes.empty(); }
    template <class Shape> std::vector<const Shape*> traverse(const Ray<T>& ray, const std::vector<Shape>& shapes) const;   // src/flat_bvh.rs:396-431

  private:
    friend class Bvh<T>;
    const Bvh<T>* owner_ = nullptr;
};

template <class T> class Bvh {
    using A = detail::Abi<T>;

  public:
    Bvh() = default;
    Bvh(Bvh&& o) noexcept : ctx_(std::move(o.ctx_)), tree_(o.tree_), n_(o.n_) { o.tree_ = nullptr; }
    Bvh& operator=(Bvh&& o) noexcept { release(); ctx_ = std::move(o.ctx_); tree_ = o.tree_; n_ = o.n_; o.tree_ = nullptr; return *this; }
    Bvh(const Bvh&) = delete;
    Bvh& operator=(const Bvh&) = delete;
    ~Bvh() { release(); }

    // Bvh::build(&mut shapes): gathers Bounded::aabb() once per shape, builds on the GPU (bit-identical tree),
    // then calls BHShape::set_bh_node_index on every shape (src/bvh/bvh_node.rs:103).
    template <class Shape> static Bvh build(std::vector<Shape>& shapes) {
        Bvh b;
        b.ctx_ = detail::default_ctx();
        b.n_ = shapes.size();
        std::vector<typename A::aabb> boxes(shapes.size());
        for (size_t i = 0; i < shapes.size(); ++i) {
            const Aabb<T> a = shapes[i].aabb();
            for (int k = 0; k < 3; ++k) { boxes[i].min[k] = a.min[k]; boxes[i].max[k] = a.max[k]; }
        }
        check(A::build(b.ctx_->h, boxes.data(), boxes.size(), BVHGPU_BUILD_EXACT_SAH, &b.tree_));
        std::vector<uint32_t> idx(shapes.size());
        check(A::nodes(b.tree_, nullptr, idx.data()));
        for (size_t i = 0; i < shapes.size(); ++i) shapes[i].set_bh_node_index(idx[i]);
        return b;
    }
    // BoundingHierarchy::build_par (src/bounding_hierarchy.rs:170-177): rayon is off the hot path, same builder.
    template <class Shape> static Bvh build_par(std::vector<Shape>& shapes) { return build(shapes); }

    // `pub nodes: Vec<BvhNode>` (src/bvh/bvh_impl.rs:27-33)
    std::vector<BvhNode<T>> nodes() const {
        std::vector<typename A::node> raw(n_ ? 2 * n_ - 1 : 0);
        check(A::nodes(tree_, raw.data(), nullptr));
        std::vector<BvhNode<T>> out(raw.size());
        for (size_t i = 0; i < raw.size(); ++i) {
            const auto& r = raw[i];
            BvhNode<T>& o = out[i];
            o.leaf = r.child_l == BVHGPU_INVALID_INDEX;
            o.parent_index = r.parent;
            o.shape_index = o.leaf ? r.shape : 0;
            o.child_l_index = o.leaf ? 0 : r.child_l;
            o.child_r_index = o.leaf ? 0 : r.child_r;
            for (int k = 0; k < 3; ++k) {
                o.child_l_aabb.min[k] = r.l_aabb.min[k]; o.child_l_aabb.max[k] = r.l_aabb.max[k];
                o.child_r_aabb.min[k] = r.r_aabb.min[k]; o.child_r_aabb.max[k] = r.r_aabb.max[k];
            }
        }
        return out;
    }

    // Bvh::flatten (src/flat_bvh.rs:312-319)
    FlatBvh<T> flatten() const {
        const size_t cap = n_ == 0 ? 0 : (n_ == 1 ? 1 : 3 * n_ - 2);
        std::vector<typename A::flat> raw(cap);
        size_t len = 0;
        check(A::flatten(tree_, raw.data(), cap, &len));
        FlatBvh<T> f;
        f.owner_ = this;
        f.nodes.resize(len);
        for (size_t i = 0; i < len; ++i) {
            for (int k = 0; k < 3; ++k) { f.nodes[i].aabb.min[k] = raw[i].aabb.min[k]; f.nodes[i].aabb.max[k] = raw[i].aabb.max[k]; }
            f.nodes[i].entry_index = raw[i].entry_index; f.nodes[i].exit_index = raw[i].exit_index; f.nodes[i].shape_index = raw[i].shape_index;
        }
        return f;
    }

    // Bvh::flatten_custom (src/flat_bvh.rs:96-143, 240-251): the caller's constructor is applied to (aabb, entry, exit, shape) of every
    // FlatNode, in the reference's emission order -- the array is the device-built FlatBvh, the constructor runs on the host.
    template <class F> auto flatten_custom(const F& constructor) const -> std::vector<decltype(constructor(std::declval<const Aabb<T>&>(), uint32_t(), uint32_t(), uint32_t()))> {
        const FlatBvh<T> f = flatten();
        std::vector<decltype(constructor(std::declval<const Aabb<T>&>(), uint32_t(), uint32_t(), uint32_t()))> out;
        out.reserve(f.nodes.size());
        for (const auto& nd : f.nodes) out.push_back(constructor(nd.aabb, nd.entry_index, nd.exit_index, nd.shape_index));
        return out;
    }

    // Batched traversal: CSR (offsets[nrays+1], shape indices in the reference's DFS order).
    void traverse_batch(const std::vector<Ray<T>>& rays, std::vector<uint32_t>& offsets, std::vector<uint32_t>& hits,
                        int mode = BVHGPU_TRAVERSE_BVH) const {
        static_assert(sizeof(Ray<T>) == sizeof(typename A::ray), "Ray layout");
        offsets.assign(rays.size() + 1, 0);
        hits.assign(4 * rays.size() + 1024, 0);
        size_t total = 0;
        const int st = A::traverse(tree_, mode, reinterpret_cast<const typename A::ray*>(rays.data()), rays.size(), offsets.data(), hits.data(), hits.size(), &total);
        if (st == BVHGPU_ERR_CAPACITY && total <= UINT32_MAX) { hits.resize(total); check(A::fetch(tree_, hits.data(), total)); }
        else { check(st); hits.resize(total); }
    }
    // Bvh::traverse (src/bvh/bvh_impl.rs:104-119)
    template <class Shape> std::vector<const Shape*> traverse(const Ray<T>& ray, const std::vector<Shape>& shapes, int mode = BVHGPU_TRAVERSE_BVH) const {
        std::vector<uint32_t> off, hits;
        traverse_batch(std::vector<Ray<T>>{ray}, off, hits, mode);
        std::vector<const Shape*> out;
        for (uint32_t h : hits) out.push_back(&shapes.at(h));
        return out;
    }
    // Bvh::traverse_iterator (src/bvh/bvh_impl.rs:128-134): same sequence; the "iterator" is the returned vector's range.
    template <class Shape> std::vector<const Shape*> traverse_iterator(const Ray<T>& ray, const std::vector<Shape>& shapes) const { return traverse(ray, shapes); }

    // every pair of shapes whose current AABBs intersect, each once: CSR indexed by shape, row s = the shapes whose leaf comes after
    // s's leaf in DFS order and whose box meets s's box (bvhgpu_overlap_pairs_*).  offsets gets n + 1 entries.
    void overlap_pairs(std::vector<uint32_t>& offsets, std::vector<uint32_t>& hits) const {
        offsets.assign(n_ + 1, 0);
        hits.resize(std::max<size_t>(4 * n_, 1024));
        size_t total = 0;
        const int st = A::overlap(tree_, offsets.data(), hits.data(), hits.size(), &total);
        if (st == BVHGPU_ERR_CAPACITY && total <= UINT32_MAX) { hits.resize(total); check(A::fetch(tree_, hits.data(), total)); }
        else { check(st); hits.resize(total); }
    }
    // every pair (a, b) of a shape of this tree and a shape of `other` whose current AABBs intersect: CSR indexed by this tree's
    // shapes, row a = other's shapes whose box meets a's, in other's DFS order (bvhgpu_overlap_trees_*).  Both trees must share a
    // context (the default one does); other may be *this.  offsets gets n + 1 entries.
    void overlap_pairs_with(const Bvh<T>& other, std::vector<uint32_t>& offsets, std::vector<uint32_t>& hits) const {
        offsets.assign(n_ + 1, 0);
        hits.resize(std::max<size_t>(4 * n_, 1024));
        size_t total = 0;
        const int st = A::overlap_trees(tree_, other.tree_, offsets.data(), hits.data(), hits.size(), &total);
        if (st == BVHGPU_ERR_CAPACITY && total <= UINT32_MAX) { hits.resize(total); check(A::fetch(tree_, hits.data(), total)); }
        else { check(st); hits.resize(total); }
    }
    // every pair of triangles (set_triangles) that meet, decided exactly: row s of overlap_pairs keeping the shapes whose closed
    // triangle has a point in common with s's (bvhgpu_triangle_pairs_*).  Excluded triangles (non-finite or degenerate) meet nothing;
    // skip_shared drops pairs that share a vertex; in f64 a triangle with a nonzero coordinate outside [2^-300, 2^300] keeps its box
    // pairs.  offsets gets n + 1 entries.
    void triangle_pairs(bool skip_shared, std::vector<uint32_t>& offsets, std::vector<uint32_t>& hits) const {
        offsets.assign(n_ + 1, 0);
        hits.resize(std::max<size_t>(4 * n_, 1024));
        size_t total = 0;
        const int st = A::tri_pairs(tree_, skip_shared ? 1 : 0, offsets.data(), hits.data(), hits.size(), &total);
        if (st == BVHGPU_ERR_CAPACITY && total <= UINT32_MAX) { hits.resize(total); check(A::fetch(tree_, hits.data(), total)); }
        else { check(st); hits.resize(total); }
    }
    // every pair (a, b) of a triangle of this tree and a triangle of `other` that meet (a shared vertex is a contact): row a of
    // overlap_pairs_with filtered the same way (bvhgpu_triangle_pairs_trees_*).  Both trees must share a context; other may be *this.
    void triangle_pairs_with(const Bvh<T>& other, std::vector<uint32_t>& offsets, std::vector<uint32_t>& hits) const {
        offsets.assign(n_ + 1, 0);
        hits.resize(std::max<size_t>(4 * n_, 1024));
        size_t total = 0;
        const int st = A::tri_pairs_trees(tree_, other.tree_, offsets.data(), hits.data(), hits.size(), &total);
        if (st == BVHGPU_ERR_CAPACITY && total <= UINT32_MAX) { hits.resize(total); check(A::fetch(tree_, hits.data(), total)); }
        else { check(st); hits.resize(total); }
    }
    // the data-parallel part of Bvh::update_shapes (src/bvh/optimization.rs:304-351): refit after shapes moved
    template <class Shape> void refit(const std::vector<Shape>& shapes) {
        std::vector<typename A::aabb> boxes(shapes.size());
        for (size_t i = 0; i < shapes.size(); ++i) {
            const Aabb<T> a = shapes[i].aabb();
            for (int k = 0; k < 3; ++k) { boxes[i].min[k] = a.min[k]; boxes[i].max[k] = a.max[k]; }
        }
        check(A::refit(tree_, boxes.data(), boxes.size()));
    }
    // Bvh::nearest_to (src/bvh/bvh_impl.rs:221-238) for shapes with `T distance_squared(const T (&point)[3]) const`
    // (PointDistance, src/point_query.rs:7-10): the device returns a short candidate list that contains the nearest shape, the
    // shape's own distance decides.  Returns {nullptr, 0} for an empty tree.
    template <class Shape> std::pair<const Shape*, T> nearest_to(const T (&point)[3], const std::vector<Shape>& shapes) const {
        uint32_t off[2] = {0, 0};
        std::vector<uint32_t> cand(1024);
        size_t total = 0;
        const int st = A::candidates(tree_, point, 1, off, cand.data(), cand.size(), &total);
        if (st == BVHGPU_ERR_CAPACITY && total <= UINT32_MAX) { cand.resize(total); check(A::fetch(tree_, cand.data(), total)); }
        else check(st);
        const Shape* best = nullptr;
        T best_d = T(0);
        for (size_t i = 0; i < total; ++i) {
            const Shape& s = shapes.at(cand[i]);
            const T d = s.distance_squared(point);
            if (!best || d < best_d) { best = &s; best_d = d; }
        }
        return {best, best ? std::sqrt(best_d) : T(0)};
    }
    // Bvh::update_shapes (src/bvh/optimization.rs:290-302): refit + in-place exact rebuild of the subtrees that grew by more
    // than `max_growth`; writes the new leaf node indices back (BHShape::set_bh_node_index).  Returns the rebuilt shape count.
    template <class Shape> size_t update_shapes(std::vector<Shape>& shapes, double max_growth = 1.5) {
        std::vector<typename A::aabb> boxes(shapes.size());
        for (size_t i = 0; i < shapes.size(); ++i) {
            const Aabb<T> a = shapes[i].aabb();
            for (int k = 0; k < 3; ++k) { boxes[i].min[k] = a.min[k]; boxes[i].max[k] = a.max[k]; }
        }
        size_t rebuilt = 0;
        check(A::optimize(tree_, boxes.data(), boxes.size(), max_growth, &rebuilt));
        if (rebuilt) {
            std::vector<uint32_t> idx(shapes.size());
            check(A::nodes(tree_, nullptr, idx.data()));
            for (size_t i = 0; i < shapes.size(); ++i) shapes[i].set_bh_node_index(idx[i]);
        }
        return rebuilt;
    }
    // Bvh::update_shapes with its own signature (src/bvh/optimization.rs:304-315): the indices of the changed shapes + the shapes.
    // Only the changed shapes' AABBs cross the boundary.  max_growth <= 0: refit only.
    template <class Shape> size_t update_shapes(const std::vector<size_t>& changed_shape_indices, std::vector<Shape>& shapes, double max_growth = 1.5) {
        std::vector<uint32_t> idx(changed_shape_indices.size());
        std::vector<typename A::aabb> boxes(changed_shape_indices.size());
        for (size_t i = 0; i < idx.size(); ++i) {
            idx[i] = (uint32_t)changed_shape_indices[i];
            const Aabb<T> a = shapes.at(changed_shape_indices[i]).aabb();
            for (int k = 0; k < 3; ++k) { boxes[i].min[k] = a.min[k]; boxes[i].max[k] = a.max[k]; }
        }
        size_t rebuilt = 0;
        check(A::update(tree_, idx.data(), boxes.data(), idx.size(), max_growth, &rebuilt));
        if (rebuilt) {
            std::vector<uint32_t> ni(shapes.size());
            check(A::nodes(tree_, nullptr, ni.data()));
            for (size_t i = 0; i < shapes.size(); ++i) shapes[i].set_bh_node_index(ni[i]);
        }
        return rebuilt;
    }
    // Closest hit per ray (what callers build from traverse + Ray::intersects_triangle, src/ray/ray_impl.rs:154-213).  Triangles: 9 T per
    // shape (a, b, c), set once; triangle == false: the shape whose AABB is entered first.
    void set_triangles(const std::vector<T>& abc9) { check(A::set_triangles(tree_, abc9.data(), abc9.size() / 9)); }
    void closest_hit(const std::vector<Ray<T>>& rays, bool triangles, std::vector<uint32_t>& shape, std::vector<T>& distance) const {
        shape.assign(rays.size(), 0); distance.assign(rays.size(), T(0));
        check(A::closest(tree_, reinterpret_cast<const typename A::ray*>(rays.data()), rays.size(), triangles ? 1 : 0, shape.data(), distance.data(), nullptr));
    }
    // Any hit per ray (occlusion: what callers build as traverse(..).iter().any(|s| ray.intersects_triangle(..).distance < tmax)):
    // shape[i] = a shape hit at a distance < tmax[i] (tmax empty: +inf for every ray), UINT32_MAX if none.  triangles == false: a shape
    // whose AABB the ray enters before tmax[i] (exact); true: a triangle whose Moeller-Trumbore distance is < tmax[i].
    void any_hit(const std::vector<Ray<T>>& rays, const std::vector<T>& tmax, bool triangles, std::vector<uint32_t>& shape) const {
        if (!tmax.empty() && tmax.size() != rays.size()) throw Error(BVHGPU_ERR_INVALID, "any_hit: one limit per ray, or none");
        shape.assign(rays.size(), 0);
        check(A::any(tree_, reinterpret_cast<const typename A::ray*>(rays.data()), rays.size(), tmax.empty() ? nullptr : tmax.data(), triangles ? 1 : 0, shape.data()));
    }
    // The first k hits per ray (transparency, several LiDAR returns, entry and exit of a wall): row i of shape / distance (k slots each,
    // row-major) lists the hits at a distance < tmax[i] (tmax empty: no limit) in ascending (distance, tie) order, then UINT32_MAX and
    // +inf.  triangle == false: the shapes whose own AABB the ray enters, by entry (exact); true: Moeller-Trumbore hits of the triangles
    // of set_triangles, with u, v in uv (2 per slot) when it is given.  k = 1 without a limit is closest_hit.  1 <= k <= 64.
    void multi_hit(const std::vector<Ray<T>>& rays, uint32_t k, const std::vector<T>& tmax, bool triangles, std::vector<uint32_t>& shape,
                   std::vector<T>& distance, std::vector<T>* uv = nullptr) const {
        if (!tmax.empty() && tmax.size() != rays.size()) throw Error(BVHGPU_ERR_INVALID, "multi_hit: one limit per ray, or none");
        shape.assign(rays.size() * k, 0); distance.assign(rays.size() * k, T(0));
        if (uv) uv->assign(2 * rays.size() * k, T(0));
        check(A::multi(tree_, reinterpret_cast<const typename A::ray*>(rays.data()), rays.size(), k, tmax.empty() ? nullptr : tmax.data(),
                       triangles ? 1 : 0, shape.data(), distance.data(), uv ? uv->data() : nullptr));
    }
    // Crossing counts per ray over the triangles of set_triangles: front[i] / back[i] = the triangles ray i crosses at a distance < tmax[i]
    // (tmax empty: no limit) through their front / back face (Ray::intersects_triangle with the winding as given / reversed).
    void count_hits(const std::vector<Ray<T>>& rays, const std::vector<T>& tmax, std::vector<uint32_t>& front, std::vector<uint32_t>& back) const {
        if (!tmax.empty() && tmax.size() != rays.size()) throw Error(BVHGPU_ERR_INVALID, "count_hits: one limit per ray, or none");
        front.assign(rays.size(), 0); back.assign(rays.size(), 0);
        check(A::count_hits(tree_, reinterpret_cast<const typename A::ray*>(rays.data()), rays.size(), tmax.empty() ? nullptr : tmax.data(),
                            front.data(), back.data()));
    }
    // Point-in-mesh over the closed mesh of set_triangles (3 T per point): inside[i] = 1 when two of three fixed rays from point i vote
    // inside under `rule` (BVHGPU_FILL_EVEN_ODD or BVHGPU_FILL_NONZERO).  Points on the surface are undefined.
    void contains(const std::vector<T>& points, int rule, std::vector<uint8_t>& inside) const {
        inside.assign(points.size() / 3, 0);
        check(A::contains(tree_, points.data(), points.size() / 3, rule, inside.data()));
    }
    // Signed distance to the closed mesh: knn_triangles with k = 1 (shape, distance, and closest point when given), the distance negated
    // where contains(rule) says inside.
    void signed_distance(const std::vector<T>& points, int rule, std::vector<uint32_t>& shape, std::vector<T>& distance,
                         std::vector<T>* closest = nullptr) const {
        const size_t n = points.size() / 3;
        shape.assign(n, 0); distance.assign(n, T(0));
        if (closest) closest->assign(3 * n, T(0));
        check(A::signed_distance(tree_, points.data(), n, rule, shape.data(), distance.data(), closest ? closest->data() : nullptr));
    }
    size_t num_shapes() const { return n_; }

    // Bvh::add_shape(shapes, new_shape_index) (src/bvh/optimization.rs:67-207): the caller has pushed the new shape, which must be the
    // last one.  No rebuild (max_growth 0): the reference's own topology.  The node index of EVERY shape may change (preorder positions
    // shift), so all of them are written back with set_bh_node_index.
    template <class Shape> void add_shape(std::vector<Shape>& shapes, size_t new_shape_index) {
        if (new_shape_index + 1 != shapes.size() || new_shape_index != n_)
            throw Error(BVHGPU_ERR_INVALID, "add_shape: the new shape must be the last one, at index num_shapes()");
        add_shapes(shapes, new_shape_index, 0.0);
    }
    // Batched add: shapes[first_new ..] are new (first_new == num_shapes()); max_growth >= 1 also rebuilds degraded subtrees.
    // Returns the number of shapes in rebuilt subtrees.
    template <class Shape> size_t add_shapes(std::vector<Shape>& shapes, size_t first_new, double max_growth = 1.5) {
        if (first_new != n_ || first_new > shapes.size()) throw Error(BVHGPU_ERR_INVALID, "add_shapes: first_new must be num_shapes()");
        std::vector<typename A::aabb> boxes(shapes.size() - first_new);
        for (size_t i = 0; i < boxes.size(); ++i) {
            const Aabb<T> a = shapes[first_new + i].aabb();
            for (int k = 0; k < 3; ++k) { boxes[i].min[k] = a.min[k]; boxes[i].max[k] = a.max[k]; }
        }
        size_t rebuilt = 0;
        check(A::add(tree_, boxes.data(), boxes.size(), max_growth, &rebuilt));
        n_ = shapes.size();
        write_node_indices(shapes);
        return rebuilt;
    }
    // Bvh::remove_shape(shapes, i, swap_shape) (src/bvh/optimization.rs:208-301).  swap_shape == true: the last shape takes index i,
    // in the tree and in `shapes` (swap_remove), as the reference does.  swap_shape == false is not representable -- device trees
    // number their shapes densely -- and throws Error(BVHGPU_ERR_UNSUPPORTED).
    template <class Shape> void remove_shape(std::vector<Shape>& shapes, size_t i, bool swap_shape) {
        if (!swap_shape) throw Error(BVHGPU_ERR_UNSUPPORTED, "remove_shape: swap_shape == false is not supported (device trees number their shapes densely)");
        remove_shapes(shapes, std::vector<size_t>{i});
    }
    // Batched remove of distinct indices: survivors with index >= n-k move into the vacated indices < n-k, smallest hole first, in the
    // tree and in `shapes`, which then loses its last k entries.  For one index this is remove_shape(i, true).
    template <class Shape> void remove_shapes(std::vector<Shape>& shapes, const std::vector<size_t>& indices) {
        if (shapes.size() != n_) throw Error(BVHGPU_ERR_INVALID, "remove_shapes: shapes.size() != num_shapes()");
        std::vector<uint32_t> idx(indices.size());
        for (size_t j = 0; j < idx.size(); ++j) idx[j] = (uint32_t)indices[j];
        check(A::remove(tree_, idx.data(), idx.size()));
        const size_t k = indices.size(), m = n_ - k;
        std::vector<char> gone(n_, 0);
        for (size_t s : indices) gone[s] = 1;
        size_t t = m;
        for (size_t h = 0; h < m; ++h) {
            if (!gone[h]) continue;
            while (gone[t]) ++t;
            std::swap(shapes[h], shapes[t++]);
        }
        shapes.erase(shapes.begin() + (std::ptrdiff_t)m, shapes.end());
        n_ = m;
        write_node_indices(shapes);
    }

  private:
    template <class Shape> void write_node_indices(std::vector<Shape>& shapes) {
        std::vector<uint32_t> idx(shapes.size());
        if (!idx.empty()) check(A::nodes(tree_, nullptr, idx.data()));
        for (size_t i = 0; i < shapes.size(); ++i) shapes[i].set_bh_node_index(idx[i]);
    }
    void release() { if (tree_) { A::free_tree(tree_); tree_ = nullptr; } }
    std::shared_ptr<detail::Ctx> ctx_;
    typename A::tree* tree_ = nullptr;
    size_t n_ = 0;
};

template <class T> template <class Shape>
std::vector<const Shape*> FlatBvh<T>::traverse(const Ray<T>& ray, const std::vector<Shape>& shapes) const {
    if (!owner_) return {};
    return owner_->traverse(ray, shapes, BVHGPU_TRAVERSE_FLAT);
}

}  // namespace bvh
