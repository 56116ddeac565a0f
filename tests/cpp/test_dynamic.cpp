// tests/cpp/test_dynamic.cpp -- the fuzz target's Add / Remove mutations (push + add_shape(len-1); remove_shape(i, true) + the
// vector's swap_remove) driven through the C++ mirror include/bvh_b200.hpp.  After every call each shape's bh_node_index must be
// the device leaf that holds it, and the tree must cover exactly the shapes in the vector.
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>

#include "bvh_b200.hpp"

struct Box {
    bvh::Aabb<float> box;
    size_t id = 0;                               // identity of the shape, follows it through swap-removes
    size_t node = ~size_t(0);
    bvh::Aabb<float> aabb() const { return box; }
    void set_bh_node_index(size_t i) { node = i; }
    size_t bh_node_index() const { return node; }
};

static int failures = 0;
#define EXPECT(c, ...) do { if (!(c)) { std::printf("FAIL %s:%d: ", __FILE__, __LINE__); std::printf(__VA_ARGS__); std::printf("\n"); ++failures; } } while (0)

static Box random_box(std::mt19937& rng, size_t id) {
    std::uniform_real_distribution<float> pos(-1000.f, 1000.f), ext(0.f, 30.f);
    Box b;
    for (int k = 0; k < 3; ++k) { b.box.min[k] = pos(rng); b.box.max[k] = b.box.min[k] + ext(rng); }
    b.id = id;
    return b;
}

static void check_indices(const bvh::Bvh<float>& tree, const std::vector<Box>& shapes, int step) {
    EXPECT(tree.num_shapes() == shapes.size(), "step %d: %zu shapes in the tree, %zu in the vector", step, tree.num_shapes(), shapes.size());
    const auto nodes = tree.nodes();
    EXPECT(nodes.size() == (shapes.empty() ? 0 : 2 * shapes.size() - 1), "step %d: %zu nodes", step, nodes.size());
    for (size_t i = 0; i < shapes.size(); ++i) {
        const size_t ni = shapes[i].bh_node_index();
        EXPECT(ni < nodes.size() && nodes[ni].leaf && nodes[ni].shape_index == i, "step %d: shape %zu has bh_node_index %zu", step, i, ni);
    }
}

int main() {
    std::mt19937 rng(12345);
    std::vector<Box> shapes;
    size_t next_id = 0;
    for (int i = 0; i < 300; ++i) shapes.push_back(random_box(rng, next_id++));
    auto tree = bvh::Bvh<float>::build(shapes);
    check_indices(tree, shapes, -1);
    for (int step = 0; step < 400; ++step) {
        const bool add = shapes.size() < 2 || (rng() % 100) < 55;
        if (add) {
            shapes.push_back(random_box(rng, next_id++));
            tree.add_shape(shapes, shapes.size() - 1);
        } else {
            const size_t i = rng() % shapes.size();
            const size_t last_id = shapes.back().id;
            tree.remove_shape(shapes, i, true);
            EXPECT(i == shapes.size() || shapes[i].id == last_id, "step %d: swap_remove did not move the last shape into %zu", step, i);
        }
        check_indices(tree, shapes, step);
        if (failures) break;
    }
    // batched forms
    std::vector<size_t> idx;
    for (size_t i = 0; i < shapes.size(); i += 3) idx.push_back(i);
    tree.remove_shapes(shapes, idx);
    check_indices(tree, shapes, 1000);
    const size_t first = shapes.size();
    for (int i = 0; i < 120; ++i) shapes.push_back(random_box(rng, next_id++));
    tree.add_shapes(shapes, first, 1.5);
    check_indices(tree, shapes, 1001);
    // swap_shape == false is not representable
    bool threw = false;
    try { tree.remove_shape(shapes, 0, false); } catch (const bvh::Error& e) { threw = e.status == BVHGPU_ERR_UNSUPPORTED; }
    EXPECT(threw, "remove_shape(swap_shape = false) must throw Error(BVHGPU_ERR_UNSUPPORTED)");
    check_indices(tree, shapes, 1002);
    if (failures) { std::printf("%d failures\n", failures); return 1; }
    std::printf("dynamic add/remove through the C++ mirror passed\n");
    return 0;
}
