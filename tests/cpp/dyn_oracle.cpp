// tests/cpp/dyn_oracle.cpp -- TEST INFRASTRUCTURE ONLY.  The oracle's restatement of the reference's sequential Bvh::add_shape /
// Bvh::remove_shape (oracle/bvh_oracle.hpp, src/bvh/optimization.rs:67-301), re-emitted in Bvh::build's preorder layout so that it
// can be compared with the device's batched add / remove node for node.  Built by tests/dynoracle.py with g++ -ffp-contract=off.
#include "../../oracle/bvh_oracle.hpp"

namespace {

// Preorder re-emission: child_l = i + 1, child_r = i + 2 n_l, Node::shape of inner nodes = shapes below; leaf shapes through `relabel`.
template <class T>
uint32_t canonical(const orc::DynBvh<T>& b, const std::vector<uint32_t>& relabel, orc::Node<T>* out, uint32_t* node_index) {
    if (b.nodes.empty()) return 0;
    std::vector<uint32_t> cnt(b.nodes.size(), 1);
    {   // shapes below every node (post order)
        std::vector<std::pair<uint32_t, int>> st{{0u, 0}};
        while (!st.empty()) {
            auto& f = st.back();
            const orc::Node<T>& nd = b.nodes[f.first];
            if (nd.is_leaf()) { st.pop_back(); continue; }
            if (f.second == 0) { f.second = 1; const uint32_t l = nd.child_l, r = nd.child_r; st.push_back({l, 0}); st.push_back({r, 0}); }
            else { cnt[f.first] = cnt[nd.child_l] + cnt[nd.child_r]; st.pop_back(); }
        }
    }
    uint32_t next = 0;
    std::vector<std::pair<uint32_t, uint32_t>> st{{0u, 0u}};                 // (old node, new parent)
    while (!st.empty()) {
        const auto [i, par] = st.back();
        st.pop_back();
        const uint32_t j = next++;
        orc::Node<T> nd = b.nodes[i];
        nd.parent = par;
        if (nd.is_leaf()) {
            nd.shape = relabel[nd.shape];
            node_index[nd.shape] = j;
        } else {
            nd.shape = cnt[i];
            nd.child_l = j + 1;
            nd.child_r = j + 2 * cnt[b.nodes[i].child_l];
            st.push_back({b.nodes[i].child_r, j});
            st.push_back({b.nodes[i].child_l, j});
        }
        out[j] = nd;
    }
    return next;
}

template <class T>
orc::DynBvh<T> load(const orc::Node<T>* nodes, uint32_t n_nodes, const uint32_t* node_index, uint32_t n) {
    orc::DynBvh<T> b;
    b.nodes.assign(nodes, nodes + n_nodes);
    b.node_index.assign(node_index, node_index + n);
    return b;
}

// shapes[0 .. n + k): the tree covers [0, n); shapes n .. n+k-1 are added one by one.  nodes / node_index sized for the result.
template <class T>
uint32_t add(orc::Node<T>* nodes, uint32_t n_nodes, uint32_t* node_index, uint32_t n, const orc::Aabb3<T>* shapes, uint32_t k) {
    orc::DynBvh<T> b = load(nodes, n_nodes, node_index, n);
    b.node_index.resize((size_t)n + k);
    std::vector<uint32_t> ident((size_t)n + k);
    for (uint32_t s = 0; s < n + k; ++s) ident[s] = s;
    for (uint32_t s = n; s < n + k; ++s) orc::add_shape(b, shapes, s);
    return canonical(b, ident, nodes, node_index);
}

// remove_shape(i, swap = false) for every index in order, then the swap rule's renumbering.
template <class T>
uint32_t remove(orc::Node<T>* nodes, uint32_t n_nodes, uint32_t* node_index, uint32_t n, const orc::Aabb3<T>* shapes, const uint32_t* idx, uint32_t k) {
    orc::DynBvh<T> b = load(nodes, n_nodes, node_index, n);
    for (uint32_t i = 0; i < k; ++i) orc::remove_shape(b, shapes, idx[i]);
    std::vector<char> rm(n, 0);
    for (uint32_t i = 0; i < k; ++i) rm[idx[i]] = 1;
    const uint32_t m = n - k;
    std::vector<uint32_t> relabel(n, orc::U32_MAX), holes;
    for (uint32_t s = 0; s < m; ++s) { if (rm[s]) holes.push_back(s); else relabel[s] = s; }
    size_t h = 0;
    for (uint32_t s = m; s < n; ++s) if (!rm[s]) relabel[s] = holes[h++];
    return canonical(b, relabel, nodes, node_index);
}

}  // namespace

extern "C" {
uint32_t dyn_add_f32(orc::Node<float>* nodes, uint32_t nn, uint32_t* ni, uint32_t n, const orc::Aabb3<float>* shapes, uint32_t k) { return add(nodes, nn, ni, n, shapes, k); }
uint32_t dyn_add_f64(orc::Node<double>* nodes, uint32_t nn, uint32_t* ni, uint32_t n, const orc::Aabb3<double>* shapes, uint32_t k) { return add(nodes, nn, ni, n, shapes, k); }
uint32_t dyn_remove_f32(orc::Node<float>* nodes, uint32_t nn, uint32_t* ni, uint32_t n, const orc::Aabb3<float>* shapes, const uint32_t* idx, uint32_t k) {
    return remove(nodes, nn, ni, n, shapes, idx, k);
}
uint32_t dyn_remove_f64(orc::Node<double>* nodes, uint32_t nn, uint32_t* ni, uint32_t n, const orc::Aabb3<double>* shapes, const uint32_t* idx, uint32_t k) {
    return remove(nodes, nn, ni, n, shapes, idx, k);
}
}
