"""tests/dimdyn.py -- restatement of the reference's sequential Bvh::add_shape / Bvh::remove_shape (src/bvh/optimization.rs:17-389),
generic in the dimension D, with numpy.float32 / numpy.float64 scalars (every operation rounds in T, in the reference's order; surface
areas are pyref._sa, a left-to-right dot).  TEST INFRASTRUCTURE: checked against the C++ oracle at D = 3 (tests/dynoracle.py, in
tests/test_dim_dynamic_cpu.py) and then used as the oracle of the 2-D and 4-D device forms.

    Dyn.add       add_shape: the descent (send_left / send_right / merge test, the slots it passes grow by the new box), the merge
                  branch (a node over {new leaf, the old node}) and the leaf split, then fix_aabbs_ascending from the split's parent
    Dyn.remove    remove_shape(i, swap_shape = false) for every index in the caller's order (connect_nodes, fix_aabbs_ascending,
                  swap_and_remove_index), then the swap rule's renumbering of a batched removal (dynoracle.swap_moves)
    Dyn.canonical the result re-emitted in Bvh::build's preorder layout (child_l = i + 1, child_r = i + 2 n_l, `shape` of an inner
                  node = shapes below it), which is the layout the device keeps: with it the trees compare node for node

The reference appends and swap-removes nodes, so its own node order is not the preorder one; canonical() is the same re-emission as
tests/cpp/dyn_oracle.cpp."""
import numpy as np

from tests.dynoracle import swap_moves
from tests.pyref import _join, _sa

U32_MAX = 0xFFFFFFFF


class Dyn:
    """The reference's node vector: per node parent, child_l, child_r, shape and the two child slots ([min], [max]) in T."""

    def __init__(self, nodes, node_index, shapes):
        self.F = nodes.dtype["l_aabb"]["min"].base.type if len(nodes) else shapes.dtype["min"].base.type
        self.dtype = nodes.dtype
        self.P = [int(x) for x in nodes["parent"]]
        self.L = [int(x) for x in nodes["child_l"]]
        self.R = [int(x) for x in nodes["child_r"]]
        self.S = [int(x) for x in nodes["shape"]]
        self.lb = [(list(a), list(b)) for a, b in zip(nodes["l_aabb"]["min"], nodes["l_aabb"]["max"])]
        self.rb = [(list(a), list(b)) for a, b in zip(nodes["r_aabb"]["min"], nodes["r_aabb"]["max"])]
        self.ni = [int(x) for x in node_index]
        self.shapes = [(list(a), list(b)) for a, b in zip(shapes["min"], shapes["max"])]
        self.D = shapes["min"].shape[1]
        self.merges = 0                                          # add_shape calls that took the merge branch

    # ---- node vector helpers ----
    def _empty(self):
        inf = self.F(np.inf)
        return ([inf] * self.D, [-inf] * self.D)

    def _push(self, p, l, r, s, lb, rb):
        self.P.append(p); self.L.append(l); self.R.append(r); self.S.append(s); self.lb.append(lb); self.rb.append(rb)
        return len(self.P) - 1

    def _leaf(self, parent, shape):
        return self._push(parent, U32_MAX, U32_MAX, shape, self._empty(), self._empty())

    def _copy(self, dst, src):
        self.P[dst], self.L[dst], self.R[dst], self.S[dst] = self.P[src], self.L[src], self.R[src], self.S[src]
        self.lb[dst], self.rb[dst] = self.lb[src], self.rb[src]

    def _box(self, i):                                           # get_node_aabb, bvh_node.rs:616-625
        return self.shapes[self.S[i]] if self.L[i] == U32_MAX else _join(self.lb[i], self.rb[i])

    @staticmethod
    def _differs(x, y):
        return any(a != b for a, b in zip(x[0], y[0])) or any(a != b for a, b in zip(x[1], y[1]))

    def _fix(self, i):                                           # fix_aabbs_ascending, optimization.rs:317-351
        while i != 0:
            p = self.P[i]
            if self.L[p] == U32_MAX:
                break
            lb, rb = self._box(self.L[p]), self._box(self.R[p])
            stop = True
            if self._differs(lb, self.lb[p]):
                stop, self.lb[p] = False, lb
            if self._differs(rb, self.rb[p]):
                stop, self.rb[p] = False, rb
            i = 0 if stop else p

    def _connect(self, child, parent, left):                     # connect_nodes, optimization.rs:34-65
        box = self._box(child)
        if left:
            self.L[parent], self.lb[parent] = child, box
        else:
            self.R[parent], self.rb[parent] = child, box
        self.P[child] = parent

    def _swap_remove(self, i):                                   # swap_and_remove_index, optimization.rs:353-389
        end = len(self.P) - 1
        if i != end:
            self._copy(i, end)
            p = self.P[i]
            if self.L[p] == end:
                self.L[p] = i
            else:
                assert self.R[p] == end
                self.R[p] = i
            if self.L[i] == U32_MAX:
                self.ni[self.S[i]] = i
            else:
                self.P[self.L[i]] = i
                self.P[self.R[i]] = i
        for a in (self.P, self.L, self.R, self.S, self.lb, self.rb):
            a.pop()

    # ---- add_shape, optimization.rs:70-206 ----
    def add(self, mn, mx):
        F = self.F
        box = ([F(v) for v in mn], [F(v) for v in mx])
        s = len(self.shapes)
        self.shapes.append(box)
        self.ni.append(0)
        if not self.P:
            self.ni[s] = self._leaf(0, s)
            return
        with np.errstate(all="ignore"):
            shape_sa = _sa(F, *box)
            i = 0
            while True:
                if self.L[i] != U32_MAX:
                    lb, rb = self.lb[i], self.rb[i]
                    le, re = _join(lb, box), _join(rb, box)
                    send_left = _sa(F, *rb) + _sa(F, *le)
                    send_right = _sa(F, *lb) + _sa(F, *re)
                    merged_box = _join(rb, lb)
                    merged = _sa(F, *merged_box) + shape_sa
                    min_send = send_left if send_left < send_right else send_right
                    if merged < min_send * F(3) / F(10):          # a node over {new leaf, this node} takes this node's place
                        l_index = self._leaf(i, s)
                        self.ni[s] = l_index
                        r_index = self._push(i, self.L[i], self.R[i], self.S[i], lb, rb)
                        self.P[self.L[i]] = r_index
                        self.P[self.R[i]] = r_index
                        self.L[i], self.lb[i], self.R[i], self.rb[i] = l_index, box, r_index, merged_box
                        self.merges += 1
                        return
                    if send_left < send_right:
                        self.lb[i] = le
                        i = self.L[i]
                    else:
                        self.rb[i] = re
                        i = self.R[i]
                else:                                            # split the leaf into a node over {new, old}
                    old = self.S[i]
                    l_index = self._leaf(i, s)
                    self.ni[s] = l_index
                    r_index = self._leaf(i, old)
                    self.ni[old] = r_index
                    self.L[i], self.R[i], self.S[i], self.lb[i], self.rb[i] = l_index, r_index, 2, box, self.shapes[old]
                    self._fix(self.P[i])
                    return

    def add_many(self, shapes):
        for mn, mx in zip(shapes["min"], shapes["max"]):
            self.add(mn, mx)

    # ---- remove_shape(i, swap_shape = false), optimization.rs:208-288, then the batched renumbering ----
    def _remove_one(self, s):
        dead = self.ni[s]
        if len(self.P) == 1:
            assert dead == 0 and self.L[0] == U32_MAX
            for a in (self.P, self.L, self.R, self.S, self.lb, self.rb):
                a.clear()
            return
        parent = self.P[dead]
        gp = self.P[parent]
        sibling = self.R[parent] if self.L[parent] == dead else self.L[parent]
        if parent == gp:                                         # a child of the root goes: the sibling becomes the root
            assert parent == 0
            if self.L[sibling] != U32_MAX:
                sl, sr = self.L[sibling], self.R[sibling]
                self._connect(sl, 0, True)
                self._connect(sr, 0, False)
            else:
                self._copy(0, sibling)
                self.P[0] = 0
                self.ni[self.S[0]] = 0
            self._swap_remove(max(sibling, dead))
            self._swap_remove(min(sibling, dead))
        else:
            self._connect(sibling, gp, self.L[gp] == parent)
            self._fix(gp)
            self._swap_remove(max(dead, parent))
            self._swap_remove(min(parent, dead))

    def remove(self, indices):
        """Removes the shapes in the caller's order and renumbers the survivors by the swap rule; returns the (new, old) moves."""
        indices = [int(i) for i in indices]
        n = len(self.shapes)
        for s in indices:
            self._remove_one(s)
        mv = swap_moves(n, indices)
        relabel = list(range(n))
        for new, old in mv:
            relabel[int(old)] = int(new)
        for i in range(len(self.P)):
            if self.L[i] == U32_MAX:
                self.S[i] = relabel[self.S[i]]
        ni = list(self.ni)
        for new, old in mv:
            self.shapes[int(new)] = self.shapes[int(old)]
            ni[int(new)] = self.ni[int(old)]
        m = n - len(indices)
        self.shapes, self.ni = self.shapes[:m], ni[:m]
        return mv

    # ---- Bvh::build's preorder layout ----
    def canonical(self):
        """(nodes, node_index) in the preorder layout, node dtype of the input."""
        nn = len(self.P)
        out = np.zeros(nn, dtype=self.dtype)
        ni = np.zeros(len(self.shapes), dtype=np.uint32)
        if nn == 0:
            return out, ni
        cnt = [1] * nn
        order, st = [], [0]
        while st:                                                # preorder of the reference's tree, then counts in reverse
            i = st.pop()
            order.append(i)
            if self.L[i] != U32_MAX:
                st.append(self.R[i]); st.append(self.L[i])
        for i in reversed(order):
            if self.L[i] != U32_MAX:
                cnt[i] = cnt[self.L[i]] + cnt[self.R[i]]
        newidx = {}
        for j, i in enumerate(order):
            newidx[i] = j
        P, L, R, S = (np.zeros(nn, dtype=np.uint32) for _ in range(4))
        lmn, lmx, rmn, rmx = (np.zeros((nn, self.D), dtype=self.F) for _ in range(4))
        for j, i in enumerate(order):
            P[j] = newidx[self.P[i]] if j else 0
            if self.L[i] == U32_MAX:
                L[j] = R[j] = U32_MAX
                S[j] = self.S[i]
                ni[self.S[i]] = j
            else:
                L[j], R[j], S[j] = j + 1, j + 2 * cnt[self.L[i]], cnt[i]
            lmn[j], lmx[j] = self.lb[i]
            rmn[j], rmx[j] = self.rb[i]
        out["parent"], out["child_l"], out["child_r"], out["shape"] = P, L, R, S
        out["l_aabb"]["min"], out["l_aabb"]["max"], out["r_aabb"]["min"], out["r_aabb"]["max"] = lmn, lmx, rmn, rmx
        return out, ni

    def shape_array(self, dtype):
        a = np.zeros(len(self.shapes), dtype=dtype)
        if len(self.shapes):
            a["min"] = np.array([b[0] for b in self.shapes], dtype=self.F)
            a["max"] = np.array([b[1] for b in self.shapes], dtype=self.F)
        return a
