// tools/sim_top.cpp -- DEV TOOL (not product): CPU model of walk_top_kernel's shared-memory wavefronts.
//   g++ -O3 -march=x86-64-v3 -ffp-contract=off -std=c++17 -I oracle tools/sim_top.cpp -o /tmp/sim_top && /tmp/sim_top
//   /tmp/sim_top 60000 5000 4 2000     (rays, tier-1 budget B1, cluster size S, tier-2 entries per CTA B2: the two-tier model)
// Model: warps of 32 lanes with the kernel's refill rule (>= 8 idle lanes -> new tickets); per warp step, an LDS.128 costs, per
// quarter-warp, the largest number of DISTINCT 16-byte chunks that fall into one of the 8 bank groups.  Variants: plain SoA
// (lo[j], hi[j]); the first H entries replicated 8 x (lane & 7 picks the copy: conflict-free).
#include "bvh_oracle.hpp"
#include <algorithm>
#include <cstdio>
using namespace orc;
struct Rec { float mn[3], mx[3]; uint32_t w3, w7; };
int main(int argc, char** argv) {
    const uint32_t n_cubes = 10000, R = argc > 1 ? atoi(argv[1]) : 200000;
    const uint32_t budget = argc > 2 ? atoi(argv[2]) : 7000;
    std::vector<float> tris; const Aabb3<float> bounds = default_bounds<float>();
    create_n_cubes(n_cubes, bounds, tris);
    const uint32_t n = n_cubes * 12, nn = 2 * n - 1;
    std::vector<Aabb3<float>> shapes(n);
    for (uint32_t i = 0; i < n; ++i) shapes[i] = triangle_aabb(&tris[9 * i], &tris[9 * i + 3], &tris[9 * i + 6]);
    std::vector<Node<float>> nodes(nn); std::vector<uint32_t> nidx(n);
    build(shapes.data(), n, nodes.data(), nidx.data());
    std::vector<uint32_t> cnt(nn);
    for (uint32_t i = nn; i-- > 0;) cnt[i] = nodes[i].is_leaf() ? 1 : cnt[nodes[i].child_l] + cnt[nodes[i].child_r];
    auto box = [&](uint32_t i, Rec& r) { const Node<float>& p = nodes[nodes[i].parent]; const Aabb3<float>& b = p.child_l == i ? p.l_aabb : p.r_aabb;
                                         for (int k = 0; k < 3; ++k) { r.mn[k] = b.min[k]; r.mx[k] = b.max[k]; } };
    std::vector<Rec> rec(nn - 1);
    for (uint32_t i = 1; i < nn; ++i) { box(i, rec[i - 1]); rec[i - 1].w3 = (i - 1) + 2 * cnt[i] - 1; rec[i - 1].w7 = nodes[i].is_leaf() ? nodes[i].shape : 0xFFFFFFFFu; }
    // choose C: largest top that fits (any C, like the device's 8 bins / octave but exact)
    uint32_t C = 2;
    for (C = 2;; ++C) { uint32_t t = 0; for (uint32_t i = 1; i < nn; ++i) t += cnt[nodes[i].parent] >= C; if (t <= budget) break; }
    std::vector<uint32_t> pre(nn + 1, 0);
    for (uint32_t i = 1; i < nn; ++i) pre[i + 1] = pre[i] + (cnt[nodes[i].parent] >= C);
    for (uint32_t i = nn; i >= 1; --i) pre[i] = pre[i];   // pre[i] = #flagged before i  (pre[i+1] computed above is "through i")
    std::vector<uint32_t> ex(nn + 1, 0);
    { uint32_t run = 0; for (uint32_t i = 0; i <= nn; ++i) { ex[i] = run; if (i >= 1 && i < nn && cnt[nodes[i].parent] >= C) ++run; } }
    const uint32_t nT = ex[nn];
    std::vector<Rec> top(nT);
    for (uint32_t i = 1; i < nn; ++i) if (cnt[nodes[i].parent] >= C) {
        Rec r; box(i, r); const uint32_t k = ex[i]; const bool leaf = nodes[i].is_leaf();
        if (!leaf && cnt[i] >= C) { r.w3 = ex[std::min(i + 2 * cnt[i] - 1, nn)]; r.w7 = 0xFFFFFFFFu; }
        else if (leaf) { r.w3 = k + 1; r.w7 = nodes[i].shape; }
        else { r.w3 = rec[i - 1].w3; r.w7 = 0x80000000u | i; }
        top[k] = r;
    }
    printf("C = %u, %u top entries\n", C, nT);
    std::vector<Ray3<float>> rays(R); uint64_t seed = 0;
    for (uint32_t i = 0; i < R; ++i) rays[i] = create_ray(seed, bounds);
    auto hit = [&](const Ray3<float>& ray, const Rec& r) { Aabb3<float> b; for (int k = 0; k < 3; ++k) { b.min[k] = r.mn[k]; b.max[k] = r.mx[k]; } return ray_intersects_aabb(ray, b); };
    if (argc > 4) {
        // Two tiers (walk_top_kernel under a cluster of S CTAs): tier 1 = T(C1) for budget B1 (argument 2), replicated; tier 2 =
        // T(C2) \ T(C1) for C2 fitting |T(C1)| + S * B2, entry t on CTA rank t % S.  Plain preorder walk (the kernel's visit order)
        // under the kernel's refill rule, one visit per lane per step, warp w on CTA rank w % S.  Reports visits per ray by tier,
        // remote (other-rank) tier-2 reads, and the share of warp steps with a lane below the tiers / a lane reading a peer, for
        // one visit per step and for the kernel's four (a group of 4 steps with one such lane in any of them).
        const uint32_t S = atoi(argv[3]), B2 = atoi(argv[4]);
        auto size_for = [&](uint32_t c) { uint32_t t = 0; for (uint32_t i = 1; i < nn; ++i) t += cnt[nodes[i].parent] >= c; return t; };
        const uint32_t n1 = nT, C1 = C;
        uint32_t C2 = C1; while (C2 > 2 && size_for(C2 - 1) <= n1 + S * B2) --C2;
        std::vector<uint32_t> tier(nn, 2), t2(nn, 0);                  // 0 tier 1, 1 tier 2, 2 below
        uint32_t n2 = 0;
        for (uint32_t i = 1; i < nn; ++i) { const uint32_t c = cnt[nodes[i].parent]; tier[i] = c >= C1 ? 0 : c >= C2 ? 1 : 2; if (tier[i] == 1) t2[i] = n2++; }
        const int W = 512;
        std::vector<uint32_t> ray(W * 32, U32_MAX), at(W * 32, 0);
        uint32_t ticket = 0; uint64_t steps = 0, v[3] = {0, 0, 0}, remote = 0, st_below = 0, st_remote = 0, grp = 0, grp_below = 0, grp_remote = 0;
        for (bool any = true; any;) {
            any = false;
            for (int w = 0; w < W; ++w) {
                uint32_t* wr = &ray[32 * w]; uint32_t* wa = &at[32 * w];
                int idle = 0; for (int l = 0; l < 32; ++l) idle += wr[l] == U32_MAX;
                if (idle >= 8 && ticket < R) for (int l = 0; l < 32 && ticket < R; ++l) if (wr[l] == U32_MAX) { wr[l] = ticket++; wa[l] = 0; }
                bool gb = false, gr = false, act = false;
                for (int u = 0; u < 4; ++u) {
                    bool sb = false, sr = false, sa = false;
                    for (int l = 0; l < 32; ++l) if (wr[l] != U32_MAX) {
                        const uint32_t i = wa[l] + 1;                     // record wa = node wa + 1
                        sa = true; ++v[tier[i]];
                        if (tier[i] == 2) sb = true;
                        if (tier[i] == 1 && t2[i] % S != (uint32_t)w % S) { sr = true; ++remote; }
                        wa[l] = hit(rays[wr[l]], rec[wa[l]]) ? wa[l] + 1 : rec[wa[l]].w3;
                        if (wa[l] >= nn - 1) wr[l] = U32_MAX;
                    }
                    if (!sa) break;
                    ++steps; st_below += sb; st_remote += sr; gb |= sb; gr |= sr; act = true;
                }
                if (act) { any = true; ++grp; grp_below += gb; grp_remote += gr; }
            }
        }
        printf("S %u  B1 %u  B2 %u: C1 %u (%u entries)  C2 %u (tier 2: %u entries, %u per CTA)\n", S, atoi(argv[2]), B2, C1, n1, C2, n2, (n2 + S - 1) / S);
        printf("  visits/ray: tier 1 %.2f  tier 2 %.2f (remote %.2f)  below %.2f  total %.3f\n", (double)v[0] / R, (double)v[1] / R, (double)remote / R,
               (double)v[2] / R, (double)(v[0] + v[1] + v[2]) / R);
        printf("  P(step has a lane below) %.3f  P(step has a remote lane) %.3f  | per 4-visit step: below %.3f  remote %.3f\n",
               (double)st_below / steps, (double)st_remote / steps, (double)grp_below / grp, (double)grp_remote / grp);
        return 0;
    }
    for (uint32_t H : {0u, 64u, 128u, 256u, 512u, 1024u}) {
        const int W = 512;
        struct Warp { uint32_t ray[32], j[32], g[32], gend[32]; };
        std::vector<Warp> warps(W);
        for (auto& w : warps) for (int l = 0; l < 32; ++l) w.ray[l] = U32_MAX;
        uint32_t ticket = 0; uint64_t steps = 0, lane_visits = 0, top_visits = 0, wf = 0, ideal = 0, hot = 0, lds = 0; bool any = true;
        while (any) {
            any = false;
            for (auto& w : warps) {
                int idle = 0; for (int l = 0; l < 32; ++l) idle += w.ray[l] == U32_MAX;
                if ((idle >= 8 || idle == 32) && ticket < R) for (int l = 0; l < 32 && ticket < R; ++l) if (w.ray[l] == U32_MAX) { w.ray[l] = ticket++; w.j[l] = 0; w.g[l] = 0; w.gend[l] = 0; }
                int na = 0; for (int l = 0; l < 32; ++l) na += w.ray[l] != U32_MAX;
                if (!na) continue;
                any = true; ++steps; lane_visits += na;
                for (int half = 0; half < 2; ++half) {          // lo, hi
                    bool anytop = false; uint32_t bytes = 0;
                    for (int q = 0; q < 4; ++q) {
                        uint32_t addr[8]; int m = 0;
                        for (int l = 8 * q; l < 8 * q + 8; ++l) if (w.ray[l] != U32_MAX && !(w.g[l] < w.gend[l])) {
                            const uint32_t j = w.j[l];
                            // chunk index in 16-byte units
                            uint32_t chunk = j < H ? (half * 8 * H + j * 8 + (l & 7)) : (16 * H + half * (nT - H) + (j - H));
                            addr[m++] = chunk; anytop = true;
                        }
                        if (!m) continue;
                        std::sort(addr, addr + m); m = std::unique(addr, addr + m) - addr;
                        int load[8] = {}; for (int k = 0; k < m; ++k) load[addr[k] & 7]++;
                        wf += *std::max_element(load, load + 8); bytes += 16 * m;
                    }
                    if (anytop) { ++lds; ideal += (bytes + 127) / 128; }
                }
                for (int l = 0; l < 32; ++l) if (w.ray[l] != U32_MAX) {
                    const Ray3<float>& ray = rays[w.ray[l]];
                    if (w.g[l] < w.gend[l]) { const Rec& r = rec[w.g[l]]; w.g[l] = hit(ray, r) ? w.g[l] + 1 : r.w3; }
                    else {
                        const Rec& r = top[w.j[l]]; ++top_visits; hot += w.j[l] < H;
                        const bool h = hit(ray, r), fringe = r.w7 != 0xFFFFFFFFu && (r.w7 & 0x80000000u);
                        if (h && fringe) { w.g[l] = r.w7 & 0x7FFFFFFFu; w.gend[l] = r.w3; }
                        w.j[l] = (h || fringe || r.w7 < 0x80000000u) ? w.j[l] + 1 : r.w3;
                    }
                    if (!(w.g[l] < w.gend[l]) && w.j[l] >= nT) w.ray[l] = U32_MAX;
                }
            }
        }
        printf("H %4u (top capacity used %5u chunks-pairs): visits/ray %.1f top %.1f (hot %.1f)  warp-steps/ray %.2f  LDS wavefronts/ray %.1f (ideal %.1f)  per LDS %.2f\n",
               H, nT + 7 * H, (double)lane_visits / R, (double)top_visits / R, (double)hot / R, (double)steps / R, (double)wf / R, (double)ideal / R, (double)wf / lds);
    }
    return 0;
}
