/*
 * oracle/gc_oracle.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of the multi-label graph cut the reference calls at
 *     imsegm/graph_cuts.py:735-744   gco.cut_general_graph(edges, edge_weights, unary_cost, pairwise_cost,
 *                                                          algorithm='expansion', n_iter=-1)
 *     imsegm/region_growing.py:148,1698,1715   (same call with n_iter=999)
 * The arithmetic lives in a third-party dependency that is NOT vendored in the reference and not installed
 * here: gco-wrapper >= 3.0.8 (requirements.txt:14; Borda/pyGCO wrapping GCO v3.0, Veksler & Delong).
 * Restated from its published behaviour:
 *   - (Python side, restated in oracle/energies.py) float energies are integerised: unary and edge weights are
 *     divided by down_weight_factor = max(|unary|.max(), |w|.max() * pairwise.max()) + 1e-10, then
 *     unary*1e5, w*1e3, pairwise*1e2, truncated to C int.
 *   - energy  E(l) = sum_i D[i][l_i] + sum_{(i,j)} w_ij * V[l_i][l_j],  64-bit totals, 32-bit terms.
 *   - labeling starts at all zeros; alpha-expansion in label order 0..K-1.
 *   - one expansion move on alpha = exact minimum of the binary (Kolmogorov-Zabih) move energy by max-flow;
 *     a site KEEPS its label iff it ends in the SINK segment, i.e. iff it can still reach the sink in the
 *     residual graph (BK's what_segment() with default SOURCE) -- the minimiser with the most sites switched
 *     to alpha.  That minimiser is unique whatever max-flow algorithm computes it, which is why a different
 *     solver (Dinic here, push-relabel on the GPU) gives identical labels.
 *   - a move is applied iff it strictly lowers the energy.
 *   - n_iter == -1: GCO's "adaptive cycles" (queue of labels that succeeded last cycle); n_iter > 0: plain
 *     cycles over all labels until the energy stops changing.
 * PARITY: pinned by the reference's tiny-graph doctests (graph_cuts.py:698-716, region_growing.py:70-76) only;
 * the adaptive-cycle bookkeeping is restated from memory of GCO v3 and matters only for K >= 3.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu legs may use this file.
 */
#include <cstdint>
#include <cstring>
#include <vector>
#include <algorithm>
#include <queue>

namespace {

struct MaxFlow {
    // arcs stored pairwise: arc a and a^1 are reverses
    int n;
    std::vector<int> head, nxt, to;
    std::vector<int64_t> cap;
    std::vector<int> level, cur;
    explicit MaxFlow(int n_) : n(n_), head(n_, -1) {}
    void add(int u, int v, int64_t c, int64_t rc)
    {
        to.push_back(v); cap.push_back(c); nxt.push_back(head[u]); head[u] = (int)to.size() - 1;
        to.push_back(u); cap.push_back(rc); nxt.push_back(head[v]); head[v] = (int)to.size() - 1;
    }
    bool bfs(int s, int t)
    {
        level.assign(n, -1);
        std::vector<int> q; q.reserve(n);
        q.push_back(s); level[s] = 0;
        for (size_t qi = 0; qi < q.size(); ++qi) {
            int u = q[qi];
            for (int a = head[u]; a >= 0; a = nxt[a])
                if (cap[a] > 0 && level[to[a]] < 0) { level[to[a]] = level[u] + 1; q.push_back(to[a]); }
        }
        return level[t] >= 0;
    }
    int64_t dfs(int s, int t)
    {
        // iterative blocking flow with current-arc pointers
        int64_t total = 0;
        std::vector<int> path; // arcs
        int u = s;
        while (true) {
            if (u == t) {
                int64_t f = INT64_MAX;
                for (int a : path) f = std::min(f, cap[a]);
                for (int a : path) { cap[a] -= f; cap[a ^ 1] += f; }
                total += f;
                // restart from the first saturated arc
                size_t k = 0;
                while (k < path.size() && cap[path[k]] > 0) ++k;
                path.resize(k);
                u = path.empty() ? s : to[path.back()];
                continue;
            }
            int& a = cur[u];
            while (a >= 0 && !(cap[a] > 0 && level[to[a]] == level[u] + 1)) a = nxt[a];
            if (a >= 0) { path.push_back(a); u = to[a]; }
            else {
                if (u == s) break;
                level[u] = -2; // dead end
                int pa = path.back(); path.pop_back();
                u = to[pa ^ 1];
            }
        }
        return total;
    }
    int64_t run(int s, int t)
    {
        int64_t flow = 0;
        while (bfs(s, t)) { cur = head; flow += dfs(s, t); }
        return flow;
    }
    // nodes that can reach t in the residual graph
    void sink_side(int t, std::vector<char>& mark)
    {
        mark.assign(n, 0);
        std::vector<int> q; q.push_back(t); mark[t] = 1;
        for (size_t qi = 0; qi < q.size(); ++qi) {
            int v = q[qi];
            // u -> v has residual iff cap[arc(u->v)] > 0; arc a from v to u has reverse a^1 from u to v
            for (int a = head[v]; a >= 0; a = nxt[a]) {
                int u = to[a];
                if (!mark[u] && cap[a ^ 1] > 0) { mark[u] = 1; q.push_back(u); }
            }
        }
    }
};

struct Problem {
    int N, K, E;
    const int32_t* edges; const int32_t* w; const int32_t* D; const int32_t* V;
    std::vector<int32_t> lab;
    int64_t energy() const
    {
        int64_t e = 0;
        for (int i = 0; i < N; ++i) e += D[(size_t)i * K + lab[i]];
        for (int k = 0; k < E; ++k) {
            int a = edges[2 * k], b = edges[2 * k + 1];
            e += (int64_t)w[k] * V[lab[a] * K + lab[b]];
        }
        return e;
    }
    // returns true iff the expansion on alpha strictly lowered the energy (and was applied)
    bool expand(int alpha, int64_t& cur_energy, int* n_flow_calls)
    {
        std::vector<int> var(N, -1);
        int nv = 0;
        for (int i = 0; i < N; ++i) if (lab[i] != alpha) var[i] = nv++;
        if (nv == 0) return false;
        std::vector<int64_t> U0(nv, 0), U1(nv, 0); // cost of x=0 (take alpha) / x=1 (keep)
        for (int i = 0; i < N; ++i) if (var[i] >= 0) {
            U0[var[i]] = D[(size_t)i * K + alpha];
            U1[var[i]] = D[(size_t)i * K + lab[i]];
        }
        const int S = nv, T = nv + 1;
        MaxFlow g(nv + 2);
        for (int k = 0; k < E; ++k) {
            int a = edges[2 * k], b = edges[2 * k + 1];
            int64_t wk = w[k];
            int va = var[a], vb = var[b];
            if (va < 0 && vb < 0) continue;
            if (va >= 0 && vb >= 0) {
                int64_t A = wk * V[alpha * K + alpha], B = wk * V[alpha * K + lab[b]];
                int64_t C = wk * V[lab[a] * K + alpha], Dd = wk * V[lab[a] * K + lab[b]];
                // E(xa,xb) = A + (C-A) xa + (Dd-C) xb + (B+C-A-Dd) (1-xa) xb
                U0[va] += A; U1[va] += C;       // A + (C-A) xa
                U1[vb] += Dd - C;               // may go negative; fixed by the min-normalisation below
                int64_t P = B + C - A - Dd;
                if (P < 0) return false;        // non-submodular: GCO raises; never happens for metric V
                if (P > 0) g.add(va, vb, P, 0); // cut when a in S (x=0), b in T (x=1)
            } else if (va >= 0) {
                U0[va] += wk * V[alpha * K + alpha];
                U1[va] += wk * V[lab[a] * K + alpha];
            } else {
                U0[vb] += wk * V[alpha * K + alpha];
                U1[vb] += wk * V[alpha * K + lab[b]];
            }
        }
        for (int v = 0; v < nv; ++v) {
            int64_t m = std::min(U0[v], U1[v]);
            int64_t c0 = U0[v] - m, c1 = U1[v] - m;
            if (c1 > 0) g.add(S, v, c1, 0); // paid when v in T (x=1)
            if (c0 > 0) g.add(v, T, c0, 0); // paid when v in S (x=0)
        }
        g.run(S, T);
        if (n_flow_calls) ++*n_flow_calls;
        std::vector<char> keep;
        g.sink_side(T, keep);
        std::vector<int32_t> old = lab;
        for (int i = 0; i < N; ++i) if (var[i] >= 0 && !keep[var[i]]) lab[i] = alpha;
        int64_t e = energy();
        if (e < cur_energy) { cur_energy = e; return true; }
        lab.swap(old);
        return false;
    }
};

} // namespace

extern "C" int oracle_alpha_expansion(int N, int K, int E, const int32_t* edges, const int32_t* w, const int32_t* unary,
                                      const int32_t* smooth, int n_iter, int32_t* labels, int64_t* energy_out, int* n_moves)
{
    Problem p{ N, K, E, edges, w, unary, smooth, std::vector<int32_t>(labels, labels + N) };
    int flows = 0;
    if (E == 0) {
        // GCO solves the no-smoothness case greedily
        for (int i = 0; i < N; ++i) {
            int best = 0;
            for (int l = 1; l < K; ++l) if (unary[(size_t)i * K + l] < unary[(size_t)i * K + best]) best = l;
            p.lab[i] = best;
        }
    } else {
        int64_t cur = p.energy();
        std::vector<int> table(K);
        for (int l = 0; l < K; ++l) table[l] = l;
        if (n_iter == -1) {
            std::vector<int> queue_sizes{ K };
            while (!queue_sizes.empty()) {
                int qsz = queue_sizes.back();
                int start = K - qsz;
                for (int next = start; next < K; ++next)
                    if (!p.expand(table[next], cur, &flows)) { std::swap(table[next], table[start]); ++start; }
                int nsz = K - start;
                if (nsz == qsz) continue;               // everything succeeded: same queue again
                if (nsz > 0) queue_sizes.push_back(nsz); // focus on the labels that succeeded
                else queue_sizes.pop_back();             // nothing succeeded: back to the larger queue, or stop
            }
        } else {
            for (int cycle = 0; cycle < n_iter; ++cycle) {
                int64_t before = cur;
                for (int l = 0; l < K; ++l) p.expand(table[l], cur, &flows);
                if (cur == before) break;
            }
        }
    }
    std::memcpy(labels, p.lab.data(), sizeof(int32_t) * (size_t)N);
    if (energy_out) *energy_out = p.energy();
    if (n_moves) *n_moves = flows;
    return 0;
}
