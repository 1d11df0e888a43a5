// alpha_expansion.cu -- multi-label GraphCut by alpha-expansion on the superpixel adjacency graph.
//
// Replaces gco.cut_general_graph(edges, edge_weights, unary, pairwise, algorithm='expansion', n_iter)
// as called from imsegm/graph_cuts.py:735-744 (and region_growing.py:148,1698,1715), on the integer energies
// pyGCO builds (see oracle/gc_oracle.cpp for the restated contract).
//
// Launch 1 (k_gc_build_csr): arc list of the undirected graph in CSR order (src, dst, reverse slot, edge id).
// Launch 2 (k_alpha_expansion): ONE THREAD-BLOCK CLUSTER of 8 CTAs (8192 threads) owns the graph for the whole
// optimisation -- GCO's cycle bookkeeping, every expansion move and every max-flow inside a single launch.
// Nodes are split into 8 contiguous index ranges (superpixel labels are raster ordered, so a range is a band of
// the image and almost every neighbour is local); a CTA keeps its nodes' excess / sink capacity / heights and the
// residuals of the arcs LEAVING its nodes in its own shared memory, and reaches the few foreign neighbours through
// distributed shared memory (cluster.map_shared_rank).  Phases are separated by cluster barriers.
//
// A move on alpha is the exact minimum of a binary submodular energy (Kolmogorov-Zabih construction):
//   x_i = 0 take alpha / x_i = 1 keep;   source->i capacity = cost(x_i=1), i->sink = cost(x_i=0),
//   i->j capacity P_ij = E01 + E10 - E00 - E11 >= 0.
// Max-flow is phase-1 push-relabel (preflow, min cut only), every pass arc-parallel:
//   * global relabel = level-synchronous backward BFS from the sink over residual arcs (exact distance labels;
//     nodes that cannot reach the sink drop out for good),
//   * sweep = node pass (push into the sink arc) | arc pass (pushes h -> h-1 against frozen heights, the amount is
//     claimed from excess[u] with atomics) | arc pass (lowest residual neighbour per stuck node) | node pass
//     (relabel into the second height buffer),
//   * terminates when no node with excess can reach the sink.
// The site keeps its label iff it can reach the sink in the final residual graph -- BK's SINK segment, the
// unique minimiser with the most sites switched -- so labels equal the oracle's whatever the flow algorithm.
// An expansion on a label that already failed on the SAME labeling is skipped (same input, same answer).
//
// When 24 N/8 + 16 max_arcs_per_CTA bytes exceed the dynamic shared memory the same code runs with the state in
// the global workspace (L2 resident) -- the per-rank base pointers then simply point into global arrays.
// This stage is latency/SMEM bound, not HBM bound: report time, not a roofline fraction (SURVEY.md section 8d).
#include "common.cuh"
#include "block_scan.cuh"
#include <cooperative_groups.h>

namespace cg = cooperative_groups;

namespace {

constexpr int NT = 1024;
constexpr int CS = 8;            // CTAs per cluster (portable maximum)
constexpr int HINF = 0x3fffffff;
constexpr int KMAX_S = 16;       // smooth-cost table cached in smem up to K = 16
constexpr int LBITS = 26;        // packed reference = rank << 26 | local index
constexpr int LMASK = (1 << LBITS) - 1;

struct GcArgs {
    int N, K, E_cap;
    const int* n_edges_dev; const int* n_nodes_dev;
    const int* edges; const int* w; const int* D; const int* V;
    int n_iter;
    int* labels;
    long long* energy_out;
    int* stats;
    // CSR arcs (built by k_gc_build_csr)
    int* off; int* fill; int* a_src; int* a_dst; int* a_rev; int* a_eid;
    long long* u0; long long* u1;
    long long* red;   // [8] cluster-wide reduction scratch
    int* newlab;
    // state in global memory (used when it does not fit in the cluster's shared memory)
    long long* g_excess; // [N]  excess
    int* g_node;      // [4][N]  tcap | h0 | h1 | hmin
    int* g_arc;       // [4][A]  res | dstp | revp | srcl
    int dyn_bytes;
};

// ---------------------------------------------------------------- CSR build (single CTA, separate launch) ---------------------------

__global__ void __launch_bounds__(NT) k_gc_build_csr(GcArgs a)
{
    const int N = a.n_nodes_dev ? min(*a.n_nodes_dev, a.N) : a.N;
    // an overflowed edge table (count > capacity) holds unspecified rows: cut nothing, the host sees the count and redoes the image
    const int E = a.n_edges_dev ? (*a.n_edges_dev > a.E_cap ? 0 : *a.n_edges_dev) : a.E_cap;
    for (int v = threadIdx.x; v < N; v += NT) a.fill[v] = 0;
    __syncthreads();
    for (int e = threadIdx.x; e < E; e += NT) { atomicAdd(&a.fill[a.edges[2 * e]], 1); atomicAdd(&a.fill[a.edges[2 * e + 1]], 1); }
    __syncthreads();
    // fill was written by the atomics above: read it past L1.  The scan's closing barrier orders the fill reset before the scatter.
    const int A = cta_scan_chunks<NT, int>(N, [&](int i) { return __ldcg(&a.fill[i]); },
                                           [&](int i, int off) { a.off[i] = off; a.fill[i] = 0; });
    if (threadIdx.x == 0) a.off[N] = A;
    for (int e = threadIdx.x; e < E; e += NT) {
        int va = a.edges[2 * e], vb = a.edges[2 * e + 1];
        int pa = a.off[va] + atomicAdd(&a.fill[va], 1);
        int pb = a.off[vb] + atomicAdd(&a.fill[vb], 1);
        a.a_src[pa] = va; a.a_dst[pa] = vb; a.a_rev[pa] = pb; a.a_eid[pa] = 2 * e;      // slot of a -> b (carries P_e)
        a.a_src[pb] = vb; a.a_dst[pb] = va; a.a_rev[pb] = pa; a.a_eid[pb] = 2 * e + 1;  // slot of b -> a (capacity 0)
    }
}

// ---------------------------------------------------------------- solver ----------------------------------------------------------

// per-rank base pointers of the distributed state (DSMEM addresses, or slices of the global arrays)
struct Peers {
    long long* excess[CS]; int* tcap[CS]; int* h[2][CS]; int* res[CS];
};

struct Ctx {
    int N, K, E, A;
    int rank, npc, n_lo, n_cnt, a_lo, a_cnt; // this CTA's node range [n_lo, n_lo+n_cnt) and arc range [a_lo, a_lo+a_cnt)
    const int* edges; const int* w; const int* D; const int* V;
    // local slices
    long long* excess; int* tcap; int* h[2]; int* hmin; int* res; int* dstp; int* revp; int* srcl;
    Peers* peers;
    int* s_V; long long* s_red; int* flags0; // flags0 = rank 0's flag words (DSMEM)
    long long* red;
};

__device__ __forceinline__ int smooth(const Ctx& c, int la, int lb) { return c.K <= KMAX_S ? c.s_V[la * c.K + lb] : c.V[la * c.K + lb]; }

// 64-bit atomic add on a node's excess (local, DSMEM or global); subtraction adds the negated amount.  Returns the old value.
__device__ __forceinline__ long long add_excess(long long* p, long long v)
{
    return (long long)atomicAdd((unsigned long long*)p, (unsigned long long)v);
}

__device__ long long block_sum_ll(long long v, long long* s_red)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    __syncthreads();
    long long t = 0;
    for (int i = 0; i < NT / 32; ++i) t += s_red[i];
    return t;
}

// cluster-wide sum through global scratch words (used a handful of times per max-flow, not per pass).  `sturn` rotates
// over three words so that the reset of a word never races with its readers or with the next round's writers.
__device__ long long cluster_sum(cg::cluster_group& cl, const Ctx& c, long long v, int& sturn)
{
    const long long b = block_sum_ll(v, c.s_red);
    const int w = sturn % 3;
    if (threadIdx.x == 0) {
        if (b != 0) atomicAdd((unsigned long long*)&c.red[w], (unsigned long long)b);
        if (c.rank == 0) c.red[(sturn + 1) % 3] = 0; // last read two barriers ago
    }
    cl.sync();
    ++sturn;
    return __ldcg(&c.red[w]);
}

// cluster-wide OR of a per-thread predicate: one DSMEM atomic per CTA, one cluster barrier.  `turn` rotates over three
// flag words so that resetting never races with readers.
__device__ bool cluster_or(cg::cluster_group& cl, const Ctx& c, int pred, int& turn)
{
    const int any = __syncthreads_or(pred);
    const int w = turn % 3;
    if (threadIdx.x == 0) {
        if (any) atomicOr(&c.flags0[w], 1);
        if (c.rank == 0) c.flags0[(turn + 1) % 3] = 0; // last read two barriers ago
    }
    cl.sync();
    const int r = *(volatile int*)&c.flags0[w];
    ++turn;
    return r != 0;
}

__device__ long long energy_of(cg::cluster_group& cl, const Ctx& c, const int* lab, int& sturn)
{
    long long e = 0;
    const int tid = c.rank * NT + threadIdx.x;
    for (int i = tid; i < c.N; i += CS * NT) e += c.D[(size_t)i * c.K + lab[i]];
    for (int k = tid; k < c.E; k += CS * NT) e += (long long)c.w[k] * smooth(c, lab[c.edges[2 * k]], lab[c.edges[2 * k + 1]]);
    return cluster_sum(cl, c, e, sturn);
}

#define HGT(buf, p) (c.peers->h[buf][(p) >> LBITS][(p)&LMASK])

// backward BFS from the sink into height buffer `cur`: 1 + distance to a node with sink capacity; unreachable = HINF.
// returns (cluster-uniform) whether any node with excess can reach the sink
__device__ bool global_relabel(cg::cluster_group& cl, const Ctx& c, int cur, int& turn, int* stats)
{
    int* h = c.h[cur];
    for (int v = threadIdx.x; v < c.n_cnt; v += NT) h[v] = (c.tcap[v] > 0) ? 1 : HINF;
    cl.sync();
    for (int level = 1;; ++level) {
        int changed = 0;
        for (int i = threadIdx.x; i < c.a_cnt; i += NT) {
            if (c.res[i] <= 0) continue;
            const int u = c.srcl[i];
            if (h[u] != HINF) continue;
            const int p = c.dstp[i];
            if (*(volatile int*)&HGT(cur, p) == level) { h[u] = level + 1; changed = 1; }
        }
        // a node labelled in this pass gets level+1, never == level: concurrent writers agree, readers never see a torn state
        if (threadIdx.x == 0 && c.rank == 0) ++stats[4];
        if (!cluster_or(cl, c, changed, turn)) break;
    }
    int active = 0;
    for (int v = threadIdx.x; v < c.n_cnt; v += NT) active |= (c.excess[v] > 0 && h[v] != HINF);
    if (threadIdx.x == 0 && c.rank == 0) ++stats[3];
    return cluster_or(cl, c, active, turn);
}

// one synchronous push-relabel sweep: heights are read from buffer `cur` (frozen), relabelled heights go to `cur ^ 1`.
// Every push goes from height h to h-1, so the labelling stays valid (h[u] <= h[v] + 1 on every residual arc).
// Returns (cluster-uniform) whether any node is still active.
__device__ bool sweep(cg::cluster_group& cl, const Ctx& c, int cur, int& turn)
{
    const int* h = c.h[cur];
    int* hn = c.h[cur ^ 1];
    // node pass: the sink arc first; foreign CTAs may already push into excess[u], so it is only touched atomically
    for (int u = threadIdx.x; u < c.n_cnt; u += NT) {
        c.hmin[u] = HINF;
        const long long ex = *(volatile long long*)&c.excess[u];
        if (ex <= 0 || h[u] == HINF) continue;
        const int tc = c.tcap[u];
        if (tc > 0) {
            const int d = ex < tc ? (int)ex : tc;
            c.tcap[u] = tc - d;
            add_excess(&c.excess[u], -(long long)d);
        }
    }
    __syncthreads();
    // arc pass: admissible pushes; the amount is claimed from excess[u] atomically (several arcs share u)
    for (int i = threadIdx.x; i < c.a_cnt; i += NT) {
        const int r = *(volatile int*)&c.res[i];
        if (r <= 0) continue;
        const int u = c.srcl[i];
        const long long ex = *(volatile long long*)&c.excess[u];
        if (ex <= 0) continue;
        const int hu = h[u];
        if (hu == HINF) continue;
        const int p = c.dstp[i];
        if (HGT(cur, p) != hu - 1) continue;
        int d = ex < r ? (int)ex : r;
        const long long old = add_excess(&c.excess[u], -(long long)d);
        if (old < d) { // over-claimed: give back what was not there
            const int have = old > 0 ? (int)old : 0;
            add_excess(&c.excess[u], d - have);
            d = have;
        }
        if (d > 0) {
            atomicSub(&c.res[i], d);
            const int q = c.revp[i];
            atomicAdd(&c.peers->res[q >> LBITS][q & LMASK], d);
            add_excess(&c.peers->excess[p >> LBITS][p & LMASK], d);
        }
    }
    cl.sync();
    // arc pass: lowest residual neighbour of every node that still holds excess and has no sink arc left
    for (int i = threadIdx.x; i < c.a_cnt; i += NT) {
        if (c.res[i] <= 0) continue;
        const int u = c.srcl[i];
        if (c.excess[u] <= 0 || c.tcap[u] > 0 || h[u] == HINF) continue;
        const int p = c.dstp[i];
        atomicMin(&c.hmin[u], HGT(cur, p));
    }
    __syncthreads();
    // node pass: relabel into the other buffer (foreign CTAs may still be reading `cur`)
    int active = 0;
    for (int u = threadIdx.x; u < c.n_cnt; u += NT) {
        const int hu = h[u];
        int nh = hu;
        if (c.excess[u] > 0 && hu != HINF) {
            active = 1;
            if (c.tcap[u] <= 0) {
                const int hm = c.hmin[u];
                if (hm == HINF) nh = HINF;       // no residual way out: source side for good
                else if (hm >= hu) nh = hm + 1;  // relabel
            }
        }
        hn[u] = nh;
    }
    return cluster_or(cl, c, active, turn);
}

__global__ void __cluster_dims__(CS, 1, 1) __launch_bounds__(NT, 1) k_alpha_expansion(GcArgs a)
{
    cg::cluster_group cl = cg::this_cluster();
    extern __shared__ __align__(16) unsigned char dyn[];
    __shared__ int s_V[KMAX_S * KMAX_S];
    __shared__ long long s_red[NT / 32];
    __shared__ int s_table[64], s_queue[64], s_failver[64], s_qn;
    __shared__ int s_stats[8];
    __shared__ int s_flags[4];
    __shared__ int s_alo[CS + 1];
    __shared__ Peers s_peers;

    Ctx c;
    c.rank = (int)cl.block_rank();
    c.N = a.n_nodes_dev ? min(*a.n_nodes_dev, a.N) : a.N;
    c.K = a.K;
    c.E = a.n_edges_dev ? (*a.n_edges_dev > a.E_cap ? 0 : *a.n_edges_dev) : a.E_cap;
    c.A = 2 * c.E;
    c.edges = a.edges; c.w = a.w; c.D = a.D; c.V = a.V;
    c.s_V = s_V; c.s_red = s_red; c.red = a.red; c.peers = &s_peers;
    const int N = c.N, K = c.K, E = c.E;
    c.npc = (N + CS - 1) / CS;
    c.n_lo = min(c.rank * c.npc, N);
    c.n_cnt = min(c.n_lo + c.npc, N) - c.n_lo;
    if (threadIdx.x <= CS) s_alo[threadIdx.x] = E > 0 ? a.off[min(threadIdx.x * c.npc, N)] : 0;
    if (threadIdx.x < 8) s_stats[threadIdx.x] = 0;
    if (threadIdx.x < 4) s_flags[threadIdx.x] = 0;
    if (K <= KMAX_S) for (int i = threadIdx.x; i < K * K; i += NT) s_V[i] = a.V[i];
    __syncthreads();
    c.a_lo = s_alo[c.rank];
    c.a_cnt = s_alo[c.rank + 1] - c.a_lo;
    int apc = 0;
    for (int r = 0; r < CS; ++r) apc = max(apc, s_alo[r + 1] - s_alo[r]);
    const size_t smem_need = sizeof(long long) * (size_t)c.npc + sizeof(int) * (4 * (size_t)c.npc + 4 * (size_t)apc);
    const bool in_smem = smem_need <= (size_t)a.dyn_bytes;
    if (in_smem) {
        // identical layout in every CTA: excess (64-bit) | tcap | h0 | h1 | hmin | res | dstp | revp | srcl
        c.excess = (long long*)dyn;
        int* q = (int*)(c.excess + c.npc);
        c.tcap = q; c.h[0] = q + c.npc; c.h[1] = q + 2 * c.npc; c.hmin = q + 3 * c.npc;
        int* s = q + 4 * c.npc;
        c.res = s; c.dstp = s + apc; c.revp = s + 2 * apc; c.srcl = s + 3 * apc;
        if (threadIdx.x < CS) {
            const int r = threadIdx.x;
            s_peers.excess[r] = cl.map_shared_rank(c.excess, r);
            s_peers.tcap[r] = cl.map_shared_rank(c.tcap, r);
            s_peers.h[0][r] = cl.map_shared_rank(c.h[0], r);
            s_peers.h[1][r] = cl.map_shared_rank(c.h[1], r);
            s_peers.res[r] = cl.map_shared_rank(c.res, r);
        }
    } else {
        int* gn = a.g_node; int* ga = a.g_arc;
        const size_t Nn = (size_t)a.N, Aa = 2 * (size_t)(a.E_cap > 0 ? a.E_cap : 1);
        c.excess = a.g_excess + c.n_lo; c.tcap = gn + c.n_lo; c.h[0] = gn + Nn + c.n_lo; c.h[1] = gn + 2 * Nn + c.n_lo;
        c.hmin = gn + 3 * Nn + c.n_lo;
        c.res = ga + c.a_lo; c.dstp = ga + Aa + c.a_lo; c.revp = ga + 2 * Aa + c.a_lo; c.srcl = ga + 3 * Aa + c.a_lo;
        if (threadIdx.x < CS) {
            const int r = threadIdx.x;
            const int nlo = min(r * c.npc, N);
            s_peers.excess[r] = a.g_excess + nlo; s_peers.tcap[r] = gn + nlo;
            s_peers.h[0][r] = gn + Nn + nlo; s_peers.h[1][r] = gn + 2 * Nn + nlo;
            s_peers.res[r] = ga + s_alo[r];
        }
    }
    c.flags0 = cl.map_shared_rank(s_flags, 0);
    __syncthreads();
    // static arc tables of this CTA: packed (rank, local) references of the head node and of the reverse slot
    for (int i = threadIdx.x; i < c.a_cnt; i += NT) {
        const int g = c.a_lo + i;
        const int v = a.a_dst[g], rv = a.a_rev[g];
        const int vr = v / c.npc;
        int rr = 0;
        while (rr + 1 < CS && rv >= s_alo[rr + 1]) ++rr;
        c.dstp[i] = (vr << LBITS) | (v - vr * c.npc);
        c.revp[i] = (rr << LBITS) | (rv - s_alo[rr]);
        c.srcl[i] = a.a_src[g] - c.n_lo;
    }
    if (c.rank == 0 && threadIdx.x == 0) { s_stats[5] = in_smem; for (int i = 0; i < 8; ++i) a.red[i] = 0; }
    cl.sync();

    int* lab = a.labels;
    long long cur_energy = 0;
    int version = 0; // bumped by every applied move
    int turn = 0;    // rotates the cluster-wide flag words
    int sturn = 0;   // rotates the cluster-wide sum words
    const int gtid = c.rank * NT + threadIdx.x;

    auto expand = [&](int alpha) -> bool {
        int any = 0;
        for (int v = threadIdx.x; v < c.n_cnt; v += NT) any |= (lab[c.n_lo + v] != alpha);
        if (!cluster_or(cl, c, any, turn)) return false;
        // unary part of the move energy
        for (int v = threadIdx.x; v < c.n_cnt; v += NT) {
            const int g = c.n_lo + v, l = lab[g];
            if (l != alpha) { a.u0[g] = c.D[(size_t)g * K + alpha]; a.u1[g] = c.D[(size_t)g * K + l]; }
            else { a.u0[g] = 0; a.u1[g] = 0; }
        }
        cl.sync();
        const int Vaa = smooth(c, alpha, alpha);
        int nonsub = 0, wide = 0;
        for (int i = threadIdx.x; i < c.a_cnt; i += NT) {
            const int g = c.a_lo + i;
            const int ed = a.a_eid[g];
            if (ed & 1) continue; // the a -> b slot does the pair's bookkeeping and initialises BOTH residuals
            const int e = ed >> 1;
            const int va = a.a_src[g], vb = a.a_dst[g];
            const int la = lab[va], lb = lab[vb];
            const long long wk = c.w[e];
            int P1 = 0, P2 = 0;
            if (la != alpha && lb != alpha) {
                const long long A = wk * Vaa, B = wk * smooth(c, alpha, lb), C = wk * smooth(c, la, alpha), Dd = wk * smooth(c, la, lb);
                // E(xa,xb) = A + (C-A) xa + (Dd-C) xb + P (1-xa) xb, and P (1-xa) xb = P1 (1-xa) xb + P2 [(1-xb) xa + xb - xa]:
                // capacity P1 on a->b, P2 on b->a (P1 + P2 = P).  Same energy function, hence the same minimisers, but residual
                // paths exist in both directions from the start (short BFS distances, far fewer sweeps).
                const long long Pl = B + C - A - Dd;
                if (Pl < 0) nonsub = 1;
                else if (Pl > 0x3fffffff) wide = 1;
                const long long p2 = Pl >> 1, p1 = Pl - p2;
                atomicAdd((unsigned long long*)&a.u0[va], (unsigned long long)A);
                atomicAdd((unsigned long long*)&a.u1[va], (unsigned long long)(C - p2));
                atomicAdd((unsigned long long*)&a.u1[vb], (unsigned long long)(Dd - C + p2));
                P1 = (int)p1; P2 = (int)p2;
            } else if (la != alpha) {
                atomicAdd((unsigned long long*)&a.u0[va], (unsigned long long)(wk * Vaa));
                atomicAdd((unsigned long long*)&a.u1[va], (unsigned long long)(wk * smooth(c, la, alpha)));
            } else if (lb != alpha) {
                atomicAdd((unsigned long long*)&a.u0[vb], (unsigned long long)(wk * Vaa));
                atomicAdd((unsigned long long*)&a.u1[vb], (unsigned long long)(wk * smooth(c, alpha, lb)));
            }
            c.res[i] = P1;
            const int q = c.revp[i];
            c.peers->res[q >> LBITS][q & LMASK] = P2;
        }
        if (cluster_or(cl, c, nonsub | wide, turn)) {
            // a non-submodular pair fails the move silently (GCO refuses it too); a pair capacity of 2^30 or more is reported in stats[7]
            if (cluster_or(cl, c, wide, turn) && threadIdx.x == 0) s_stats[7] = 1;
            return false;
        }
        int big = 0;
        for (int v = threadIdx.x; v < c.n_cnt; v += NT) {
            const int g = c.n_lo + v;
            const long long x0 = __ldcg(&a.u0[g]), x1 = __ldcg(&a.u1[g]);
            const long long m = x0 < x1 ? x0 : x1;
            const bool act = lab[g] != alpha;
            const long long ex = act ? x1 - m : 0, tc = act ? x0 - m : 0;
            if (ex > 0x1fffffff || tc > 0x1fffffff) big = 1;
            c.excess[v] = ex;
            c.tcap[v] = (int)tc;
        }
        // sink capacities are 32-bit: a terminal capacity of 2^29 or more refuses the move and is reported in stats[6].  The excess
        // is 64-bit: it never exceeds the node's terminal capacity plus its incoming pair capacities (each below 2^30), whatever the degree
        if (cluster_or(cl, c, big, turn)) { if (threadIdx.x == 0) s_stats[6] = 1; return false; }
        // ---- max-flow (phase 1) ----
        if (threadIdx.x == 0) ++s_stats[1];
        int cur = 0;
        while (global_relabel(cl, c, cur, turn, s_stats)) {
            for (int s = 0; s < 96; ++s) {
                if (threadIdx.x == 0) ++s_stats[2];
                const bool more = sweep(cl, c, cur, turn);
                cur ^= 1;
                if (!more) break;
            }
        }
        // ---- candidate labeling: keep iff the site can still reach the sink ----
        for (int v = threadIdx.x; v < c.n_cnt; v += NT) {
            const int g = c.n_lo + v;
            a.newlab[g] = (lab[g] != alpha && c.h[cur][v] == HINF) ? alpha : lab[g];
        }
        cl.sync();
        const long long e_new = energy_of(cl, c, a.newlab, sturn);
        if (e_new < cur_energy) {
            for (int v = gtid; v < N; v += CS * NT) lab[v] = a.newlab[v];
            cur_energy = e_new;
            if (threadIdx.x == 0) ++s_stats[0];
            cl.sync();
            return true;
        }
        return false;
    };

    // expansion with the "same labeling, same answer" shortcut (identical decisions in every CTA)
    auto try_label = [&](int alpha) -> bool {
        __syncthreads();
        if (s_failver[alpha] == version) return false;
        const bool ok = expand(alpha);
        __syncthreads();
        if (ok) ++version;
        else if (threadIdx.x == 0) s_failver[alpha] = version;
        __syncthreads();
        return ok;
    };

    if (E == 0) {
        // no smoothness: GCO's special case, independent argmin per site
        for (int v = gtid; v < N; v += CS * NT) {
            int best = 0;
            for (int l = 1; l < K; ++l) if (c.D[(size_t)v * K + l] < c.D[(size_t)v * K + best]) best = l;
            lab[v] = best;
        }
        cl.sync();
    } else {
        cur_energy = energy_of(cl, c, lab, sturn);
        const int KT = K < 64 ? K : 64; // label table lives in smem; K > 64 is rejected on the host
        if (threadIdx.x == 0) { for (int l = 0; l < KT; ++l) { s_table[l] = l; s_failver[l] = -1; } s_qn = 1; s_queue[0] = KT; }
        __syncthreads();
        if (a.n_iter == -1) {
            // GCO adaptive cycles (see oracle/gc_oracle.cpp); every CTA keeps its own identical copy of the bookkeeping
            while (true) {
                __syncthreads();
                if (s_qn == 0) break;
                const int qsz = s_queue[s_qn - 1];
                int start = KT - qsz;
                for (int next = start; next < KT; ++next) {
                    __syncthreads();
                    const bool ok = try_label(s_table[next]);
                    if (!ok) {
                        if (threadIdx.x == 0) { int t = s_table[next]; s_table[next] = s_table[start]; s_table[start] = t; }
                        ++start;
                    }
                }
                __syncthreads();
                const int nsz = KT - start;
                if (threadIdx.x == 0) {
                    if (nsz == qsz) { /* all succeeded: run the same queue again */ }
                    else if (nsz > 0) { if (s_qn < 64) s_queue[s_qn++] = nsz; }
                    else --s_qn;
                }
            }
        } else {
            for (int cycle = 0; cycle < a.n_iter; ++cycle) {
                const long long before = cur_energy;
                for (int l = 0; l < KT; ++l) try_label(l);
                if (cur_energy == before) break;
            }
        }
        __syncthreads();
    }
    const long long e_fin = energy_of(cl, c, lab, sturn);
    if (c.rank == 0 && threadIdx.x == 0) {
        if (a.energy_out) *a.energy_out = e_fin;
        if (a.stats) for (int i = 0; i < 8; ++i) a.stats[i] = s_stats[i];
    }
    cl.sync(); // no CTA may exit while a peer can still address its shared memory
}

struct GcWs {
    int* off; int* fill; int* a_src; int* a_dst; int* a_rev; int* a_eid; long long* u0; long long* u1; long long* red; int* newlab;
    long long* g_excess; int* g_node; int* g_arc;
};

static size_t carve_gc(GcWs& w, void* ws, size_t bytes, int N, int E)
{
    WsCarver c(ws, bytes);
    size_t e = E > 0 ? E : 1;
    w.off = c.take<int>((size_t)N + 1); w.fill = c.take<int>(N);
    w.a_src = c.take<int>(2 * e); w.a_dst = c.take<int>(2 * e); w.a_rev = c.take<int>(2 * e); w.a_eid = c.take<int>(2 * e);
    w.u0 = c.take<long long>(N); w.u1 = c.take<long long>(N); w.red = c.take<long long>(8);
    w.newlab = c.take<int>(N);
    w.g_excess = c.take<long long>(N);
    w.g_node = c.take<int>(4 * (size_t)N);
    w.g_arc = c.take<int>(4 * 2 * e);
    return isb_align(c.off);
}

} // namespace

extern "C" size_t isb_alpha_expansion_workspace_bytes(int N, int K, int E)
{
    GcWs w;
    return carve_gc(w, nullptr, 0, N, E);
}

extern "C" int isb_alpha_expansion(int N, const int32_t* n_nodes_dev, int K, int E, const int32_t* n_edges_dev, const int32_t* edges,
                                   const int32_t* edge_wi, const int32_t* unary_i, const int32_t* smooth_i, int n_iter, int32_t* labels,
                                   int64_t* energy_out, int32_t* stats_out, void* ws, size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(edges && edge_wi && unary_i && smooth_i && labels && ws, "null pointer");
    ISB_REQUIRE(N > 0 && K > 0 && K <= 64 && E >= 0, "bad sizes (K must be <= 64)");
    ISB_REQUIRE(n_iter == -1 || n_iter > 0, "n_iter must be -1 (adaptive cycles) or positive");
    ISB_REQUIRE((N + CS - 1) / CS < (1 << LBITS) && 2LL * E < (1LL << LBITS), "graph too large for the packed references");
    GcWs w;
    size_t need = carve_gc(w, ws, ws_bytes, N, E);
    ISB_REQUIRE(need <= ws_bytes, "workspace too small");
    GcArgs a;
    a.N = N; a.K = K; a.E_cap = E; a.n_edges_dev = n_edges_dev; a.n_nodes_dev = n_nodes_dev;
    a.edges = edges; a.w = edge_wi; a.D = unary_i; a.V = smooth_i; a.n_iter = n_iter;
    a.labels = labels; a.energy_out = (long long*)energy_out; a.stats = stats_out;
    a.off = w.off; a.fill = w.fill; a.a_src = w.a_src; a.a_dst = w.a_dst; a.a_rev = w.a_rev; a.a_eid = w.a_eid;
    a.u0 = w.u0; a.u1 = w.u1; a.red = w.red; a.newlab = w.newlab;
    a.g_excess = w.g_excess; a.g_node = w.g_node; a.g_arc = w.g_arc;
    // always launch with the full dynamic smem: the kernel decides from the REAL node/edge counts (device scalars)
    // whether the flow state fits in the cluster's shared memory or stays in the global workspace
    const size_t smem_max = 227 * 1024 - 8 * 1024; // leave room for the static arrays
    a.dyn_bytes = (int)smem_max;
    {   // the attribute is per device: set it once for every device this process launches on
        static bool attr_set[64] = {};
        int dev = 0;
        ISB_CUDA_CHECK(cudaGetDevice(&dev));
        if (dev < 0 || dev >= 64 || !attr_set[dev]) {
            ISB_CUDA_CHECK(cudaFuncSetAttribute(k_alpha_expansion, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max));
            if (dev >= 0 && dev < 64) attr_set[dev] = true;
        }
    }
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope prof(ISB_PROF_GC, st);
    if (E > 0) {
        k_gc_build_csr<<<1, NT, 0, st>>>(a);
        ISB_LAUNCH_CHECK();
    }
    k_alpha_expansion<<<CS, NT, smem_max, st>>>(a);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}
