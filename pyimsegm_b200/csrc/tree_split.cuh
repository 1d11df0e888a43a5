// tree_split.cuh -- the constants and FP64 expressions of scikit-learn 1.9's Gini tree builder (_criterion.pyx, _partitioner.pxd,
// _tree.pyx) shared by both tree fits: forest_fit.cu (exact splits, level by level) and extra_trees_fit.cu (random splits, depth
// first).  The library is built with -fmad=false, so each expression is evaluated in scikit-learn's order without FMA contraction.
#pragma once

namespace {

constexpr int FF_KMAX = 64;                  // classes (isb_forest_predict_proba's limit)
constexpr int FF_DMAX = 2048;                // feature columns
constexpr long long FF_WMAX = 1ll << 26;     // total count of a tree: squared class counts stay below 2^52, exact in float64
constexpr float FEATURE_THRESHOLD = 1e-7f;   // _partitioner.pxd: a float32 constant, added in float32
constexpr double FF_EPSILON = 2.220446049250313e-16;  // np.finfo('double').eps of _tree.pyx

// Gini.node_impurity / children_impurity from the sum of squared (integer) class counts and the weight
__device__ __forceinline__ double gini_of(unsigned long long sq, double w)
{
    return 1.0 - (double)sq / (w * w);
}

// Criterion.proxy_impurity_improvement
__device__ __forceinline__ double gini_proxy(unsigned long long sql, double wl, unsigned long long sqr, double wr)
{
    return -wr * gini_of(sqr, wr) - wl * gini_of(sql, wl);
}

// Criterion.impurity_improvement: wn the node's weight, W the tree's, imp the node's impurity, il / ir the children's
__device__ __forceinline__ double impurity_improvement(double wn, double W, double imp, double wl, double il, double ir)
{
    const double wr = wn - wl;
    return (wn / W) * (imp - (wr / wn * ir) - (wl / wn * il));
}

} // namespace
