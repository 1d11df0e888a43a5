"""numpy restatement of ``isb_forest_fit_groups`` (``forest_fit._fit_arrays_groups``): every tree built alone by the single-forest
oracle (``oracle.forest.build_tree``) from its group's rows and parameters; ``n_levels`` is that of the deepest tree, as the device
reports it for the whole call."""
from oracle import forest as of


def fit_arrays_groups(Xs, y, K, counts, seeds, tree_group, max_features, min_samples_split, min_samples_leaf, max_depth,
                      min_impurity_decrease):
    trees = [of.build_tree(Xs[g], y, counts[t], K, int(seeds[t]), int(max_features[g]), int(min_samples_split[g]),
                           int(min_samples_leaf[g]), max_depth, min_impurity_decrease) for t, g in enumerate(tree_group)]
    levels = max(t['n_levels'] for t in trees)
    for t in trees:
        t['n_levels'] = levels
    return trees
