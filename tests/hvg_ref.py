"""Float64 restatement of scanpy 1.10.1 ``highly_variable_genes(flavor="cell_ranger", n_top_genes=…)`` on a dense matrix, written
the way scanpy writes it (``_get_mean_var``, ``pd.cut`` bins, ``groupby(...).agg(median, statsmodels mad)``, ``_nth_highest``),
so that the device path in dance_b200/transforms/pp.py is checked against an independent route to the same numbers."""
import numpy as np
import pandas as pd


def _mad(a):
    a = np.asarray(a, np.float64)
    return np.median(np.abs(a - np.median(a)) / 0.6744897501960817)


def cell_ranger(X, n_top_genes: int) -> pd.DataFrame:
    X = np.asarray(X, np.float64)
    n = X.shape[0]
    mean = X.mean(axis=0)
    var = (np.multiply(X, X).mean(axis=0) - mean**2) * (n / (n - 1))
    mean[mean == 0] = 1e-12
    disp = var / mean
    df = pd.DataFrame({"means": mean, "dispersions": disp})
    df["mean_bin"] = pd.cut(df["means"], np.r_[-np.inf, np.percentile(df["means"], np.arange(10, 105, 5)), np.inf])
    stats = df.groupby("mean_bin", observed=True)["dispersions"].agg(avg="median", dev=_mad)
    stats = stats.loc[df["mean_bin"]].set_index(df.index)
    with np.errstate(divide="ignore", invalid="ignore"):
        df["dispersions_norm"] = (df["dispersions"] - stats["avg"]) / stats["dev"]
    dn = df["dispersions_norm"].to_numpy()
    x = dn[~np.isnan(dn)]
    k = min(n_top_genes, X.shape[1], x.size)
    cut = np.sort(x)[::-1][k - 1]
    df["highly_variable"] = np.nan_to_num(dn, nan=-np.inf) >= cut
    return df
