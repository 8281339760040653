from dance_b200.transforms import pp as _pp


def log1p(adata, *args, **kwargs):
    return _pp.log1p(adata, *args, **kwargs)


def normalize_total(adata, *args, **kwargs):
    return _pp.normalize_total(adata, *args, **kwargs)


def filter_genes(data, *args, **kwargs):
    return _pp.filter_genes(data, *args, **kwargs)


def filter_cells(data, *args, **kwargs):
    return _pp.filter_cells(data, *args, **kwargs)


def highly_variable_genes(adata, *args, **kwargs):
    return _pp.highly_variable_genes(adata, *args, **kwargs)
