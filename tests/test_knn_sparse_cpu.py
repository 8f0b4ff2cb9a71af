"""`_to_device_csr`: any scipy.sparse matrix becomes the canonical CSR the sparse k-NN and pair-distance kernels
require (int64 indptr, int32 indices sorted within each row, fp32 values, duplicates summed)."""
import numpy as np
import scipy.sparse as sp
import torch

from pymde_b200.preprocess import data_matrix as dm


def _check(data, dense):
    (indptr, indices, values), shape = dm._to_device_csr(data, "cpu")
    assert shape == dense.shape
    assert indptr.dtype == torch.int64 and indices.dtype == torch.int32 and values.dtype == torch.float32
    ip, ix, v = indptr.numpy(), indices.numpy(), values.numpy()
    assert ip[0] == 0 and ip[-1] == len(ix) == len(v) and (np.diff(ip) >= 0).all()
    for r in range(shape[0]):
        row = ix[ip[r]:ip[r + 1]]
        assert (np.diff(row) > 0).all() and (row >= 0).all() and (row < shape[1]).all()
    got = sp.csr_matrix((v, ix, ip), shape=shape).toarray()
    np.testing.assert_array_equal(got, dense.astype(np.float32))


def test_coo_with_duplicates_is_summed():
    r = np.array([0, 2, 0, 2, 1, 0])
    c = np.array([3, 1, 3, 1, 0, 2])
    v = np.array([1.0, 2.0, 0.5, -1.0, 4.0, 7.0])
    A = sp.coo_matrix((v, (r, c)), shape=(3, 5))
    dense = np.zeros((3, 5))
    np.add.at(dense, (r, c), v)
    _check(A, dense)
    (indptr, indices, _), _ = dm._to_device_csr(A, "cpu")
    assert int(indptr[-1]) == 4  # (0, 3) and (2, 1) appear once each


def test_unsorted_csr_is_sorted():
    A = sp.csr_matrix((np.array([1.0, 2.0, 3.0, 4.0], np.float32), np.array([4, 0, 2, 1]), np.array([0, 3, 4])),
                      shape=(2, 5))
    assert not A.has_sorted_indices
    _check(A, A.toarray())
    # the caller's matrix is left as it was
    assert list(A.indices) == [4, 0, 2, 1]


def test_csc_int32_float64_and_empty_rows():
    rng = np.random.default_rng(0)
    dense = rng.standard_normal((40, 30)) * (rng.random((40, 30)) < 0.2)
    dense[[3, 17, 39]] = 0.0  # empty rows, including the last one
    _check(sp.csc_matrix(dense), dense)
    _check(sp.csr_matrix(dense.astype(np.float64)), dense)
    _check(sp.csr_matrix((dense != 0).astype(np.int32) * 3), (dense != 0) * 3.0)


def test_all_empty_matrix():
    _check(sp.csr_matrix((6, 9), dtype=np.float32), np.zeros((6, 9)))
