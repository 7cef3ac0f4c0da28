"""similarity retriever (SURVEY.md section 8f rank 4: the pair-selection step in front of the hot path).

Drop-in for gtsfm/retriever/similarity_retriever.py:35-182 (`SimilarityRetriever`): same constructor, `get_image_pairs`
contract (ValueError without descriptors, RuntimeError above MAX_NUM_IMAGES, pairs (i1 < i2) per query image best first),
`set_num_matched`, `repr`.  The similarity matrix G G^T and the per-row top-`num_matched` selection run in
libgtsfm_b200.so (`b2_similarity_pairs_host`); the descriptors come from `gtsfm_b200.global_descriptor` (NetVLAD) or the reference's.
Difference: the returned similarity matrix is full (the reference fills the upper BLOCK triangle only, :104-111), which
`compute_pairs_from_similarity_matrix` never looks at (:176-177 masks the lower triangle).
"""
from __future__ import annotations

from pathlib import Path
from typing import List, Optional, Tuple

import numpy as np

from . import _lib
from .gtsfm_api import RetrieverBase

MAX_NUM_IMAGES = 10000  # similarity_retriever.py:23


class B200SimilarityRetriever(RetrieverBase):
    def __init__(self, num_matched: int, min_score: float = 0.1, blocksize: int = 50, device: int = 0) -> None:
        self._num_matched = num_matched
        self._blocksize = blocksize  # kept for the constructor contract: the device computes the matrix in one launch
        self._min_score = min_score
        self._device = device
        self._ctx: Optional[_lib.Context] = None
        self._latest_similarity_matrix: Optional[np.ndarray] = None

    def __repr__(self) -> str:
        return f"""
        B200SimilarityRetriever:
            Num. frames matched: {self._num_matched}
            Block size: {self._blocksize}
            Minimum score: {self._min_score}
        """

    def __getstate__(self):  # device state is created lazily on the worker (picklable like the other plugins)
        d = dict(self.__dict__)
        d["_ctx"] = None
        return d

    def set_num_matched(self, n) -> None:
        self._num_matched = n

    def _context(self) -> _lib.Context:
        if self._ctx is None:
            self._ctx = _lib.Context(self._device)
        return self._ctx

    def similarity_and_partners(self, global_descriptors, want_sim: bool = True) -> Tuple[Optional[np.ndarray], np.ndarray]:
        g = np.ascontiguousarray(np.asarray(global_descriptors, np.float32))
        if g.ndim != 2:
            raise ValueError("global descriptors must all have the same length")
        n, dim = g.shape
        if n > MAX_NUM_IMAGES:
            raise RuntimeError("Cannot construct similarity matrix of this size.")
        pad = (-dim) % 64  # zero columns do not change G G^T
        if pad:
            g = np.ascontiguousarray(np.pad(g, ((0, 0), (0, pad))))
        k = min(int(self._num_matched), n)
        partners = np.full((n, max(k, 1)), -1, np.int32)
        sim = np.empty((n, n), np.float32) if want_sim else None
        ctx = self._context()
        rc = ctx.lib.b2_similarity_pairs_host(ctx.handle, _lib.ptr(g), n, dim + pad, max(k, 1), float(self._min_score), _lib.ptr(partners),
                                              _lib.ptr(sim) if want_sim else None)
        ctx.check(rc, "similarity_pairs")
        return sim, partners[:, :k]

    def get_image_pairs(self, global_descriptors: Optional[List[np.ndarray]], image_fnames: List[str],
                        plots_output_dir: Optional[Path] = None) -> List[Tuple[int, int]]:
        if global_descriptors is None:
            raise ValueError("Global descriptors need to be provided")
        if len(global_descriptors) == 0:
            return []
        sim, partners = self.similarity_and_partners(global_descriptors)
        self._latest_similarity_matrix = sim
        rows, ranks = np.nonzero(partners >= 0)  # row-major: query ascending, best partner first (:255-259)
        return [(int(i), int(partners[i, r])) for i, r in zip(rows, ranks)]
