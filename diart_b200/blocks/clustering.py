"""``OnlineSpeakerClustering`` (mirrors reference ``src/diart/blocks/clustering.py:10-218``).

Constrained incremental clustering: cosine distances of the local speakers' embeddings to the
running centroids, optimal assignment, threshold ``delta_new``, centroid update (sum) for long
speakers and creation of new centroids while there is room.  State (float64 centroids, active set)
lives on the GPU inside a ``dg_cluster`` handle; ``centers`` / ``active_centers`` read it back.
"""
from __future__ import annotations

import ctypes as C
from typing import Iterable, List, Optional, Tuple

import numpy as np
import torch

from .. import _lib
from ..core import SlidingWindowFeature
from ..mapping import SpeakerMap


# scipy.spatial.distance.cdist metrics (reference mapping.py:175) evaluated in float64 by the clustering kernel
METRICS = {"cosine": 0, "euclidean": 1, "sqeuclidean": 2, "cityblock": 3, "chebyshev": 4}


class OnlineSpeakerClustering:
    def __init__(self, tau_active: float, rho_update: float, delta_new: float,
                 metric: Optional[str] = "cosine", max_speakers: int = 20,
                 device: Optional[torch.device] = None):
        if metric not in METRICS:
            raise ValueError(f"metric must be one of {sorted(METRICS)} (scipy cdist names), got {metric!r}")
        self.tau_active, self.rho_update, self.delta_new = tau_active, rho_update, delta_new
        self.metric, self.max_speakers = metric, max_speakers
        self.device = torch.device(device) if device is not None else torch.device("cuda")
        if self.device.type == "cuda" and self.device.index is None and torch.cuda.is_available():
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.blocked_centers = set()   # reference clustering.py:46 -- never populated there either
        self._h: Optional[C.c_void_p] = None
        self._dim: Optional[int] = None
        self._seed: Optional[np.ndarray] = None   # initial centroids (n, D) written when the handle is created

    # ------------------------------------------------------------------ handle management
    def _handle(self, dim: int) -> C.c_void_p:
        if self._h is None:
            if self._seed is not None and self._seed.shape[1] != dim:
                raise ValueError(f"the known speakers' centroids have dimension {self._seed.shape[1]}, the embeddings "
                                 f"{dim}")
            _lib.require_cuda(self.device)
            h = C.c_void_p()
            _lib.check(_lib.lib().dg_cluster_create(self.max_speakers, dim, self.tau_active, self.rho_update,
                                                    self.delta_new, self.device.index, C.byref(h)))
            if METRICS[self.metric]:
                _lib.check(_lib.lib().dg_cluster_set_metric(h, METRICS[self.metric]))
            self._h, self._dim = h, dim
            if self._seed is not None:
                self._write_seed()
        assert dim == self._dim, "embedding dimension changed"
        return self._h

    def seed(self, centroids: Optional[np.ndarray]):
        """the initial state before the first step: centres 0 .. n - 1 hold ``centroids`` (float64 (n, D)) and are active,
        and the state is initialised, so the first step takes the reference's distance path.  None or n = 0: the fresh
        state (not initialised).  Written now if the handle exists, else when it is created (the dimension is checked
        then, before any launch)."""
        c = None if centroids is None or len(centroids) == 0 else np.ascontiguousarray(centroids, dtype=np.float64)
        if c is not None and len(c) > self.max_speakers:
            raise ValueError(f"{len(c)} known speakers, at most max_speakers = {self.max_speakers}")
        if c is not None and self._h is not None and c.shape[1] != self._dim:
            raise ValueError(f"the known speakers' centroids have dimension {c.shape[1]}, the embeddings {self._dim}")
        self._seed = c
        if self._h is not None:
            if c is None:
                self.reset()
            else:
                self._write_seed()

    def _write_seed(self):
        centers = np.zeros((self.max_speakers, self._dim))
        centers[:len(self._seed)] = self._seed
        self._set_state(centers, range(len(self._seed)), True)

    def __del__(self):
        try:
            if self._h is not None:
                _lib.lib().dg_cluster_destroy(self._h)
        except Exception:  # noqa: BLE001
            pass

    def _state(self):
        if self._h is None:
            return None, set(), False
        centers = np.zeros((self.max_speakers, self._dim))
        active = np.zeros(self.max_speakers, dtype=np.int32)
        init = C.c_int()
        _lib.check(_lib.lib().dg_cluster_get_state(self._h, centers.ctypes.data, active.ctypes.data, C.byref(init)))
        return centers, set(int(i) for i in np.where(active)[0]), bool(init.value)

    def _set_state(self, centers: np.ndarray, active: Iterable[int], initialized: bool = True):
        h = self._handle(centers.shape[1])
        mask = np.zeros(self.max_speakers, dtype=np.int32)
        mask[list(active)] = 1
        c = np.ascontiguousarray(centers, dtype=np.float64)
        _lib.check(_lib.lib().dg_cluster_set_state(h, c.ctypes.data, mask.ctypes.data, int(initialized)))

    # ------------------------------------------------------------------ reference attributes
    @property
    def centers(self) -> Optional[np.ndarray]:
        centers, _, init = self._state()
        return centers if init else None

    @property
    def active_centers(self) -> set:
        return self._state()[1]

    @property
    def num_known_speakers(self) -> int:
        return len(self.active_centers)

    @property
    def num_blocked_speakers(self) -> int:
        return len(self.blocked_centers)

    @property
    def num_free_centers(self) -> int:
        return self.max_speakers - self.num_known_speakers - self.num_blocked_speakers

    @property
    def inactive_centers(self) -> List[int]:
        active = self.active_centers
        return [c for c in range(self.max_speakers) if c not in active or c in self.blocked_centers]

    def get_next_center_position(self) -> Optional[int]:
        active = self.active_centers
        for center in range(self.max_speakers):
            if center not in active and center not in self.blocked_centers:
                return center
        return None

    def init_centers(self, dimension: int):
        self._set_state(np.zeros((self.max_speakers, dimension)), [], True)
        self.blocked_centers = set()

    def update(self, assignments: Iterable[Tuple[int, int]], embeddings: np.ndarray):
        centers, active, init = self._state()
        if init:
            for l_spk, g_spk in assignments:
                assert g_spk in active, "Cannot update unknown centers"
                centers[g_spk] += embeddings[l_spk]
            self._set_state(centers, active, True)

    def add_center(self, embedding: np.ndarray) -> int:
        centers, active, _ = self._state()
        center = self.get_next_center_position()
        centers[center] = embedding
        active.add(center)
        self._set_state(centers, active, True)
        return center

    def reset(self):
        if self._h is not None:
            _lib.check(_lib.lib().dg_cluster_reset(self._h))

    # ------------------------------------------------------------------ the step
    def step_batch(self, segmentation: torch.Tensor, embeddings: torch.Tensor, want_permuted: bool = False):
        """Processes B consecutive chunks in order on the device.

        segmentation (B,F,K), embeddings (B,K,D): float32 tensors (moved to the device if needed).
        Returns ``(maps int32 (B,K) on device, permuted float32 (B,F,M) on device or None)``.
        """
        _lib.require_cuda(self.device)
        seg = segmentation.to(self.device, torch.float32).contiguous()
        emb = embeddings.to(self.device, torch.float32).contiguous()
        B, F, K = seg.shape
        assert emb.shape[0] == B and emb.shape[1] == K
        h = self._handle(emb.shape[2])
        maps = torch.empty((B, K), device=self.device, dtype=torch.int32)
        perm = torch.empty((B, F, self.max_speakers), device=self.device) if want_permuted else None
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().dg_cluster_step(h, seg.data_ptr(), emb.data_ptr(), B, F, K, maps.data_ptr(),
                                                  _lib.ptr(perm), _lib.stream_ptr(self.device)))
        return maps, perm

    def identify(self, segmentation: SlidingWindowFeature, embeddings: torch.Tensor) -> SpeakerMap:
        data = segmentation.data if isinstance(segmentation, SlidingWindowFeature) else np.asarray(segmentation)
        seg = torch.from_numpy(np.ascontiguousarray(data, dtype=np.float32)).unsqueeze(0)
        emb = torch.as_tensor(embeddings).detach().float()
        if emb.ndim == 2:
            emb = emb.unsqueeze(0)
        maps, _ = self.step_batch(seg, emb)
        amap = maps[0].cpu().numpy()
        self._state()   # surfaces the reference's "Cannot update unknown centers" assertion, if it fired
        return SpeakerMap(amap, self.max_speakers)

    def __call__(self, segmentation: SlidingWindowFeature, embeddings: torch.Tensor) -> SlidingWindowFeature:
        return SlidingWindowFeature(self.identify(segmentation, embeddings).apply(segmentation.data),
                                    segmentation.sliding_window)
