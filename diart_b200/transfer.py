"""A live stream's whole state, to move it between servers (``MultiStreamDiarization.export`` / ``restore``, and the same on
``MultiStreamVoiceActivityDetection``).

A :class:`StreamState` is one stream of one server after its last tick: the packed device state of ``dg_multi_export`` (audio
from the next window on, staged samples included, the 16 kHz frames a resampled stream's next windows read, the aggregation
history, the clustering state and the gallery claims) and what the server keeps on the host (timestamp shift, counters,
labels, latency, source rate).  It also records what the stream's results depend on -- fingerprints of the models and of
the gallery it is named from, and the configuration values the networks, clustering and post-path read -- so that a server
refuses a state it could not continue exactly.  ``save`` / ``load`` write and read it as a versioned ``.npz``."""
from __future__ import annotations

import hashlib
import json
from typing import Any, Dict

import numpy as np
import torch

VERSION = 1   # of the .npz and of the packed state (dg_multi_export's format version)


def model_fingerprint(model) -> str:
    """a hash of a native model (``B200PyanNet`` / ``B200XVectorSincNet``): its class, ``pool_mode`` / ``powerset`` and every
    tensor of its state dict; computed once per model object"""
    fp = getattr(model, "_transfer_fingerprint", None)
    if fp is None:
        h = hashlib.sha256(type(model).__name__.encode())
        h.update(repr((getattr(model, "pool_mode", None), getattr(model, "powerset", None))).encode())
        for name in sorted(model._state):
            value = model._state[name]
            arr = value.detach().cpu().numpy() if isinstance(value, torch.Tensor) else np.asarray(value)
            arr = np.ascontiguousarray(arr)
            h.update(f"{name}|{arr.dtype.str}|{arr.shape}".encode())
            h.update(arr.tobytes())
        fp = h.hexdigest()
        model._transfer_fingerprint = fp
    return fp


def gallery_fingerprint(gallery) -> str:
    """a hash of a ``SpeakerGallery``'s names and float64 centroids (not its threshold: a stream keeps its own)"""
    fp = getattr(gallery, "_transfer_fingerprint", None)
    if fp is None:
        h = hashlib.sha256("\0".join(gallery.names).encode())
        h.update(np.ascontiguousarray(gallery.known.centroids, dtype=np.float64).tobytes())
        fp = h.hexdigest()
        gallery._transfer_fingerprint = fp
    return fp


class StreamState:
    """One exported stream (``server.export``), to ``server.restore`` on this or any compatible server.  Its contents are
    private; ``kind``, ``sample_rate``, ``latency`` and ``nbytes`` describe it."""

    def __init__(self, blob: np.ndarray, meta: Dict[str, Any]):
        self._blob = np.ascontiguousarray(blob, dtype=np.uint8)
        self._meta = dict(meta)

    @property
    def kind(self) -> str:
        """``"diarization"`` or ``"vad"``"""
        return self._meta["kind"]

    @property
    def sample_rate(self) -> int:
        """the stream's source rate in Hz"""
        return int(self._meta["rate"])

    @property
    def latency(self) -> float:
        return float(self._meta["latency"])

    @property
    def nbytes(self) -> int:
        """bytes of the packed device state"""
        return int(self._blob.nbytes)

    def __eq__(self, other) -> bool:
        return (isinstance(other, StreamState) and self._meta == other._meta and
                np.array_equal(self._blob, other._blob))

    def save(self, path):
        """writes the state to ``path`` (a ``.npz``)"""
        meta = np.frombuffer(json.dumps(self._meta, sort_keys=True).encode(), dtype=np.uint8)
        np.savez(path, version=np.int64(VERSION), blob=self._blob, meta=meta)

    @classmethod
    def load(cls, path) -> "StreamState":
        """reads a state ``save`` wrote; ValueError for another format version or a file that is not one"""
        with np.load(path, allow_pickle=False) as z:
            if not {"version", "blob", "meta"} <= set(z.files):
                raise ValueError(f"{path} is not a saved stream state")
            version = int(z["version"])
            if version != VERSION:
                raise ValueError(f"{path} holds a stream state of format version {version}; this build reads {VERSION}")
            blob, meta = z["blob"], json.loads(z["meta"].tobytes().decode())
        if blob.dtype != np.uint8 or blob.ndim != 1 or meta.get("version") != VERSION:
            raise ValueError(f"{path} is not a saved stream state of format version {VERSION}")
        return cls(blob, meta)
