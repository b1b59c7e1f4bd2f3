"""Cached-replay data format (SURVEY §8f-2): the on-disk detections / embeddings that sit either side of the hot path,
and a runner that replays many cached sequences through one multi-stream GPU tracker.

Reference behaviour restated here (nothing is imported from the reference):

* ``NpyAppender``       -- `boxmot/data/cache.py:140-260` (`AppendableNpyWriter`): a standard NPY v2.0 file whose row
  count is rewritten in place after every append.  The header is the one numpy writes (`numpy/lib/_format_impl.py`
  `_write_array_header`: sorted dict, growth padding for the first axis, 64-byte alignment), so the files are
  byte-identical to the reference's and either side can append to the other's file.
* ``SequenceCache``     -- `boxmot/data/dataset.py:307-368, 373-430` (`MOTSequence._prepare/_build_det_index/__iter__`):
  dets rows are `(frame_id, x1, y1, x2, y2, conf, cls)` float32 sorted by frame, embeddings are row-aligned,
  `target_fps` thinning by `compute_fps_mask` (`dataset.py:127-132`).
* ``replay_sequences``  -- the frame loop of `boxmot/engine/eval/replay.py:311-350` (`process_sequence`): confidence
  filter on the cached rows, frames without detections are NOT passed to the tracker, embeddings/detections row
  mismatch is an error, rows formatted by `convert_to_mot_format` (`engine/tracking/mot.py:255-271`).
* ``fill_embeddings``   -- the embeddings-only fill of `engine/eval/cache.py:252-308`: an existing detections cache gets its
  row-aligned embeddings file from any `get_features(boxes, frame)` backend (a `B200ReID` keeps that on the GPU).
* ``cache_paths``       -- the directory layout of `engine/eval/cache.py:371-424, 503-512` / `data/dataset.py:154-175`.

B200 angle: sequences are independent units, so S cached sequences advance together as the S streams of one
`MultiStreamTracker` (one launch sequence per step for all of them).  A stream that has run out of frames is fed
empty detections; its (empty) outputs are ignored, which cannot change the rows already produced.
"""
from __future__ import annotations

import os
import struct
from pathlib import Path
from typing import Callable, Iterator, List, Optional, Sequence, Tuple

import numpy as np

_MAGIC = b"\x93NUMPY"
_ALIGN = 64          # numpy ARRAY_ALIGN
_GROWTH_DIGITS = 21  # numpy GROWTH_AXIS_MAX_DIGITS: spare room so the first axis can grow in place


def _descr(dtype: np.dtype) -> str:
    dtype = np.dtype(dtype)
    if dtype.fields is not None or dtype.hasobject:
        raise TypeError("only plain numeric dtypes are cached")
    return dtype.str


def npy_header(rows: int, trailing: Tuple[int, ...], dtype=np.float32, version=(2, 0)) -> bytes:
    """The exact header bytes numpy writes for a C-ordered `(rows, *trailing)` array (NPY 1.0 or 2.0)."""
    shape = (int(rows), *[int(t) for t in trailing])
    body = "{'descr': %r, 'fortran_order': False, 'shape': %r, }" % (_descr(dtype), shape)
    body += " " * (_GROWTH_DIGITS - len(repr(shape[0])))
    raw = body.encode("latin1")
    fmt = "<H" if tuple(version) == (1, 0) else "<I"
    hlen = len(raw) + 1
    pad = _ALIGN - ((len(_MAGIC) + 2 + struct.calcsize(fmt) + hlen) % _ALIGN)
    return _MAGIC + bytes(version) + struct.pack(fmt, hlen + pad) + raw + b" " * pad + b"\n"


def read_npy_header(fp) -> Tuple[Tuple[int, int], Tuple[int, ...], np.dtype, int]:
    """(version, shape, dtype, data offset) of an open NPY file; C order only."""
    import ast

    fp.seek(0)
    head = fp.read(8)
    if head[:6] != _MAGIC:
        raise ValueError("not an NPY file")
    version = (head[6], head[7])
    if version == (1, 0):
        (hlen,) = struct.unpack("<H", fp.read(2))
    elif version == (2, 0):
        (hlen,) = struct.unpack("<I", fp.read(4))
    else:
        raise ValueError(f"Unsupported npy version for append: {version}")
    d = ast.literal_eval(fp.read(hlen).decode("latin1"))
    if d.get("fortran_order"):
        raise ValueError("Fortran-order npy append is not supported")
    return version, tuple(d["shape"]), np.dtype(d["descr"]), fp.tell()


class NpyAppender:
    """Append row chunks to a standard `.npy` file without buffering the whole array
    (same constructor, `append`, `close`, `rows` and file bytes as the reference's `AppendableNpyWriter`)."""

    def __init__(self, path, *, dtype=np.float32, trailing_shape: Optional[Tuple[int, ...]] = None,
                 empty_trailing_shape: Optional[Tuple[int, ...]] = None):
        self.path = Path(path)
        self.dtype = np.dtype(dtype)
        self.trailing_shape = tuple(trailing_shape) if trailing_shape is not None else None
        self.empty_trailing_shape = (tuple(empty_trailing_shape) if empty_trailing_shape is not None
                                     else self.trailing_shape)
        self.rows = 0
        self._fp = None
        self._data_offset = None
        self._version = (2, 0)
        if self.path.exists():
            self._open_existing()
        elif self.trailing_shape is not None:
            self._create(self.trailing_shape)

    def _create(self, trailing) -> None:
        self.path.parent.mkdir(parents=True, exist_ok=True)
        self.trailing_shape = tuple(trailing)
        self._fp = open(self.path, "wb+")
        self._fp.write(npy_header(self.rows, self.trailing_shape, self.dtype, (2, 0)))
        self._data_offset = self._fp.tell()

    def _open_existing(self) -> None:
        self._fp = open(self.path, "rb+")
        self._version, shape, self.dtype, offset = read_npy_header(self._fp)
        self.rows = int(shape[0]) if len(shape) > 0 else 0
        self.trailing_shape = tuple(shape[1:]) if len(shape) > 1 else ()
        if self.rows == 0 and self.trailing_shape == (0,):
            # placeholder written for an empty sequence: start over with the real width
            self._fp.close()
            self._fp = None
            self.trailing_shape = None
            self.path.unlink(missing_ok=True)
            return
        self._data_offset = offset
        self._fp.seek(0, os.SEEK_END)

    def _sync_header(self) -> None:
        if self._fp is None:
            return
        head = npy_header(self.rows, self.trailing_shape, self.dtype, self._version)
        if len(head) != self._data_offset:
            raise RuntimeError(f"NPY header resize changed data offset for {self.path}: "
                               f"{self._data_offset} -> {len(head)}")
        self._fp.seek(0)
        self._fp.write(head)
        self._fp.flush()

    def append(self, arr) -> None:
        arr = np.asarray(arr, dtype=self.dtype)
        if arr.size == 0:
            return
        if arr.ndim == 1:
            arr = arr.reshape(1, -1)
        if self.trailing_shape is None:
            self._create(tuple(arr.shape[1:]))
        elif tuple(arr.shape[1:]) != self.trailing_shape:
            raise ValueError(f"Appended array shape mismatch for {self.path}: "
                             f"expected (*, {self.trailing_shape}), got {arr.shape}")
        arr = np.ascontiguousarray(arr, dtype=self.dtype)
        self._fp.seek(0, os.SEEK_END)
        self._fp.write(arr.tobytes(order="C"))
        self.rows += int(arr.shape[0])
        self._sync_header()

    def close(self) -> None:
        if self._fp is None:
            if self.empty_trailing_shape is None:
                return
            self._create(self.empty_trailing_shape)
        self._sync_header()
        self._fp.close()
        self._fp = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def cache_paths(project, detector: str, seq: str, *, benchmark: Optional[str] = None, split: Optional[str] = None,
                reid_key: Optional[str] = None, preprocess: str = "resize") -> Tuple[Path, Optional[Path]]:
    """`<project>/dets_n_embs[/<benchmark>][/<split>]/<detector>/dets/<seq>.npy` and
    `.../<detector>/embs/<reid_key>/<preprocess>/<seq>.npy` (None without a ReID key)."""
    base = Path(project) / "dets_n_embs"
    if benchmark:
        base = base / benchmark
    if split:
        base = base / split
    base = base / (Path(detector).stem if Path(detector).suffix else str(detector))
    dets = base / "dets" / f"{seq}.npy"
    embs = base / "embs" / reid_key / preprocess / f"{seq}.npy" if reid_key else None
    return dets, embs


def fps_mask(frames: np.ndarray, orig_fps: int, target_fps: int) -> np.ndarray:
    """Rows whose frame id survives thinning from `orig_fps` to `target_fps` (`dataset.py:127-132`)."""
    tgt = min(orig_fps, target_fps)
    step = orig_fps / tgt
    wanted = set(np.arange(1, int(frames.max()) + 1, step).astype(int))
    return np.isin(frames.astype(int), list(wanted))


class SequenceCache:
    """One cached sequence: `(frame_id, x1, y1, x2, y2, conf, cls)` rows + row-aligned embeddings.  `frame_hw`: the
    `(H, W)` of the sequence's images (the reference hands every update a frame of that size; SFSORT's margins read it)."""

    def __init__(self, dets, embs=None, *, frame_ids: Optional[Sequence[int]] = None, name: str = "",
                 orig_fps: Optional[int] = None, target_fps: Optional[int] = None,
                 frame_hw: Optional[Tuple[int, int]] = None):
        self.name = name
        self.frame_hw = None if frame_hw is None else (int(frame_hw[0]), int(frame_hw[1]))
        self.dets = np.load(dets, mmap_mode="r") if isinstance(dets, (str, os.PathLike)) else np.asarray(dets)
        if self.dets.ndim != 2 or (self.dets.shape[0] and self.dets.shape[1] != 7):
            raise ValueError(f"dets cache of {name!r} must be (rows, 7): frame_id, x1, y1, x2, y2, conf, cls")
        self.embs = None
        if embs is not None:
            self.embs = np.load(embs, mmap_mode="r") if isinstance(embs, (str, os.PathLike)) else np.asarray(embs)
            if self.dets.shape[0] != self.embs.shape[0]:
                raise ValueError(f"Row mismatch in {name}")
        ids = None if frame_ids is None else np.asarray(frame_ids, dtype=np.int64)
        if target_fps and orig_fps and self.dets.shape[0] > 0:
            keep = fps_mask(self.dets[:, 0], orig_fps, target_fps)
            self.dets = self.dets[keep]
            if self.embs is not None:
                self.embs = self.embs[keep]
            if ids is not None:
                kept = set(self.dets[:, 0].astype(int).tolist())
                ids = np.asarray([f for f in ids.tolist() if f in kept], dtype=np.int64)
        self.index = self._build_index()
        # the reference iterates the sequence's image list; without one, every frame id present in the cache
        self.frame_ids = ids if ids is not None else np.asarray(list(self.index), dtype=np.int64)

    def _build_index(self):
        """frame id -> (start, end) row range; rows of one frame are contiguous (runs, as the reference scans them)."""
        index = {}
        n = self.dets.shape[0]
        if n == 0:
            return index
        fids = np.asarray(self.dets[:, 0]).astype(int)
        cuts = np.flatnonzero(fids[1:] != fids[:-1]) + 1
        starts = np.concatenate(([0], cuts))
        ends = np.concatenate((cuts, [n]))
        for s, e in zip(starts.tolist(), ends.tolist()):
            index[int(fids[s])] = (s, e)   # a frame id that re-appears later overwrites, like the reference's dict
        return index

    def __len__(self) -> int:
        return len(self.frame_ids)

    def frames(self) -> Iterator[Tuple[int, np.ndarray, np.ndarray]]:
        """(frame_id, dets (n, 6), embs (n, D) or (n, 0)) for every frame of the sequence, empty frames included."""
        width = 6
        for fid in self.frame_ids.tolist():
            if fid in self.index:
                s, e = self.index[fid]
                d = np.array(self.dets[s:e, 1:])
                m = np.array(self.embs[s:e]) if self.embs is not None else np.zeros((e - s, 0))
            else:
                d = np.empty((0, width), dtype=np.float32)
                m = np.empty((0, 0), dtype=np.float32)
            yield int(fid), d, m


def to_mot_rows(tracks: np.ndarray, frame_id: int) -> np.ndarray:
    """`(frame, id, left, top, width, height, conf, cls + 1, det_ind)` rows of one frame
    (`convert_to_mot_format`, numpy branch: the box is rounded AFTER the width/height subtraction)."""
    tracks = np.asarray(tracks)
    if tracks.size == 0:
        return np.empty((0, 9), dtype=np.float32)
    ltwh = np.array(tracks[:, 0:4], copy=True)
    ltwh[:, 2] = ltwh[:, 2] - ltwh[:, 0]
    ltwh[:, 3] = ltwh[:, 3] - ltwh[:, 1]
    n = len(tracks)
    return np.column_stack((
        np.full((n, 1), frame_id, dtype=np.int32),
        tracks[:, 4].reshape(-1, 1).astype(np.int32),
        ltwh.round().astype(np.int32),
        tracks[:, 5].reshape(-1, 1),
        (tracks[:, 6] + 1).reshape(-1, 1).astype(np.int32),
        tracks[:, 7].reshape(-1, 1).astype(np.int32),
    ))


def _frame_inputs(cache: SequenceCache, conf_threshold: float):
    """The (frame_id, dets, embs) triples `process_sequence` hands to `tracker.update`: confidence filter applied,
    frames left without detections dropped (the reference skips the call), row mismatch raised."""
    for fid, d, m in cache.frames():
        if d.size and conf_threshold > 0:
            keep = d[:, 4] >= conf_threshold
            d = d[keep]
            m = m[keep] if m.size else m
        if not d.size:
            continue
        if m.size and d.shape[0] != m.shape[0]:
            raise ValueError(f"Detection/embedding count mismatch for {cache.name} frame {fid}: "
                             f"dets={d.shape[0]} embs={m.shape[0]}")
        yield fid, d, (m if m.size else None)


def replay_sequences(tracker, caches: Sequence[SequenceCache], conf_threshold: float = 0.0,
                     on_step: Optional[Callable[[int], None]] = None, timing=None) -> List[np.ndarray]:
    """Replay `len(caches)` cached sequences through `tracker`, a multi-stream tracker with one stream per cache
    (`MultiStreamTracker.update(dets_list, imgs, embs_list) -> rows_list`).  Returns one MOT array per sequence.

    Every stream consumes its own non-empty frames in order; the streams advance together, one tracker step for all
    of them.  A stream that has finished receives empty detections and its outputs are discarded.

    `timing`: optional `runtime.TimingStats`-like object; every step adds the engine's CUDA-event ReID / association
    durations (`tracker.last_device_ms()`), the split `process_sequence` reports as ReID time vs tracker-rest time
    (`replay.py:333-335`)."""
    S = len(caches)
    if getattr(tracker, "n_streams", S) != S:
        raise ValueError(f"tracker has {tracker.n_streams} streams for {S} sequences")
    feeds = [_frame_inputs(c, conf_threshold) for c in caches]
    if getattr(tracker, "kind", None) == "sfsort":   # each stream's margins come from its sequence's frame size
        for i, c in enumerate(caches):
            if c.frame_hw is not None:
                tracker.set_frame_size(i, c.frame_hw)
    rows: List[List[np.ndarray]] = [[] for _ in range(S)]
    feat_dim = int(getattr(tracker, "feat_dim", 0))
    wants_embs = bool(getattr(tracker, "with_reid", False))
    empty_d = np.empty((0, 6), dtype=np.float32)
    step = 0
    while True:
        dets, embs, fids = [], [], []
        for feed in feeds:
            item = next(feed, None)
            if item is None:
                dets.append(empty_d)
                embs.append(None)
                fids.append(None)
            else:
                fid, d, m = item
                if wants_embs and m is None:
                    raise ValueError("this tracker associates on appearance: the cache has no embeddings "
                                     "(replay never re-embeds from stub images)")
                if wants_embs and m.shape[1] != feat_dim:
                    raise ValueError(f"cached embeddings are {m.shape[1]}-d, the tracker was built for {feat_dim}-d")
                dets.append(np.ascontiguousarray(d, dtype=np.float32))
                embs.append(np.ascontiguousarray(m, dtype=np.float32) if wants_embs else None)
                fids.append(fid)
        if all(f is None for f in fids):
            break
        out = tracker.update(dets, None, embs if wants_embs else None)
        if timing is not None and hasattr(tracker, "last_device_ms"):
            timing.add_device_times(*tracker.last_device_ms())
            timing.frames += 1
        for i, fid in enumerate(fids):
            if fid is not None and len(out[i]):
                rows[i].append(to_mot_rows(np.asarray(out[i]), fid))
        step += 1
        if on_step is not None:
            on_step(step)
    if getattr(tracker, "kind", None) == "occluboost":   # online GTA gap rows at the end, as process_sequence
        for i in range(S):
            gta = tracker.flush_gta(i)
            if gta.size:
                rows[i].append(np.asarray(gta, dtype=np.float32))
    return [np.concatenate(r, axis=0) if r else np.empty((0, 9), dtype=np.float32) for r in rows]


def write_cache(dets_path, embs_path, frames: Sequence[Tuple[int, np.ndarray, Optional[np.ndarray]]]) -> None:
    """Write a sequence the way the reference's generator does (`engine/eval/cache.py:702-717, 895-928`): one appended
    chunk per non-empty frame, the frame id prepended to the `(x1, y1, x2, y2, conf, cls)` rows, the embeddings chunk
    written BEFORE the detections chunk so an interrupted run never leaves more detection rows than embedding rows."""
    dw = NpyAppender(dets_path, dtype=np.float32, trailing_shape=(7,), empty_trailing_shape=(7,))
    ew = (NpyAppender(embs_path, dtype=np.float32, trailing_shape=None, empty_trailing_shape=(0,))
          if embs_path is not None else None)
    try:
        for fid, d, m in frames:
            d = np.asarray(d, dtype=np.float32).reshape(-1, 6)
            if not len(d):
                continue
            if ew is not None:
                if m is None or len(m) != len(d):
                    raise ValueError(f"frame {fid}: embeddings must be row-aligned with detections")
                ew.append(np.asarray(m).astype(np.float32, copy=False))
            dw.append(np.column_stack((np.full((len(d), 1), fid, dtype=np.float32), d)))
    finally:
        dw.close()
        if ew is not None:
            ew.close()


def fill_embeddings(dets_path, embs_path, reid_model, load_frame: Callable[[int], Optional[np.ndarray]],
                    on_progress: Optional[Callable[[int, int], None]] = None) -> int:
    """Embeddings-only fill of a cached sequence (`engine/eval/cache.py:252-308`): the detections file is immutable; its
    rows are read back in stored order, each run of equal frame id is embedded with one
    `reid_model.get_features(boxes (n, 4), frame)` call (a `B200ReID` keeps crops, network and normalisation on the
    GPU) and appended to `embs_path` row-aligned with the detections.  `load_frame(frame_id)` returns the BGR frame or
    None (such frames are skipped, as the reference does for unreadable images).  Returns the rows written."""
    dets = np.load(dets_path).astype(np.float32, copy=False)
    if dets.ndim != 2 or dets.shape[0] == 0:
        return 0
    writer = NpyAppender(embs_path, dtype=np.float32, trailing_shape=None, empty_trailing_shape=(0,))
    written = 0
    try:
        n_rows, i = dets.shape[0], 0
        while i < n_rows:
            fid = int(dets[i, 0])
            j = i
            while j < n_rows and int(dets[j, 0]) == fid:
                j += 1
            boxes = dets[i:j, 1:5].copy()
            img = load_frame(fid)
            if img is not None:
                feats = np.asarray(reid_model.get_features(boxes, img), dtype=np.float32)
                if feats.ndim == 1:
                    feats = feats.reshape(1, -1) if feats.size else feats
                if feats.shape[0] != boxes.shape[0]:
                    raise RuntimeError(f"Embedding count mismatch during fill for {Path(dets_path).stem}: "
                                       f"dets={boxes.shape[0]} embs={feats.shape[0]}")
                writer.append(feats)
                written += boxes.shape[0]
            if on_progress is not None:
                on_progress(j, n_rows)
            i = j
    finally:
        writer.close()
    return written


def write_mot_results(txt_path, mot_rows: np.ndarray) -> None:
    """Append MOT rows to a result file exactly as the reference does (`engine/tracking/mot.py:318-344`): the file is
    created even when there is nothing to write; 9-column rows use `%d,%d,%d,%d,%d,%d,%.6f,%d,%d`."""
    if mot_rows is None:
        return
    txt_path = Path(txt_path)
    txt_path.parent.mkdir(parents=True, exist_ok=True)
    txt_path.touch(exist_ok=True)
    mot_rows = np.asarray(mot_rows)
    if mot_rows.size == 0:
        return
    if mot_rows.ndim == 1:
        mot_rows = mot_rows.reshape(1, -1)
    with open(str(txt_path), "a") as f:
        if mot_rows.shape[1] == 9:
            np.savetxt(f, mot_rows, fmt="%d,%d,%d,%d,%d,%d,%.6f,%d,%d")
        else:
            np.savetxt(f, mot_rows, fmt="%g", delimiter=",")
