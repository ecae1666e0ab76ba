"""PlayerTracker on the CUDA engine — same API as reference trackers/players_tracker/players_tracker.py
(Player :14-197, Players :199-263, PlayerTracker :266-383)."""
from __future__ import annotations

from pathlib import Path
from typing import Iterable, Optional, Type

import numpy as np

from ..engine.yolo_engine import ResultBlock, YoloEngine
from . import sv_compat as sv
from .tracker import NoPredictFrames, Object, Tracker


class Player:
    """players_tracker.py:14-197.  Built either from a one-row `Detections` (the reference's constructor) or, on the
    fast path, straight from the row's values (`from_row`): slicing a Detections per player costs more than the
    ByteTrack update of the whole frame, and rank 0 does it for every frame of every shard."""

    def __init__(self, detection, projection: Optional[tuple[int, int]] = None):
        self._detection = detection
        self.projection = projection
        self.xyxy = detection.xyxy[0]
        tid = detection.tracker_id
        self.id = int(tid[0]) if tid is not None and len(tid) else None
        self.class_id = int(detection.class_id[0])
        self.confidence = float(detection.confidence[0])

    @classmethod
    def from_row(cls, xyxy, tracker_id, class_id, confidence, projection=None) -> "Player":
        p = cls.__new__(cls)
        p._detection = None
        p.projection = projection
        p.xyxy = xyxy
        p.id = None if tracker_id is None else int(tracker_id)
        p.class_id = int(class_id)
        p.confidence = float(confidence)
        return p

    @property
    def detection(self):
        if self._detection is None:
            self._detection = sv.Detections(xyxy=np.asarray(self.xyxy).reshape(1, 4),
                                            confidence=np.array([self.confidence], dtype=np.float32),
                                            class_id=np.array([self.class_id]),
                                            tracker_id=None if self.id is None else np.array([self.id]))
        return self._detection

    @property
    def top_left(self):
        return tuple(int(p) for p in self.xyxy[:2])

    @property
    def bottom_right(self):
        return tuple(int(p) for p in self.xyxy[2:])

    @property
    def height(self):
        return self.bottom_right[1] - self.top_left[1]

    @property
    def width(self):
        return self.bottom_right[0] - self.top_left[0]

    @property
    def midpoint(self):
        return int(self.top_left[0] + self.width / 2), int(self.top_left[1] + self.height / 2)

    @property
    def feet(self):
        return int(self.top_left[0] + self.width / 2), int(self.bottom_right[1])

    @classmethod
    def from_json(cls, x: dict):
        det = sv.Detections(xyxy=np.array([x["xyxy"]]), confidence=np.array([x["confidence"]]),
                            tracker_id=None if x.get("id") is None else np.array([x["id"]]),
                            class_id=np.array([x["class_id"]]))
        return cls(detection=det, projection=x.get("projection"))

    def serialize(self) -> dict:
        return {"id": self.id, "xyxy": [float(p) for p in self.xyxy], "projection": self.projection,
                "class_id": self.class_id, "confidence": self.confidence}

    def draw(self, frame, video_info=None, annotator="rectangle_bounding_box", show_confidence=True):
        import cv2

        cv2.rectangle(frame, self.top_left, self.bottom_right, (0, 200, 255), 2)
        label = f"{self.id}" + (f" {self.confidence:.2f}" if show_confidence else "")
        cv2.putText(frame, label, (self.top_left[0], max(0, self.top_left[1] - 4)), cv2.FONT_HERSHEY_SIMPLEX, 0.5,
                    (0, 200, 255), 1)
        return frame

    def draw_projection(self, frame):
        """The player on the mini court (players_tracker.py:171-190): a filled circle at `projection` and the id."""
        import cv2

        if not self.projection:
            raise ValueError("Inexistent projection.")
        cv2.circle(frame, self.projection, 8, (0, 0, 255), -1)
        cv2.putText(frame, str(self.id), (self.projection[0], self.projection[1] - 10), cv2.FONT_HERSHEY_SIMPLEX, 0.9,
                    (0, 0, 255), 2)
        return frame


class Players(Object):
    """All tracked players of one frame (players_tracker.py:199-263).  Array-backed like PlayersKeypoints: the tracker
    hands in the frame's rows (xyxy, id, class, confidence) and the Player objects are materialised when `players` is
    read."""

    def __init__(self, players: list[Player] | None = None, _rows=None):
        super().__init__()
        self._list = players
        self._rows = _rows  # (xyxy (n,4) float32, ids (n,) int | None, class_id (n,), confidence (n,))

    @classmethod
    def from_rows(cls, xyxy, ids, class_id, confidence) -> "Players":
        return cls(None, _rows=(xyxy, ids, class_id, confidence))

    @property
    def players(self) -> list[Player]:
        if self._list is None:
            xyxy, ids, cid, conf = self._rows
            self._list = [Player.from_row(xyxy[i], None if ids is None else ids[i], cid[i], conf[i])
                          for i in range(len(xyxy))]
        return self._list

    @classmethod
    def from_json(cls, x: list[dict]) -> "Players":
        return cls([Player.from_json(p) for p in x])

    def serialize(self) -> list[dict]:
        return [p.serialize() for p in self.players]

    def __len__(self):
        return len(self._rows[0]) if self._list is None else len(self._list)

    def __iter__(self):
        return iter(self.players)

    def __getitem__(self, i):
        return self.players[i]

    def draw(self, frame, video_info=None, annotator="rectangle_bounding_box", show_confidence=True):
        for p in self.players:
            frame = p.draw(frame, video_info, annotator, show_confidence)
        return frame


class PlayerTracker(Tracker):
    stage = "detect"
    CONF = 0.5
    IOU = 0.7
    IMGSZ = 640

    def __init__(self, model_path, polygon_zone, batch_size: int, annotator: str = "rectangle_bounding_box",
                 show_confidence: bool = True, load_path: Optional[str | Path] = None,
                 save_path: Optional[str | Path] = None):
        super().__init__(load_path=load_path, save_path=save_path)
        self.model = YoloEngine(model_path, max_batch=batch_size)  # reference: YOLO(model_path) (:303)
        self.polygon_zone = polygon_zone
        self.batch_size = batch_size
        self.annotator = annotator
        self.show_confidence = show_confidence

    def video_info_post_init(self, video_info) -> "PlayerTracker":
        self.video_info = video_info
        self.byte_track = sv.ByteTrack(frame_rate=video_info.fps)
        return self

    def object(self) -> Type[Object]:
        return Players

    def draw_kwargs(self) -> dict:
        return {"video_info": self.video_info, "annotator": self.annotator, "show_confidence": self.show_confidence}

    def __str__(self) -> str:
        return "players_tracker"

    def restart(self) -> None:
        self.results.restart()
        self.byte_track.reset()

    def to(self, device: str) -> None:
        self.model.to(device)

    def detect_sample_async(self, sample):
        """Enqueue the model stage (boxes in frame pixels); returns a callable yielding the raw results (see
        YoloEngine.predict_frames_async)."""
        return self.model.predict_frames_async(sample, "letterbox_q1", conf=self.CONF, iou=self.IOU,
                                               imgsz=self.IMGSZ, classes=[0])

    def postprocess(self, results, frame_hw=None) -> list[Players]:
        """Polygon filter + ByteTrack ids (players_tracker.py:362-378); sequential, frame order matters.  The boxes
        are already in frame pixels, so `frame_hw` is not needed."""
        if isinstance(results, ResultBlock) and hasattr(self.byte_track, "update_many"):
            return self._postprocess_block(results)
        out = []
        for result in results:
            det = sv.Detections.from_ultralytics(result)
            if self.polygon_zone is not None:
                det = det[self.polygon_zone.trigger(det)]
            det = self.byte_track.update_with_detections(detections=det)
            out.append(Players.from_rows(det.xyxy, det.tracker_id, det.class_id, det.confidence))
        return out

    def _postprocess_block(self, block: ResultBlock) -> list[Players]:
        """The same stage over a dense block of frames: one polygon test over all detections, one native ByteTrack call
        for all frames (`pb_bytetrack_update_many`), result objects as views into the surviving rows."""
        n, cap = block.rows.shape[:2]
        counts = block.counts.astype(np.int64)
        valid = np.arange(cap)[None, :] < counts[:, None]  # (n, cap) row-major = frame order, score order within
        det = block.rows[valid]  # (total, rowlen)
        frame_of = np.repeat(np.arange(n), counts)
        if self.polygon_zone is not None and len(det):
            keep = self.polygon_zone.trigger(sv.Detections(xyxy=det[:, :4]))
            det, frame_of = det[keep], frame_of[keep]
        xyxy = np.ascontiguousarray(det[:, :4])
        conf = np.ascontiguousarray(det[:, 4])
        per_frame = np.bincount(frame_of, minlength=n).astype(np.int32)
        ids = self.byte_track.update_many(xyxy, conf, per_frame)
        tracked = ids != -1
        xyxy, conf, ids = xyxy[tracked], conf[tracked], ids[tracked].astype(int)
        cid = det[tracked, 5].astype(int)
        ends = np.cumsum(np.bincount(frame_of[tracked], minlength=n)).tolist()
        out, a = [], 0
        for b in ends:
            out.append(Players.from_rows(xyxy[a:b], ids[a:b], cid[a:b], conf[a:b]))
            a = b
        return out

    def predict_sample(self, sample: Iterable[np.ndarray], **kwargs) -> list[Players]:
        return self.postprocess(self.detect_sample(sample))

    def predict_frames(self, frame_generator, **kwargs):
        raise NoPredictFrames()
