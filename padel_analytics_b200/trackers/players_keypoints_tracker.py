"""PlayerKeypointsTracker on the CUDA engine — API of
/root/reference/trackers/players_keypoints_tracker/players_keypoints_tracker.py (:15-327)."""
from __future__ import annotations

from pathlib import Path
from typing import Iterable, Optional, Type

import numpy as np

from ..engine.yolo_engine import ResultBlock, YoloEngine
from .tracker import NoPredictFrames, Object, Tracker


class PlayerKeypoint:
    """One named keypoint of one player (players_keypoints_tracker.py:15-57).  A plain __slots__ class: a frame holds
    ~200 of them and rank 0 builds them for every frame of every shard."""
    __slots__ = ("id", "name", "xy")

    def __init__(self, id: int, name: str, xy: tuple[float, float]):
        self.id = id
        self.name = name
        self.xy = xy

    def __eq__(self, other):
        return isinstance(other, PlayerKeypoint) and (self.id, self.name, self.xy) == (other.id, other.name, other.xy)

    def __repr__(self):
        return f"PlayerKeypoint(id={self.id}, name={self.name!r}, xy={self.xy})"

    def asint(self):
        return tuple(int(v) for v in self.xy)

    @classmethod
    def from_json(cls, x: dict):
        return cls(**x)

    def serialize(self) -> dict:
        return {"id": self.id, "name": self.name, "xy": self.xy}

    def draw(self, frame):
        import cv2

        cv2.circle(frame, self.asint(), radius=2, color=(255, 0, 0), thickness=-1)
        return frame


class PlayerKeypoints:
    KEYPOINTS_NAMES = ["left_foot", "right_foot", "torso", "right_shoulder", "left_shoulder", "head", "neck",
                       "left_hand", "right_hand", "right_knee", "left_knee", "right_elbow", "left_elbow"]
    CONNECTIONS = [("left_foot", "left_knee"), ("left_knee", "torso"), ("right_foot", "right_knee"),
                   ("right_knee", "torso"), ("torso", "left_shoulder"), ("torso", "right_shoulder"),
                   ("left_hand", "left_elbow"), ("left_elbow", "left_shoulder"), ("left_shoulder", "neck"),
                   ("neck", "head"), ("right_hand", "right_elbow"), ("right_elbow", "right_shoulder"),
                   ("right_shoulder", "neck")]

    def __init__(self, player_keypoints: list[PlayerKeypoint]):
        self.player_keypoints = player_keypoints
        self._by_name = None

    @property
    def keypoints_by_name(self) -> dict:
        if self._by_name is None:
            self._by_name = {k.name: k for k in self.player_keypoints}
        return self._by_name

    @classmethod
    def from_json(cls, x: dict):
        return cls([PlayerKeypoint.from_json(k) for k in x["player_keypoints"]])

    def serialize(self) -> dict:
        return {"player_keypoints": [k.serialize() for k in self.player_keypoints]}

    def __len__(self):
        return len(self.player_keypoints)

    def __iter__(self):
        return iter(self.player_keypoints)

    def __getitem__(self, name: str) -> PlayerKeypoint:
        assert name in self.KEYPOINTS_NAMES
        return self.keypoints_by_name[name]

    def draw(self, frame):
        import cv2

        pts = {k.name: k.asint() for k in self.player_keypoints}
        if not pts:
            return frame
        for a, b in self.CONNECTIONS:
            cv2.line(frame, pts[a], pts[b], color=(255, 0, 0), thickness=2)
        return frame


class PlayersKeypoints(Object):
    """All players' keypoints of one frame (players_keypoints_tracker.py:165-205).  Array-backed: the tracker hands in
    the frame's (players, 13, 2) coordinates and the PlayerKeypoints / PlayerKeypoint objects (~200 per frame) are only
    materialised when `players_keypoints` is read -- rank 0 assembles every frame of every shard, and a consumer that
    only serialises or counts never pays for the objects."""

    def __init__(self, players_keypoints: list[PlayerKeypoints] | None = None, _xy: list | None = None) -> None:
        super().__init__()
        self._list = players_keypoints
        self._xy = _xy  # (players, 13, 2) float64 ndarray when built by the tracker

    @classmethod
    def from_xy(cls, xy: list) -> "PlayersKeypoints":
        return cls(None, _xy=xy)

    @property
    def players_keypoints(self) -> list[PlayerKeypoints]:
        if self._list is None:
            names = PlayerKeypoints.KEYPOINTS_NAMES
            self._list = [PlayerKeypoints([PlayerKeypoint(i, names[i], (x, y)) for i, (x, y) in enumerate(det)])
                          for det in self._xy.tolist()]
        return self._list

    @classmethod
    def from_json(cls, x) -> "PlayersKeypoints":
        return cls([PlayerKeypoints.from_json(p) for p in x])

    def serialize(self) -> list[dict]:
        if self._list is None:  # straight from the coordinates, same JSON as the objects would give
            names = PlayerKeypoints.KEYPOINTS_NAMES
            return [{"player_keypoints": [{"id": i, "name": names[i], "xy": (x, y)} for i, (x, y) in enumerate(det)]}
                    for det in self._xy.tolist()]
        return [p.serialize() for p in self._list]

    def __len__(self):
        return len(self._xy) if self._list is None else len(self._list)

    def __iter__(self):
        return iter(self.players_keypoints)

    def __getitem__(self, i):
        return self.players_keypoints[i]

    def draw(self, frame):
        for p in self.players_keypoints:
            frame = p.draw(frame)
        return frame


class PlayerKeypointsTracker(Tracker):
    stage = "detect"
    CONF = 0.25
    IOU = 0.7

    def __init__(self, model_path, train_image_size: int, batch_size: int, load_path: Optional[str | Path] = None,
                 save_path: Optional[str | Path] = None):
        super().__init__(load_path=load_path, save_path=save_path)
        self.model = YoloEngine(model_path, max_batch=batch_size)  # reference: YOLO(model_path) (:238)
        assert train_image_size in (640, 1280)
        self.train_image_size = train_image_size
        self.batch_size = batch_size

    def video_info_post_init(self, video_info) -> "PlayerKeypointsTracker":
        return self

    def object(self) -> Type[Object]:
        return PlayersKeypoints

    def draw_kwargs(self) -> dict:
        return {}

    def __str__(self) -> str:
        return "players_keypoints_tracker"

    def restart(self) -> None:
        self.results.restart()

    def to(self, device: str) -> None:
        self.model.to(device)

    def detect_sample_async(self, sample):
        return self.model.predict_frames_async(sample, "pil_square", conf=self.CONF, iou=self.IOU,
                                               imgsz=self.train_image_size, classes=[0])

    def postprocess(self, results, frame_hw) -> list[PlayersKeypoints]:
        """players_keypoints_tracker.py:276-318.  The reference's `.squeeze(0)` / `len()==2` juggling crashes for
        exactly one or two detected players (SURVEY App. E q4); here every detection count is handled uniformly."""
        ratio_x = frame_hw[1] / self.train_image_size
        ratio_y = frame_hw[0] / self.train_image_size
        out = []
        names = PlayerKeypoints.KEYPOINTS_NAMES
        if isinstance(results, ResultBlock):  # the same arithmetic over the whole block of frames at once
            xy = results.keypoints[..., :2].astype(np.float64) * np.array([ratio_x, ratio_y])
            return [PlayersKeypoints.from_xy(xy[i, :c]) for i, c in enumerate(results.counts.tolist())]
        for result in results:
            # float32 -> Python float (exact) * Python float ratio, as `keypoint[0].item() * ratio_x` does (:306-309)
            xy = result.keypoints.xy.numpy().astype(np.float64) * np.array([ratio_x, ratio_y])
            out.append(PlayersKeypoints.from_xy(xy.reshape(-1, len(names), 2)))
        return out

    def predict_sample(self, sample: Iterable[np.ndarray], **kwargs) -> list[PlayersKeypoints]:
        return self.postprocess(self.detect_sample(sample), sample[0].shape[:2])

    def predict_frames(self, frame_generator, **kwargs):
        raise NoPredictFrames()
