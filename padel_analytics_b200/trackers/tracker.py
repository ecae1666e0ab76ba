"""Tracker abstractions with the public surface of /root/reference/trackers/tracker.py:15-330 (same names, ctor
arguments, JSON cache behaviour and batching semantics), so code written against the reference keeps working."""
from __future__ import annotations

import json
from abc import ABC, abstractmethod
from dataclasses import dataclass, field
from pathlib import Path
from typing import Iterable, Optional, Type

import numpy as np
import torch


class NoPredictSample(Exception):
    """The tracker consumes the whole frame generator (predict_frames), not samples — tracker.py:15-20."""


class NoPredictFrames(Exception):
    """The tracker consumes samples of batch_size frames (predict_sample) — tracker.py:22-27."""


class Object(ABC):
    """A tracked thing in one frame (players, ball, ...) with a JSON round trip — tracker.py:30-65."""

    @classmethod
    def from_json(cls, x):
        raise NotImplementedError

    def serialize(self):
        raise NotImplementedError

    def draw(self, frame: np.ndarray, **kwargs) -> np.ndarray:
        return frame


@dataclass
class TrackingResults:
    """Per-frame predictions accumulated over a video — tracker.py:67-120."""

    predictions: list = field(default_factory=list)
    sample_predictions: list = field(default_factory=list)
    counter: int = 0

    def load(self, predictions: list) -> None:
        self.predictions, self.sample_predictions, self.counter = predictions, [], 0

    def update(self, predictions: list) -> None:
        self.predictions += predictions
        self.sample_predictions = predictions
        self.counter += 1

    def restart(self) -> None:
        self.predictions, self.sample_predictions, self.counter = [], [], 0

    def __len__(self) -> int:
        return len(self.predictions)

    def __getitem__(self, i: int):
        return self.predictions[i]

    def __iter__(self):
        return iter(self.predictions)


def sampler(generator: Iterable[np.ndarray], sequence_length: int):
    """Chunk a frame iterator into lists of `sequence_length` frames, last partial chunk kept — tracker.py:290-312."""
    chunk = []
    for frame in generator:
        chunk.append(frame)
        if len(chunk) == sequence_length:
            yield chunk
            chunk = []
    if chunk:
        yield chunk


class Tracker(ABC):
    batch_size: int
    # How TrackingRunner drives the tracker:
    #   "ball"   -- windows streamed through BallTracker's device pipeline (stream_begin / stream_push_async)
    #   "detect" -- detect_sample_async(batch), then postprocess(results, frame_hw), the order-dependent host stage
    #   "fixed"  -- `fixed_detection` repeated for every frame
    #   "frames" -- predict_and_update only
    stage: str = "frames"
    fixed_detection: Optional[Object] = None

    def __init__(self, load_path: Optional[str | Path] = None, save_path: Optional[str | Path] = None) -> None:
        self.results = TrackingResults()
        self.load_path = load_path
        self.save_path = save_path
        self.load_predictions()  # tracker.py:141-146 (ctor order kept, SURVEY App. E q9)

    @abstractmethod
    def video_info_post_init(self, video_info) -> "Tracker": ...

    @abstractmethod
    def object(self) -> Type[Object]: ...

    @abstractmethod
    def draw_kwargs(self) -> dict: ...

    @property
    def DEVICE(self) -> str:  # tracker.py:172-174
        return "cuda" if torch.cuda.is_available() else "cpu"

    @abstractmethod
    def restart(self) -> None: ...

    def __len__(self) -> int:
        return len(self.results)

    @abstractmethod
    def __str__(self) -> str: ...

    def save_predictions(self) -> None:  # tracker.py:200-220
        if self.save_path:
            with open(self.save_path, "w") as f:
                json.dump([o.serialize() for o in self.results.predictions], f)
            print(f"{self}: {len(self)} predictions saved.")

    def load_predictions(self) -> None:  # tracker.py:222-241
        if self.load_path:
            with open(self.load_path, "r") as f:
                raw = json.load(f)
            self.results.load([self.object().from_json(o) for o in raw])
        print(f"{self}: {len(self)} predictions loaded.")

    def to(self, device: str) -> None:
        pass

    def detect_sample(self, sample):
        """A "detect" tracker's model stage on one sample: the engine's raw results, no sequential state."""
        return self.detect_sample_async(sample)()

    @abstractmethod
    def predict_sample(self, sample: Iterable[np.ndarray], **kwargs): ...

    @abstractmethod
    def predict_frames(self, frame_generator: Iterable[np.ndarray], **kwargs): ...

    def predict_and_update(self, frame_generator: Iterable[np.ndarray], **kwargs) -> TrackingResults:
        """tracker.py:280-330: try predict_frames on the whole generator, else batch through predict_sample."""
        try:
            self.results.predictions = self.predict_frames(frame_generator, **kwargs)
        except NoPredictFrames:
            for sample in sampler(frame_generator, self.batch_size):
                self.results.update(self.predict_sample(sample, **kwargs))
        print(f"{self}: {len(self.results)} predictions.")
        return self.results
