"""KeypointsTracker (court, 12 keypoints) on the CUDA engine — API of
/root/reference/trackers/keypoints_tracker/keypoints_tracker.py (:18-315): model_type="yolo" (YOLOv8-pose, predict_sample),
model_type="resnet" (torchvision ResNet50 regressor :158-167, predict_frames :276-312, input pipeline
keypoints_tracker/iterable.py:10-41) and the fixed-keypoints short-circuit."""
from __future__ import annotations

from pathlib import Path
from typing import Iterable, Optional, Type

import numpy as np

from ..engine.yolo_engine import ResultBlock, YoloEngine
from .tracker import NoPredictFrames, NoPredictSample, Object, Tracker


class Keypoint:
    def __init__(self, id: int, xy: tuple[float, float]):
        self.id = id
        self.xy = xy

    @classmethod
    def from_json(cls, x: dict):
        return cls(**x)

    def serialize(self) -> dict:
        return {"id": self.id, "xy": self.xy}

    def asint(self):
        return tuple(int(v) for v in self.xy)

    def draw(self, frame):
        import cv2

        x, y = self.asint()
        cv2.putText(frame, str(self.id + 1), (x + 5, y - 5), cv2.FONT_HERSHEY_SIMPLEX, 0.4, (255, 255, 255), 1)
        cv2.circle(frame, (x, y), radius=6, color=(255, 0, 0), thickness=-1)
        return frame


class Keypoints(Object):
    def __init__(self, keypoints: list[Keypoint]):
        super().__init__()
        self.keypoints = sorted(keypoints, key=lambda k: k.id)
        self.keypoints_by_id = {k.id: k for k in keypoints}

    @classmethod
    def from_json(cls, x: list[dict]) -> "Keypoints":
        return cls([Keypoint.from_json(k) for k in x])

    def serialize(self) -> list[dict]:
        return [k.serialize() for k in self.keypoints]

    def __len__(self):
        return len(self.keypoints)

    def __iter__(self):
        return iter(self.keypoints)

    def __getitem__(self, id: int) -> Keypoint:
        return self.keypoints_by_id[id]

    def draw(self, frame):
        for k in self.keypoints:
            frame = k.draw(frame)
        return frame


class KeypointsTracker(Tracker):
    NUMBER_KEYPOINTS = 12
    TRAIN_IMAGE_SIZE = 640
    CONF = 0.5
    IOU = 0.7
    POINTS_MAPPER = {0: 10, 1: 11, 2: 1, 3: 0, 4: 7, 5: 9, 6: 8, 7: 5, 8: 6, 9: 2, 10: 4, 11: 3}  # :214-227

    def __init__(self, model_path, batch_size: int, model_type: str = "yolo",
                 fixed_keypoints_detection: Optional[Keypoints] = None, load_path: Optional[str | Path] = None,
                 save_path: Optional[str | Path] = None):
        super().__init__(load_path=load_path, save_path=save_path)
        self.batch_size = batch_size
        self.model_type = model_type
        if model_type == "yolo":
            self.model = YoloEngine(model_path, max_batch=batch_size) if model_path is not None else None
        elif model_type == "resnet":
            # reference: models.resnet50(pretrained=True) with fc -> 24, then load_state_dict(torch.load(model_path))
            # (:158-166); the checkpoint (torchvision key names) is all that is needed here
            import torch

            from ..engine.resnet_engine import ResNet50Engine

            sd = model_path if isinstance(model_path, dict) else torch.load(model_path, map_location="cpu")
            self.model = ResNet50Engine(sd, max_batch=batch_size)
        else:
            raise ValueError("Unknown model type")
        self.fixed_keypoints_detection = fixed_keypoints_detection

    def video_info_post_init(self, video_info) -> "KeypointsTracker":
        return self

    def object(self) -> Type[Object]:
        return Keypoints

    def draw_kwargs(self) -> dict:
        return {}

    def __str__(self) -> str:
        return "keypoints_tracker"

    def restart(self) -> None:
        self.results.restart()

    def to(self, device: str) -> None:
        if self.model is not None:
            self.model.to(device)

    @property
    def stage(self) -> str:
        """The runner stage: "fixed" with a fixed detection, "detect" for a YOLO model, else "frames" (the ResNet
        regressor runs through predict_frames, as the reference's does)."""
        if self.fixed_keypoints_detection is not None:
            return "fixed"
        return "detect" if self.model_type == "yolo" and self.model is not None else "frames"

    @property
    def fixed_detection(self) -> Optional[Keypoints]:
        return self.fixed_keypoints_detection

    def detect_sample_async(self, sample):
        return self.model.predict_frames_async(sample, "pil_square", conf=self.CONF, iou=self.IOU,
                                               imgsz=self.TRAIN_IMAGE_SIZE, classes=None,
                                               max_det=self.NUMBER_KEYPOINTS)

    def postprocess(self, results, frame_hw) -> list[Keypoints]:
        """keypoints_tracker.py:229-260: the reference assumes exactly one court detection (`squeeze(0)`, q5); we take
        the highest-confidence detection (NMS output is score-sorted) and return no keypoints when there is none."""
        ratio_x = frame_hw[1] / self.TRAIN_IMAGE_SIZE
        ratio_y = frame_hw[0] / self.TRAIN_IMAGE_SIZE
        out = []
        if isinstance(results, ResultBlock):  # the same arithmetic over the whole block of frames at once
            top = (results.keypoints[:, 0, :, :2].astype(np.float64) * np.array([ratio_x, ratio_y])).tolist()
            for c, xy in zip(results.counts.tolist(), top):
                out.append(Keypoints([Keypoint(id=self.POINTS_MAPPER[i], xy=(x, y)) for i, (x, y) in enumerate(xy)]
                                     if c else []))
            return out
        for result in results:
            kps = []
            if len(result.keypoints.xy):
                xy = result.keypoints.xy[0].numpy().astype(np.float64) * np.array([ratio_x, ratio_y])
                for i, (x, y) in enumerate(xy.tolist()):
                    kps.append(Keypoint(id=self.POINTS_MAPPER[i], xy=(x, y)))
            out.append(Keypoints(kps))
        return out

    def predict_sample(self, sample: Iterable[np.ndarray], **kwargs) -> list[Keypoints]:
        if self.fixed_keypoints_detection is not None:
            return [self.fixed_keypoints_detection for _ in range(len(sample))]
        if self.model_type != "yolo":
            raise NoPredictSample()
        return self.postprocess(self.detect_sample(sample), sample[0].shape[:2])

    def predict_frames(self, frame_generator, **kwargs):
        if self.fixed_keypoints_detection is not None:
            return [self.fixed_keypoints_detection for _ in frame_generator]
        if self.model_type == "yolo":
            raise NoPredictFrames()
        # ResNet50 regressor (:276-312): batches of frames -> sigmoid outputs (n, 12, 2) in [0,1]^2 -> frame pixels;
        # keypoint ids are the output order (no points_mapper on this branch)
        from .tracker import sampler

        out = []
        for chunk in sampler(frame_generator, self.batch_size):
            h_frame, w_frame = chunk[0].shape[:2]
            p = self.model.predict_frames(chunk).reshape(len(chunk), self.NUMBER_KEYPOINTS, 2)
            for det in p:
                out.append(Keypoints([Keypoint(i, (float(k[0] * w_frame), float(k[1] * h_frame)))
                                      for i, k in enumerate(det)]))
        return out
