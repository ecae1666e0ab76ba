"""Court projection and data collection of the render pass: the API of the reference's analytics/projected_court.py
(ProjectedCourt :201-668) and analytics/data_analytics.py (DataAnalytics :87-302), restated.

`ProjectedCourt` holds the mini-court geometry drawn in the top-right corner of every rendered frame, the homography
that maps frame pixels onto it, and the per-frame homography update policy.  `DataAnalytics` collects the players'
projected positions (metres, origin at the middle of the court) frame by frame and derives distance, velocity and
acceleration tables from them.

Documented deviations from reference quirks:
  q8  `DataPoint.validate` deletes players whose id is not 1-4 by their index in a copy of the list, so with two or
      more such players it deletes the wrong ones or raises IndexError.  ByteTrack ids grow past 4 whenever a track is
      lost and found again, so here every such player is dropped and the others kept, which is what the reference
      does whenever it has at most one of them.
  No per-frame prints ("player/s missing", "Missing data for players projection", ...).
"""
from __future__ import annotations

import copy
from dataclasses import dataclass
from typing import Optional

import numpy as np

# court dimensions in metres (the reference's constants/court_dimensions.py)
BASE_LINE = 10
SIDE_LINE = 20
SERVICE_SIDE_LINE = 3
NET_SIDE_LINE = 10


class InconsistentPredictedKeypoints(Exception):
    pass


class InvalidDataPoint(Exception):
    pass


def meters_to_pixels(meters: float, reference_in_meters: float, reference_in_pixels: int) -> int:
    return int(meters * reference_in_pixels / reference_in_meters)


def pixels_to_meters(pixels: float, reference_in_meters: float, reference_in_pixels: int) -> float:
    return pixels * reference_in_meters / reference_in_pixels


@dataclass
class Rectangle:
    top_left: tuple[int, int]
    bottom_right: tuple[int, int]

    @property
    def width(self) -> int:
        return self.bottom_right[0] - self.top_left[0]

    @property
    def height(self) -> int:
        return self.bottom_right[1] - self.top_left[1]


class ProjectedCourtKeypoints:
    """The 12 mini-court points (k1 bottom-left ... k12 top-right, rows k1-k2 base line, k3-k5 service line, k6-k7 net,
    k8-k10 service line, k11-k12 base line) and the origin used for positions in metres (the middle of k6-k7)."""

    NAMES = tuple(f"k{i}" for i in range(1, 13))
    EXTRA = {18: ("k1", "k2", "k6", "k7", "k11", "k12"),
             22: ("k1", "k2", "k3", "k5", "k6", "k7", "k8", "k10", "k11", "k12")}

    def __init__(self, points: dict[str, tuple[int, int]]):
        self.points = dict(points)
        k6, k7 = self.points["k6"], self.points["k7"]
        self.origin = (k6[0] + int((k7[0] - k6[0]) / 2), k6[1] + int((k7[1] - k6[1]) / 2))

    def __getattr__(self, name):
        points = self.__dict__.get("points")
        if points is not None and name in points:
            return points[name]
        raise AttributeError(name)

    @property
    def width(self) -> int:
        return self.k7[0] - self.k6[0]

    @property
    def height(self) -> int:
        return self.k1[1] - self.k11[1]

    def keypoints_xy(self, number_keypoints: int) -> np.ndarray:
        """(n, 2) float64 destination points of the homography: k1..k12, then the repeated points of the 18- and
        22-keypoint layouts."""
        names = list(self.NAMES) + list(self.EXTRA.get(number_keypoints, ()))
        return np.array([[float(v) for v in self.points[n]] for n in names])

    def draw_points(self) -> list[tuple[tuple[int, int], tuple[int, int, int]]]:
        """(centre, RGB colour) of the circles drawn on the mini court: the 12 points red, then the origin green."""
        return [(self.points[n], (255, 0, 0)) for n in self.NAMES] + [(self.origin, (0, 255, 0))]

    def lines(self) -> list[tuple[tuple[int, int], tuple[int, int]]]:
        p = self.points
        return [(p["k1"], p["k2"]), (p["k3"], p["k5"]), (p["k6"], p["k7"]), (p["k8"], p["k10"]),
                (p["k11"], p["k12"]), (p["k1"], p["k11"]), (p["k4"], p["k9"]), (p["k2"], p["k12"])]

    def shift_point_origin(self, point: tuple[float, float], dimension: str) -> tuple[float, float]:
        """`point` relative to the origin, in pixels or (dimension="meters") in metres along the base line scale."""
        shifted = [float(point[0] - self.origin[0]), float(point[1] - self.origin[1])]
        if dimension == "meters":
            shifted = [pixels_to_meters(v, BASE_LINE, self.width) for v in shifted]
        return tuple(shifted)


class ProjectedCourt:
    """The mini court of the rendered video and the homography onto it (projected_court.py:201-668)."""

    WIDTH_MULTIPLIER = 0.14
    HEIGHT_MULTIPLIER = 0.47
    BUFFER = 50
    PADDING = 20
    ALPHA = 0.5

    def __init__(self, video_info):
        self.video_info = video_info
        self.WIDTH = int(self.WIDTH_MULTIPLIER * video_info.width)
        self.HEIGHT = int(self.HEIGHT_MULTIPLIER * video_info.height)
        # background: a WIDTH x HEIGHT box BUFFER pixels from the top-right corner
        end_x, end_y = video_info.width - self.BUFFER, self.BUFFER + self.HEIGHT
        self.background_position = Rectangle((int(end_x - self.WIDTH), int(end_y - self.HEIGHT)),
                                             (int(end_x), int(end_y)))
        # court: PADDING inside the background, height from the court's aspect ratio
        x0 = self.background_position.top_left[0] + self.PADDING
        y0 = self.background_position.top_left[1] + self.PADDING
        x1 = self.background_position.bottom_right[0] - self.PADDING
        y1 = y0 + meters_to_pixels(SIDE_LINE, BASE_LINE, x1 - x0)
        self.court_position = Rectangle((int(x0), int(y0)), (int(x1), int(y1)))
        c = self.court_position
        service = meters_to_pixels(SERVICE_SIDE_LINE, BASE_LINE, c.width)
        mid_x = int(c.top_left[0] + c.width / 2)
        mid_y = int(c.top_left[1] + c.height / 2)
        (left, top), (right, bottom) = c.top_left, c.bottom_right
        self.court_keypoints = ProjectedCourtKeypoints({
            "k1": (left, bottom), "k2": (right, bottom),
            "k3": (left, bottom - service), "k4": (mid_x, bottom - service), "k5": (right, bottom - service),
            "k6": (left, mid_y), "k7": (right, mid_y),
            "k8": (left, top + service), "k9": (mid_x, top + service), "k10": (right, top + service),
            "k11": (left, top), "k12": (right, top)})
        self.H = None

    # ---- homography ----------------------------------------------------------------------------------------------
    def homography_matrix(self, keypoints_detection) -> np.ndarray:
        """cv2.findHomography from the detected court keypoints (in id order) to the mini-court points."""
        import cv2

        kps = keypoints_detection.keypoints
        if len(kps) not in (12, 18, 22):
            raise ValueError("Unhandled number of keypoints detected")
        src = np.array([k.xy for k in kps])
        dst = self.court_keypoints.keypoints_xy(len(kps))
        if src.shape != dst.shape:
            raise InconsistentPredictedKeypoints("Don't have enough source points")
        H, _ = cv2.findHomography(src, dst)
        return H

    def update_homography(self, keypoints_detection, is_fixed_keypoints: bool) -> Optional[np.ndarray]:
        """The per-frame policy of projected_court.py:633-647: computed on the first frame with keypoints; after that
        kept as is when the keypoints are fixed, else recomputed every frame and None on a frame without keypoints."""
        if self.H is None:
            if keypoints_detection:
                self.H = self.homography_matrix(keypoints_detection)
        elif not is_fixed_keypoints:
            self.H = self.homography_matrix(keypoints_detection) if keypoints_detection else None
        return self.H

    @staticmethod
    def project_point(point, homography_matrix: np.ndarray) -> tuple[float, float]:
        assert homography_matrix.shape == (3, 3)
        src = np.array([float(point[0]), float(point[1]), 1.0])
        dst = np.matmul(homography_matrix, src)
        dst = dst / dst[2]
        return dst[0], dst[1]

    def project_players(self, players_detection, homography_matrix: np.ndarray,
                        data_analytics: Optional["DataAnalytics"] = None) -> list:
        """Copies of the players with `projection` set (the tracker's results are left alone); each position is
        recorded in `data_analytics` in metres."""
        out = []
        for player in players_detection:
            p = copy.copy(player)
            p.projection = tuple(int(v) for v in self.project_point(player.feet, homography_matrix))
            if data_analytics is not None:
                pos = self.court_keypoints.shift_point_origin(tuple(float(v) for v in p.projection), "meters")
                data_analytics.add_player_position(id=p.id, position=pos)
            out.append(p)
        return out

    def project_ball(self, ball_detection, homography_matrix: np.ndarray):
        b = copy.copy(ball_detection)
        b.projection = tuple(int(v) for v in self.project_point(ball_detection.asint(), homography_matrix))
        return b

    # ---- drawing on a host frame (RGB, as the reference draws) ---------------------------------------------------
    def blend_lut(self) -> np.ndarray:
        """The background blend as a byte table: cv2.addWeighted(v, ALPHA, 255, 1 - ALPHA, 0) for every v."""
        import cv2

        v = np.arange(256, dtype=np.uint8).reshape(1, 256)
        return cv2.addWeighted(v, self.ALPHA, np.full_like(v, 255), 1 - self.ALPHA, 0).reshape(256)

    def draw_background_single_frame(self, frame: np.ndarray) -> np.ndarray:
        """A copy of `frame` with the background box blended halfway to white."""
        import cv2

        shapes = np.zeros_like(frame, np.uint8)
        cv2.rectangle(shapes, self.background_position.top_left, self.background_position.bottom_right,
                      (255, 255, 255), -1)
        out = frame.copy()
        mask = shapes.astype(bool)
        out[mask] = cv2.addWeighted(out, self.ALPHA, shapes, 1 - self.ALPHA, 0)[mask]
        return out

    def draw_projected_court_single_frame(self, frame: np.ndarray) -> np.ndarray:
        import cv2

        for centre, colour in self.court_keypoints.draw_points():
            cv2.circle(frame, centre, 5, colour, -1)
        for a, b in self.court_keypoints.lines():
            cv2.line(frame, a, b, (0, 0, 0), 2)
        return frame

    def draw_projections_and_collect_data(self, frame: np.ndarray, keypoints_detection, players_detection,
                                          ball_detection, data_analytics: Optional["DataAnalytics"] = None,
                                          is_fixed_keypoints: bool = False):
        """projected_court.py:608-668 on a host RGB frame: background, mini court, homography update, projected
        players (recorded in `data_analytics`) and ball.  Returns (frame, data_analytics)."""
        out = self.draw_projected_court_single_frame(self.draw_background_single_frame(frame))
        H = self.update_homography(keypoints_detection, is_fixed_keypoints)
        if H is not None and players_detection:
            for p in self.project_players(players_detection, H, data_analytics):
                out = p.draw_projection(out)
        if H is not None and ball_detection:
            out = self.project_ball(ball_detection, H).draw_projection(out)
        return out, data_analytics


# ---- data collection ---------------------------------------------------------------------------------------------
@dataclass
class PlayerPosition:
    id: int
    position: tuple[float, float]

    @property
    def key(self) -> str:
        return f"player{self.id}"


@dataclass
class DataPoint:
    frame: Optional[int] = None
    players_position: Optional[list[PlayerPosition]] = None

    def validate(self) -> None:
        if self.frame is None:
            raise InvalidDataPoint("Unknown frame")
        if self.players_position is None:
            return
        self.players_position = [p for p in self.players_position if p.id in (1, 2, 3, 4)]  # q8
        ids = [p.id for p in self.players_position]
        if len(ids) != len(set(ids)):
            raise InvalidDataPoint("N-plicate player id")

    def add_player_position(self, player_position: PlayerPosition) -> None:
        if self.players_position is None:
            self.players_position = [player_position]
        else:
            self.players_position.append(player_position)

    def sort_players_position(self) -> Optional[list[PlayerPosition]]:
        return sorted(self.players_position, key=lambda p: p.id) if self.players_position else None


class DataAnalytics:
    """Per-frame player positions (data_analytics.py:87-302).  `frames` starts as [0]; every `step` closes the current
    data point and opens the next frame's."""

    PLAYER_IDS = (1, 2, 3, 4)
    FRAME_INTERVALS = (1, 2, 3, 4)

    def __init__(self):
        self.frames = [0]
        self.current_datapoint = DataPoint(frame=self.frames[-1])
        self.datapoints: list[DataPoint] = []

    def restart(self) -> None:
        self.__init__()

    def __len__(self) -> int:
        return len(self.frames)

    def step(self, x: int = 1) -> None:
        new_frame = self.frames[-1] + 1
        assert new_frame not in self.frames
        self.frames.append(new_frame)
        self.current_datapoint.validate()
        self.datapoints.append(self.current_datapoint)
        self.current_datapoint = DataPoint(frame=self.frames[-1])

    def add_player_position(self, id: int, position: tuple[float, float]) -> None:
        self.current_datapoint.add_player_position(PlayerPosition(id=id, position=position))

    @classmethod
    def from_dict(cls, data: dict) -> "DataAnalytics":
        inst = cls()
        inst.frames = data["frame"]
        inst.datapoints = []
        for i, frame in enumerate(data["frame"]):
            pos = [PlayerPosition(id=p, position=(data[f"player{p}_x"][i], data[f"player{p}_y"][i]))
                   for p in cls.PLAYER_IDS
                   if data[f"player{p}_x"][i] is not None and data[f"player{p}_y"][i] is not None]
            inst.datapoints.append(DataPoint(frame=frame, players_position=pos or None))
        inst.current_datapoint = None
        return inst

    def into_dict(self) -> dict[str, list]:
        """{"frame": [...], "player{i}_x" / "player{i}_y": [...]} with None where a player is missing."""
        data = {"frame": []}
        for p in self.PLAYER_IDS:
            data[f"player{p}_x"], data[f"player{p}_y"] = [], []
        for dp in self.datapoints:
            data["frame"].append(dp.frame)
            have = {pp.id: pp.position for pp in (dp.sort_players_position() or [])}
            for p in self.PLAYER_IDS:
                xy = have.get(p)
                data[f"player{p}_x"].append(None if xy is None else xy[0])
                data[f"player{p}_y"].append(None if xy is None else xy[1])
        return data

    def into_dataframe(self, fps: float):
        """The positions plus, per frame interval k in 1..4: delta_time{k}; per player and axis the displacement
        delta{x,y}{k}, velocity V{x,y}{k}, velocity change deltaV{x,y}{k} and acceleration A{x,y}{k}; per player the
        distance moved since the previous frame and the velocity and acceleration norms Vnorm{k}, Anorm{k}."""
        import warnings

        import pandas as pd

        with warnings.catch_warnings():  # column by column on purpose: the reference's column order
            warnings.simplefilter("ignore", pd.errors.PerformanceWarning)
            return self._dataframe(pd.DataFrame(self.into_dict()), fps)

    def _dataframe(self, df, fps: float):
        for p in self.PLAYER_IDS:  # a player never seen is an all-None column: make it NaN like a partial one
            for ax in "xy":
                df[f"player{p}_{ax}"] = df[f"player{p}_{ax}"].astype("float64")
        df["time"] = df["frame"] * (1 / fps)

        def norm(a, b):
            return np.sqrt(a ** 2 + b ** 2)

        for k in self.FRAME_INTERVALS:
            dt = df["time"].diff(k)
            df[f"delta_time{k}"] = dt
            for p in self.PLAYER_IDS:
                pre = f"player{p}_"
                for ax in "xy":
                    d = df[f"{pre}{ax}"].diff(k)
                    df[f"{pre}delta{ax}{k}"] = d
                    v = d / dt
                    df[f"{pre}V{ax}{k}"] = v
                    dv = v.diff(k)
                    df[f"{pre}deltaV{ax}{k}"] = dv
                    df[f"{pre}A{ax}{k}"] = dv / dt
                df[f"{pre}distance"] = norm(df[f"{pre}deltax1"], df[f"{pre}deltay1"])
                df[f"{pre}Vnorm{k}"] = norm(df[f"{pre}Vx{k}"], df[f"{pre}Vy{k}"])
                df[f"{pre}Anorm{k}"] = norm(df[f"{pre}Ax{k}"], df[f"{pre}Ay{k}"])
        return df
