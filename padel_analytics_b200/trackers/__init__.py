"""Drop-in tracker classes (same names / constructor arguments / results API as /root/reference/trackers/__init__.py:1-6)
whose model forwards run on the CUDA engine."""
from .players_tracker import Player, Players, PlayerTracker
from .ball_tracker import Ball, BallTracker
from .keypoints_tracker import Keypoint, Keypoints, KeypointsTracker
from .players_keypoints_tracker import PlayerKeypoint, PlayerKeypoints, PlayersKeypoints, PlayerKeypointsTracker
from .tracker import NoPredictFrames, NoPredictSample, Object, Tracker, TrackingResults
from .runner import TrackingRunner

__all__ = ["Player", "Players", "PlayerTracker", "Ball", "BallTracker", "Keypoint", "Keypoints", "KeypointsTracker",
           "PlayerKeypoint", "PlayerKeypoints", "PlayersKeypoints", "PlayerKeypointsTracker", "TrackingRunner",
           "Tracker", "TrackingResults", "Object", "NoPredictFrames", "NoPredictSample"]
