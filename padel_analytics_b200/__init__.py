"""padel_analytics_b200 — H100-native (sm_90a) inference engine for the padel_analytics tracker hot path."""
__version__ = "0.1.0"
