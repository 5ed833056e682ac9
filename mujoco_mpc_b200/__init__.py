"""H100-native (sm_90a) rollout engine behind MJPC's planner/task surface (see DESIGN.md)."""
__version__ = "0.1.0"
