"""tensorlink_b200 — H100-native shard executor behind tensorlink's DistributedModel API."""
__version__ = "0.1.0"
