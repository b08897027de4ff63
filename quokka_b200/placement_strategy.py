"""Where an operator's channels live.  The names and constructor arguments are the reference's
(pyquokka/placement_strategy.py), because user code passes them to `stateful_transform` and
`TaskGraph.new_*_node`; the meaning is re-mapped onto GPUs: a "node" is one rank (one GPU), and every
strategy answers one question for the SPMD driver -- `owners(world_size)`: which ranks own a channel."""
from __future__ import annotations

from dataclasses import dataclass


class PlacementStrategy:
    def owners(self, world_size: int) -> list:
        """Ranks that own a channel of the operator (the kernels use a whole GPU, so one channel per rank)."""
        return list(range(world_size))

    @property
    def single(self) -> bool:
        return False


class SingleChannelStrategy(PlacementStrategy):
    """Exactly one channel, on rank 0: final ungrouped aggregates, top-k."""

    def owners(self, world_size: int) -> list:
        return [0]

    @property
    def single(self) -> bool:
        return True


@dataclass
class CustomChannelsStrategy(PlacementStrategy):
    channels_per_node: int = 1        # accepted for compatibility; > 1 is folded into the one channel per GPU

    def __init__(self, channels) -> None:
        if int(channels) < 1:
            raise ValueError("channels must be >= 1")
        self.channels_per_node = int(channels)


@dataclass
class DatasetStrategy(PlacementStrategy):
    total_channels: int = 1

    def __init__(self, total_channels) -> None:
        self.total_channels = int(total_channels)

    def owners(self, world_size: int) -> list:
        return list(range(min(world_size, max(1, self.total_channels))))


@dataclass
class TaggedCustomChannelsStrategy(CustomChannelsStrategy):
    tag: str = ""

    def __init__(self, channels, tag) -> None:
        super().__init__(channels)
        self.tag = tag
