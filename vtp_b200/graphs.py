"""Capture, replay and release of every CUDA graph in the package (model entry points, training and evaluation steps)."""
import torch

from . import lib


class StepGraph:
    """One CUDA graph of a function that reads and writes only static device buffers.  A replay adds the kernels of ours
    captured in it to `lib.LAUNCHES`, as an eager call of the function does."""

    def __init__(self, device, enabled: bool = True):
        self.device, self.enabled = torch.device(device), enabled
        self.graph, self.launches, self.calls = None, 0, 0

    def capture(self, fn, warmup: int = 0):
        """`warmup` real calls of fn on a side stream, then one call captured without executing; returns its result."""
        cur = torch.cuda.current_stream(self.device)
        side = torch.cuda.Stream(self.device)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            for _ in range(warmup):
                fn()
        cur.wait_stream(side)
        torch.cuda.synchronize(self.device)
        l0 = lib.LAUNCHES
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = fn()
        self.graph, self.launches = graph, lib.LAUNCHES - l0
        return out

    def replay(self) -> None:
        self.graph.replay()
        lib.LAUNCHES += self.launches

    def __call__(self, fn) -> None:
        """First call eager, second captured; every call from the second on replays.  Only the capture synchronises."""
        self.calls += 1
        if self.graph is None and (not self.enabled or self.calls == 1):
            return fn()
        if self.graph is None:
            self.capture(fn)
        self.replay()

    def release(self) -> None:
        """Wait for the device and destroy the graph (NCCL communicators it captured can be torn down afterwards)."""
        if self.graph is not None:
            torch.cuda.synchronize(self.device)
            self.graph.reset()
            self.graph = None
