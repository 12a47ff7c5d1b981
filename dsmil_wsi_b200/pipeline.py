"""Host-buffer front end: bags that live in (pinned) HOST memory are streamed through the GPU
aggregator with copies overlapped with compute (two device slots, a copy stream and the compute
stream, CUDA events between them).  This is the call an inference caller makes when features come
off disk (train_tcga.py:62 loads every bag from a .pt file to the GPU; attention_map.py:80-85 stacks
features on the host) -- and it is what bench.py times as the end-to-end (`e2e`) number.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import torch


class HostBagPipeline:
    def __init__(self, milnet, max_rows: int, feature_size: int, num_classes: int, depth: int = 4,
                 device: torch.device | None = None, copy_streams: int = 2):
        self.net = milnet.eval()
        self.dev = device or next(milnet.parameters()).device
        if self.dev.type != "cuda":
            raise RuntimeError("HostBagPipeline needs the model on a CUDA device (no CPU path)")
        self.depth = depth
        self.D, self.C = feature_size, num_classes
        with torch.cuda.device(self.dev):
            self.slots = [torch.empty(max_rows, feature_size, dtype=torch.float32, device=self.dev)
                          for _ in range(depth)]
            # two H2D streams, four slots: consecutive bags are in flight on two copy engines (the host link is the bound)
            self.copy_streams = [torch.cuda.Stream(device=self.dev) for _ in range(max(1, copy_streams))]
            self.h2d_done = [torch.cuda.Event() for _ in range(depth)]
            self.slot_free = [torch.cuda.Event() for _ in range(depth)]
        # pinned result staging (classes, pred, A, B per bag), grown on demand
        self._host_out: List[Tuple[torch.Tensor, ...]] = []

    def _host_result(self, i: int, N: int):
        while len(self._host_out) <= i:
            self._host_out.append(())
        cur = self._host_out[i]
        if not cur or cur[0].shape[0] < N:
            pin = lambda *s: torch.empty(*s, dtype=torch.float32).pin_memory()
            cur = (pin(N, self.C), pin(1, self.C), pin(N, self.C), pin(1, self.C, self.D))
            self._host_out[i] = cur
        return cur

    @torch.no_grad()
    def run(self, host_bags: Sequence[torch.Tensor]):
        """host_bags: CPU fp32 [N_i, D] tensors (pinned for full overlap).  Returns per bag
        (classes, prediction_bag, A, B) as HOST tensors; synchronises once at the end.

        The returned tensors are VIEWS of this pipeline's pinned result buffers, which the next `run()` overwrites
        (asynchronously): consume or `.clone()` them before calling `run()` again."""
        results = []
        with torch.cuda.device(self.dev):
            compute = torch.cuda.current_stream()
            for s in range(self.depth):
                self.slot_free[s].record(compute)
            for i, hb in enumerate(host_bags):
                s = i % self.depth
                N = hb.shape[0]
                cs = self.copy_streams[i % len(self.copy_streams)]
                with torch.cuda.stream(cs):
                    cs.wait_event(self.slot_free[s])                        # slot drained by its last forward
                    self.slots[s][:N].copy_(hb, non_blocking=True)
                    self.h2d_done[s].record(cs)
                compute.wait_event(self.h2d_done[s])
                classes, pred, A, B = self.net(self.slots[s][:N])
                self.slot_free[s].record(compute)
                hc, hp, hA, hB = self._host_result(i, N)
                hc[:N].copy_(classes, non_blocking=True)
                hp.copy_(pred, non_blocking=True)
                hA[:N].copy_(A, non_blocking=True)
                hB.copy_(B, non_blocking=True)
                results.append((hc[:N], hp, hA[:N], hB))
            compute.synchronize()
        return results

    def bytes_per_bag(self, N: int) -> Tuple[int, int]:
        """(h2d, d2h) bytes moved for one bag of N rows."""
        return 4 * N * self.D, 4 * (2 * N * self.C + self.C + self.C * self.D)
