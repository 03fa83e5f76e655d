"""Object sharding of ONE video stream over the ranks of a process group (SURVEY.md section 8(e).2, DESIGN.md section 6.2).

Every rank runs the image encoder, the key projection, the memory keys, top-k, usage and long-term maintenance for all
objects (replicated); each object's value arrays, sensory state, object summaries, pixel fusion, object transformer,
decoder and mask encoder run on the one rank that owns it.  Two kinds of per-frame exchange couple the objects: the
foreground test of the object transformer and the tail of `CUTIE.segment` both aggregate over all objects, so the
owners all-gather their logits first (`ObjectGroup.gather`).

Ownership is a function of the sequence of add / delete calls alone, so every rank holds the same table without
communicating: a new object goes to the rank that owns the fewest live objects (ties: the lowest rank) and never moves;
deleting it frees the slot.
"""
from typing import Dict, List, Sequence

import torch
import torch.distributed as dist


class ObjectShards:
    """Which rank of `group` owns each live object (by object id)."""

    def __init__(self, group):
        self.group = group
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.owner: Dict[int, int] = {}
        self._groups: Dict[tuple, 'ObjectGroup'] = {}

    def add(self, obj_ids: Sequence[int]) -> None:
        """Place every object of `obj_ids` (in that order) that has no owner yet."""
        for o in obj_ids:
            if o not in self.owner:
                load = [0] * self.world
                for r in self.owner.values():
                    load[r] += 1
                self.owner[o] = load.index(min(load))
                self._groups.clear()

    def retain(self, live_ids: Sequence[int]) -> None:
        """Forget the objects not in `live_ids` (deleted objects free their slots)."""
        live = set(live_ids)
        if any(o not in live for o in self.owner):
            self.owner = {o: r for o, r in self.owner.items() if o in live}
            self._groups.clear()

    def local(self, obj_ids: Sequence[int]) -> List[int]:
        """The objects of `obj_ids` this rank owns, in the order of `obj_ids`."""
        return [o for o in obj_ids if self.owner[o] == self.rank]

    def group_of(self, obj_ids: Sequence[int]) -> 'ObjectGroup':
        """The exchange over the objects `obj_ids` (tmp-id order: the order of the object axis of the full tensors)."""
        key = tuple(obj_ids)
        g = self._groups.get(key)
        if g is None:
            g = self._groups[key] = ObjectGroup(self, key)
        return g

    def broadcast(self, tensors: Sequence[torch.Tensor]) -> List[torch.Tensor]:
        """Rank 0's copy of `tensors` (same shapes on every rank, concatenated along dim 1 for one collective)."""
        buf = torch.cat(list(tensors), dim=1)
        dist.broadcast(buf, group=self.group, group_src=0)
        return [t.contiguous() for t in buf.split([t.shape[1] for t in tensors], dim=1)]


class ObjectGroup:
    """One object list and its all-gather: every rank contributes the rows of the objects it owns (in list order) and
    receives the full list's rows, padded to the largest local count on the wire."""

    def __init__(self, shards: ObjectShards, obj_ids: tuple):
        self.shards = shards
        self.ids = list(obj_ids)
        owner = [shards.owner[o] for o in self.ids]
        self.positions = [j for j, r in enumerate(owner) if r == shards.rank]
        self.local_ids = [self.ids[j] for j in self.positions]
        counts = [owner.count(r) for r in range(shards.world)]
        self.pad = max(counts)
        seen = [0] * shards.world
        self._order = []                     # row of the gathered [world * pad] block that holds list entry j
        for r in owner:
            self._order.append(r * self.pad + seen[r])
            seen[r] += 1
        self._dev = {}

    def positions_tensor(self, device) -> torch.Tensor:
        """int32 positions of this rank's objects in the list (kernels.qt_aux_fg)."""
        t = self._dev.get(('pos', device))
        if t is None:
            t = self._dev[('pos', device)] = torch.tensor(self.positions, dtype=torch.int32, device=device)
        return t

    def gather(self, x_local: torch.Tensor) -> torch.Tensor:
        """x_local [B, len(local_ids), ...] -> [B, len(ids), ...], identical on every rank."""
        B, n, *rest = x_local.shape
        assert n == len(self.local_ids)
        world, dev = self.shards.world, x_local.device
        send = x_local.new_zeros(B, self.pad, *rest)
        send[:, :n] = x_local
        recv = x_local.new_empty(world * B, self.pad, *rest)
        dist.all_gather_into_tensor(recv, send, group=self.shards.group)
        order = self._dev.get(('order', dev))
        if order is None:
            order = self._dev[('order', dev)] = torch.tensor(self._order, dtype=torch.int64, device=dev)
        rows = recv.view(world, B, self.pad, *rest).transpose(0, 1).reshape(B, world * self.pad, *rest)
        return rows.index_select(1, order)
