"""Peer-mapped memory windows -- the H100-native replacement of the reference's MPI RMA window
(MPI_Alloc_mem + MPI_Win_create, /root/reference/dmnist/event/event.cpp:170-179).

Every rank owns one device slab with an identical layout on all ranks (so "the same offset in
my neighbour's slab" is the reference's `target_disp`).  Slabs are exported with CUDA IPC
(native runtime: csrc/ipc.cu), the 64-byte handles are exchanged once through the process
group, and each rank maps its peers' slabs.  A kernel-side `st.global` to a mapped address is
the `MPI_Put`: it crosses NVLink 4 / NVSwitch directly into the peer's HBM.

Two bootstraps implement the same interface:
  DistBootstrap   one process per GPU (torchrun); handles travel via all_gather_object
  LocalBootstrap  R virtual ranks inside ONE process on ONE GPU (peer pointer == the other
                  virtual rank's local pointer).  Used by the single-GPU tests to exercise the
                  complete cross-rank protocol (flags, acks, pushes) without torchrun.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch

class _RawCuda:
    """Minimal __cuda_array_interface__ holder so torch can alias raw device memory."""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1",
                                         "data": (ptr, False), "version": 2}


def tensor_from_ptr(ptr: int, nbytes: int, device: torch.device) -> torch.Tensor:
    """uint8 tensor aliasing [ptr, ptr+nbytes) on `device` (no copy, no ownership)."""
    t = torch.as_tensor(_RawCuda(ptr, nbytes), device=device)
    assert t.data_ptr() == ptr, "as_tensor copied instead of aliasing"
    return t


class Layout:
    """Named, 256-byte aligned sections inside a slab."""

    def __init__(self):
        self.sections: Dict[str, Tuple[int, int]] = {}
        self.size = 0

    def add(self, name: str, nbytes: int) -> None:
        off = (self.size + 255) // 256 * 256
        self.sections[name] = (off, nbytes)
        self.size = off + nbytes

    def offset(self, name: str) -> int:
        return self.sections[name][0]

    def nbytes(self, name: str) -> int:
        return self.sections[name][1]


class Window:
    """One rank's slab + the mapped views of its peers."""

    def __init__(self, layout: Layout, rank: int, world: int, device: torch.device):
        from ..ops import ext
        self._C = ext()
        self.layout, self.rank, self.world, self.device = layout, rank, world, device
        with torch.cuda.device(device):
            self.ptr, self.handle = self._C.ipc_alloc(max(256, layout.size))
        self.raw = tensor_from_ptr(self.ptr, max(256, layout.size), device)
        self.peer_ptrs: List[int] = [0] * world
        self.peer_ptrs[rank] = self.ptr
        self._opened: List[int] = []
        self._closed = False

    # ---- local views ------------------------------------------------------------------
    def view(self, name: str, dtype: torch.dtype) -> torch.Tensor:
        off, nb = self.layout.sections[name]
        return self.raw[off: off + nb].view(dtype)

    def addr(self, name: str, rank: Optional[int] = None) -> int:
        base = self.ptr if rank is None else self.peer_ptrs[rank]
        if base == 0:
            raise RuntimeError(f"peer {rank} not mapped")
        return base + self.layout.offset(name)

    # ---- mapping ----------------------------------------------------------------------
    def connect_handles(self, handles: List[bytes]) -> None:
        with torch.cuda.device(self.device):
            for r, h in enumerate(handles):
                if r == self.rank:
                    continue
                try:
                    p = self._C.ipc_open(h)
                except RuntimeError as e:
                    raise RuntimeError(
                        f"rank {self.rank}: cannot map the window of rank {r} ({e}). The p2p backend needs "
                        "CUDA IPC + peer access between all GPUs of the node (NVLink/NVSwitch or PCIe P2P, one "
                        "process per GPU in the same IPC namespace); use --backend nccl otherwise.") from e
                self.peer_ptrs[r] = p
                self._opened.append(p)

    def connect_local(self, ptrs: List[int]) -> None:
        for r, p in enumerate(ptrs):
            self.peer_ptrs[r] = p

    def close(self) -> None:
        if self._closed:
            return
        self._closed = True
        try:
            torch.cuda.synchronize(self.device)
            with torch.cuda.device(self.device):
                for p in self._opened:
                    self._C.ipc_close(p)
                self.raw = None
                self._C.ipc_free(self.ptr)
        except Exception:
            pass


class SymmWindow(Window):
    """EXPERIMENTAL (EGB_NVLS=1): the slab lives in torch symmetric memory instead of cudaMalloc + CUDA IPC.
    The rendezvous maps every peer's slab (same role as the IPC handles) AND, on NVSwitch systems, a
    MULTICAST address of the slab: a `multimem.ld_reduce` on it is reduced inside the switch and a
    `multimem.st` is delivered to all ranks -- the NVLS path of csrc/allreduce_nvls.cu.  Everything else
    (layout, views, peer addresses) is identical to `Window`, so all other kernels run unchanged."""

    def __init__(self, layout: Layout, rank: int, world: int, device: torch.device):
        import torch.distributed._symmetric_memory as symm
        from ..ops import ext
        self._C = ext()
        self.layout, self.rank, self.world, self.device = layout, rank, world, device
        nbytes = max(256, layout.size)
        self._t = symm.empty(nbytes, dtype=torch.uint8, device=device)
        self._t.zero_()                                   # window starts zeroed, like ipc_alloc
        torch.cuda.synchronize(device)
        self.raw = self._t
        self.ptr = self._t.data_ptr()
        self.handle = None
        self.peer_ptrs: List[int] = [0] * world
        self.peer_ptrs[rank] = self.ptr
        self.mc_ptr = 0
        self._hdl = None
        self._opened: List[int] = []
        self._closed = False

    def rendezvous(self, group=None) -> None:
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm
        group = group if group is not None else dist.group.WORLD
        try:
            symm.enable_symm_mem_for_group(group.group_name)
        except Exception:
            pass                                          # newer torch enables groups implicitly
        hdl = symm.rendezvous(self._t, group)
        ptrs = [int(p) for p in hdl.buffer_ptrs]
        if len(ptrs) != self.world or ptrs[self.rank] != self.ptr:
            raise RuntimeError("symmetric-memory rendezvous returned an unexpected peer table")
        self.peer_ptrs = ptrs
        self.mc_ptr = int(getattr(hdl, "multicast_ptr", 0) or 0)
        self._hdl = hdl

    def mc_addr(self, name: str) -> int:
        """Multicast address of a section (0 when the fabric has no multicast support)."""
        return 0 if not self.mc_ptr else self.mc_ptr + self.layout.offset(name)

    def close(self) -> None:
        if self._closed:
            return
        self._closed = True
        try:
            torch.cuda.synchronize(self.device)
        except Exception:
            pass
        self.raw = self._t = self._hdl = None


def wants_symm_window(env) -> bool:
    import os
    return os.environ.get("EGB_NVLS", "0") == "1" and env.world > 1 and getattr(env, "backend", "") != "local"


class DistBootstrap:
    def __init__(self, env, group=None):
        self.rank, self.world, self.group = env.rank, env.world, group

    def all_gather_object(self, obj):
        if self.world == 1:
            return [obj]
        import torch.distributed as dist
        out = [None] * self.world
        dist.all_gather_object(out, obj, group=self.group)
        return out

    def connect(self, win: Window) -> None:
        if isinstance(win, SymmWindow):
            win.rendezvous(self.group)
        else:
            handles = self.all_gather_object(win.handle)
            win.connect_handles(handles)
        if self.world > 1:
            import torch.distributed as dist
            dist.barrier(group=self.group)

    def barrier(self) -> None:
        if self.world > 1:
            import torch.distributed as dist
            dist.barrier(group=self.group)


class LocalBootstrap:
    """Rendezvous board shared by R virtual ranks living in the same process."""

    def __init__(self, world: int):
        self.world = world
        self.board: Dict[str, Dict[int, object]] = {}

    def for_rank(self, rank: int) -> "_LocalRankView":
        return _LocalRankView(self, rank)


class _LocalRankView:
    def __init__(self, parent: LocalBootstrap, rank: int):
        self.parent, self.rank, self.world = parent, rank, parent.world

    def publish(self, key: str, obj) -> None:
        self.parent.board.setdefault(key, {})[self.rank] = obj

    def collect(self, key: str):
        b = self.parent.board.get(key, {})
        if len(b) != self.world:
            raise RuntimeError(f"local rendezvous '{key}': {len(b)}/{self.world} ranks published")
        return [b[r] for r in range(self.world)]

    def connect(self, win: Window) -> None:
        win.connect_local(self.collect("window_ptr"))

    def barrier(self) -> None:
        pass
