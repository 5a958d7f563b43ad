"""Host-buffer pipeline: run a kernel of this library over a batch that lives in HOST memory.

The kernels move 24 B per output pixel at HBM speed (terabytes per second); a batch that starts and ends in host memory is
bound by the PCIe link instead (tens of GB/s per direction), so what matters end to end is that (a) the host-to-device copy
of chunk i+1, the kernel of chunk i and the device-to-host copy of chunk i-1 overlap, and (b) the pinned host pages live on
the NUMA node the GPU hangs off: ranks whose buffers sit on the other socket share its interconnect and lose much of the
PCIe bandwidth.  This module is that pipeline as a library feature:

* :func:`bind_to_device_numa_node` pins the calling process (CPU affinity + preferred memory node) to the GPU's node;
* :class:`HostPipeline` owns three streams, a ring of device staging buffers and the event choreography;
* :func:`warp_perspective_host` / :func:`apply_host` are the calls a user makes with host tensors.

Reference context: the reference has no such stage -- its users call ``.cuda()`` / ``.cpu()`` around
``kornia.geometry.transform.warp_perspective`` (imgwarp.py:69) and pay the copies serially.
"""
from __future__ import annotations

import ctypes
import os
from typing import Callable, Optional, Sequence

import torch

__all__ = ["bind_to_device_numa_node", "device_numa_node", "pinned_empty", "HostPipeline", "apply_host", "join", "warp_perspective_host",
           "host_ring_samples"]


# ------------------------------------------------------------------------------------------ NUMA placement
def _read(path: str) -> Optional[str]:
    try:
        with open(path) as f:
            return f.read().strip()
    except OSError:
        return None


def parse_cpulist(text: str) -> list[int]:
    """'0-31,64-95' -> [0..31, 64..95] (the format of /sys/devices/system/node/nodeN/cpulist)."""
    cpus: list[int] = []
    for part in text.split(","):
        part = part.strip()
        if not part:
            continue
        if "-" in part:
            a, b = part.split("-")
            cpus.extend(range(int(a), int(b) + 1))
        else:
            cpus.append(int(part))
    return cpus


def pci_bus_id(device_index: int) -> Optional[str]:
    """'0000:1b:00.0'-style address of a CUDA device (sysfs spelling: lower case, 4-digit domain)."""
    try:
        p = torch.cuda.get_device_properties(device_index)
        return f"{p.pci_domain_id:04x}:{p.pci_bus_id:02x}:{p.pci_device_id:02x}.0"
    except Exception:
        return None


def device_numa_node(device_index: int, sysfs: str = "/sys") -> Optional[int]:
    """NUMA node the GPU's PCIe root hangs off, from sysfs; None when the platform does not say (single node, VM)."""
    bus = pci_bus_id(device_index)
    if bus is None:
        return None
    text = _read(f"{sysfs}/bus/pci/devices/{bus}/numa_node")
    try:
        node = int(text) if text is not None else -1
    except ValueError:
        node = -1
    return node if node >= 0 else None


def node_cpus(node: int, sysfs: str = "/sys") -> list[int]:
    text = _read(f"{sysfs}/devices/system/node/node{node}/cpulist")
    return parse_cpulist(text) if text else []


_MPOL_PREFERRED = 1
_SYS_SET_MEMPOLICY = 238  # x86_64


def _prefer_memory_node(node: int) -> bool:
    """set_mempolicy(MPOL_PREFERRED, {node}) for the calling thread (pages pinned afterwards come from that node when it has
    room).  Raw syscall: libnuma is not assumed.  Returns whether the kernel accepted it."""
    try:
        libc = ctypes.CDLL(None, use_errno=True)
        nbits = 1024
        mask = (ctypes.c_ulong * (nbits // (8 * ctypes.sizeof(ctypes.c_ulong))))()
        mask[node // (8 * ctypes.sizeof(ctypes.c_ulong))] |= 1 << (node % (8 * ctypes.sizeof(ctypes.c_ulong)))
        rc = libc.syscall(_SYS_SET_MEMPOLICY, _MPOL_PREFERRED, ctypes.byref(mask), ctypes.c_ulong(nbits))
        return rc == 0
    except Exception:
        return False


_BOUND: dict = {}
_BINDING_DISABLED = os.environ.get("KB200_NO_NUMA_BIND", "") == "1"  # read once: measurement aid (the unbound contrast run)


def bind_to_device_numa_node(device_index: int, sysfs: str = "/sys") -> dict:
    """Bind the calling process to the NUMA node of ``cuda:device_index``: CPU affinity = that node's cores, memory policy =
    prefer that node.  Call it BEFORE allocating pinned buffers (one process per GPU: right after ``set_device``).  Returns
    what was done, e.g. ``{"node": 0, "cpus": 64, "affinity": True, "mempolicy": True}``; all-None/False when the platform
    gives no answer (nothing is changed then).  Idempotent per process."""
    if device_index in _BOUND:
        return _BOUND[device_index]
    info = {"node": None, "cpus": 0, "affinity": False, "mempolicy": False}
    if _BINDING_DISABLED:
        info["disabled"] = True
        _BOUND[device_index] = info
        return info
    node = device_numa_node(device_index, sysfs)
    if node is not None:
        cpus = node_cpus(node, sysfs)
        info.update(node=node, cpus=len(cpus))
        if cpus and hasattr(os, "sched_setaffinity"):
            try:
                allowed = os.sched_getaffinity(0)
                use = set(cpus) & allowed or set(cpus)
                os.sched_setaffinity(0, use)
                info["affinity"] = True
                info["cpus"] = len(use)
            except OSError:
                pass
        info["mempolicy"] = _prefer_memory_node(node)
    _BOUND[device_index] = info
    return info


def pinned_empty(shape: Sequence[int], dtype: torch.dtype = torch.float32, device_index: Optional[int] = None) -> torch.Tensor:
    """Page-locked host tensor; when ``device_index`` is given the process is first bound to that GPU's NUMA node so the
    pages are local to its PCIe root."""
    if device_index is not None:
        bind_to_device_numa_node(device_index)
    return torch.empty(tuple(shape), dtype=dtype, pin_memory=True)


def host_ring_samples(batch: int, chunk: int, bytes_per_sample: int, available_bytes: Optional[int] = None, local_ranks: Optional[int] = None) -> int:
    """How many samples each rank keeps in pinned host memory (``bytes_per_sample`` = source + destination bytes of one
    sample): all of them when a third of this rank's share of the available host memory holds the buffers, else the largest
    whole number of chunks that does (at least one chunk)."""
    if available_bytes is None:
        try:
            import psutil

            available_bytes = psutil.virtual_memory().available
        except Exception:
            return batch
    if local_ranks is None:
        local_ranks = int(os.environ.get("LOCAL_WORLD_SIZE", os.environ.get("WORLD_SIZE", "1")))
    fit = int(available_bytes / max(local_ranks, 1) / 3) // max(bytes_per_sample, 1)
    if fit >= batch:
        return batch
    return max(chunk, fit // chunk * chunk) if batch > chunk else batch


# ------------------------------------------------------------------------------------------ the pipeline
class HostPipeline:
    """Three-stream pipeline over dim-0 chunks of host tensors: H2D copy | kernel | D2H copy.

    ``fn(chunk_inputs..., start, stop)`` runs on the compute stream with device views of the chunk's inputs and returns
    the chunk's device result (any shape with the chunk length in dim 0).  Inputs are copied from (ideally pinned) host
    tensors; the result lands in ``out`` (host).  ``nbuf`` staging slots per input keep the three stages busy; slot reuse is
    ordered with events (a slot's input may be overwritten once its kernel finished, its output once the D2H copy left).
    The pipeline holds its device buffers between calls, so steady-state calls allocate nothing but the kernel's result."""

    def __init__(self, device, chunk: int = 16, nbuf: int = 3, bind_numa: bool = True):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("kornia_b200.streaming: the pipeline feeds a CUDA device; there is no CPU path")
        self.index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self.chunk, self.nbuf = int(chunk), int(nbuf)
        self.numa = bind_to_device_numa_node(self.index) if bind_numa else None
        self.s_in, self.s_k, self.s_out = (torch.cuda.Stream(self.device) for _ in range(3))
        self._stage: dict = {}
        self._ev = None

    def _staging(self, inputs: Sequence[torch.Tensor]):
        key = tuple((tuple(t.shape[1:]), t.dtype) for t in inputs)
        st = self._stage.get(key)
        if st is None:
            st = [[torch.empty((self.chunk,) + shp, dtype=dt, device=self.device) for shp, dt in key] for _ in range(self.nbuf)]
            self._stage = {key: st}  # one shape family at a time: a new family replaces the old buffers
        if self._ev is None:
            self._ev = [[torch.cuda.Event() for _ in range(self.nbuf)] for _ in range(3)]
        return st

    def join(self) -> None:
        """Make the caller's current stream wait for everything the pipeline has queued (copies included)."""
        cur = torch.cuda.current_stream(self.device)
        for s in (self.s_in, self.s_k, self.s_out):
            cur.wait_stream(s)

    def run(self, fn: Callable[..., torch.Tensor], inputs: Sequence[torch.Tensor], out: torch.Tensor, batch: Optional[int] = None,
            join: bool = True) -> torch.Tensor:
        """One pass over ``batch`` samples (default: the length of the host tensors).  ``inputs``: host tensors sharing dim 0;
        when they are shorter than ``batch`` they are a pinned ring that is read (and ``out`` written) cyclically -- the ring
        length must then be a whole number of chunks.  ``join=False`` leaves the caller's stream free: back-to-back passes then
        overlap (the first copies of pass n+1 run under the last kernels and copies of pass n; slots are ordered by events
        across passes) and the caller calls :meth:`join` once at the end."""
        hb = inputs[0].shape[0]
        batch = hb if batch is None else int(batch)
        if batch > hb and hb % self.chunk != 0:
            raise ValueError(f"a host ring of {hb} samples must be a whole number of {self.chunk}-sample chunks")
        if out.shape[0] != hb or any(t.shape[0] != hb for t in inputs):
            raise ValueError("inputs and out must share their first dimension")
        stage = self._staging(inputs)
        ev_in, ev_k, ev_out = self._ev
        if getattr(self, "_results", None) is None:
            self._results = [None] * self.nbuf  # kept across passes: a result may still be on its way out when the next pass starts
        results = self._results
        cur = torch.cuda.current_stream(self.device)
        # only the compute stream depends on the caller's stream (device tensors the caller produced, e.g. the matrices); the
        # copies read / write host memory and are ordered among themselves by the slot events
        self.s_k.wait_stream(cur)
        for i, b0 in enumerate(range(0, batch, self.chunk)):
            j = i % self.nbuf
            n = min(self.chunk, batch - b0)
            h0 = b0 % hb
            with torch.cuda.stream(self.s_in):
                self.s_in.wait_event(ev_k[j])  # the kernel that last read this slot is done
                for dst, src in zip(stage[j], inputs):
                    dst[:n].copy_(src[h0:h0 + n], non_blocking=True)
                ev_in[j].record(self.s_in)
            with torch.cuda.stream(self.s_k):
                self.s_k.wait_event(ev_in[j])
                self.s_k.wait_event(ev_out[j])  # the previous result of this slot has left the device
                results[j] = fn(*[t[:n] for t in stage[j]], b0, b0 + n)
                ev_k[j].record(self.s_k)
            with torch.cuda.stream(self.s_out):
                self.s_out.wait_event(ev_k[j])
                out[h0:h0 + n].copy_(results[j], non_blocking=True)
                results[j].record_stream(self.s_out)  # allocated on the compute stream, read here: tell the caching allocator
                ev_out[j].record(self.s_out)
        if join:
            self.join()
        return out


_PIPELINES: dict = {}


def _pipeline(device, chunk: int) -> HostPipeline:
    key = (str(torch.device(device)), int(chunk))
    p = _PIPELINES.get(key)
    if p is None:
        p = _PIPELINES[key] = HostPipeline(device, chunk=chunk)
    return p


def join(device="cuda", chunk: int = 16) -> None:
    """Wait (on the caller's current stream) for the passes issued with ``join=False`` on this device's pipeline."""
    _pipeline(device, chunk).join()


def apply_host(fn: Callable[..., torch.Tensor], inputs: Sequence[torch.Tensor], out: torch.Tensor, device="cuda", chunk: int = 16,
               logical_batch: Optional[int] = None, synchronize: bool = True, join: bool = True) -> torch.Tensor:
    """``out[b] = fn(inputs[b]...)`` for host tensors, chunked and pipelined on ``device`` (see :class:`HostPipeline`).
    ``logical_batch`` > len(inputs[0]) streams that many samples through the (shorter) host ring cyclically -- what a
    benchmark or a producer/consumer loop does when the whole batch cannot be page-locked at once."""
    for t in list(inputs) + [out]:
        if t.is_cuda:
            raise RuntimeError("kornia_b200.streaming: inputs and out are HOST tensors; call the op directly for device tensors")
    pipe = _pipeline(device, chunk)
    pipe.run(fn, inputs, out, batch=logical_batch, join=join or synchronize)
    if synchronize:
        torch.cuda.current_stream(pipe.device).synchronize()
    return out


def warp_perspective_host(src: torch.Tensor, M: torch.Tensor, dsize: tuple[int, int], mode: str = "bilinear", padding_mode: str = "zeros",
                          align_corners: bool = True, fill_value: Optional[torch.Tensor] = None, *, out: Optional[torch.Tensor] = None,
                          device="cuda", chunk: int = 16, logical_batch: Optional[int] = None, synchronize: bool = True,
                          join: bool = True) -> torch.Tensor:
    """``warp_perspective`` (imgwarp.py:69 semantics) for a batch in host memory: ``src`` (B,C,H,W) fp32 host tensor (pinned
    for full speed: :func:`pinned_empty`) or interleaved uint8 (B,H,W,C) decoder frames (3 B/pixel over PCIe instead of 12,
    converted and warped in one kernel: ``warp_perspective_from_uint8``); ``M`` (B,3,3) on the host or already on the
    device.  Returns ``out`` (host, (B,C,h,w) fp32; allocated pinned when not given)."""
    from .geometry.transform import warp_perspective
    from .geometry.transform.ingest import warp_perspective_from_uint8

    dev = torch.device(device)
    B = src.shape[0]
    n_log = B if logical_batch is None else int(logical_batch)
    u8 = src.dtype == torch.uint8
    C = src.shape[3] if u8 else src.shape[1]
    if out is None:
        out = pinned_empty((B, C, int(dsize[0]), int(dsize[1])), torch.float32, dev.index if dev.index is not None else torch.cuda.current_device())
    M_dev = M.to(dev, non_blocking=True)
    if M_dev.shape[0] < n_log:
        raise ValueError(f"M holds {M_dev.shape[0]} matrices for {n_log} samples")
    op = warp_perspective_from_uint8 if u8 else warp_perspective

    def step(chunk_src, b0, b1):
        return op(chunk_src, M_dev[b0:b1], dsize, mode, padding_mode, align_corners, fill_value)

    return apply_host(step, [src], out, device=dev, chunk=chunk, logical_batch=logical_batch, synchronize=synchronize, join=join)
