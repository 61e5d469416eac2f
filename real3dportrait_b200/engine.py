"""FrameEngine — the per-GPU frame loop of a clip (the caller side of the hot path, inference/real3d_infer.py:480-492,515-521):
a batch of tri-planes + cameras + jitter in, 512^2 frames out, one process per GPU.  Frames are independent (SURVEY.md §8e), so the
only exchange between ranks is the reassembly of the output clip:

  exchange='allgather'  every step's frames are all-gathered with NCCL on a side stream (every rank ends up with every frame)
  exchange='p2p'        every rank PUSHES its frames straight into the clip buffer on rank 0 at their global frame index with a
                        copy-engine peer copy (CUDA IPC mapping of rank 0's buffer; no SM is taken from the conv kernels, no staging copy,
                        and the clip needs no reassembly pass) - video writing only needs the clip on one rank
  exchange='none'       frames stay on their rank

With out_uint8 the last SR epilogue writes uint8 HWC video frames (the reference's ((x+1)/2*255).int() conversion, real3d_infer.py:519),
4x fewer bytes to exchange or copy to the host."""
from __future__ import annotations

import contextlib
import os
from typing import Callable, Dict, Optional

import torch

from . import _capi as capi
from .renderer import PlanesCL
from .synthesis import RenderHead


@contextlib.contextmanager
def gpu_local_cpus(device_index: int = 0, report: Optional[dict] = None):
    """Run the body on CPUs of the GPU's NUMA node (as far as the process may use them), then restore the affinity.

    Pinned host buffers are placed on the node of the allocating thread; staging buffers on the far socket cost a third of the
    PCIe rate on two-socket hosts.  Wrap only the ALLOCATION: `with gpu_local_cpus(i): buf = torch.empty(..., pin_memory=True)`.
    Anything unexpected (no sysfs entry, empty intersection, no permission) leaves the affinity untouched; `report` (a dict) receives
    what happened: the GPU's NUMA node, whether the affinity was narrowed, and why not if it was not."""
    old = None
    info = {'gpu_numa_node': None, 'pinned_to_gpu_node': False, 'reason': ''}
    try:
        pr = torch.cuda.get_device_properties(device_index)
        addr = f'{pr.pci_domain_id:04x}:{pr.pci_bus_id:02x}:{pr.pci_device_id:02x}.0'
        try:
            info['gpu_numa_node'] = int(open(f'/sys/bus/pci/devices/{addr}/numa_node').read().strip())
        except Exception:
            pass
        txt = open(f'/sys/bus/pci/devices/{addr}/local_cpulist').read().strip()
        local = set()
        for part in txt.split(','):
            if part:
                lo, _, hi = part.partition('-')
                local.update(range(int(lo), int(hi or lo) + 1))
        cur = os.sched_getaffinity(0)
        both = cur & local
        if not both:
            info['reason'] = 'the process may not run on any CPU of the GPU node (affinity/cgroup): buffers land on the current node'
        elif both == cur:
            info['pinned_to_gpu_node'], info['reason'] = True, 'process already confined to the GPU node'
        else:
            os.sched_setaffinity(0, both)
            old = cur
            info['pinned_to_gpu_node'] = True
    except Exception as e:                                             # noqa: BLE001
        old = None
        info['reason'] = f'{type(e).__name__}: {e}'
    if report is not None:
        report.update(info)
    try:
        yield
    finally:
        if old is not None:
            try:
                os.sched_setaffinity(0, old)
            except Exception:
                pass


def default_sr_mode() -> str:
    try:
        from . import sr_tc  # noqa: F401
        return 'tc' if sr_tc.available() else 'fp32'
    except ImportError:
        return 'fp32'


def _ptr_key(t) -> int:
    if t is None:
        return 0
    if isinstance(t, PlanesCL):
        return t.data.data_ptr()
    if isinstance(t, (tuple, list)):
        return hash(tuple(_ptr_key(x) for x in t))
    return t.data_ptr()


def _frames_of(planes) -> int:
    if isinstance(planes, (tuple, list)):
        return max(_frames_of(p) for p in planes)
    return planes.dims[0] if isinstance(planes, PlanesCL) else planes.shape[0]


class FrameEngine:
    """batch: frames per step; static_styles: the SR styles are constant (Real3D passes ws == 1, img2plane_baseline.py:142) so
    the folded fp16 weights are prepared once per parameter load; use_graph: replay the whole step as ONE CUDA graph."""

    def __init__(self, batch: int = 4, sr_mode: str = 'fp32', device=None, world: int = 1, rank: int = 0, dist=None, hp: Optional[dict] = None,
                 static_styles: bool = True, use_graph: bool = True, out_uint8: bool = False, exchange: str = 'allgather'):
        assert exchange in ('allgather', 'p2p', 'none')
        self.batch, self.world, self.rank, self.dist = batch, world, rank, dist
        self.device = device if device is not None else torch.device('cuda', torch.cuda.current_device())
        self.head = RenderHead(hp=hp, sr_mode=sr_mode).to(self.device).eval()
        self.static_styles, self.use_graph = static_styles, use_graph
        self.out_uint8 = bool(out_uint8)
        if self.out_uint8 and sr_mode not in ('tc', 'tc_exact'):
            raise NotImplementedError('uint8 frames are written by the tensor-core SR epilogue (sr_mode="tc")')
        self.exchange = exchange if world > 1 else 'none'
        self.graph = None
        self.launches_per_step = 0
        self.s_in = None                  # static graph inputs (planes, cameras, u_coarse, u_fine)
        self.s_out = None
        self.inplace = {}                 # input pointers -> (graph, output, the inputs kept alive): see prepare()
        self._pool = None
        self._clip = None

    # ---- output geometry -------------------------------------------------------------------------------------------------------------
    def frame_shape(self):
        return (512, 512, 3) if self.out_uint8 else (3, 512, 512)

    def frame_dtype(self):
        return torch.uint8 if self.out_uint8 else torch.float32

    def load_params(self, decoder_params: Dict[str, torch.Tensor], sr_params: Dict[str, torch.Tensor]) -> None:
        sd = {'decoder.' + k: v for k, v in decoder_params.items()}
        sd.update({'superresolution.' + k: v for k, v in sr_params.items()})
        self.head.load_state_dict(sd, strict=True)
        self.graph = None
        self.inplace = {}
        sr = self.head.superresolution
        sr.static_prepared = None
        if self.static_styles and sr.sr_mode in ('tc', 'tc_exact') and not self.head.torso:
            from . import sr_tc
            ones = torch.ones(1, 3, self.head.hparams['w_dim'], device=self.device)
            with torch.no_grad():
                sr.static_prepared = sr_tc.Prepared(sr, ones, sr.sr_mode == 'tc_exact')

    @torch.no_grad()
    def _body(self, planes, cameras, u_coarse, u_fine=None) -> torch.Tensor:
        over = {'u_coarse': u_coarse}
        if u_fine is not None:
            over['u_fine'] = u_fine
        return self.head.synthesis(planes, cameras, lean=True, out_uint8=self.out_uint8, **over)['image']

    def _capture_graph(self, planes, cameras, u_coarse, u_fine=None):
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):                                       # warm-up outside capture: lazy inits (func attributes, driver entry points)
                self._body(planes, cameras, u_coarse, u_fine)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        if self._pool is None:
            self._pool = torch.cuda.graph_pool_handle()               # all step graphs share one pool: they never run concurrently
        c0 = capi.lib().r3dp_launch_count()
        with torch.cuda.graph(g, pool=self._pool):
            out = self._body(planes, cameras, u_coarse, u_fine)
        self.launches_per_step = int(capi.lib().r3dp_launch_count() - c0)      # libr3dp kernels inside one replay
        return g, out

    def _needs_fine(self) -> bool:
        return int(self.head.rendering_kwargs['depth_resolution_importance'] or 0) > 0

    def _draw(self, n, device, u_coarse, u_fine):
        """Jitter in the reference's order and shapes (renderer.py:226,281) when the caller does not supply it."""
        S, Si = self.head.rendering_kwargs['depth_resolution'], int(self.head.rendering_kwargs['depth_resolution_importance'] or 0)
        M = self.head.neural_rendering_resolution ** 2
        if u_coarse is None:
            u_coarse = torch.rand(n, M, S, 1, device=device)
        if u_fine is None and Si > 0:
            u_fine = torch.rand(n * M, Si, device=device)
        return u_coarse, u_fine

    @torch.no_grad()
    def prepare(self, inputs, max_graphs: int = 64) -> int:
        """Zero-copy steps for RESIDENT inputs: capture one step graph per (planes, cameras, u_coarse[, u_fine]) tuple that reads those very
        buffers, so `step()` on them replays without first copying the planes into static graph inputs.  `planes` may be the reference's
        [B,3,32,H,W] tensor (repacked inside the step), a PlanesCL the producer wrote channels-last (no repack), or a (cano, secc) pair.
        The tensors are kept referenced (their addresses stay valid); refill them in place between steps.  Returns the number of graphs held."""
        if not self.use_graph:
            return 0
        for item in inputs:
            planes, cameras, u_coarse = item[:3]
            u_fine = item[3] if len(item) > 3 else None
            k = (_ptr_key(planes), cameras.data_ptr(), u_coarse.data_ptr(), _ptr_key(u_fine))
            if k in self.inplace or len(self.inplace) >= max_graphs or _frames_of(planes) not in (self.batch, 1):
                continue
            if self._needs_fine() and u_fine is None:
                raise ValueError('this head renders with importance samples: prepare() needs u_fine [B*M, S_imp] in every input tuple')
            g, out = self._capture_graph(planes, cameras, u_coarse, u_fine)
            self.inplace[k] = (g, out, (planes, cameras, u_coarse, u_fine))
        return len(self.inplace)

    @torch.no_grad()
    def step(self, planes, cameras: torch.Tensor, u_coarse: Optional[torch.Tensor] = None, u_fine: Optional[torch.Tensor] = None,
             frame_index: Optional[int] = None) -> torch.Tensor:
        """planes [B,3,32,256,256] | PlanesCL | (cano, secc); cameras [B,25]; u_coarse [B,4096,S,1], u_fine [B*4096,S_imp] (drawn here if None)
        -> this rank's frames: fp32 [B,3,512,512] in [-1,1] or uint8 [B,512,512,3]; with exchange='allgather' the gathered
        [world*B,...] (rank-major); with exchange='p2p' the frames are additionally pushed into the open clip at `frame_index`.
        The returned tensor is reused by the next step."""
        drawn = u_coarse is None or (u_fine is None and self._needs_fine())
        u_coarse, u_fine = self._draw(cameras.shape[0], cameras.device, u_coarse, u_fine)
        graphable = self.use_graph and capi.PROF is None and cameras.shape[0] == self.batch
        key = (_ptr_key(planes), cameras.data_ptr(), u_coarse.data_ptr(), _ptr_key(u_fine))
        hit = self.inplace.get(key) if (graphable and self.inplace and not drawn) else None
        if hit is not None:
            hit[0].replay()
            out = hit[1]
        elif graphable and isinstance(planes, torch.Tensor):
            if self.graph is None:
                self.s_in = (planes.clone(), cameras.clone(), u_coarse.clone(), None if u_fine is None else u_fine.clone())
                self.graph, self.s_out = self._capture_graph(*self.s_in)
            for dst, src in zip(self.s_in, (planes, cameras, u_coarse, u_fine)):
                if dst is not None and src.data_ptr() != dst.data_ptr():
                    dst.copy_(src, non_blocking=True)
            self.graph.replay()
            out = self.s_out
        else:
            out = self._body(planes, cameras, u_coarse, u_fine)
        if self.exchange == 'allgather':
            if capi.PROF is not None:                                   # profiling pass: serial, so the region time is the collective's own
                gathered = torch.empty((self.world * self.batch,) + tuple(out.shape[1:]), dtype=out.dtype, device=self.device)
                with capi.region('exchange'):
                    self.dist.all_gather_into_tensor(gathered, out.contiguous())
                return gathered
            return self._gather_async(out)
        if self.exchange == 'p2p' and self._clip is not None and frame_index is not None:
            with capi.region('exchange'):
                self._push(out, frame_index)
        return out

    # ---- exchange: NCCL all-gather on a side stream --------------------------------------------------------------------------------------
    def _gather_async(self, out: torch.Tensor) -> torch.Tensor:
        """Frame exchange of step i on a side stream so it runs under the compute of step i+1: the step's frames are copied to one of two
        staging slots (the graph's output buffer is rewritten by the next replay), NCCL all-gathers slot -> gathered[slot] on `comm`.
        The returned tensor is complete once `wait_gather()` (or a device sync) has run; a slot is reused two steps later."""
        if getattr(self, '_ga', None) is None:
            shape = (self.world * self.batch,) + tuple(out.shape[1:])
            self._ga = {'comm': torch.cuda.Stream(device=self.device), 'k': 0,
                        'stage': [torch.empty_like(out) for _ in range(2)],
                        'dst': [torch.empty(shape, dtype=out.dtype, device=self.device) for _ in range(2)],
                        'done': [torch.cuda.Event() for _ in range(2)], 'ready': [torch.cuda.Event() for _ in range(2)]}
            cur0 = torch.cuda.current_stream()
            for e in self._ga['done']:
                e.record(cur0)
        ga = self._ga
        k = ga['k'] & 1
        ga['k'] += 1
        cur = torch.cuda.current_stream()
        cur.wait_event(ga['done'][k])                                   # the collective that last used this slot has finished
        ga['stage'][k].copy_(out, non_blocking=True)
        ga['ready'][k].record(cur)
        with torch.cuda.stream(ga['comm']):
            ga['comm'].wait_event(ga['ready'][k])
            self.dist.all_gather_into_tensor(ga['dst'][k], ga['stage'][k])
            ga['done'][k].record(ga['comm'])
        return ga['dst'][k]

    def wait_gather(self) -> None:
        """Make the current stream wait for every frame exchange issued so far (call before consuming step()'s result when world > 1)."""
        if getattr(self, '_ga', None) is not None:
            torch.cuda.current_stream().wait_stream(self._ga['comm'])
        if getattr(self, '_p2p', None) is not None:
            torch.cuda.current_stream().wait_stream(self._p2p['stream'])

    # ---- exchange: peer pushes into the clip on rank 0 -----------------------------------------------------------------------------------
    def open_clip(self, frames_per_rank: int) -> Optional[torch.Tensor]:
        """Allocate the output clip [world*frames_per_rank, ...] on rank 0 and map it into every other rank (CUDA IPC); returns the clip on
        rank 0, None elsewhere.  Frame f of rank r lands at clip[r*frames_per_rank + f].  With world == 1 the clip is a local buffer."""
        shape = (self.world * frames_per_rank,) + self.frame_shape()
        self._fpr = frames_per_rank
        if self.world == 1 or self.exchange != 'p2p':
            self._clip = torch.empty(shape, dtype=self.frame_dtype(), device=self.device) if self.rank == 0 else None
            self._clip_view = self._clip
            self._p2p = None
            return self._clip
        from torch.multiprocessing.reductions import reduce_tensor
        payload = [None]
        if self.rank == 0:
            self._clip = torch.empty(shape, dtype=self.frame_dtype(), device=self.device)
            payload = [reduce_tensor(self._clip)]
        self.dist.broadcast_object_list(payload, src=0)
        if self.rank == 0:
            self._clip_view = self._clip
        else:
            fn, args = payload[0]
            self._clip_view = fn(*args)                                # rank 0's buffer, mapped into this process (lives on rank 0's device)
            self._clip = self._clip_view                               # pushes only; never read here
        self._p2p = {'stream': torch.cuda.Stream(device=self.device), 'k': 0, 'stage': None,
                     'done': [torch.cuda.Event() for _ in range(2)], 'ready': [torch.cuda.Event() for _ in range(2)]}
        for e in self._p2p['done']:
            e.record(torch.cuda.current_stream())
        return self._clip if self.rank == 0 else None

    def _push(self, out: torch.Tensor, frame_index: int) -> None:
        n = min(out.shape[0], self._fpr - frame_index)
        if n <= 0:
            return
        dst = self._clip_view[self.rank * self._fpr + frame_index: self.rank * self._fpr + frame_index + n]
        if self._p2p is None:                                          # single rank / local clip: plain device copy on the compute stream
            dst.copy_(out[:n], non_blocking=True)
            return
        p = self._p2p
        k = p['k'] & 1
        p['k'] += 1
        cur = torch.cuda.current_stream()
        if p['stage'] is None:
            p['stage'] = [torch.empty_like(out) for _ in range(2)]
        cur.wait_event(p['done'][k])
        p['stage'][k].copy_(out, non_blocking=True)                     # the graph's output buffer is rewritten by the next replay
        p['ready'][k].record(cur)
        with torch.cuda.stream(p['stream']):
            p['stream'].wait_event(p['ready'][k])
            src = p['stage'][k][:n]
            # peer copy over NVLink by the copy engine (no SMs), enqueued directly: torch's cross-device copy_ brackets every copy with
            # event record/wait pairs on BOTH devices' current streams (measured: 1.3 ms/step of host-side stalls at 2 GPUs)
            capi.check(capi.lib().r3dp_peer_copy(dst.data_ptr(), dst.device.index, src.data_ptr(), src.device.index,
                                                 src.numel() * src.element_size(), capi.stream()))
            p['done'][k].record(p['stream'])

    def close_clip(self) -> Optional[torch.Tensor]:
        """Wait until every rank's pushes have landed; returns the finished clip on rank 0."""
        self.wait_gather()
        torch.cuda.synchronize(self.device)
        if self.world > 1 and self.dist is not None:
            self.dist.barrier()
        clip = self._clip if self.rank == 0 else None
        if self.rank != 0 and getattr(self, '_p2p', None) is not None:      # drop this process's mapping of rank 0's buffer before rank 0 may free it
            self._clip_view = self._clip = None
            torch.cuda.ipc_collect()
        if self.world > 1 and self.dist is not None and getattr(self, '_p2p', None) is not None:
            self.dist.barrier()
            if self.rank == 0:
                torch.cuda.ipc_collect()                                      # the consumers' references are gone: drop the producer-side IPC bookkeeping
        return clip

    # ---- host-buffer entry point: H2D / compute / D2H of consecutive steps overlap on three streams -----------------------
    def _host_pipeline(self):
        if getattr(self, '_hp', None) is None:
            dev = self.device
            self._hp = {
                'copy_in': torch.cuda.Stream(device=dev), 'copy_out': torch.cuda.Stream(device=dev), 'k': 0,
                'in_ready': [torch.cuda.Event() for _ in range(2)], 'in_free': [torch.cuda.Event() for _ in range(2)],
                'out_ready': [torch.cuda.Event() for _ in range(2)], 'out_free': [torch.cuda.Event() for _ in range(2)],
                'stage': [None, None], 'out': [None, None],
            }
        return self._hp

    @torch.no_grad()
    def step_host(self, h_planes: torch.Tensor, h_cameras: torch.Tensor, h_u: torch.Tensor, h_out: torch.Tensor,
                  h_u_fine: Optional[torch.Tensor] = None) -> None:
        """Same step, from PINNED HOST tensors to a pinned host output (frames of THIS rank), fully asynchronous: the call
        enqueues H2D (copy-in stream) -> step (current stream) -> D2H (copy-out stream) and returns; with two staging slots the
        copy of step i+1 runs under the compute of step i.  Call `sync_host()` before reading `h_out`."""
        hp = self._host_pipeline()
        k = hp['k'] & 1
        hp['k'] += 1
        cur = torch.cuda.current_stream()
        hosts = (h_planes, h_cameras, h_u) + ((h_u_fine,) if h_u_fine is not None else ())
        if hp['stage'][k] is None:
            hp['stage'][k] = tuple(torch.empty_like(h, device=self.device) for h in hosts)
            hp['out'][k] = torch.empty((self.batch,) + self.frame_shape(), dtype=self.frame_dtype(), device=self.device)
            for dst, src in zip(hp['stage'][k], hosts):
                dst.copy_(src)                                         # warm-up / capture run on REAL inputs (uninitialised cameras give NaN depths)
            self.prepare([hp['stage'][k]])                             # the step reads the staging slot in place (no device-side input copy)
            hp['in_free'][k].record(cur); hp['out_free'][k].record(cur)
        stage = hp['stage'][k]
        with torch.cuda.stream(hp['copy_in']):
            hp['copy_in'].wait_event(hp['in_free'][k])                 # the step that last read this slot is done
            for dst, src in zip(stage, hosts):
                dst.copy_(src, non_blocking=True)
            hp['in_ready'][k].record(hp['copy_in'])
        cur.wait_event(hp['in_ready'][k])
        out = self.step(*stage)
        self.wait_gather()
        hp['in_free'][k].record(cur)
        cur.wait_event(hp['out_free'][k])
        mine = out[self.rank * self.batch:(self.rank + 1) * self.batch] if out.shape[0] > self.batch else out
        hp['out'][k].copy_(mine, non_blocking=True)
        hp['out_ready'][k].record(cur)
        with torch.cuda.stream(hp['copy_out']):
            hp['copy_out'].wait_event(hp['out_ready'][k])
            h_out.copy_(hp['out'][k], non_blocking=True)
            hp['out_free'][k].record(hp['copy_out'])

    def sync_host(self) -> None:
        hp = self._host_pipeline()
        hp['copy_in'].synchronize(); hp['copy_out'].synchronize(); torch.cuda.current_stream().synchronize()

    def static_inputs(self):
        """(planes, cameras, u_coarse, u_fine) static buffers of the captured graph: a producer may write its outputs straight into them
        and call step() with these very tensors to skip the copy-in."""
        return self.s_in

    def profile_steps(self, inputs: Callable[[int], tuple], first: int, steps: int) -> Dict:
        """Re-run `steps` steps eagerly with CUDA events around every stage (on the launching stream)."""
        capi.PROF = capi.Profiler()
        self.step(*inputs(first))                                   # eager warm-up: one-time lazy initialisations stay out of the stage times
        torch.cuda.synchronize()
        capi.PROF = capi.Profiler()
        L = capi.lib()
        tc = self.head.superresolution.sr_mode in ('tc', 'tc_exact')
        if tc:
            L.r3dp_sr_tc_prof(1)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for i in range(steps):
            self.step(*inputs(first + i))
        b.record()
        torch.cuda.synchronize()
        stages = capi.PROF.totals()
        capi.PROF = None
        conv_ms, conv_n = None, 0
        if tc:
            import ctypes as C
            ms, n = C.c_float(0), C.c_int(0)
            capi.check(L.r3dp_sr_tc_prof_read(C.byref(ms), C.byref(n)))
            L.r3dp_sr_tc_prof(0)
            conv_ms, conv_n = float(ms.value), int(n.value)
        kernel = 'conv_tc3_kernel<1> (wgmma implicit-GEMM conv)' if tc else 'conv_taps_kernel (fp32 CUDA-core direct conv)'
        return {'stages': stages, 'sr_conv_ms': stages.get('sr_conv', float('nan')), 'total_ms': a.elapsed_time(b), 'sr_kernel': kernel,
                'conv_kernel_ms': conv_ms, 'conv_launches': conv_n}
