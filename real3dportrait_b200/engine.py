"""FrameEngine — the per-GPU frame loop of a clip (the caller side of the hot path, inference/real3d_infer.py:480-492,515-521):
a batch of tri-planes + cameras + jitter in, 512^2 frames out, one process per GPU.  Frames are independent (SURVEY.md §8e), so the
only exchange between ranks is the reassembly of the output clip:

  exchange='allgather'  every step's frames are all-gathered with NCCL on a side stream (every rank ends up with every frame)
  exchange='p2p'        every rank PUSHES its frames straight into the clip buffer on rank 0 at their global frame index with a
                        copy-engine peer copy (CUDA IPC mapping of rank 0's buffer; no SM is taken from the conv kernels, no staging copy,
                        and the clip needs no reassembly pass) - video writing only needs the clip on one rank
  exchange='none'       frames stay on their rank

With out_uint8 the last SR epilogue writes uint8 HWC video frames (the reference's ((x+1)/2*255).int() conversion, real3d_infer.py:519),
4x fewer bytes to exchange or copy to the host.

With torso_model=... the engine runs the torso head (OSAvatarSECC_Img2plane_Torso, SuperresolutionHybrid8XDC_Warp): begin_clip() takes the
constants of a clip (ref_torso_img, bg_img, segmap, kp_s; real3d_infer.py:463-467) and every step takes the frames' kp_d.  The torso warper is
the caller's PyTorch module; it need not be capturable: by default a step replays two graphs around an eager warper call.

With out_mode='concat_debug' every frame is the reference's default debug strip [512,2560,3] (real3d_infer.py:494-521): source | driving
SECC | raw render | depth | final, see debug_frames.py.  The depth panel is normalised over the whole clip, so close_clip() writes it."""
from __future__ import annotations

import contextlib
import os
from typing import Callable, Dict, Optional

import torch

from . import _capi as capi
from .debug_frames import FRAME_SHAPE as DEBUG_FRAME_SHAPE, RES as DEBUG_RES, debug_panels, depth_panel
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
    """The SR mode a run takes when none is asked for: the tensor-core path, which the library always builds."""
    return 'tc'


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


class _TorsoGraphs:
    """One torso step as two CUDA graphs around an eager torso_model call: graph A (render, SR prep, block0, the warper's inputs), the
    warper on the current stream, its three outputs copied into graph B's static inputs (the caching allocator does not keep their
    addresses), graph B (the rest of the head).  Under weight_fuse=False graph B reads neither rgb_torso nor occlusion_2; they are copied
    all the same (two small copies) so that every configuration keeps one step layout."""

    def __init__(self, sr, a, st, b_in, b):
        self.sr, self.a, self.st, self.b_in, self.b = sr, a, st, b_in, b

    def replay(self) -> None:
        self.a.replay()
        rgb_torso, ret = self.sr.run_torso(self.st)
        for dst, src in zip(self.b_in, (rgb_torso, ret['deformed_torso_hid'], ret['occlusion_2'])):
            dst.copy_(src)
        self.b.replay()


class FrameEngine:
    """batch: frames per step; static_styles: the SR styles are constant (Real3D passes ws == 1, img2plane_baseline.py:142) so
    the folded fp16 weights are prepared once per parameter load or move; use_graph: replay the step as CUDA graphs.
    torso_model: run the torso head with this warper (WarpBasedTorsoModelMediaPipe or a module with its forward signature);
    warper_in_graph: capture the warper inside the step's single graph (only for capturable warpers; the default runs it eagerly
    between two graphs).  torso_stage2='cuda': the warper's stage 2 on this library's kernels, its appearance features cached per clip by
    begin_clip() (SuperresolutionHybrid8XDC_Warp.set_torso_stage2).  torso_motion='cuda' (needs torso_stage2='cuda'): the warper's
    motion-field estimator on this library's 3-D convolutions too (SuperresolutionHybrid8XDC_Warp.set_torso_motion).
    secc2plane: a SegFormerSECC2PlaneBackbone; the engine then runs it inside the step (captured in the step's graph, graph A of the torso
    split): begin_planes(cano_planes, cond_cano, cond_src) once per clip, then step(None, cameras, ..., cond_tgt=drv_secc) renders
    cano_planes + backbone(cat[cano, src, tgt]) (secc_img2plane.py:64-81) without materialising either plane set; prepare() tuples and
    step_host() take the driving SECC image [B,3,H,W] in the planes slot.
    secc_renderer (with secc2plane): a SECC_Renderer; the engine then renders the SECC images itself from 3DMM coefficients [id | exp] at zero
    pose (real3d_infer.py:391-405): begin_planes(cano_planes, coeff_src=c [1,144]) renders the clip's two images, and step(None, cameras, ...,
    coeff=c [B,144]) renders the driving image inside the step (and its graph), in front of the backbone.  Each step is one renderer call, so
    face 0 is background in the first frame of every step, i.e. every `batch`-th frame of the clip.  The reference renders a clip in 50-frame
    calls and loses face 0 only in frames 0, 50, 100, ...: the engine's frames differ from it where face 0 wins in the other frames that start a
    step (one triangle, a few pixels).  prepare() tuples and step_host() then carry the coefficients in the planes slot.
    blink (with secc_renderer): the engine also closes the eyes of each driving image as real3d_infer.py's default blink_mode='period' does
    (blink_eye_for_secc): coefficient rows become [B, n_id + n_exp + 2] = [id | exp | t | T] (fp32; period_blink_schedule gives (t, T), T = 0
    leaves a frame untouched) and the edit runs in place between the render and the backbone, inside the step's graph.  blink_faults() counts
    the frames on which the reference would raise (left unedited).  begin_planes() is unchanged: the reference blinks only the driving images.
    img2plane (with secc2plane): an Img2PlaneModel; begin_planes(img=ref_head_img [1,3,512,512], ...) then makes the clip's canonical planes
    from the source image (cal_cano_plane, secc_img2plane.py:50-62) straight into the engine's canonical buffer, once per clip and outside
    the step's graph, in place of begin_planes(cano_planes, ...).
    out_mode='concat_debug' (with secc2plane and out_uint8=True): frames are the reference's default debug strips uint8 [512,2560,3]
    (real3d_infer.py:494-521).  open_clip(frames_per_rank, ref_gt_img=...) takes the source image of panel 0, every step needs the open clip
    and its frame_index, and close_clip() writes the depth panel, normalised over the whole clip.  Panel 1 is the SECC image the step used
    (cond_tgt, or the rendered and blinked image).  Needs exchange='p2p' at world > 1; step_host() is not built for it."""

    def __init__(self, batch: int = 4, sr_mode: str = 'fp32', device=None, world: int = 1, rank: int = 0, dist=None, hp: Optional[dict] = None,
                 static_styles: bool = True, use_graph: bool = True, out_uint8: bool = False, exchange: str = 'allgather',
                 torso_model: Optional[torch.nn.Module] = None, warper_in_graph: bool = False, torso_stage2: str = 'torch',
                 torso_motion: str = 'torch', secc2plane: Optional[torch.nn.Module] = None, secc_renderer: Optional[torch.nn.Module] = None,
                 blink: bool = False, img2plane: Optional[torch.nn.Module] = None, out_mode: str = 'final'):
        assert exchange in ('allgather', 'p2p', 'none')
        if out_mode not in ('final', 'concat_debug'):
            raise ValueError(f"out_mode must be 'final' or 'concat_debug', got {out_mode!r}")
        if out_mode == 'concat_debug':
            if secc2plane is None:
                raise ValueError("out_mode='concat_debug' shows the driving SECC image: FrameEngine(secc2plane=..., out_mode='concat_debug')")
            if not out_uint8:
                raise ValueError("out_mode='concat_debug' writes uint8 video frames: FrameEngine(out_uint8=True, out_mode='concat_debug')")
            if world > 1 and exchange != 'p2p':
                raise NotImplementedError("out_mode='concat_debug' at world > 1 collects the clip on rank 0 with exchange='p2p' only")
            if (hp or {}).get('mask_invalid_rays', False):
                raise NotImplementedError("out_mode='concat_debug' reads the lean render path, which mask_invalid_rays does not take")
        self.debug = out_mode == 'concat_debug'
        self.out_mode = out_mode
        if secc2plane is not None and (hp or {}).get('phase1_plane_fusion_mode', 'add') != 'add':
            raise NotImplementedError('secc2plane: only phase1_plane_fusion_mode="add" (cano + secc, secc_img2plane.py:76-77) is built')
        self.batch, self.world, self.rank, self.dist = batch, world, rank, dist
        self.device = device if device is not None else torch.device('cuda', torch.cuda.current_device())
        self.head = RenderHead(hp=hp, sr_mode=sr_mode, torso_model=torso_model).to(self.device).eval()
        self.head.superresolution.static_styles = bool(static_styles)
        self.use_graph = use_graph
        self.torso, self.warper_in_graph = self.head.torso, bool(warper_in_graph)
        if torso_stage2 != 'torch':
            if not self.torso:
                raise ValueError('torso_stage2 is an option of the torso head: FrameEngine(torso_model=...)')
            self.head.superresolution.set_torso_stage2(torso_stage2)
        if torso_motion != 'torch':
            if not self.torso:
                raise ValueError('torso_motion is an option of the torso head: FrameEngine(torso_model=...)')
            self.head.superresolution.set_torso_motion(torso_motion)
        self.secc = secc2plane.to(self.device).eval() if secc2plane is not None else None
        self._cano_cl = None              # secc2plane: the clip's canonical planes, 'hwpc' [1,H,W,3,C] (begin_planes)
        if secc_renderer is not None and secc2plane is None:
            raise ValueError('secc_renderer renders the input of the SECC -> plane backbone: FrameEngine(secc2plane=..., secc_renderer=...)')
        self.secc_r = secc_renderer.to(self.device) if secc_renderer is not None else None
        if blink and self.secc_r is None:
            raise ValueError('blink edits the images the SECC renderer draws: FrameEngine(secc2plane=..., secc_renderer=..., blink=True)')
        self.blink = bool(blink)
        if img2plane is not None and secc2plane is None:
            raise ValueError('img2plane makes the canonical planes of a secc2plane clip: FrameEngine(secc2plane=..., img2plane=...)')
        self.img2p = img2plane.to(self.device).eval() if img2plane is not None else None
        self.out_uint8 = bool(out_uint8)
        if self.out_uint8 and self.head.superresolution.sr_mode not in ('tc', 'tc_exact'):     # the head's effective mode: a torso head maps 'fp32' to 'tc'
            raise NotImplementedError('uint8 frames are written by the tensor-core SR epilogue (sr_mode="tc")')
        # fuse mode v3 thresholds the head mask at a host-side quantile (sr_with_ref.py:141-143): its steps cannot be captured
        self.eager_reason = ('fuse mode v3 reads a host-side quantile of the head mask every step'
                             if self.torso and self.head.superresolution.fuse_mode == 'v3' else None)
        self._consts = None               # torso head: the clip's constants (begin_clip)
        self.exchange = exchange if world > 1 else 'none'
        self.graph = None
        self.launches_per_step = 0
        self.s_in = None                  # static graph inputs (planes, cameras, u_coarse, u_fine)
        self.s_out = None
        self.inplace = {}                 # input pointers -> (graph, output, the inputs kept alive): see prepare()
        self._pool = None
        self._clip = None
        self._ref_gt = None               # concat_debug: panel 0's source image [1,3,512,512] (open_clip)
        self._clip_depth = None           # concat_debug: the clip's depths [world*frames_per_rank,64,64] on rank 0

    # ---- output geometry -------------------------------------------------------------------------------------------------------------
    def frame_shape(self):
        if self.debug:
            return DEBUG_FRAME_SHAPE
        return (512, 512, 3) if self.out_uint8 else (3, 512, 512)

    def frame_dtype(self):
        return torch.uint8 if self.out_uint8 else torch.float32

    def load_params(self, decoder_params: Dict[str, torch.Tensor], sr_params: Dict[str, torch.Tensor]) -> None:
        sd = {'decoder.' + k: v for k, v in decoder_params.items()}
        sd.update({'superresolution.' + k: v for k, v in sr_params.items()})
        self.head.load_state_dict(sd, strict=True)
        self.graph = None
        self.inplace = {}
        self._consts = None                                            # loading dropped the head's per-clip cache: begin_clip() again
        self.head.superresolution.prepared_styles()                    # folded now, so that no step or captured graph does it

    # ---- torso head: per-clip constants --------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def begin_clip(self, ref_torso_img: torch.Tensor, bg_img: torch.Tensor, segmap: torch.Tensor, kp_s: torch.Tensor) -> None:
        """The constants of a clip (real3d_infer.py:463-467): ref_torso_img, bg_img [1,3,512,512], segmap [1,6,512,512], kp_s [1,68,3].
        Runs the head's per-clip cache (bg_encoder(bg_img), the two antialiased resizes) and keeps the [batch,...] broadcasts every step
        reads.  A later begin_clip() refills these buffers in place, so graphs captured for an earlier clip render the new one."""
        if not self.torso:
            raise ValueError('begin_clip() is for the torso head: FrameEngine(torso_model=...)')
        if not (ref_torso_img.shape[0] == bg_img.shape[0] == segmap.shape[0] == kp_s.shape[0] == 1):
            raise ValueError('one set of clip constants: ref_torso_img, bg_img, segmap and kp_s have batch size 1')
        B = self.batch
        if not self.head.superresolution.begin_clip(ref_torso_img, bg_img, batch=B, in_place=True, segmap=segmap.to(self.device)):
            self.graph, self.inplace = None, {}                       # new constant buffers: graphs captured earlier read the old ones
        bc = {'segmap': segmap.expand(B, -1, -1, -1), 'kp_s': kp_s.expand(B, -1, -1)}
        if self._consts is None:
            self._consts = {k: v.to(self.device, torch.float32).contiguous() for k, v in bc.items()}
        else:
            for k, v in bc.items():
                self._consts[k].copy_(v)
        self._consts.update({'ref_torso_img': ref_torso_img, 'bg_img': bg_img})

    @torch.no_grad()
    def begin_planes(self, cano_planes: Optional[torch.Tensor] = None, cond_cano: Optional[torch.Tensor] = None,
                     cond_src: Optional[torch.Tensor] = None, *, coeff_src: Optional[torch.Tensor] = None,
                     img: Optional[torch.Tensor] = None) -> None:
        """secc2plane engines: the clip's canonical planes [1,3,32,256,256] and the backbone's per-clip SECC images [1,3,H,W] (cond_src only in
        'cano_src_tgt').  With a secc_renderer the images come from the source frame's coefficients coeff_src [1,144] = [id | exp] instead:
        cond_src = r(id, exp), cond_cano = r(id, 0 exp), zero pose (real3d_infer.py:404-405).  With FrameEngine(img2plane=...), img = the
        source head image [1,3,512,512] in place of cano_planes: the backbone writes the canonical planes straight into the engine's buffer.
        A later begin_planes() refills the same buffers in place, so graphs captured for an earlier clip render the new one."""
        if self.secc is None:
            raise ValueError('begin_planes() needs FrameEngine(secc2plane=...)')
        if (cano_planes is None) == (img is None):
            raise ValueError('begin_planes: pass exactly one of cano_planes and img (the source image, with FrameEngine(img2plane=...))')
        if img is not None and self.img2p is None:
            raise ValueError('begin_planes(img=...) needs FrameEngine(secc2plane=..., img2plane=Img2PlaneModel)')
        if img is not None and (img.ndim != 4 or img.shape[0] != 1):
            raise ValueError(f'begin_planes: img must be one source image [1,3,H,W], got {tuple(img.shape)}')
        if self.secc_r is not None:
            if coeff_src is None or cond_cano is not None or cond_src is not None:
                raise ValueError('secc_renderer engine: begin_planes(cano_planes, coeff_src=c [1,144]) (the engine renders cond_cano / cond_src)')
            c = capi.f32(coeff_src.to(self.device))
            if c.ndim != 2 or c.shape[0] != 1:
                raise ValueError(f'begin_planes: coeff_src must be [1,{self.secc_r.n_id + self.secc_r.n_exp}], got {tuple(c.shape)}')
            cano_c = c.clone()
            cano_c[:, self.secc_r.n_id:] = 0
            cond_src = self.secc_r.render(c)[1]
            cond_cano = self.secc_r.render(cano_c)[1]
        elif coeff_src is not None:
            raise ValueError('coeff_src needs FrameEngine(secc_renderer=...)')
        elif cond_cano is None:
            raise ValueError('begin_planes(cano_planes, cond_cano, cond_src)')
        if img is not None:
            img = img.to(self.device)
            H2 = img.shape[-1] // 2
            old = self._cano_cl
            keep = old is not None and tuple(old.data.shape) == (1, H2, H2, 3, 32)
            cl = self.img2p.planes_cl(img, out=old.data if keep else None)
            if not keep:
                self._cano_cl = cl
                self.graph, self.inplace = None, {}
        else:
            from .secc2plane import canonical_planes_cl
            cl = canonical_planes_cl(cano_planes.to(self.device))
            if self._cano_cl is not None and self._cano_cl.data.shape == cl.data.shape:
                self._cano_cl.data.copy_(cl.data)
            else:
                self._cano_cl = cl
                self.graph, self.inplace = None, {}
        self.secc.begin_clip(cond_cano.to(self.device), None if cond_src is None else cond_src.to(self.device))

    def _planes(self, planes):
        """The render's plane sets: with secc2plane, `planes` is the driving SECC image (or, with a secc_renderer, the coefficients it is
        rendered from) and the backbone runs here (inside the capture)."""
        if self.secc is None:
            return planes
        if self._cano_cl is None:
            raise RuntimeError('secc2plane: call begin_planes(cano_planes, cond_cano, cond_src) before the first step')
        if self.secc_r is not None:
            secc = self.secc_r.render(planes)[1]
            if self.blink:
                self.secc_r.blink(secc, rows=planes[:, self.secc_r.n_id + self.secc_r.n_exp:])
            planes = secc
        if self.debug:
            self._secc_used = planes                                   # the step's driving SECC image: panel 1 of its debug frames
        return (self._cano_cl, self.secc.planes_cl(planes))

    def blink_faults(self) -> int:
        """blink=True engines: the frames left unedited since the last call because the reference raises on them (resets; one sync)."""
        if not self.blink:
            raise ValueError('blink_faults() is for FrameEngine(..., blink=True)')
        return self.secc_r.blink_faults()

    def end_clip(self) -> None:
        """Release the clip's constants, and the graphs that read them."""
        if self.torso:
            self.head.superresolution.end_clip()
        self._consts = None
        self.graph, self.inplace = None, {}

    def _cond(self, kp_d: torch.Tensor) -> Dict[str, torch.Tensor]:
        c = self._consts
        return {'ref_torso_img': c['ref_torso_img'], 'bg_img': c['bg_img'], 'segmap': c['segmap'], 'kp_s': c['kp_s'], 'kp_d': kp_d}

    def _check_kp_d(self, kp_d) -> None:
        if not self.torso:
            if kp_d is not None:
                raise ValueError('kp_d is the per-frame condition of the torso head: this engine runs the plain head (no torso_model)')
            return
        if self._consts is None:
            raise RuntimeError('torso head: call begin_clip(ref_torso_img, bg_img, segmap, kp_s) before the first step')
        if kp_d is None:
            raise ValueError('torso head: every step needs kp_d [B,68,3]')

    @staticmethod
    def _over(u_coarse, u_fine) -> Dict[str, torch.Tensor]:
        over = {'u_coarse': u_coarse}
        if u_fine is not None:
            over['u_fine'] = u_fine
        return over

    @torch.no_grad()
    def _body(self, planes, cameras, u_coarse, u_fine=None, kp_d=None) -> torch.Tensor:
        cond = self._cond(kp_d) if self.torso else None
        if self.debug:
            ret = self.head.synthesis(self._planes(planes), cameras, cond=cond, lean=True, keep_render=True, **self._over(u_coarse, u_fine))
            return self._debug_frames(ret['image'], ret['render_feat'], ret['render_depth'], self._secc_used)
        return self.head.synthesis(self._planes(planes), cameras, cond=cond, lean=True, out_uint8=self.out_uint8, **self._over(u_coarse, u_fine))['image']

    def _debug_frames(self, image, feat, depth, secc):
        """concat_debug: the step's strips with panels 0, 1, 2 and 4 (panel 3 is written into the clip by close_clip), and its depths
        [B,64,64] for the clip.  image: the SR's clamped fp32 frames; the panel kernel converts them as the reference's float64 cat does."""
        B = image.shape[0]
        frames = torch.empty((B,) + DEBUG_FRAME_SHAPE, dtype=torch.uint8, device=self.device)
        debug_panels(self._ref_gt, capi.f32(secc), feat, capi.f32(image), frames)
        return frames, depth.view(B, DEBUG_RES, DEBUG_RES)

    def _capture_graph(self, planes, cameras, u_coarse, u_fine=None, kp_d=None):
        if self.torso and not self.warper_in_graph:
            g, out = self._capture_split(planes, cameras, u_coarse, u_fine, kp_d)
        else:
            g, out = self._capture_whole(planes, cameras, u_coarse, u_fine, kp_d)
        # the renderer's buffers the graph reads and writes (basis, faces, NCC code, key buffer) belong to the graph too: another engine built on
        # the same renderer, or a .to() of it, then cannot free memory the graph keeps writing to
        g.keep_alive = self.secc_r.graph_buffers(_frames_of(planes), blink=self.blink) if self.secc_r is not None else ()
        return g, out

    def _capture_whole(self, planes, cameras, u_coarse, u_fine=None, kp_d=None):
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):                                       # warm-up outside capture: lazy inits (func attributes, driver entry points)
                self._body(planes, cameras, u_coarse, u_fine, kp_d)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        if self._pool is None:
            self._pool = torch.cuda.graph_pool_handle()               # all step graphs share one pool: they never run concurrently
        c0 = capi.lib().r3dp_launch_count()
        with torch.cuda.graph(g, pool=self._pool):
            out = self._body(planes, cameras, u_coarse, u_fine, kp_d)
        self.launches_per_step = int(capi.lib().r3dp_launch_count() - c0)      # libr3dp kernels inside one replay
        return g, out

    def _capture_split(self, planes, cameras, u_coarse, u_fine, kp_d):
        """Torso step as graph A -> eager warper -> graph B (see _TorsoGraphs); returns (graphs, output buffer)."""
        sr, over = self.head.superresolution, self._over(u_coarse, u_fine)
        if self.debug:                                               # graph B writes the debug frames: graph A's render and SECC image stay alive in st
            over['keep_render'] = True

        def pre():
            st = self.head.torso_pre(self._planes(planes), cameras, self._cond(kp_d), self.out_uint8 and not self.debug, **over)
            if self.debug:
                st['debug_secc'] = self._secc_used
            return st

        def post(st, rgb_torso, ret):
            out = sr.forward_post(st, rgb_torso, ret)
            return self._debug_frames(out, st['render_feat'], st['render_depth'], st['debug_secc']) if self.debug else out
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side), torch.no_grad():
            for _ in range(2):                                       # warm-up outside capture, as in _capture_graph
                st = pre()
                rgb_torso, ret = sr.run_torso(st)
                post(st, rgb_torso, ret)
            b_in = tuple(capi.f32(t).clone() for t in (rgb_torso, ret['deformed_torso_hid'], ret['occlusion_2']))
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        if self._pool is None:
            self._pool = torch.cuda.graph_pool_handle()
        a, b = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
        c0 = capi.lib().r3dp_launch_count()
        with torch.no_grad():
            with torch.cuda.graph(a, pool=self._pool):
                st = pre()
            with torch.cuda.graph(b, pool=self._pool):
                out = post(st, b_in[0], {'deformed_torso_hid': b_in[1], 'occlusion_2': b_in[2]})
        self.launches_per_step = int(capi.lib().r3dp_launch_count() - c0)
        return _TorsoGraphs(sr, a, st, b_in, b), out

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
        The tensors are kept referenced (their addresses stay valid); refill them in place between steps.  Returns the number of graphs held.
        The torso head takes (planes, cameras, u_coarse, u_fine, kp_d) tuples; its graphs read kp_d [B,68,3] in place too.  Under fuse mode v3
        the steps run eagerly (see `eager_reason`) and nothing is captured."""
        if not self.use_graph or self.eager_reason is not None:
            return 0
        if self.debug and self._ref_gt is None:
            raise RuntimeError("out_mode='concat_debug': open_clip(frames_per_rank, ref_gt_img=...) before prepare()")
        for item in inputs:
            planes, cameras, u_coarse = item[:3]
            u_fine = item[3] if len(item) > 3 else None
            kp_d = item[4] if len(item) > 4 else None
            self._check_kp_d(kp_d)
            k = (_ptr_key(planes), cameras.data_ptr(), u_coarse.data_ptr(), _ptr_key(u_fine))
            if self.torso:
                k += (kp_d.data_ptr(),)
            if k in self.inplace or len(self.inplace) >= max_graphs or _frames_of(planes) not in (self.batch, 1):
                continue
            if self._needs_fine() and u_fine is None:
                raise ValueError('this head renders with importance samples: prepare() needs u_fine [B*M, S_imp] in every input tuple')
            g, out = self._capture_graph(planes, cameras, u_coarse, u_fine, kp_d)
            self.inplace[k] = (g, out, (planes, cameras, u_coarse, u_fine, kp_d))
        return len(self.inplace)

    @torch.no_grad()
    def step(self, planes, cameras: torch.Tensor, u_coarse: Optional[torch.Tensor] = None, u_fine: Optional[torch.Tensor] = None,
             frame_index: Optional[int] = None, *, kp_d: Optional[torch.Tensor] = None, cond_tgt: Optional[torch.Tensor] = None,
             coeff: Optional[torch.Tensor] = None) -> torch.Tensor:
        """planes [B,3,32,256,256] | PlanesCL | (cano, secc); cameras [B,25]; u_coarse [B,4096,S,1], u_fine [B*4096,S_imp] (drawn here if None)
        -> this rank's frames: fp32 [B,3,512,512] in [-1,1] or uint8 [B,512,512,3]; with exchange='allgather' the gathered
        [world*B,...] (rank-major); with exchange='p2p' the frames are additionally pushed into the open clip at `frame_index`.
        out_mode='concat_debug': this rank's debug strips uint8 [B,512,2560,3], pushed with their depths into the open clip at `frame_index`
        (both required).  Their panel 3 is NOT written: it is normalised over the whole clip, and close_clip() writes it into the clip.
        kp_d [B,68,3]: the frames' driving key points, the torso head's only per-frame condition (torso engines only).
        cond_tgt [B,3,H,W]: the driving SECC image, in place of planes (pass None), for FrameEngine(secc2plane=...).
        coeff [B,144]: the frames' [id | exp] coefficients, in place of cond_tgt, for FrameEngine(secc2plane=..., secc_renderer=...);
        [B,146] = [id | exp | t | T] with blink=True.
        The returned tensor is reused by the next step."""
        if self.secc_r is not None:
            if planes is not None or cond_tgt is not None or coeff is None:
                raise ValueError('secc_renderer engine: step(None, cameras, ..., coeff=c [B,144])')
            K = self.secc_r.n_id + self.secc_r.n_exp + (2 if self.blink else 0)
            if coeff.ndim != 2 or coeff.shape[1] != K:
                raise ValueError(f'step: coeff must be [B,{K}]{" (id | exp | t | T)" if self.blink else ""}, got {tuple(coeff.shape)}')
            planes = coeff
        elif coeff is not None:
            raise ValueError('coeff needs FrameEngine(secc2plane=..., secc_renderer=...)')
        elif self.secc is not None:
            if planes is not None or cond_tgt is None:
                raise ValueError('secc2plane engine: step(None, cameras, ..., cond_tgt=drv_secc)')
            planes = cond_tgt
        elif cond_tgt is not None:
            raise ValueError('cond_tgt needs FrameEngine(secc2plane=...)')
        self._check_kp_d(kp_d)
        if self.debug and (self._clip is None or frame_index is None or not 0 <= frame_index < self._fpr):
            raise RuntimeError("out_mode='concat_debug': every step needs an open clip (open_clip(frames_per_rank, ref_gt_img=...)) and its "
                               f"frame_index in [0, frames_per_rank), got frame_index={frame_index}")
        drawn = u_coarse is None or (u_fine is None and self._needs_fine())
        u_coarse, u_fine = self._draw(cameras.shape[0], cameras.device, u_coarse, u_fine)
        graphable = self.use_graph and capi.PROF is None and cameras.shape[0] == self.batch and self.eager_reason is None
        key = (_ptr_key(planes), cameras.data_ptr(), u_coarse.data_ptr(), _ptr_key(u_fine))
        if self.torso:
            key += (kp_d.data_ptr(),)
        hit = self.inplace.get(key) if (graphable and self.inplace and not drawn) else None
        if hit is not None:
            hit[0].replay()
            out = hit[1]
        elif graphable and isinstance(planes, torch.Tensor):
            if self.graph is None:
                self.s_in = (planes.clone(), cameras.clone(), u_coarse.clone(), None if u_fine is None else u_fine.clone())
                if self.torso:
                    self.s_in += (kp_d.clone(),)
                self.graph, self.s_out = self._capture_graph(*self.s_in)
            for dst, src in zip(self.s_in, (planes, cameras, u_coarse, u_fine, kp_d)):
                if dst is not None and src.data_ptr() != dst.data_ptr():
                    dst.copy_(src, non_blocking=True)
            self.graph.replay()
            out = self.s_out
        else:
            out = self._body(planes, cameras, u_coarse, u_fine, kp_d)
        if self.debug:
            frames, depth = out
            with capi.region('exchange'):
                self._push(frames, frame_index, depth)
            return frames
        if self.exchange == 'allgather':
            if capi.PROF is not None:                                   # profiling pass: serial, so the region time is the collective's own
                gathered = torch.empty((self.world * self.batch,) + tuple(out.shape[1:]), dtype=out.dtype, device=self.device)
                with capi.region('exchange'):
                    self.dist.all_gather_into_tensor(gathered, out.contiguous())
                return gathered
            return self._gather_async(out)
        if (self.exchange == 'p2p' or self.world == 1) and self._clip is not None and frame_index is not None:      # world 1: the clip is local
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
    def open_clip(self, frames_per_rank: int, ref_gt_img: Optional[torch.Tensor] = None) -> Optional[torch.Tensor]:
        """Allocate the output clip [world*frames_per_rank, ...] on rank 0 and map it into every other rank (CUDA IPC); returns the clip on
        rank 0, None elsewhere.  Frame f of rank r lands at clip[r*frames_per_rank + f].  With world == 1 the clip is a local buffer.
        out_mode='concat_debug': ref_gt_img [1,3,512,512] is the source image of panel 0 (real3d_infer.py's ref_gt_img), and rank 0 also
        holds the clip's depths [world*frames_per_rank,64,64] for close_clip()."""
        if self.debug:
            if ref_gt_img is None or tuple(ref_gt_img.shape) != (1, 3, 512, 512):
                raise ValueError("out_mode='concat_debug': open_clip(frames_per_rank, ref_gt_img=[1,3,512,512]), got "
                                 f"{None if ref_gt_img is None else tuple(ref_gt_img.shape)}")
            if self._ref_gt is None:
                self._ref_gt = torch.empty(1, 3, 512, 512, device=self.device)
            self._ref_gt.copy_(ref_gt_img)                             # in place: graphs captured for an earlier clip read the new image
        elif ref_gt_img is not None:
            raise ValueError("ref_gt_img is panel 0 of the debug frames: FrameEngine(out_mode='concat_debug')")
        shape = (self.world * frames_per_rank,) + self.frame_shape()
        dshape = (self.world * frames_per_rank, DEBUG_RES, DEBUG_RES)
        self._fpr = frames_per_rank
        if self.world == 1 or self.exchange != 'p2p':
            self._clip = torch.empty(shape, dtype=self.frame_dtype(), device=self.device) if self.rank == 0 else None
            self._clip_view = self._clip
            self._clip_depth = torch.empty(dshape, device=self.device) if self.debug and self.rank == 0 else None
            self._p2p = None
            return self._clip
        from torch.multiprocessing.reductions import reduce_tensor
        payload = [None]
        if self.rank == 0:
            self._clip = torch.empty(shape, dtype=self.frame_dtype(), device=self.device)
            self._clip_depth = torch.empty(dshape, device=self.device) if self.debug else None
            payload = [(reduce_tensor(self._clip), None if self._clip_depth is None else reduce_tensor(self._clip_depth))]
        self.dist.broadcast_object_list(payload, src=0)
        if self.rank == 0:
            self._clip_view = self._clip
        else:
            (fn, args), dep = payload[0]
            self._clip_view = fn(*args)                                # rank 0's buffer, mapped into this process (lives on rank 0's device)
            self._clip = self._clip_view                               # pushes only; never read here
            self._clip_depth = dep[0](*dep[1]) if dep is not None else None
        self._p2p = {'stream': torch.cuda.Stream(device=self.device), 'k': 0, 'stage': None,
                     'done': [torch.cuda.Event() for _ in range(2)], 'ready': [torch.cuda.Event() for _ in range(2)]}
        for e in self._p2p['done']:
            e.record(torch.cuda.current_stream())
        return self._clip if self.rank == 0 else None

    def _push(self, out: torch.Tensor, frame_index: int, depth: Optional[torch.Tensor] = None) -> None:
        """Frames (and, for concat_debug, their depths [B,64,64]) into the clip at this rank's frame_index."""
        n = min(out.shape[0], self._fpr - frame_index)
        if n <= 0:
            return
        g0 = self.rank * self._fpr + frame_index
        pairs = [(out, self._clip_view)] + ([(depth, self._clip_depth)] if depth is not None else [])
        if self._p2p is None:                                          # single rank / local clip: plain device copy on the compute stream
            for src, clip in pairs:
                clip[g0:g0 + n].copy_(src[:n], non_blocking=True)
            return
        p = self._p2p
        k = p['k'] & 1
        p['k'] += 1
        cur = torch.cuda.current_stream()
        if p['stage'] is None:
            p['stage'] = [[torch.empty_like(src) for src, _ in pairs] for _ in range(2)]
        cur.wait_event(p['done'][k])
        for stage, (src, _) in zip(p['stage'][k], pairs):
            stage[:src.shape[0]].copy_(src, non_blocking=True)         # the graph's output buffer is rewritten by the next replay
        p['ready'][k].record(cur)
        with torch.cuda.stream(p['stream']):
            p['stream'].wait_event(p['ready'][k])
            for stage, (_, clip) in zip(p['stage'][k], pairs):
                dst, src = clip[g0:g0 + n], stage[:n]
                # peer copy over NVLink by the copy engine (no SMs), enqueued directly: torch's cross-device copy_ brackets every copy with
                # event record/wait pairs on BOTH devices' current streams (measured: 1.3 ms/step of host-side stalls at 2 GPUs)
                capi.check(capi.lib().r3dp_peer_copy(dst.data_ptr(), dst.device.index, src.data_ptr(), src.device.index,
                                                     src.numel() * src.element_size(), capi.stream()))
            p['done'][k].record(p['stream'])

    def close_clip(self) -> Optional[torch.Tensor]:
        """Wait until every rank's pushes have landed; returns the finished clip on rank 0.  concat_debug: rank 0 then writes every frame's
        depth panel, normalised by the min and max over the whole clip (two launches on the current stream)."""
        self.wait_gather()
        torch.cuda.synchronize(self.device)
        if self.world > 1 and self.dist is not None:
            self.dist.barrier()
        clip = self._clip if self.rank == 0 else None
        if self.debug and self.rank == 0 and clip is not None:
            depth_panel(self._clip_depth, clip)
        if self.rank != 0 and getattr(self, '_p2p', None) is not None:      # drop this process's mapping of rank 0's buffer before rank 0 may free it
            self._clip_view = self._clip = self._clip_depth = None
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
                  h_u_fine: Optional[torch.Tensor] = None, h_kp_d: Optional[torch.Tensor] = None) -> None:
        """Same step, from PINNED HOST tensors to a pinned host output (frames of THIS rank), fully asynchronous: the call
        enqueues H2D (copy-in stream) -> step (current stream) -> D2H (copy-out stream) and returns; with two staging slots the
        copy of step i+1 runs under the compute of step i.  Call `sync_host()` before reading `h_out`.  h_kp_d: the torso head's kp_d."""
        if self.debug:
            raise NotImplementedError("out_mode='concat_debug' collects a device-resident clip; step_host() has no clip design for it")
        self._check_kp_d(h_kp_d)
        hp = self._host_pipeline()
        k = hp['k'] & 1
        hp['k'] += 1
        cur = torch.cuda.current_stream()
        hosts = (h_planes, h_cameras, h_u) + ((h_u_fine,) if h_u_fine is not None else ())
        if self.torso:
            hosts = hosts[:3] + (h_u_fine, h_kp_d)                     # prepare()'s torso tuple: u_fine may be None
        if hp['stage'][k] is None:
            hp['stage'][k] = tuple(None if h is None else torch.empty_like(h, device=self.device) for h in hosts)
            hp['out'][k] = torch.empty((self.batch,) + self.frame_shape(), dtype=self.frame_dtype(), device=self.device)
            for dst, src in zip(hp['stage'][k], hosts):
                if dst is not None:
                    dst.copy_(src)                                     # warm-up / capture run on REAL inputs (uninitialised cameras give NaN depths)
            self.prepare([hp['stage'][k]])                             # the step reads the staging slot in place (no device-side input copy)
            hp['in_free'][k].record(cur); hp['out_free'][k].record(cur)
        stage = hp['stage'][k]
        with torch.cuda.stream(hp['copy_in']):
            hp['copy_in'].wait_event(hp['in_free'][k])                 # the step that last read this slot is done
            for dst, src in zip(stage, hosts):
                if dst is not None:
                    dst.copy_(src, non_blocking=True)
            hp['in_ready'][k].record(hp['copy_in'])
        cur.wait_event(hp['in_ready'][k])
        # secc2plane: h_planes is the driving SECC image, or the coefficients it is rendered from with a secc_renderer
        p0, tgt = (None, {'coeff' if self.secc_r is not None else 'cond_tgt': stage[0]}) if self.secc is not None else (stage[0], {})
        out = self.step(p0, *stage[1:4], kp_d=stage[4], **tgt) if self.torso else self.step(p0, *stage[1:], **tgt)
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
        kernel = 'conv_tc3_kernel (wgmma implicit-GEMM conv, 2-row tiles)' if tc else 'conv_taps_kernel (fp32 CUDA-core direct conv)'
        return {'stages': stages, 'sr_conv_ms': stages.get('sr_conv', float('nan')), 'total_ms': a.elapsed_time(b), 'sr_kernel': kernel,
                'conv_kernel_ms': conv_ms, 'conv_launches': conv_n}
