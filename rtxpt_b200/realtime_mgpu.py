"""BASELINE configs[2] (realtime mode + NEE-AT + ReBLUR + tone map) on several GPUs: the frame recipe of include/rtxpt_b200.h ("The realtime frame on several GPUs"), SURVEY.md §8e.
Every rank traces the screen tiles it owns; three kinds of per-pixel images cross ranks, each as ONE all-gather of packed tiles:
    guides (depth, specular hit distance, per plane branch ID + normal: what the guide filter and the disocclusion relaxation read of a pixel's neighbours) -> per plane the seven NRD input images -> the merged output colour.
ReBLUR runs on the whole frame on every rank (2.8 ms at 1080p against 32 ms of tracing on one GPU): all ranks feed it the same inputs, so their histories stay identical
and no history exchange is needed.  `LocalGroup` drives all ranks from one process (contexts on one or several devices, the exchange is a device copy: tests, single-GPU
emulation); `DistGroup` is one rank of a torchrun job (torch.distributed.all_gather_into_tensor over NCCL)."""
import numpy as np
from . import structs as S

GUIDES = [S.BUFFER_DEPTH_F32, S.BUFFER_SPECULAR_HITT_F32, S.BUFFER_STABLE_PLANE_NEIGHBOUR_GUIDES]
NRD_INPUTS = [S.BUFFER_DENOISER_VIEWSPACE_Z_F32, S.BUFFER_DENOISER_MOTION_VECTORS_F16, S.BUFFER_DENOISER_NORMAL_ROUGHNESS_R10G10B10A2, S.BUFFER_DENOISER_DIFF_RADIANCE_HITDIST_F16,
              S.BUFFER_DENOISER_SPEC_RADIANCE_HITDIST_F16, S.BUFFER_DENOISER_DISOCCLUSION_MIX_R8, S.BUFFER_COMBINED_HISTORY_CLAMP_RELAX_R8]
OUTPUT = [S.BUFFER_OUTPUT_COLOR_F16]


class LocalGroup:
    """All ranks in this process: `contexts[r]` was created with tile_rank = r, tile_world = len(contexts)."""
    def __init__(self, contexts):
        import torch
        self.torch = torch; self.ctxs = list(contexts); self.world = len(self.ctxs); self.buf = {}

    def each(self, fn):
        for c in self.ctxs: fn(c)

    def exchange(self, buffers):
        key = tuple(buffers); n = self.ctxs[0].exchange_bytes(buffers)
        if key not in self.buf: self.buf[key] = self.torch.empty((self.world, n), dtype=self.torch.uint8, device="cuda")
        g = self.buf[key]
        for c in self.ctxs: c.synchronize()                       # nobody is still reading the previous exchange out of this buffer
        for r, c in enumerate(self.ctxs): c.exchange_pack(buffers, g[r].data_ptr())
        for c in self.ctxs: c.synchronize()                       # the copies of all ranks are in place before anyone reads them
        for c in self.ctxs: c.exchange_unpack(buffers, g.data_ptr())
        return self.world * n


class DistGroup:
    """One rank of a torch.distributed job (backend nccl); `stream` = the torch stream all of this rank's GPU work is queued on - it must also be torch's CURRENT stream
    (torch.cuda.set_stream), because NCCL orders the all-gather against the current stream."""
    def __init__(self, ctx, stream=None):
        import torch, torch.distributed as dist
        self.torch = torch; self.dist = dist; self.ctxs = [ctx]; self.world = dist.get_world_size(); self.buf = {}
        self.stream = stream.cuda_stream if stream is not None else None

    def each(self, fn):
        fn(self.ctxs[0])

    def exchange(self, buffers):
        c = self.ctxs[0]; key = tuple(buffers); n = c.exchange_bytes(buffers)
        if key not in self.buf: self.buf[key] = (self.torch.empty(n, dtype=self.torch.uint8, device="cuda"), self.torch.empty(self.world * n, dtype=self.torch.uint8, device="cuda"))
        send, gathered = self.buf[key]
        c.exchange_pack(buffers, send.data_ptr(), self.stream)
        self.dist.all_gather_into_tensor(gathered, send)
        c.exchange_unpack(buffers, gathered.data_ptr(), self.stream)
        return self.world * n


def realtime_frame(group, denoiser_constants, reblur_frame, tone_mapping=None, feedback=False, planes=3, reblur_settings=None):
    """One frame of Sample::Render in realtime mode on `group`'s ranks (constants, view and realtime constants already set on every context).  Returns the bytes all-gathered.
    reblur_settings (structs.ReblurSettings, RTXPT's m_ui.ReblurSettings): applied on every rank before this frame, so that their histories stay identical."""
    stream = getattr(group, "stream", None); moved = 0
    if reblur_settings is not None: group.each(lambda c: c.set_reblur_settings(reblur_settings))
    if feedback: group.each(lambda c: c.neeat_update_begin(stream))
    group.each(lambda c: c.path_trace_realtime(False, stream))
    moved += group.exchange(GUIDES)
    group.each(lambda c: c.denoise_spec_hit_t(stream))
    first = True
    for plane in range(planes - 1, -1, -1):
        group.each(lambda c: c.denoiser_prepare_inputs(plane, first, denoiser_constants, stream))
        moved += group.exchange(NRD_INPUTS)
        group.each(lambda c: c.reblur_denoise(plane, reblur_frame, stream))
        group.each(lambda c: c.denoiser_final_merge(plane, stream=stream, identity=False))
        first = False
    moved += group.exchange(OUTPUT)
    if tone_mapping is not None: group.each(lambda c: c.tone_map(tone_mapping, stream=stream))
    return moved
