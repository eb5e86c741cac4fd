"""Restoration-forward pipeline = the reference's `RefRestorationModel.test()`
(mmsr/models/ref_restoration_model.py:271-279): extractor -> correspondence -> restoration,
as one object that bench.py, smoke() and the tests drive.  One instance per process/GPU."""
import torch
import torch.nn.functional as F

from mmsr.models.archs.contras_extractor_arch import ContrasExtractorSep
from mmsr.models.archs.corres_generation_arch import CorrespondenceGenerationArch
from mmsr.models.archs.ref_restoration_arch import RestorationNet


def synthetic_pair(seed, batch, lr_size, ref_size, device='cpu', generator_device='cpu'):
    """SURVEY.md §8(d) recipe: LR ~ U[0,1), `img_in_up` = bicubic x4 of LR clamped to [0,1], Ref ~ U[0,1)
    zero-padded bottom/right to the HR size (as the dataset does, ref_cufed_dataset.py:106-114)."""
    g = torch.Generator(device=generator_device).manual_seed(seed)
    hr = 4 * lr_size
    img_lq = torch.rand(batch, 3, lr_size, lr_size, generator=g, device=generator_device)
    ref = torch.rand(batch, 3, ref_size, ref_size, generator=g, device=generator_device)
    img_up = F.interpolate(img_lq, scale_factor=4, mode='bicubic', align_corners=False).clamp_(0, 1)
    img_ref = F.pad(ref, (0, hr - ref_size, 0, hr - ref_size))
    return img_lq.to(device), img_up.to(device), img_ref.to(device)


class RestorationPipeline:

    def __init__(self, device, ngf=64, n_blocks=16, groups=8, channels_last=False, allow_tf32=False, cuda_graph=False):
        self.device = torch.device(device)
        if self.device.type != 'cuda':
            raise RuntimeError('RestorationPipeline needs a CUDA device (no CPU fallback for the H100 hot path)')
        self.net_extractor = ContrasExtractorSep()
        self.net_map = CorrespondenceGenerationArch(3, 1, ['relu1_1', 'relu2_1', 'relu3_1'], 'vgg19')
        self.net_g = RestorationNet(ngf=ngf, n_blocks=n_blocks, groups=groups)
        self.channels_last = channels_last
        self.allow_tf32 = allow_tf32
        # cuda_graph: the ~190 launches of a forward are captured once per input shape and replayed (no change in the
        # arithmetic: bit-identical results; removes the launch gaps between the dependent kernels, ~2 % of a step)
        self.cuda_graph = bool(cuda_graph)
        self._graphs = {}
        self._graph_stream = None
        self._placed = False

    def nets(self):
        return self.net_extractor, self.net_map, self.net_g

    def load_state_dicts(self, sd_extractor=None, sd_map=None, sd_g=None, strict=True):
        for net, sd in zip(self.nets(), (sd_extractor, sd_map, sd_g)):
            if sd is not None:
                net.load_state_dict(sd, strict=strict)
        return self

    def place(self):
        mf = torch.channels_last if self.channels_last else torch.contiguous_format
        for net in self.nets():
            net.to(self.device).eval()
            if self.channels_last:
                net.to(memory_format=mf)
        self._placed = True
        return self

    @torch.no_grad()
    def forward(self, img_in_lq, img_in_up, img_ref, return_idx=False, check_finite=False):
        """Device tensors in, SR device tensor out.  check_finite: synchronise and raise if the result contains inf / NaN
        (a packed-split activation that left the fp16 range shows up there; off on the timed path)."""
        if not self._placed:
            self.place()
        prev = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = self.allow_tf32
        try:
            if self.channels_last:
                img_in_lq = img_in_lq.contiguous(memory_format=torch.channels_last)
                img_in_up = img_in_up.contiguous(memory_format=torch.channels_last)
                img_ref = img_ref.contiguous(memory_format=torch.channels_last)
            feats = self.net_extractor(img_in_up, img_ref)
            pre_offset, ref_feat = self.net_map(feats, img_ref)
            sr = self.net_g(img_in_lq, pre_offset, ref_feat)
        finally:
            torch.backends.cudnn.allow_tf32 = prev
        if check_finite and not bool(torch.isfinite(sr).all()):
            raise RuntimeError('non-finite SR output: an activation left the fp16 range of the packed-split layout '
                               '(see c2m_b200.ops.suggest_sa) or the inputs were not finite')
        return (sr, pre_offset.max_idx) if return_idx else sr

    # -- CUDA-graph replay of the forward (opt-in)
    def _capture(self, shapes, static_in):
        # two eager passes first (weight packing, scale-exponent calibration, allocator warm-up), then a quiet device
        torch.cuda.synchronize(self.device)
        gs = self._graph_stream
        gs.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(gs):
            for _ in range(2):
                self.forward(*static_in)
            torch.cuda.synchronize(self.device)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=gs):
                static_out = self.forward(*static_in, return_idx=True)
        torch.cuda.current_stream(self.device).wait_stream(gs)
        torch.cuda.synchronize(self.device)
        ent = (g, static_in, static_out)
        self._graphs[shapes] = ent
        return ent

    @torch.no_grad()
    def forward_graphed(self, img_in_lq, img_in_up, img_ref, return_idx=False):
        """`forward` through a CUDA graph captured per input-shape triple.  The first call for a shape captures (with
        these inputs as calibration data if nothing ran before); the returned tensors are the graph's static outputs
        and are overwritten by the next replay of the same shape."""
        if not self._placed:
            self.place()
        shapes = tuple(tuple(t.shape) for t in (img_in_lq, img_in_up, img_ref))
        ent = self._graphs.get(shapes)
        if ent is None:
            static_in = [t.detach().to(self.device, torch.float32).clone() for t in (img_in_lq, img_in_up, img_ref)]
            if self._graph_stream is None:
                self._graph_stream = torch.cuda.Stream(self.device)
            ent = self._capture(shapes, static_in)
        g, static_in, (sr, idx) = ent
        for dst, src in zip(static_in, (img_in_lq, img_in_up, img_ref)):
            if dst.data_ptr() != src.data_ptr():
                dst.copy_(src, non_blocking=True)
        g.replay()
        return (sr, idx) if return_idx else sr

    @torch.no_grad()
    def run_host(self, img_in_lq, img_in_up, img_ref, out=None):
        """Public end-to-end call: (pinned) HOST tensors in -> HOST SR tensor out; the H2D and
        D2H copies are part of the call."""
        nb = dict(non_blocking=True)
        if self.cuda_graph:
            # H2D straight into the graph's static inputs, replay, D2H
            shapes = tuple(tuple(t.shape) for t in (img_in_lq, img_in_up, img_ref))
            if shapes not in self._graphs:
                self.forward_graphed(img_in_lq.to(self.device, **nb), img_in_up.to(self.device, **nb),
                                     img_ref.to(self.device, **nb))
            g, static_in, (sr, _) = self._graphs[shapes]
            for dst, src in zip(static_in, (img_in_lq, img_in_up, img_ref)):
                dst.copy_(src, non_blocking=True)
            g.replay()
        else:
            sr = self.forward(img_in_lq.to(self.device, **nb), img_in_up.to(self.device, **nb),
                              img_ref.to(self.device, **nb))
        if out is None:
            out = torch.empty(sr.shape, dtype=sr.dtype, pin_memory=True)
        out.copy_(sr, non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        return out
