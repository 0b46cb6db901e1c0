"""Meta-architectures with the reference's forward() contracts.

GeneralizedRCNN       -- detector/generalized_rcnn.py:16-65 (single frame)
GeneralizedRCNNMEGA   -- detector/generalized_rcnn_mega.py:21-225 (per-video state machine)
GeneralizedRCNNRDN    -- detector/generalized_rcnn_rdn.py:20-190 (per-video state machine, 37-frame window)
GeneralizedRCNNFGFA   -- detector/generalized_rcnn_fgfa.py:19-219 (flow-guided aggregation over a 19-frame window)
GeneralizedRCNNDFF    -- detector/generalized_rcnn_dff.py:19-138 (key-frame features warped along FlowNetS flow)

`forward(images)` returns `list[BoxList]` (fields `scores`, `labels`) exactly like the reference in
eval mode -- under MODEL.RPN_ONLY (single-frame, FGFA and DFF) the proposals instead, field `objectness`, in descending
objectness order (generalized_rcnn.py:51-55, rpn/rpn.py:186-197); the arithmetic runs in the B200 engine built lazily from this module's own state_dict
(so weights loaded with load_state_dict / DetectronCheckpointer are what the kernels use).
"""
import torch
from torch import nn

from ..nets import EmbedNet, FlowNetS, build_backbone, build_roi_heads, build_rpn, engine_config_from
from ...b200 import engine as _engine
from ...structures.bounding_box import BoxList
from ...structures.image_list import to_image_list


class _EngineBacked(nn.Module):
    engine_cls = None

    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg.clone()
        self.device = torch.device(cfg.MODEL.DEVICE)
        self.backbone = build_backbone(cfg)
        self.rpn = build_rpn(cfg, self.backbone.out_channels)
        self.roi_heads = build_roi_heads(cfg, self.backbone.out_channels)
        extractor = (self.roi_heads["box"].feature_extractor,) if self.roi_heads else ()
        for sub in (self.backbone, self.rpn) + extractor:
            if hasattr(sub, "_bind"):        # callable sub-modules (model.rpn(...), feature_extractor(..., pre_calculate=True))
                sub._bind(self)
        self._engine = None
        self._sd_override = None
        self.d2h_bytes_per_frame = 0

    def adopt_state_dict(self, sd):
        self._sd_override = {k: v for k, v in sd.items()}
        self._engine = None

    def load_state_dict(self, *a, **k):
        self._engine = None
        return super().load_state_dict(*a, **k)

    @property
    def engine(self):
        if self._engine is None:
            if self.device.type != "cuda":
                raise RuntimeError("mega_core (B200 build) runs on CUDA only; MODEL.DEVICE=%s" % self.device)
            sd = self._sd_override if self._sd_override is not None else self.state_dict()
            self._engine = self.engine_cls(sd, engine_config_from(self.cfg), self.device)
        return self._engine

    def _to_boxlist(self, det, im_w, im_h):
        n = int(det.count.item())
        out = BoxList(det.boxes[:n].clone(), (int(im_w), int(im_h)), mode="xyxy")
        if isinstance(det, _engine.Proposals):
            out.add_field("objectness", det.objectness[:n].clone())
            self.d2h_bytes_per_frame = 4 + n * (16 + 4)
            return out
        out.add_field("scores", det.scores[:n].clone())
        out.add_field("labels", det.labels[:n].clone())
        self.d2h_bytes_per_frame = 4 + n * (16 + 4 + 8)
        return out

    def _dev(self, t):
        t = t.tensors if hasattr(t, "tensors") else t
        if t.dim() == 3:
            t = t[None]
        return t.to(self.device, non_blocking=True).float().contiguous()


class GeneralizedRCNN(_EngineBacked):
    engine_cls = _engine.BaseEngine

    def forward(self, images, targets=None):
        if self.training:
            raise NotImplementedError("the B200 build covers inference (eval mode) only")
        images = to_image_list(images)
        out = []
        with torch.no_grad():
            for i, (h, w) in enumerate(images.image_sizes):
                det = self.engine.forward(self._dev(images.tensors[i][:, :h, :w]), w, h)
                out.append(self._to_boxlist(det, w, h))
        return out


class GeneralizedRCNNMEGA(_EngineBacked):
    engine_cls = _engine.MegaEngine

    def forward(self, images, targets=None):
        """images: the dict VIDMEGADataset._get_test builds (data/datasets/vid_mega.py:132-140):
        cur, ref_l, ref_g, frame_category, seg_len, pattern, img_dir, transforms. Optional extra key
        `lookahead` (list of 12 pre-staged frames) replaces the disk reads of frame 0
        (generalized_rcnn_mega.py:183-193) for synthetic / benchmark streams."""
        if self.training:
            raise NotImplementedError("the B200 build covers inference (eval mode) only")
        if targets is not None:
            raise ValueError("In testing mode, targets should be None")
        cur = to_image_list(images["cur"])
        im_h, im_w = cur.image_sizes[0]
        eng = self.engine
        with torch.no_grad():
            if images["frame_category"] == 0:
                self.seg_len, self.end_id = images["seg_len"], 0
                look = images.get("lookahead")
                if look is None:
                    look = self._read_lookahead(images, eng.L - eng.cfg.key_frame_location - 1)
                det = eng.start_video(self._dev(cur), [self._dev(x) for x in look],
                                      [self._dev(g) for g in images["ref_g"]], im_w, im_h)
            else:
                self.end_id = min(getattr(self, "end_id", 0) + 1, getattr(self, "seg_len", 1) - 1)
                assert len(images["ref_l"]) == 1 and len(images["ref_g"]) == 1, \
                    "steady-state frames carry one look-ahead local frame and one global frame"
                pair = eng.static_input((2,) + tuple(cur.tensors.shape[1:]))
                pair[0].copy_(self._host(images["ref_l"][0]), non_blocking=True)
                pair[1].copy_(self._host(images["ref_g"][0]), non_blocking=True)
                det = eng.step_batched(pair, im_w, im_h)
        return [self._to_boxlist(det, im_w, im_h)]

    def forward_frames(self, images_list, prefetch=None):
        """Offline streams (tools/test_net.py reads every frame from disk, so the frames after `cur` are at hand):
        n consecutive steady-state frames (each the dict forward() takes, frame_category 1) in ONE call. The per-frame
        branch -- backbone / RPN / res5 / ROIAlign / l_fcs[0], a pure function of each frame -- runs as one batch of
        2n images (MegaEngine.stepn_batched), the n aggregations in order. Returns n results, each what forward()
        returns for that frame; n <= MegaEngine.MAX_FRAMES_PER_STEP.
        prefetch: the images_list of the NEXT call (or None at the end of the stream). The per-frame branch of those frames
        then runs WHILE this call's frames are aggregated (MegaEngine.stepn_pipelined: two streams sharing the GPU by SMs),
        and the next call -- which must be given exactly that list -- finds it done."""
        if self.training:
            raise NotImplementedError("the B200 build covers inference (eval mode) only")
        eng = self.engine
        n = len(images_list)
        assert all(im["frame_category"] == 1 and len(im["ref_l"]) == 1 and len(im["ref_g"]) == 1 for im in images_list), \
            "forward_frames takes steady-state frames (one look-ahead local frame and one global frame each)"
        cur = to_image_list(images_list[0]["cur"])
        im_h, im_w = cur.image_sizes[0]

        def stage(lst):
            buf = eng.static_input((2 * len(lst),) + tuple(cur.tensors.shape[1:]))
            for i, im in enumerate(lst):
                buf[2 * i].copy_(self._host(im["ref_l"][0]), non_blocking=True)
                buf[2 * i + 1].copy_(self._host(im["ref_g"][0]), non_blocking=True)
            return buf

        with torch.no_grad():
            for _ in images_list:
                self.end_id = min(getattr(self, "end_id", 0) + 1, getattr(self, "seg_len", 1) - 1)
            pending = getattr(self, "_prefetched", 0)
            if prefetch is None and not pending:
                dets = eng.stepn_batched(stage(images_list), im_w, im_h)
            else:
                if not pending:                                   # first call of a pipelined stream: its own branch now
                    eng.stepn_pipelined(stage(images_list), im_w, im_h)
                else:
                    assert pending == n, "this call's frames are not the ones the previous call prefetched"
                dets = eng.stepn_pipelined(stage(prefetch) if prefetch else None, im_w, im_h)
                self._prefetched = len(prefetch) if prefetch else 0
        out, d2h = [], 0
        for det in dets:
            out.append([self._to_boxlist(det, im_w, im_h)])
            d2h += self.d2h_bytes_per_frame
        self.d2h_bytes_per_frame = d2h / n
        return out

    @staticmethod
    def _host(t):
        t = t.tensors if hasattr(t, "tensors") else t
        return t[0] if t.dim() == 4 else t

    def _read_lookahead(self, infos, n):
        """frame 0 of a video: the reference opens the next frames from disk inside the model"""
        from PIL import Image
        names = []
        for _ in range(n):
            self.end_id = min(self.end_id + 1, self.seg_len - 1)
            names.append(infos["img_dir"] % (infos["pattern"] % self.end_id))
        transform = infos["transforms"]
        if getattr(transform, "jpeg_decode", "pil") == "device":           # MODEL.B200.JPEG_DECODE: one decode batch
            from ...data.transforms import EncodedImage
            encoded = []
            for name in names:
                with open(name, "rb") as f:
                    encoded.append(EncodedImage(f.read()))
            images = transform.decode_batch(encoded)
        else:
            images = (Image.open(name).convert("RGB") for name in names)
        frames = []
        for img in images:
            img = transform(img)
            if isinstance(img, tuple):
                img = img[0]
            frames.append(img.view(1, *img.shape))
        return frames


class GeneralizedRCNNRDN(GeneralizedRCNNMEGA):
    engine_cls = _engine.RdnEngine

    def forward(self, images, targets=None):
        """images: the dict VIDRDNDataset._get_test builds (data/datasets/vid_rdn.py): cur, ref (one look-ahead
        frame for frame_category 1), frame_category, seg_len, pattern, img_dir, transforms; optional `lookahead`
        (list of 18 pre-staged frames) replaces the disk reads of frame 0 (generalized_rcnn_rdn.py:154-164)."""
        if self.training:
            raise NotImplementedError("the B200 build covers inference (eval mode) only")
        if targets is not None:
            raise ValueError("In testing mode, targets should be None")
        cur = to_image_list(images["cur"])
        im_h, im_w = cur.image_sizes[0]
        eng = self.engine
        with torch.no_grad():
            if images["frame_category"] == 0:
                self.seg_len, self.end_id = images["seg_len"], 0
                look = images.get("lookahead")
                if look is None:
                    look = self._read_lookahead(images, eng.L - eng.cfg.key_frame_location - 1)
                det = eng.start_video(self._dev(cur), [self._dev(x) for x in look], im_w, im_h)
            else:
                self.end_id = min(getattr(self, "end_id", 0) + 1, getattr(self, "seg_len", 1) - 1)
                assert len(images["ref"]) == 1, "steady-state frames carry one look-ahead frame"
                buf = eng.static_input((1,) + tuple(cur.tensors.shape[1:]))
                buf[0].copy_(self._host(images["ref"][0]), non_blocking=True)
                det = eng.step(buf, im_w, im_h)
        return [self._to_boxlist(det, im_w, im_h)]


class GeneralizedRCNNFGFA(GeneralizedRCNNRDN):
    """same call contract as the RDN detector (images dict with cur / ref / frame_category / ...); the module tree
    additionally holds `flownet` and `embednet` (detector/generalized_rcnn_fgfa.py:30-35)"""
    engine_cls = _engine.FgfaEngine

    def __init__(self, cfg):
        super().__init__(cfg)
        self.flownet = FlowNetS(cfg)
        self.embednet = EmbedNet(cfg)


class GeneralizedRCNNDFF(_EngineBacked):
    """images: the dict VIDDFFDataset._get_test builds (data/datasets/vid_dff.py:48-67): `cur` and `is_key_frame`"""
    engine_cls = _engine.DffEngine

    def __init__(self, cfg):
        super().__init__(cfg)
        self.flownet = FlowNetS(cfg)

    def forward(self, images, targets=None):
        if self.training:
            raise NotImplementedError("the B200 build covers inference (eval mode) only")
        if targets is not None:
            raise ValueError("In testing mode, targets should be None")
        cur = to_image_list(images["cur"])
        im_h, im_w = cur.image_sizes[0]
        with torch.no_grad():
            det = self.engine.forward(self._dev(cur), bool(images["is_key_frame"]), im_w, im_h)
        return [self._to_boxlist(det, im_w, im_h)]
