"""ImageNet-VID / DET datasets, test-time side, with the reference's class names and item contracts
(data/datasets/vid.py, vid_mega.py, vid_rdn.py, vid_fgfa.py, vid_dff.py). Host-side file handling only: frame lists,
XML annotations (cached as <data_dir>/cache/<image_set>_anno.pkl like the reference), PIL decoding, and the per-method
dict `model(images)` consumes. One module instead of five files: the four video methods differ only in which extra
frames a test item carries. Training items (`_get_train` with random reference frames) are not provided."""
import os
import pickle
import xml.etree.ElementTree as ET

import numpy as np
import torch
import torch.utils.data
from PIL import Image

from ...config import cfg
from ...structures.bounding_box import BoxList
from ...utils.comm import is_main_process
from ..transforms.jpeg import EncodedImage

_NAMES = ("__background__ airplane antelope bear bicycle bird bus car cattle dog domestic_cat elephant fox giant_panda "
          "hamster horse lion lizard monkey motorcycle rabbit red_panda sheep snake squirrel tiger train turtle watercraft "
          "whale zebra").split()
_WNIDS = ("__background__ n02691156 n02419796 n02131653 n02834778 n01503061 n02924116 n02958343 n02402425 n02084071 "
          "n02121808 n02503517 n02118333 n02510455 n02342885 n02374451 n02129165 n01674464 n02484322 n03790512 n02324045 "
          "n02509815 n02411705 n01726692 n02355227 n02129604 n04468005 n01662784 n04530566 n02062744 n02391049").split()


class VIDDataset(torch.utils.data.Dataset):
    """single-frame items (method "base"): (image, target, idx) -- data/datasets/vid.py:21-231"""
    classes = list(_NAMES)
    classes_map = list(_WNIDS)

    def __init__(self, image_set, data_dir, img_dir, anno_path, img_index, transforms, is_train=True):
        self.det_vid = image_set.split("_")[0]
        self.image_set, self.transforms, self.is_train = image_set, transforms, is_train
        self.data_dir, self.img_dir, self.anno_path, self.img_index = data_dir, img_dir, anno_path, img_index
        self._img_dir = os.path.join(img_dir, "%s.JPEG")
        self._anno_path = os.path.join(anno_path, "%s.xml")
        with open(img_index) as f:
            rows = [line.strip().split(" ") for line in f.readlines()]
        if len(rows[0]) == 2:                              # DET-style list: "<name> <frame id>"
            self.image_set_index = [r[0] for r in rows]
            self.frame_id = [int(r[1]) for r in rows]
        else:                                              # video list: "<video dir> <frame id> <index in video> <length>"
            self.image_set_index = ["%s/%06d" % (r[0], int(r[2])) for r in rows]
            self.pattern = [r[0] + "/%06d" for r in rows]
            self.frame_id = [int(r[1]) for r in rows]
            self.frame_seg_id = [int(r[2]) for r in rows]
            self.frame_seg_len = [int(r[3]) for r in rows]
        if is_train:
            raise NotImplementedError("mega_core.data (B200 build): test-time datasets only")
        self.classes_to_ind = dict(zip(self.classes_map, range(len(self.classes_map))))
        self.categories = dict(zip(range(len(self.classes)), self.classes))
        self.annos = self.load_annos(os.path.join(self.cache_dir, image_set + "_anno.pkl"))

    def __len__(self):
        return len(self.image_set_index)

    def __getitem__(self, idx):
        return self._get_test(idx)

    # ---- images
    def _open(self, name):
        if getattr(self.transforms, "jpeg_decode", "pil") == "device":       # MODEL.B200.JPEG_DECODE
            with open(self._img_dir % name, "rb") as f:
                return EncodedImage(f.read())
        return Image.open(self._img_dir % name).convert("RGB")

    def _transformed(self, idx, img, extra):
        """(current image, target) and every list of extra frames through the transform, as the reference's items do"""
        target = self.get_groundtruth(idx).clip_to_image(remove_empty=True)
        if isinstance(img, EncodedImage):                   # every frame of the item in one decode batch
            frames = self.transforms.decode_batch([img] + [f for k in extra for f in extra[k]])
            img, rest = frames[0], iter(frames[1:])
            extra = {k: [next(rest) for _ in extra[k]] for k in extra}
        if self.transforms is not None:
            img, target = self.transforms(img, target)
            extra = {k: [self.transforms(f, None)[0] for f in frames] for k, frames in extra.items()}
        return img, target, extra

    def _get_test(self, idx):
        img, target, _ = self._transformed(idx, self._open(self.image_set_index[idx]), {})
        return img, target, idx

    def _index_video_starts(self):
        """positions of every video's frame 0: what VIDTestDistributedSampler cuts the dataset at (vid_rdn.py:11-16)"""
        self.start_index = [i for i, name in enumerate(self.image_set_index) if int(name.split("/")[-1]) == 0]

    def _video_fields(self, idx):
        return {"seg_len": self.frame_seg_len[idx], "pattern": self.pattern[idx], "img_dir": self._img_dir,
                "transforms": self.transforms}

    # ---- annotations
    def _preprocess_annotation(self, root):
        size = root.find("size")
        im_info = (int(size.find("height").text), int(size.find("width").text))
        boxes, labels = [], []
        for obj in root.findall("object"):
            name = obj.find("name").text
            if name not in self.classes_to_ind:
                continue
            bb = obj.find("bndbox")
            boxes.append([max(float(bb.find("xmin").text), 0), max(float(bb.find("ymin").text), 0),
                          min(float(bb.find("xmax").text), im_info[1] - 1), min(float(bb.find("ymax").text), im_info[0] - 1)])
            labels.append(self.classes_to_ind[name.lower().strip()])
        return {"boxes": torch.tensor(boxes, dtype=torch.float32).reshape(-1, 4), "labels": torch.tensor(labels),
                "im_info": im_info}

    def load_annos(self, cache_file):
        if os.path.exists(cache_file):
            with open(cache_file, "rb") as f:
                return pickle.load(f)
        annos = [self._preprocess_annotation(ET.parse(self._anno_path % name).getroot()) for name in self.image_set_index]
        if is_main_process():
            with open(cache_file, "wb") as f:
                pickle.dump(annos, f)
        return annos

    @property
    def cache_dir(self):
        path = os.path.join(self.data_dir, "cache")
        os.makedirs(path, exist_ok=True)
        return path

    def get_img_info(self, idx):
        h, w = self.annos[idx]["im_info"]
        return {"height": h, "width": w}

    def get_groundtruth(self, idx):
        a = self.annos[idx]
        h, w = a["im_info"]
        target = BoxList(a["boxes"].reshape(-1, 4), (w, h), mode="xyxy")
        target.add_field("labels", a["labels"])
        return target

    @staticmethod
    def map_class_id_to_class_name(class_id):
        return VIDDataset.classes[class_id]


class _LookaheadDataset(VIDDataset):
    """RDN / FGFA test items (vid_rdn.py:50-83, vid_fgfa.py:50-83): the current frame plus the frame MAX_OFFSET ahead
    (clamped to the video); frame 0 of a video has frame_category 0 and the model reads the frames in between itself"""
    section = None

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._index_video_starts()

    def _get_test(self, idx):
        name = self.image_set_index[idx]
        frame_id = int(name.split("/")[-1])
        ahead = min(self.frame_seg_len[idx] - 1, frame_id + cfg.MODEL.VID[self.section].MAX_OFFSET)
        img, target, extra = self._transformed(idx, self._open(name), {"ref": [self._open(self.pattern[idx] % ahead)]})
        images = {"cur": img, "ref": extra["ref"], "frame_category": 0 if frame_id == 0 else 1}
        images.update(self._video_fields(idx))
        return images, target, idx


class VIDRDNDataset(_LookaheadDataset):
    section = "RDN"


class VIDFGFADataset(_LookaheadDataset):
    section = "FGFA"


class VIDMEGADataset(VIDDataset):
    """vid_mega.py:8-142, test side: look-ahead local frame + global frames drawn from a per-video (shuffled) order"""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        m = cfg.MODEL.VID.MEGA
        self.start_index, self.start_id, self.shuffled_index = [], [], {}
        for i, name in enumerate(self.image_set_index):
            if int(name.split("/")[-1]) == 0:
                self.start_index.append(i)
                if m.GLOBAL.ENABLE:
                    order = np.arange(self.frame_seg_len[i])
                    if m.GLOBAL.SHUFFLE:
                        np.random.shuffle(order)           # the reference's global numpy RNG (vid_mega.py:22-24)
                    self.shuffled_index[str(i)] = order
            self.start_id.append(self.start_index[-1])

    def _get_test(self, idx):
        m = cfg.MODEL.VID.MEGA
        name = self.image_set_index[idx]
        frame_id = int(name.split("/")[-1])
        img = self._open(name)
        ahead = min(self.frame_seg_len[idx] - 1, frame_id + m.MAX_OFFSET)
        extra = {"ref_l": [self._open(self.pattern[idx] % ahead)], "ref_g": []}
        if m.GLOBAL.ENABLE:
            order = self.shuffled_index[str(self.start_id[idx])]
            for i in range(m.GLOBAL.SIZE if frame_id == 0 else 1):
                g = self._open(self.pattern[idx] % order[(idx - self.start_id[idx] + m.GLOBAL.SIZE - i - 1) % self.frame_seg_len[idx]])
                extra["ref_g"].append(g)
                # faithful to the reference: its loop re-binds `img` (vid_mega.py:119), so the tensor under "cur" is the
                # LAST global frame; the model reads "cur" only for frame_category 0 (INTEGRATION.md)
                img = g
        img, target, extra = self._transformed(idx, img, extra)
        images = {"cur": img, "ref_l": extra["ref_l"], "ref_g": extra["ref_g"], "frame_category": 0 if frame_id == 0 else 1}
        images.update(self._video_fields(idx))
        return images, target, idx


class VIDDFFDataset(VIDDataset):
    """vid_dff.py:48-67: every 10th frame is a key frame"""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._index_video_starts()

    def _get_test(self, idx):
        name = self.image_set_index[idx]
        img, target, _ = self._transformed(idx, self._open(name), {})
        return {"cur": img, "is_key_frame": int(name.split("/")[-1]) % 10 == 0}, target, idx
