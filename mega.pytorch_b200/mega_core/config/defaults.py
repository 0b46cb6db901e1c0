"""Configuration tree for the inference hot path.

Same key names and default values as the reference's config/defaults.py for everything the VID
inference path reads (MODEL.*, MODEL.VID.* defaults.py:393-463, INPUT.*, TEST.*); training / mask
/ keypoint / retinanet / FBNet keys are not carried. `CfgNode` is a small stand-alone
implementation (yacs is not a dependency): attribute access, merge_from_file (YAML),
merge_from_list, freeze/defrost, clone.
"""
import ast
import copy
import os


class CfgNode(dict):
    def __init__(self, init=None):
        super().__init__()
        object.__setattr__(self, "_frozen", False)
        for k, v in (init or {}).items():
            self[k] = CfgNode(v) if isinstance(v, dict) and not isinstance(v, CfgNode) else v

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)

    def __setattr__(self, k, v):
        if object.__getattribute__(self, "_frozen"):
            raise AttributeError("config is frozen: cannot set %s" % k)
        self[k] = v

    def _each(self):
        for v in self.values():
            if isinstance(v, CfgNode):
                yield v

    def freeze(self):
        object.__setattr__(self, "_frozen", True)
        for n in self._each():
            n.freeze()

    def defrost(self):
        object.__setattr__(self, "_frozen", False)
        for n in self._each():
            n.defrost()

    def clone(self):
        return copy.deepcopy(self)

    def __deepcopy__(self, memo):
        new = CfgNode()
        for k, v in self.items():
            dict.__setitem__(new, k, copy.deepcopy(v, memo))
        object.__setattr__(new, "_frozen", object.__getattribute__(self, "_frozen"))
        return new

    @staticmethod
    def _fit(new, old):
        if isinstance(new, str):
            try:
                new = ast.literal_eval(new)
            except (ValueError, SyntaxError):
                pass
        if isinstance(old, tuple) and isinstance(new, list):
            new = tuple(new)
        if isinstance(old, float) and isinstance(new, int) and not isinstance(new, bool):
            new = float(new)
        return new

    def merge_from_dict(self, d, strict=False):
        for k, v in d.items():
            if isinstance(v, dict):
                if k not in self:
                    if strict:
                        raise KeyError("unknown config section %s" % k)
                    self[k] = CfgNode()
                self[k].merge_from_dict(v, strict)
            else:
                self[k] = self._fit(v, self.get(k))

    def merge_from_file(self, path):
        import yaml
        with open(path) as fh:
            self.merge_from_dict(yaml.safe_load(fh) or {})

    def merge_from_list(self, lst):
        assert len(lst) % 2 == 0, "opts must be KEY VALUE pairs"
        for key, v in zip(lst[0::2], lst[1::2]):
            node = self
            parts = key.split(".")
            for p in parts[:-1]:
                node = node[p]
            node[parts[-1]] = self._fit(v, node.get(parts[-1]))


_C = CfgNode({
    "MODEL": {
        "DEVICE": "cuda", "META_ARCHITECTURE": "GeneralizedRCNN", "WEIGHT": "", "RPN_ONLY": False, "MASK_ON": False,
        "KEYPOINT_ON": False, "RETINANET_ON": False, "CLS_AGNOSTIC_BBOX_REG": False,
        "BACKBONE": {"CONV_BODY": "R-50-C4", "FREEZE_CONV_BODY_AT": 2},
        "RESNETS": {"NUM_GROUPS": 1, "WIDTH_PER_GROUP": 64, "STRIDE_IN_1X1": True, "TRANS_FUNC": "BottleneckWithFixedBatchNorm",
                    "STEM_FUNC": "StemWithFixedBatchNorm", "RES5_DILATION": 1, "BACKBONE_OUT_CHANNELS": 1024,
                    "RES2_OUT_CHANNELS": 256, "STEM_OUT_CHANNELS": 64, "STAGE_WITH_DCN": (False, False, False, False),
                    "WITH_MODULATED_DCN": False, "DEFORMABLE_GROUPS": 1},
        "RPN": {"USE_FPN": False, "ANCHOR_SIZES": (32, 64, 128, 256, 512), "ANCHOR_STRIDE": (16,),
                "ASPECT_RATIOS": (0.5, 1.0, 2.0), "STRADDLE_THRESH": 0, "PRE_NMS_TOP_N_TRAIN": 12000,
                "PRE_NMS_TOP_N_TEST": 6000, "POST_NMS_TOP_N_TRAIN": 2000, "POST_NMS_TOP_N_TEST": 1000, "NMS_THRESH": 0.7,
                "MIN_SIZE": 0, "FPN_POST_NMS_TOP_N_TRAIN": 2000, "FPN_POST_NMS_TOP_N_TEST": 2000,
                "FPN_POST_NMS_PER_BATCH": True, "RPN_HEAD": "SingleConvRPNHead"},
        "ROI_HEADS": {"USE_FPN": False, "BBOX_REG_WEIGHTS": (10.0, 10.0, 5.0, 5.0), "SCORE_THRESH": 0.05, "NMS": 0.5,
                      "DETECTIONS_PER_IMG": 100, "BATCH_SIZE_PER_IMAGE": 512},
        "ROI_BOX_HEAD": {"FEATURE_EXTRACTOR": "ResNet50Conv5ROIFeatureExtractor", "PREDICTOR": "FastRCNNPredictor",
                         "POOLER_RESOLUTION": 14, "POOLER_SAMPLING_RATIO": 0, "POOLER_SCALES": (1.0 / 16,),
                         "NUM_CLASSES": 81, "MLP_HEAD_DIM": 1024, "USE_GN": False},
        "VID": {"ENABLE": False, "METHOD": "base", "IGNORE": False,
                "RPN": {"REF_PRE_NMS_TOP_N": 6000, "REF_POST_NMS_TOP_N": 75},
                "ROI_BOX_HEAD": {"REDUCE_CHANNEL": False,
                                 "ATTENTION": {"ENABLE": False, "EMBED_DIM": 64, "GROUP": 16, "STAGE": 2,
                                               "ADVANCED_STAGE": 0}},
                "RDN": {"MIN_OFFSET": -18, "MAX_OFFSET": 18, "ALL_FRAME_INTERVAL": 37, "KEY_FRAME_LOCATION": 18,
                        "REF_NUM": 2, "RATIO": 0.2},
                "MEGA": {"MIN_OFFSET": -12, "MAX_OFFSET": 12, "ALL_FRAME_INTERVAL": 25, "KEY_FRAME_LOCATION": 12,
                         "REF_NUM_LOCAL": 2, "RATIO": 0.2, "SHUFFLED_CUR_TEST": False,
                         "MEMORY": {"ENABLE": True, "SIZE": 25},
                         "GLOBAL": {"ENABLE": True, "RES_STAGE": 1, "SIZE": 10, "SHUFFLE": True}},
                "FGFA": {"MIN_OFFSET": -9, "MAX_OFFSET": 9, "ALL_FRAME_INTERVAL": 19, "KEY_FRAME_LOCATION": 9,
                         "REF_NUM": 2}},
        # B200 build only: arithmetic of the tensor-core contractions -- "f16" (fp16 operands / storage, throughput
        # mode), "tf32" (fp32 storage, TF32 operands), "fp32x3" (3xTF32 split, strict parity with the fp32 reference)
        # SEQ_NMS (B200 build only): Seq-NMS over whole videos after the detection loop (mega_core.engine.seq_nms) --
        # boxes of consecutive frames link at IoU > LINK_IOU, a chain suppresses IoU > NMS_IOU in its frames, its boxes
        # get the chain's "avg" or "max" score
        "B200": {"PRECISION": "f16",
                 "SEQ_NMS": {"ENABLED": False, "LINK_IOU": 0.5, "NMS_IOU": 0.3, "RESCORE": "avg"}},
    },
    "INPUT": {"MIN_SIZE_TRAIN": (800,), "MAX_SIZE_TRAIN": 1333, "MIN_SIZE_TEST": 800, "MAX_SIZE_TEST": 1333,
              "PIXEL_MEAN": [102.9801, 115.9465, 122.7717], "PIXEL_STD": [1.0, 1.0, 1.0], "TO_BGR255": True},
    "DATASETS": {"TRAIN": (), "TEST": ()},
    "DATALOADER": {"NUM_WORKERS": 4, "SIZE_DIVISIBILITY": 0, "ASPECT_RATIO_GROUPING": True},
    "SOLVER": {"BASE_LR": 0.001, "WEIGHT_DECAY": 0.0005, "STEPS": (30000,), "MAX_ITER": 40000, "IMS_PER_BATCH": 16,
               "WARMUP_ITERS": 500},
    "TEST": {"EXPECTED_RESULTS": [], "EXPECTED_RESULTS_SIGMA_TOL": 4, "IMS_PER_BATCH": 8, "DETECTIONS_PER_IMG": 100,
             # test-time box augmentation (config/defaults.py:511-526), single-frame method only
             # (mega_core.engine.bbox_aug)
             "BBOX_AUG": {"ENABLED": False, "H_FLIP": False, "SCALES": (), "MAX_SIZE": 4000, "SCALE_H_FLIP": False}},
    "OUTPUT_DIR": ".", "DTYPE": "float32", "AMP_VERBOSE": False,
    "PATHS_CATALOG": os.path.join(os.path.dirname(os.path.abspath(__file__)), "paths_catalog.py"),
})
