"""`build_transforms(cfg, is_train)` with the reference's name and config keys (data/transforms/build.py:5-49)."""
from .transforms import DeviceTestTransform


def build_transforms(cfg, is_train=True, device="cuda"):
    """Test-time pipeline of the reference -- Resize(MIN_SIZE_TEST, MAX_SIZE_TEST) -> ToTensor -> Normalize(PIXEL_MEAN,
    PIXEL_STD, TO_BGR255); colour jitter and the flips have probability / strength 0 at test time (build.py:16-24) --
    as ONE kernel on the device. Training-time augmentation is outside the inference hot path and is not provided."""
    if is_train:
        raise NotImplementedError("mega_core.data.transforms (B200 build) provides the test-time transform only")
    b200 = getattr(getattr(cfg, "MODEL", None), "B200", None)       # a config that carries only INPUT decodes with PIL
    return DeviceTestTransform(cfg.INPUT.MIN_SIZE_TEST, cfg.INPUT.MAX_SIZE_TEST, cfg.INPUT.PIXEL_MEAN,
                               cfg.INPUT.PIXEL_STD, cfg.INPUT.TO_BGR255, device=device,
                               jpeg_decode=getattr(b200, "JPEG_DECODE", "pil"))
