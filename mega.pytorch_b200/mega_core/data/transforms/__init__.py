from .build import build_transforms  # noqa: F401
from .jpeg import EncodedImage, decode_jpeg_exact  # noqa: F401
from .transforms import DeviceTestTransform, decode_jpeg, get_size, resample_tables  # noqa: F401
