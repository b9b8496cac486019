"""comic-text-detector_b200: H100-native engine behind the reference's inference path
(page -> block boxes + text-line map + segmentation mask).  Import as `ctd_b200`
(the directory name carries a hyphen; ctd_b200.py at the repository root aliases it)."""
from . import compiler  # noqa: F401
from .binding import Engine, CtdError, load_library, LIB_PATH  # noqa: F401
from . import binding, multigpu, onnx_model, textblock  # noqa: F401
from .inference import TextDetector, REFINEMASK_INPAINT, REFINEMASK_ANNOTATION  # noqa: F401
from .basemodel import TextDetBase  # noqa: F401
from .jpeg import JpegDecoder, JpegEncoder, jpeg_probe  # noqa: F401
from .png import PngDecoder, PngEncoder, png_probe  # noqa: F401
from .textmask import MaskRefiner, refine_mask, refine_undetected_mask  # noqa: F401
from .regions import RegionCropper  # noqa: F401
from .postprocess import PostProcessor  # noqa: F401
from .preprocess import NetworkDetector, Preprocessor, preprocess_img  # noqa: F401
