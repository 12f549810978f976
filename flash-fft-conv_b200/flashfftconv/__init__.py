from .conv import FlashFFTConv  # noqa: F401  (reference flashfftconv/__init__.py:1)
from .depthwise_1d import FlashDepthWiseConv1d  # noqa: F401  (reference flashfftconv/__init__.py:2)
from .gated import gated_long_conv, hyena_mixer, hyena_operator  # noqa: F401
from .sparse_conv import PartialFFTConv, FrequencySparseFFTConv  # noqa: F401  (reference flashfftconv/sparse_conv.py)
from .block_conv import blocked_long_conv  # noqa: F401
from .decode import HyenaDecoder, LongConvDecoder  # noqa: F401
from .docs import DocumentTable  # noqa: F401
from .modal import ModalFilter, log_vandermonde, log_vandermonde_transpose  # noqa: F401
from .fir_conv import FirFilter, fir_conv, fir_mixer  # noqa: F401
