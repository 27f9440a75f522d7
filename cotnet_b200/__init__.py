"""cotnet_b200 -- H100-native (sm_90a) CoT-block hot path behind the reference's operator API.

Public surface mirrors JDAI-CV/CoTNet's ``cupy_layers`` / ``models.cotnet`` names for this path only
(SURVEY.md section 8): LocalConvolution, aggregation_zeropad, aggregation_zeropad_mix, CotLayer, CoXtLayer, and the
remaining ``cupy_layers`` variants (refpad, dilate, mix_merge: section 8f rank 4).
"""
from .aggregation_zeropad import AggregationZeropad, LocalConvolution, aggregation_zeropad  # noqa: F401
from .aggregation_zeropad_mix import (AggregationZeropadMix, LocalConvolutionMix,  # noqa: F401
                                      aggregation_zeropad_mix)
from .aggregation_refpad import AggregationRefpad, aggregation_refpad  # noqa: F401
from .aggregation_zeropad_dilate import (AggregationZeropadDilate, LocalConvolutionDilate,  # noqa: F401
                                         aggregation_zeropad_dilate)
from .aggregation_zeropad_mix_merge import (AggregationZeropadMixMerge, LocalConvolutionMixMerge,  # noqa: F401
                                            aggregation_zeropad_mix_merge)

__version__ = "0.1.0"
