"""implicit_b200: an H100-native (sm_90a) ALS fit / recommend hot path behind benfred/implicit's API.

    from implicit_b200 import AlternatingLeastSquares
    model = AlternatingLeastSquares(factors=64, use_cg=False)
    model.fit(user_items)                       # scipy CSR, users x items
    ids, scores = model.recommend(userid, user_items[userid], N=10)

Python host code calls hand-written CUDA through the C-ABI in include/als_b200.h (ctypes); there is
no PyTorch and no CPU fallback in this package.
"""
from .als import AlternatingLeastSquares
from .utils import ModelFitError, ParameterWarning

__version__ = "0.1.0"
__all__ = ["AlternatingLeastSquares", "ModelFitError", "ParameterWarning", "__version__"]
