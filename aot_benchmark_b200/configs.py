"""Model configuration objects with the reference's attribute names.

The drop-in engines read ``cfg.MODEL_*`` / ``cfg.TEST_*`` exactly as the reference does
(configs/default.py:5-138 merged with configs/models/<model>.py).  When the reference's own
``configs`` package is on PYTHONPATH (tools/eval.py drop-in) its objects are used unchanged;
this module provides the same keys for stand-alone use (bench, tests, GPU box)."""
from __future__ import annotations

# (vos, engine, encoder, encoder_dim, lstt_num, align_corners, test_long_gap)
_MODELS = {
    # configs/models/default.py:5-27 + aott.py / aots.py / aotb.py / aotl.py
    "aott": ("aot", "mobilenetv2", [24, 32, 96, 1280], 1, True, 9999),
    "aots": ("aot", "mobilenetv2", [24, 32, 96, 1280], 2, True, 9999),
    "aotb": ("aot", "mobilenetv2", [24, 32, 96, 1280], 3, True, 9999),
    "aotl": ("aot", "mobilenetv2", [24, 32, 96, 1280], 3, True, 5),
    # configs/models/r50_aotl.py:7-16
    "r50_aotl": ("aot", "resnet50", [256, 512, 1024, 1024], 3, True, 5),
    # configs/models/r101_aotl.py, rs101_aotl.py
    "r101_aotl": ("aot", "resnet101", [256, 512, 1024, 1024], 3, True, 5),
    "rs101_aotl": ("aot", "resnest101", [256, 512, 1024, 1024], 3, True, 5),
    # configs/models/default_deaot.py:9-17 + deaot*.py
    "deaott": ("deaot", "mobilenetv2", [24, 32, 96, 1280], 1, True, 9999),
    "deaots": ("deaot", "mobilenetv2", [24, 32, 96, 1280], 2, True, 9999),
    "deaotb": ("deaot", "mobilenetv2", [24, 32, 96, 1280], 3, True, 9999),
    "deaotl": ("deaot", "mobilenetv2", [24, 32, 96, 1280], 3, True, 5),
    # configs/models/r50_deaotl.py
    "r50_deaotl": ("deaot", "resnet50", [256, 512, 1024, 1024], 3, True, 5),
    # configs/models/swinb_aotl.py:9-18, swinb_deaotl.py:9-18
    "swinb_aotl": ("aot", "swin_base", [128, 256, 512, 512], 3, False, 5),
    "swinb_deaotl": ("deaot", "swin_base", [128, 256, 512, 512], 3, False, 5),
}


class EngineConfig:
    """Stand-alone equivalent of ``configs.default.DefaultEngineConfig(exp, model)``."""

    def __init__(self, exp_name: str = "default", model: str = "r50_aotl"):
        if model not in _MODELS:
            raise NotImplementedError(f"model config '{model}' is not on the H100 hot path "
                                      f"(available: {sorted(_MODELS)})")
        vos, enc, enc_dim, lstt, ac, gap = _MODELS[model]
        deaot = vos == "deaot"
        self.MODEL_NAME = model
        self.EXP_NAME = exp_name + "_" + model
        self.MODEL_VOS = vos
        self.MODEL_ENGINE = vos + "engine"
        self.MODEL_ALIGN_CORNERS = ac
        self.MODEL_ENCODER = enc
        self.MODEL_ENCODER_DIM = list(enc_dim)
        self.MODEL_ENCODER_EMBEDDING_DIM = 256
        self.MODEL_DECODER_INTERMEDIATE_LSTT = not deaot
        self.MODEL_FREEZE_BN = True
        self.MODEL_FREEZE_BACKBONE = False
        self.MODEL_MAX_OBJ_NUM = 10
        self.MODEL_SELF_HEADS = 1 if deaot else 8
        self.MODEL_ATT_HEADS = 1 if deaot else 8
        self.MODEL_LSTT_NUM = lstt
        self.MODEL_EPSILON = 1e-5
        self.MODEL_USE_PREV_PROB = False
        self.TRAIN_LONG_TERM_MEM_GAP = 2 if gap == 5 else 9999
        self.TEST_LONG_TERM_MEM_GAP = gap
        self.TEST_SHORT_TERM_MEM_SKIP = 1
        # test-time augmentation and the frame size rule (configs/default.py:97-100); TTAInferEngine defaults to the first two
        self.TEST_FLIP = False
        self.TEST_MULTISCALE = [1]
        self.TEST_MAX_SHORT_EDGE = None
        self.TEST_MAX_LONG_EDGE = 800 * 1.3
        # keys the reference model constructors read (all inactive in eval)
        self.TRAIN_ENCODER_FREEZE_AT = 2
        self.TRAIN_LSTT_EMB_DROPOUT = 0.
        self.TRAIN_LSTT_ID_DROPOUT = 0.
        self.TRAIN_LSTT_DROPPATH = 0.1
        self.TRAIN_LSTT_DROPPATH_SCALING = False
        self.TRAIN_LSTT_DROPPATH_LST = False
        self.TRAIN_LSTT_LT_DROPOUT = 0.
        self.TRAIN_LSTT_ST_DROPOUT = 0.
