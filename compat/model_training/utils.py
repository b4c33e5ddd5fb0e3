"""reference path: model_training/utils.py -- the helpers the inference / demo path imports (demo_utils.py:9,
losses/*.py): index-set loading (model_training/utils.py:56-105), the logger factory (:22-43) and ``indices_reweighing``
(:108-117).  hydra / omegaconf / coloredlogs are not needed here (they only serve the training entry point)."""
import logging
import os
from typing import Any, Dict, List

from dad_3dheads_b200.flame_assets import get_list_of_npy_files, indices_reweighing, load_indices_from_npy  # noqa: F401


def create_logger(name: str, msg_format: str = "") -> logging.Logger:
    logger = logging.Logger(name)
    handler = logging.StreamHandler()
    level = logging.DEBUG if os.environ.get("DEBUG") else logging.INFO
    handler.setLevel(level)
    handler.setFormatter(logging.Formatter(msg_format or "%(asctime)s %(name)s %(levelname)s - %(message)s"))
    logger.addHandler(handler)
    logger.setLevel(level)
    return logger


logger = create_logger(__name__)


def load_2d_indices(config: Dict[str, Any]) -> List[int]:
    """model_training/utils.py:56-78: sorted .npy files of a subset folder -> one flat index list."""
    if config["2d_subset_name"] == "multipie_keypoints":
        return None
    indices = []
    for filename in sorted(get_list_of_npy_files(config)):
        if os.path.exists(filename):
            indices += load_indices_from_npy(filename)
        else:
            raise ValueError(f"[{filename.split('.')[0].split('/')[-1]}] class of keypoints doesn't exist")
    return indices
