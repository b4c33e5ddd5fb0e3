"""The keypoint path of albumentations 1.0.0 that the reference's FlameDataset builds (flame_dataset.py:173-192,202-208), on
top of the image-only albumentations stand-in the reference harness puts on ``sys.path`` (TEST INFRASTRUCTURE ONLY).

``keypoint_albumentations()`` swaps, for the duration of a ``with`` block, the module's ``Compose``, ``LongestMaxSize``,
``PadIfNeeded`` and ``Normalize`` for subclasses that also carry keypoints, and adds ``KeypointParams``; on exit the module
is as it was, so the predictor's image-only path is untouched.  A pipeline built inside the block keeps working after it.
Restated from 1.0.0 in the same Python scalar arithmetic:
  * ``Compose`` with ``KeypointParams("xy", remove_invisible=False)`` turns each keypoint row into ``(x, y, 0.0, 0.0)``
    (``convert_keypoints_to_albumentations``) and back into ``(x, y)`` after the transforms;
  * each transform takes its parameters from the image as it arrives: ``LongestMaxSize`` applies
    ``keypoint_scale(kp, s, s)`` with ``s = max_size / max([rows, cols])``, ``PadIfNeeded`` adds ``(pad_left, pad_top)``,
    ``Normalize`` leaves keypoints alone.
With float32 keypoints and Python scalars, numpy's promotion rules decide the arithmetic exactly as in the package."""
import contextlib
import math


class KeypointParams:
    def __init__(self, format, label_fields=None, remove_invisible=True, angle_in_degrees=True,
                 check_each_transform=True):
        if format != "xy" or remove_invisible:
            raise NotImplementedError("only KeypointParams('xy', remove_invisible=False) is restated")
        self.format, self.remove_invisible, self.angle_in_degrees = format, remove_invisible, angle_in_degrees


class _Keypoints:
    def __call__(self, **data):
        rows, cols = data["image"].shape[:2]
        data = super().__call__(**data)
        if "keypoints" in data:
            data["keypoints"] = [self.apply_to_keypoint(tuple(kp[:4]), rows, cols) + tuple(kp[4:])
                                 for kp in data["keypoints"]]
        return data

    def apply_to_keypoint(self, keypoint, rows, cols):
        return keypoint


def _pads(t, rows, cols):
    """PadIfNeeded.update_params of 1.0.0: (pad_top, pad_left)."""
    top = int((t.min_height - rows) / 2.0) if rows < t.min_height else 0
    left = int((t.min_width - cols) / 2.0) if cols < t.min_width else 0
    return top, left


def _classes(A):
    class LongestMaxSize(_Keypoints, A.LongestMaxSize):
        def apply_to_keypoint(self, keypoint, rows, cols):
            scale = self.max_size / max([rows, cols])
            x, y, angle, kp_scale = keypoint[:4]                  # functional.keypoint_scale(keypoint, scale, scale)
            return x * scale, y * scale, angle, kp_scale * max(scale, scale)

    class PadIfNeeded(_Keypoints, A.PadIfNeeded):
        def apply_to_keypoint(self, keypoint, rows, cols):
            top, left = _pads(self, rows, cols)
            x, y, angle, scale = keypoint[:4]
            return x + left, y + top, angle, scale

    class Normalize(_Keypoints, A.Normalize):
        pass

    class Compose(A.Compose):
        def __init__(self, transforms, bbox_params=None, keypoint_params=None, additional_targets=None, p=1.0):
            super().__init__(transforms)
            self.keypoint_params = keypoint_params

        def __call__(self, **data):
            kp = self.keypoint_params is not None and "keypoints" in data
            if kp:
                angle = math.radians(0.0) % (2 * math.pi)
                data["keypoints"] = [(k[0], k[1], angle, 0.0) for k in (tuple(k) for k in data["keypoints"])]
            data = super().__call__(**data)
            if kp:
                data["keypoints"] = [(k[0], k[1]) + tuple(k[4:]) for k in data["keypoints"]]
            return data

    return {"LongestMaxSize": LongestMaxSize, "PadIfNeeded": PadIfNeeded, "Normalize": Normalize, "Compose": Compose,
            "KeypointParams": KeypointParams}


@contextlib.contextmanager
def keypoint_albumentations():
    """Within the block, the harness's ``albumentations`` module carries keypoints (call after ``ref_harness.activate()``)."""
    import albumentations as A
    new = _classes(A)
    old = {k: getattr(A, k) for k in new}
    for k, v in new.items():
        setattr(A, k, v)
    try:
        yield A
    finally:
        for k, v in old.items():
            setattr(A, k, v)
