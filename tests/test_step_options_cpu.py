"""CPU: StepOptions, the checked and canonical options of one predict_batch step, which with the input's shape and dtype
keys the captured graphs of predict_batch_graphed and BatchStream."""
import dataclasses

import pytest

from dad_3dheads_b200.overlay import OVERLAY_KINDS
from dad_3dheads_b200.predictor import FRAME_RENDER_KEYS, RENDER_KEYS, StepOptions


@pytest.mark.parametrize("kw, want", [
    (dict(), dict(landmark_subset="445", to_2d=True, fast_decode=True, render=(), frame_render=(), overlay=(),
                  rpy=False, rois=None, extend=None)),
    (dict(to_2d=False, render="lit"), dict(render=("lit",))),
    (dict(to_2d=False, render=["lit", "depth", "pncc", "depth"]), dict(render=("pncc", "depth", "lit"))),
    (dict(to_2d=False, render=list(reversed(RENDER_KEYS))), dict(render=RENDER_KEYS)),
    (dict(rois=3, to_2d=False, frame_render=("head_index", "pncc")), dict(frame_render=("pncc", "head_index"))),
    (dict(rois=3, to_2d=False, frame_render=list(reversed(FRAME_RENDER_KEYS))), dict(frame_render=FRAME_RENDER_KEYS)),
    (dict(rois=3, overlay="pose"), dict(overlay=("pose",))),
    (dict(rois=3, overlay=("face_mesh", "68_landmarks")), dict(overlay=("68_landmarks", "face_mesh"))),
    (dict(rois=3, overlay=list(reversed(OVERLAY_KINDS))), dict(overlay=OVERLAY_KINDS)),
    (dict(render=None, frame_render=None, overlay=None), dict(render=(), frame_render=(), overlay=())),
    (dict(rpy=1), dict(rpy=True)),
    (dict(rpy=0), dict(rpy=False)),
    (dict(rois=0), dict(rois=0, extend=(0.0, 0.0, 0.0, 0.0))),
    (dict(rois=5, extend=0.1), dict(rois=5, extend=(0.1, 0.1, 0.1, 0.1))),
    (dict(rois=5, extend=(0.1, 0.2)), dict(extend=(0.1, 0.1, 0.2, 0.2))),
    (dict(rois=5, extend=[0.1, 0.2, 0.3, 0.4]), dict(extend=(0.1, 0.2, 0.3, 0.4))),
    (dict(rois=5, extend=(1, 2, 3, 4)), dict(extend=(1.0, 2.0, 3.0, 4.0))),
    (dict(extend=0.3), dict(extend=None)),                           # ignored without boxes, as predict_batch does
    (dict(extend=(0.1, 0.2, 0.3)), dict(extend=None)),
    (dict(landmark_subset=None, fast_decode=False), dict(landmark_subset=None, fast_decode=False)),
])
def test_canonical_record(kw, want):
    opts = StepOptions(**kw)
    got = dataclasses.asdict(opts)
    for k, v in want.items():
        assert got[k] == v and type(got[k]) is type(v), (k, got[k], v)
    assert all(type(x) is float for x in opts.extend or ())
    assert StepOptions(**got) == opts                                # canonical form is a fixed point


def test_equal_options_give_one_key():
    a = StepOptions(to_2d=False, rois=4, extend=0.1, frame_render=["lit", "pncc"], overlay="pose", rpy=1)
    b = StepOptions(to_2d=False, rois=4, extend=(0.1, 0.1, 0.1, 0.1), frame_render=("pncc", "lit"), overlay=["pose"],
                    rpy=True)
    assert a == b and hash(a) == hash(b) and len({a, b}) == 1
    assert {(a, (4, 64, 80, 3)): 1}[(b, (4, 64, 80, 3))] == 1
    with pytest.raises(dataclasses.FrozenInstanceError):
        a.rpy = False


def test_each_option_changes_the_key():
    base = dict(to_2d=False, rois=4, frame_render=("pncc",))
    variants = [dict(landmark_subset="191"), dict(landmark_subset=None), dict(to_2d=True, frame_render=None),
                dict(fast_decode=False), dict(frame_render=("depth",)), dict(overlay="pose"), dict(rpy=True),
                dict(rois=5), dict(extend=0.1), dict(rois=None, frame_render=None),
                dict(rois=None, frame_render=None, render="pncc")]
    keys = {StepOptions(**base)} | {StepOptions(**{**base, **v}) for v in variants}
    assert len(keys) == 1 + len(variants)


@pytest.mark.parametrize("kw", [
    dict(to_2d=False, render="normals"),                             # unknown names
    dict(to_2d=False, render=("pncc", "normals")),
    dict(rois=2, to_2d=False, frame_render=("pncc", "normals")),
    dict(rois=2, overlay="mesh"),
    dict(rois=2, overlay=("pose", "3d_mesh")),
    dict(render="pncc"),                                             # render / frame_render need to_2d=False
    dict(render=("lit",), to_2d=True),
    dict(rois=2, frame_render="pncc"),
    dict(rois=2, frame_render=FRAME_RENDER_KEYS, to_2d=True),
    dict(to_2d=False, frame_render="pncc"),                          # frame_render / overlay need boxes
    dict(to_2d=False, frame_render="lit"),
    dict(overlay="pose"),
    dict(overlay=OVERLAY_KINDS, rpy=True),
    dict(rois=2, to_2d=False, render="pncc"),                        # render with boxes
    dict(rois=0, to_2d=False, render=("depth",)),
    dict(rois=2, to_2d=False, render="pncc", frame_render="pncc"),
    dict(rois=2, extend=(0.1, 0.2, 0.3)),                            # extend: 1, 2 or 4 values
    dict(rois=2, extend=()),
])
def test_rejected(kw):
    with pytest.raises(ValueError):
        StepOptions(**kw)


def test_stream_without_rois_rejects_frame_outputs():
    """BatchStream builds its record from its own arguments: rois=None is a stream without boxes."""
    for kw in (dict(to_2d=False, frame_render="pncc"), dict(overlay=("68_landmarks",))):
        with pytest.raises(ValueError):
            StepOptions(rois=None, **kw)
        StepOptions(rois=8, **kw)
