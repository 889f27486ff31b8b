"""Clip-level result egress (siammot_b200/egress.py) against the reference's own code: ``boxlists_to_entities`` is imported
verbatim (over stand-ins for gluoncv's two container classes), ``DatasetInference._postprocess_tracks`` is executed from its
source text (its module needs motmetrics & co. to import).  What they return for the seeded results below is stored by
tests/golden/make_reference_vectors.py."""
import ast
import os
import sys
import textwrap

import numpy as np
import pytest
import torch

VIDEOS = [(1280, 720), (1920, 1080), (2560, 1408)]


def entity_tuple(e):
    return (tuple(e.bbox), e.confidence, e.labels, e.id, e.frame_num, e.time)


def entity_key(e):
    return (e.id, e.frame_num, tuple(e.bbox))


class PostprocessSelf(object):
    """The two attributes DatasetInference._postprocess_tracks reads from its instance."""
    _track_len, _track_conf = 5, 0.7


def _random_results(seed, n_frames=12, net=(1280, 704)):
    from siammot_b200.structures import BoxList
    g = torch.Generator().manual_seed(seed)
    out = []
    for t in range(n_frames):
        n = int(torch.randint(0, 9, (1,), generator=g))
        xy = torch.rand(n, 2, generator=g) * torch.tensor([net[0] * 0.8, net[1] * 0.8])
        wh = torch.rand(n, 2, generator=g) * 200 + 5
        bl = BoxList(torch.cat([xy, xy + wh], 1), net, "xyxy")
        bl.add_field("scores", torch.rand(n, generator=g) * 0.5 + 0.5)
        bl.add_field("ids", torch.randint(-1, 4, (n,), generator=g))
        bl.add_field("labels", torch.randint(1, 3, (n,), generator=g))
        out.append(bl)
    return out


@pytest.mark.parametrize("video", VIDEOS)
def test_clip_to_tracks_and_entities_equal_the_reference_path(video):
    from helpers import ref_vectors
    from siammot_b200 import egress
    results = _random_results(video[0])
    # the reference path, per frame (inferencer.py:64-70): BoxList.resize -> convert("xywh") -> boxlists_to_entities
    ref_entities = ref_vectors()["egress"][video]
    tracks = egress.clip_to_tracks(results, video[0], video[1], first_frame_idx=100, timestamps=[0.04 * (100 + t) for t in range(len(results))])
    got = egress.to_entities(tracks, class_table=["person", "vehicle"])
    assert len(got) == len(ref_entities) == len(tracks)
    assert [entity_tuple(e) for e in got] == ref_entities


def _reference_postprocess():
    """DatasetInference._postprocess_tracks, literally, from the reference file."""
    from oracle import reference_loader
    reference_loader.load()
    path = os.path.join(reference_loader.REFERENCE_ROOT, "siammot", "engine", "inferencer.py")
    src = open(path).read()
    tree = ast.parse(src)
    for node in ast.walk(tree):
        if isinstance(node, ast.FunctionDef) and node.name == "_postprocess_tracks":
            code = textwrap.dedent(ast.get_source_segment(src, node))
            break
    else:
        raise AssertionError("_postprocess_tracks not found")
    from gluoncv.torch.data.gluoncv_motion_dataset.dataset import DataSample
    ns = {"np": np, "DataSample": DataSample}
    exec(code, ns)
    return ns["_postprocess_tracks"], DataSample


def test_postprocess_tracks_equals_the_reference_filter():
    from helpers import ref_vectors
    from siammot_b200 import egress
    results = _random_results(7, n_frames=40)
    tracks = egress.clip_to_tracks(results, 1280, 720)
    ref = ref_vectors()["egress"]["postprocess"]      # _postprocess_tracks(PostprocessSelf(), <these tracks>), sorted keys
    got = egress.to_entities(egress.postprocess_tracks(tracks, PostprocessSelf._track_len, PostprocessSelf._track_conf),
                             ["person", "vehicle"])
    assert len(ref) > 0 and ref == sorted(map(entity_key, got))
    assert all(e.id >= 0 for e in got)
    # grouped by id, frames ascending
    assert [(e.id, e.frame_num) for e in got] == sorted((e.id, e.frame_num) for e in got)
