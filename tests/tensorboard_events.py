"""Read the TensorBoard event files of a model directory back (tensorboard's LegacyEventFileLoader: the events as written,
without the loader's migration to tensor summaries)."""
import glob
import os
from collections import defaultdict

from gms_b200 import io_image


def event_files(model_dir: str) -> list:
    """The directory's event files, oldest first (by the wall time of each file's first event)."""
    from tensorboard.backend.event_processing.event_file_loader import LegacyEventFileLoader
    files = glob.glob(os.path.join(model_dir, "events.out.tfevents.*"))
    return sorted(files, key=lambda f: (next(iter(LegacyEventFileLoader(f).Load())).wall_time, f))


def read_events(path: str) -> dict:
    """tag -> [(step, value)] in file order: a float for a scalar, the decoded uint8 [H,W,3] image, or the HistogramProto."""
    from tensorboard.backend.event_processing.event_file_loader import LegacyEventFileLoader
    tags = defaultdict(list)
    for e in LegacyEventFileLoader(path).Load():
        for v in e.summary.value:
            kind = v.WhichOneof("value")
            if kind == "simple_value":
                tags[v.tag].append((e.step, v.simple_value))
            elif kind == "image":
                tags[v.tag].append((e.step, io_image.decode_png(v.image.encoded_image_string)))
            elif kind == "histo":
                tags[v.tag].append((e.step, v.histo))
            else:
                raise AssertionError(f"unexpected summary {kind} for {v.tag}")
    return dict(tags)
