"""Where the suite's measured errors go: one JSON file per topic under OUT, one key per check."""
import json
import os

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.join(ROOT, "gpurun_out")


def record(file, name, payload, echo=False):
    """store payload under name in OUT/file, keeping the other keys; an unreadable file starts afresh"""
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, file)
    data = {}
    if os.path.exists(path):
        try:
            data = json.load(open(path))
        except Exception:
            data = {}
    data[name] = payload
    json.dump(data, open(path, "w"), indent=1, default=float)
    if echo:
        print(name, json.dumps(payload, default=float))
