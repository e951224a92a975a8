"""TEST INFRASTRUCTURE ONLY -- fixtures for the front-door and configuration tests.

    python oracle/make_golden_frontdoor.py       (build container: needs the reference tree, see oracle/refshim.py)

Copies the reference's token table, speaker table and inference text (data, 21 KB) to tests/golden/frontdoor/ and writes
tests/golden/config_yaml.json: the `model` section, n_mels and segment_size of the reference's config.yaml as read by
emotivoice_b200.config.load_yaml_config -- what tests/test_host_logic.py compares the default configuration against."""
import json
import os
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from emotivoice_b200.config import load_yaml_config  # noqa: E402
from oracle.refshim import REF_ROOT  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def main():
    out = os.path.join(GOLDEN, "frontdoor")
    os.makedirs(out, exist_ok=True)
    for src, dst in (("data/youdao/text/tokenlist", "tokenlist"), ("data/youdao/text/speaker2", "speaker2"),
                     ("data/inference/text", "inference_text")):
        shutil.copyfile(os.path.join(REF_ROOT, src), os.path.join(out, dst))
    y = load_yaml_config(os.path.join(REF_ROOT, "config/joint/config.yaml"))
    with open(os.path.join(GOLDEN, "config_yaml.json"), "w") as f:
        json.dump({"model": dict(y.model), "n_mels": y.n_mels, "segment_size": y.segment_size}, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
