"""Records what the unmodified reference launcher (llm-d-fast-model-actuation, inference_server/launcher/) answers to the
request scripts of tests/test_node_agent_differential.py, so that the node agent is compared with it without the
reference being present:

    python tests/golden/make_launcher_golden.py <reference checkout>/inference_server/launcher

writes tests/golden/reference_launcher.json.  Each script runs against a freshly started launcher (as each test gets a
fresh agent), with the config-0 stand-in children and the kubernetes import stub of scripts/."""
import json
import os
import shutil
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests import test_node_agent_differential as T  # noqa: E402


def main(launcher_dir: str) -> None:
    recorded = {}
    scripts = (("rest_contract", lambda svc: T._script(svc, T._port())), ("watch_stream", T._watch_sequence),
               ("stopped_event", T._stopped_event))
    with tempfile.TemporaryDirectory() as work:
        copy = os.path.join(work, "launcher")      # the launcher runs in its own directory: keep the source tree untouched
        shutil.copytree(launcher_dir, copy)
        for key, script in scripts:
            svc = T.Service(os.path.join(copy, "launcher.py"), work)
            try:
                recorded[key] = script(svc)
            finally:
                svc.close()
    with open(T.GOLDEN, "w") as f:
        json.dump(recorded, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main(sys.argv[1])
