"""Generates tests/golden/reference_pins.json (see reference_pins.py) from the reference's own library,
oracle/_ref/libvbx_ref.so.  Run it where that library was built; it needs no GPU:

    python tests/golden/make_reference_pins.py [key prefix ...]

With key prefixes, only the keys that start with one of them are recomputed; the others are kept as recorded.
It also runs the restatement on every case and reports where the two differ."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from oracle import pyoracle as po  # noqa: E402
from tests import test_block_sizes_gpu as tb  # noqa: E402
from tests import test_esdf_fe_gpu as tfe  # noqa: E402
from tests import test_esdf_fixed_point_gpu as tfp  # noqa: E402
from tests import test_esdf_options_gpu as teo  # noqa: E402
from tests import test_esdf_reference_gpu as te  # noqa: E402
from tests import test_fast_reference_gpu as tf  # noqa: E402
from tests import test_icp_cpu as tic  # noqa: E402
from tests import test_icp_degenerate_gpu as tid  # noqa: E402
from tests import test_icp_gpu as ti  # noqa: E402
from tests import test_merged_reference_gpu as tm  # noqa: E402
from tests import test_mesh_cpu as tmc  # noqa: E402
from tests import test_oracle_pin as to  # noqa: E402
from tests import test_tsdf_edges_gpu as tte  # noqa: E402
from tests import test_tsdf_ground_truth_gpu as tg  # noqa: E402
from tests.golden import reference_pins as pins  # noqa: E402


def _joined(digests):
    return pins.array_digest(np.frombuffer("".join(digests).encode(), np.uint8))


def cases():
    """key -> function(lib) returning what the tests check under that key."""
    out = {"mesh/mc_tables": tmc.reference_table_digest, "icp/shuffle": tic.shuffle_digest}
    for name in tm.CASES:
        out[f"merged/{name}"] = lambda lib, n=name: tm.reference_side(n, lib)[2]
    for key in te.PIN_KEYS:
        out[f"esdf/{key}"] = lambda lib, k=key: te.reference_side(k, lib)[2]
    for key in teo.PIN_KEYS:
        out[f"esdf_options/{key}"] = lambda lib, k=key: teo.reference_side(k, lib)[2]
    for key in tfp.PIN_KEYS:
        out[f"esdf_fixed_point/{key}"] = lambda lib, k=key: tfp.reference_side(k, lib)[1]
    for key in tfe.PIN_KEYS:
        if key.startswith("synthetic/"):
            out[f"esdf_fe/{key}"] = lambda lib, k=key: tfe.synthetic_reference_side(k.split("/", 1)[1], lib)[1]
        else:
            out[f"esdf_fe/{key}"] = lambda lib, k=key: tfe.reference_side(k, lib)[1]
    for key in tte.PIN_KEYS:
        out[f"tsdf_edges/{key}"] = lambda lib, k=key: tte.reference_side(k, lib)[3]
    for key in tg.PIN_KEYS:
        out[f"tsdf_ground_truth/{key}"] = lambda lib, k=key: tg.reference_side(k, lib)[1]
    for key in ti.PIN_KEYS:
        out[f"icp/{key}"] = lambda lib, k=key: ti.reference_side(k, lib)[2]
    for key in tid.PIN_KEYS:
        out[f"icp_degenerate/{key}"] = lambda lib, k=key: tid.reference_side(k, lib)[1]
    for key in tb.PIN_KEYS:
        out[f"block_sizes/{key}"] = lambda lib, k=key: tb.reference_side(k, lib)[2]
    for key in tf.PIN_KEYS:
        # (reference_side primes the library's process-wide Fast reset counter first)
        out[f"fast_reference/{key}"] = lambda lib, k=key: tf.reference_side(k, lib)[2]
    for name, fn in to.REFERENCE_CASES.items():
        out[f"oracle_pin/{name}"] = lambda lib, f=fn: _joined(f(lib))
    return out


def main(prefixes=()):
    ref, port = po.OracleLib("reference"), po.OracleLib("port")
    pinned = json.load(open(pins.PATH)) if prefixes else {}
    for key, fn in cases().items():
        if prefixes and not key.startswith(tuple(prefixes)):
            continue
        pinned[key] = fn(ref)
        if key.startswith(("icp/refine", "icp_degenerate/", "block_sizes/icp/")):
            same = fn(port)["map"] == pinned[key]["map"]   # the restatement's ICP is compared at 1e-5, not bit for bit
        elif key == "mesh/mc_tables":
            same = True                                     # the restatement owns no copy of the table
        else:
            same = fn(port) == pinned[key]
        print(f"{key:45s} restatement {'==' if same else '!='} reference", flush=True)
    with open(pins.PATH, "w") as f:
        json.dump(pinned, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", pins.PATH)


if __name__ == "__main__":
    main(sys.argv[1:])
