"""Convert the reference's example problems into portable .npz fixtures.

Needs a checkout of the reference:  python tests/golden/make_problem_fixtures.py <reference checkout>
bench.py and the tests read these files, so they run without the reference
(examples/README.md in the reference documents the provenance of the .mat files).
Only the raw problem data (At, b, c, K) is stored -- no reference code.
"""
import os
import sys

import numpy as np
import scipy.io as sio
import scipy.sparse as sp

REF = os.path.join(sys.argv[1], "examples")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "problems")
NAMES = ["arch0", "control07", "nb", "trto3"]

os.makedirs(OUT, exist_ok=True)
for name in NAMES:
    d = sio.loadmat(os.path.join(REF, name + ".mat"))
    At = sp.csc_matrix(d["At"] if "At" in d else d["A"], dtype=np.float64)
    At.sort_indices()
    b = np.asarray(d["b"].todense() if sp.issparse(d["b"]) else d["b"], dtype=np.float64).ravel()
    c = np.asarray(d["c"].todense() if sp.issparse(d["c"]) else d["c"], dtype=np.float64).ravel()
    Kraw = d["K"]
    K = {"K_" + n: np.asarray(Kraw[n][0, 0], dtype=np.float64).ravel() for n in Kraw.dtype.names}
    np.savez_compressed(os.path.join(OUT, name + ".npz"), At_data=At.data, At_indices=At.indices.astype(np.int32),
                        At_indptr=At.indptr.astype(np.int64), At_shape=np.array(At.shape), b=b, c=c, **K)
    print(name, At.shape, At.nnz, {k: v[:4] for k, v in K.items()}, file=sys.stderr)
