"""GPU: the per-environment row blocks' lending (csrc/env_rows.h) replays tests/golden/env_rows_transcript.json.gz exactly: every verb accepted or
refused with the same message, the same row pointers present after it, and the same qpos, qvel and obs digests after every launch verb."""
import gzip
import json
import os
import sys

import pytest

from conftest import GOLDEN, product

sys.path.insert(0, GOLDEN)
import make_env_rows_transcript as T  # noqa: E402


@pytest.mark.gpu
def test_transcript_replays_exactly():
    P = product()
    with gzip.open(os.path.join(GOLDEN, 'env_rows_transcript.json.gz'), 'rt') as f:
        want = json.load(f)
    assert tuple(want['rows']) == T.ROWS and want['n_env'] == T.N_ENV
    for c in want['cases']:
        got = T.run_copy_case(P, c['verbs']) if c['copy'] else T.run_case(P, c['model'], c['prec'], c['verbs'])
        for i, (g, w) in enumerate(zip(got, c['log'])):
            assert g == w, (c['model'], c['prec'], c['verbs'], i)
        assert len(got) == len(c['log'])
