#!/usr/bin/env python
"""Experiment builds of the library (never the default one): lib/libn2nmn_b200_<name>.so, selected
at run time with N2NMN_LIB=<path>. Builds need no GPU.

    python tools/build_variants.py timeline            # clock64 stamps for tools/timeline.py
    python tools/build_variants.py epilogue            # the four builds of gpu_epilogue_attrib.sh
"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from n2nmn_b200 import build as b

SETS = {
    'timeline': [('timeline', ['N2NMN_EXP_TIMELINE'])],
    'epilogue': [('e_nostore', ['N2NMN_EXP_EPI_NOSTORE']), ('e_nomath', ['N2NMN_EXP_EPI_NOMATH']),
                 ('e_nostmath', ['N2NMN_EXP_EPI_NOSTORE', 'N2NMN_EXP_EPI_NOMATH']),
                 ('e_none', ['N2NMN_EXP_EPI_NONE'])],
    'rings': [('a3b3', ['N2NMN_EXP_STAGES_A=3', 'N2NMN_EXP_STAGES_B=3']),
              ('a5b2', ['N2NMN_EXP_STAGES_A=5', 'N2NMN_EXP_STAGES_B=2'])],
}
for which in (sys.argv[1:] or ['timeline']):
    for name, defs in SETS[which]:
        print(b.build_variant(name, defs))
