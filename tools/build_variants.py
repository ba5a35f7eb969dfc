#!/usr/bin/env python
"""Experiment builds of the library (never the default one): lib/libn2nmn_b200_<name>.so, selected
at run time with N2NMN_LIB=<path>. Builds need no GPU.

    python tools/build_variants.py timeline   # clock64 stamps (N2NMN_EXP_TIMELINE, common.cuh)
    python tools/build_variants.py attrib     # the contraction with one part removed, and its
                                              # 2-CTA cluster form, timed by tools/proj_bench.py
                                              # (proj_wgmma.cuh)
"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from n2nmn_b200 import build as b

SETS = {
    'timeline': [('timeline', ['N2NMN_EXP_TIMELINE'])],
    'attrib': [('no_epi', ['N2NMN_EXP_PROJ_NO_EPI']), ('no_b', ['N2NMN_EXP_PROJ_NO_B']),
               ('no_mma', ['N2NMN_EXP_PROJ_NO_MMA']), ('no_store', ['N2NMN_EXP_PROJ_NO_STORE']),
               ('no_find', ['N2NMN_EXP_PROJ_NO_FIND']),
               ('pairs', ['N2NMN_EXP_PROJ_PAIRS']),
               ('pairs_no_epi', ['N2NMN_EXP_PROJ_PAIRS', 'N2NMN_EXP_PROJ_NO_EPI']),
               ('pairs_no_b', ['N2NMN_EXP_PROJ_PAIRS', 'N2NMN_EXP_PROJ_NO_B'])],
}
for which in (sys.argv[1:] or ['timeline']):
    for name, defs in SETS[which]:
        print(b.build_variant(name, defs))
