"""oracle/ -- TEST INFRASTRUCTURE (checkers), never imported by edgedict_b200.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / ``--impl reference``
leg may import this package.  It holds

* ``loss``       ctypes front-end to oracle/liboracle.so (plain-C restatement of the
                 warp-transducer loss) and to oracle/_ref/libwarprnnt_ref.so (the reference's
                 own CPU library compiled from a warp-transducer tree, when present);
* ``model_np``   numpy restatement of the reference model forward (rnnt/models.py:16-269) and
                 of the streaming greedy loop (rnnt/stream.py:93-120);
* ``model_torch`` functional torch restatement (fp32/fp64, autograd) used for gradient
                 parity and as the CPU baseline arm.
"""
