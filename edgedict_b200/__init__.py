"""edgedict_b200 -- H100-native (sm_90a) RNN-Transducer engine behind the reference's
``rnnt.models`` / ``rnnt.stream`` / ``warprnnt_pytorch`` interfaces.  See DESIGN.md."""
__version__ = "0.1.0"
