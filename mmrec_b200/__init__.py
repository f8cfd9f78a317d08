"""mmrec_b200: H100-native (sm_90a) hot path of MMRec -- sparse graph propagation, modality projection and
full-catalog scoring + top-k -- behind the reference's model API.  See DESIGN.md."""
__version__ = "0.1.0"
