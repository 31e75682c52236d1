"""tha4_b200 -- H100-native (sm_90a) drop-in for the THA4 poser hot path (teacher mode_07 / mode_12, student mode_14).

Host side mirrors the reference's Python surface (`Poser`, `GeneralPoser02`, `create_poser`, the seven
`nn.Module`s and their state_dict layout); all device work happens in hand-written sm_90a CUDA kernels behind
the C ABI of libtha4_b200.so (include/tha4_b200.h).  There is no CPU or PyTorch-op fallback: using a module or
poser without the compiled library and an H100 (compute capability 9.0) raises.
"""
__version__ = '0.1.0'
