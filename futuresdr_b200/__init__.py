"""futuresdr_b200 -- H100-native (sm_90a) backend for FutureSDR's FIR / decimator / resampler /
FFT / Apply / PfbArbResampler hot path, and the stream plumbing of branching flowgraphs.

Python host layer above the C ABI (include/b200sdr.h).  Class and method names mirror the
reference's Rust API for this path (futuredsp::{FirFilter, DecimatingFirFilter,
PolyphaseResamplingFir}, futuredsp::{firdes::{hilbert, lowpass}, windows::hamming}, futuresdr::blocks::{Fir,
FirBuilder, Fft, Apply, PfbArbResampler, SignalSource, SignalSourceBuilder, FixedPointPhase, Head,
Combine, Split, Delay, StreamDuplicator, StreamDeinterleaver}, the WLAN / M17 receivers' MovingAverage, the ZigBee
receiver's ClockRecoveryMm and Decoder, the keyfob receiver's Decoder, ApplyNM and the SSB example's oscillator mixers,
the LoRa Transmitter, the WLAN and ZigBee transmit chains,
runtime::mocker::Mocker) so the parity tests read like the reference's own tests.
Importing this package loads libb200sdr.so and raises if it is missing: no CPU fallback.
"""
from ._lib import (  # noqa: F401
    B200SdrError,
    INSUFFICIENT_INPUT, INSUFFICIENT_OUTPUT, BOTH_SUFFICIENT,
    ALGO_AUTO, ALGO_DIRECT, ALGO_TENSOR, ALGO_FFT, ALGO_SCAN,
)
from .context import Context, default_context  # noqa: F401
from .filters import (  # noqa: F401
    ComputationStatus, FirFilter, DecimatingFirFilter, PolyphaseResamplingFir, IirFilter,
)
from .blocks import (  # noqa: F401
    FixedPointPhase, Head, SignalSource, SignalSourceBuilder, SignalWave,
    Combine, CombineOp, Delay, Split, SplitOp, StreamDeinterleaver, StreamDuplicator, MovingAverage,
    AdsbDemod, ClockRecoveryMm, ZigbeeDecoder, KeyfobDecoder, KEYFOB_CODE, ApplyNM, ApplyNMOp, Mixer, MixOp,
    LoraTransmitter, LORA_BURST, WlanTransmitter, WLAN_BURST, ZigbeeTransmitter, ZIGBEE_BURST,
)
from . import adsb, firdes, keyfob, lora, ssb, windows, wlan, zigbee  # noqa: F401
# host edges (VectorSource/Sink, FileSource/Sink, H2D/D2H ring, run_chain, Flowgraph): futuresdr_b200.edges
