// handles.cpp -- compile-time checks of the C++ host layer (include/b200sdr.hpp): every class that owns a library
// object is move-only, so a copy can never destroy the object twice.  Compiled (syntax only, no GPU, no library) by
// tests/test_cpp_handles.py.
#include <type_traits>

#include "b200sdr.hpp"

using namespace b2s;

static_assert(!std::is_copy_constructible_v<Instance>);
static_assert(!std::is_copy_constructible_v<DecimatingFirFilter<float, float>>);
static_assert(!std::is_copy_constructible_v<FirFilter<Complex32, float>>);
static_assert(!std::is_copy_constructible_v<PolyphaseResamplingFir<Complex32>>);
static_assert(!std::is_copy_constructible_v<IirFilter<float>>);
static_assert(!std::is_copy_constructible_v<SignalSource<float>>);
static_assert(!std::is_copy_constructible_v<Fft>);
static_assert(!std::is_copy_constructible_v<Apply<Complex32, float>>);
static_assert(!std::is_copy_constructible_v<PfbArbResampler>);
static_assert(!std::is_copy_constructible_v<Rotator>);
static_assert(!std::is_copy_constructible_v<MovingAvg>);
static_assert(!std::is_copy_constructible_v<SpectrumPipe>);
// the filter cores and the rotator carry no device buffers of their own: they can still be moved
static_assert(std::is_move_constructible_v<DecimatingFirFilter<float, float>>);
static_assert(std::is_move_constructible_v<IirFilter<float>>);
static_assert(std::is_move_constructible_v<Rotator>);
