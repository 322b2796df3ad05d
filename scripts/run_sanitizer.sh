# memcheck of the kernels touched this round on small shapes (sanitizer slows kernels ~50x)
export B2S_SANITIZE=1
timeout 300 compute-sanitizer --tool memcheck --print-limit 5 python -m pytest tests/test_gpu_fir_tensor.py -m gpu -q -x -k "parity and (256 or 129 or 17) or unaligned" 2>&1 | tail -8
timeout 300 compute-sanitizer --tool memcheck --print-limit 5 python -m pytest tests/test_gpu_blocks.py tests/test_gpu_fir.py -m gpu -q -x -k "resampler or decim" 2>&1 | tail -8
timeout 300 compute-sanitizer --tool memcheck --print-limit 5 python -m pytest tests/test_gpu_spectrum.py tests/test_gpu_channelizer.py -m gpu -q -x -k "not tone" 2>&1 | tail -8
timeout 300 compute-sanitizer --tool memcheck --print-limit 5 python -m pytest tests/test_gpu_stream_blocks.py -m gpu -q -x -k "not 1048579 and not 1048577 and not 65541" 2>&1 | tail -8
timeout 300 compute-sanitizer --tool memcheck --print-limit 5 python -m pytest tests/test_gpu_boxavg.py -m gpu -q -x -k "ragged or word_offset or seams or refusals" 2>&1 | tail -8
timeout 600 compute-sanitizer --tool memcheck --print-limit 5 python -m pytest tests/test_gpu_zigbee.py -m gpu -q -x -k "not 64mi and not front_end and not 100_00" 2>&1 | tail -8
timeout 600 compute-sanitizer --tool racecheck --print-limit 5 python -m pytest tests/test_gpu_zigbee.py -m gpu -q -x -k "not 64mi and not front_end and not 100_00 and not steps" 2>&1 | tail -8
timeout 600 compute-sanitizer --tool memcheck --print-limit 5 python -m pytest tests/test_gpu_keyfob.py -m gpu -q -x -k "not 64mi and not front_end and not dense and not 2_pow_32 and not 100_003 and not 1048576" 2>&1 | tail -8
timeout 600 compute-sanitizer --tool racecheck --print-limit 5 python -m pytest tests/test_gpu_keyfob.py -m gpu -q -x -k "not 64mi and not front_end and not dense and not 2_pow_32 and not steps and not 100_003 and not 1048576" 2>&1 | tail -8
timeout 600 compute-sanitizer --tool memcheck --print-limit 5 python -m pytest tests/test_gpu_ssb.py -m gpu -q -x -k "not 40mi and not loopback and not graph" 2>&1 | tail -8
timeout 600 compute-sanitizer --tool racecheck --print-limit 5 python -m pytest tests/test_gpu_ssb.py -m gpu -q -x -k "not 40mi and not loopback and not graph and not random" 2>&1 | tail -8
timeout 600 compute-sanitizer --tool memcheck --print-limit 5 python -m pytest tests/test_gpu_lora.py -m gpu -q -x -k "slicing or sync_word or finish or refuses" 2>&1 | tail -8
timeout 600 compute-sanitizer --tool racecheck --print-limit 5 python -m pytest tests/test_gpu_lora.py -m gpu -q -x -k "sync_word or finish" 2>&1 | tail -8
timeout 600 compute-sanitizer --tool memcheck --print-limit 5 python -m pytest tests/test_gpu_wlan.py -m gpu -q -x -k "slicing or pads or refusals or finish or stale" 2>&1 | tail -8
timeout 600 compute-sanitizer --tool racecheck --print-limit 5 python -m pytest tests/test_gpu_wlan.py -m gpu -q -x -k "slicing or pads" 2>&1 | tail -8
