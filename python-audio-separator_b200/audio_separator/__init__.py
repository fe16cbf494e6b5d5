"""Drop-in `audio_separator` package whose separation hot path runs on the H100-native engine (libb200sep.so)."""
