# The reference's model quantiser (src/quantize.cpp), compiled in place like the rest of oracle/_ref
# (test and measurement infrastructure; nothing here is linked into the product).
#
#   make -C oracle -f quantize.mk   -> oracle/_ref/quantize_ref      the reference tool over the reference's
#                                                                      lib/ggml.c: the CPU oracle of
#                                                                      fastllama_b200/quantize.py
#                                   -> oracle/_ref/quantize_ref.o    also linked by fastllama_b200/csrc/Makefile
#                                                                      over libggml_b200 (the drop-in quantize)
#
# Kept beside Makefile rather than in it so the recipe of the existing oracle targets stays as it is; it
# reuses that recipe's flags and its ggml_ref.o / llama_ref.o rules.  Without the reference sources it
# does nothing, and whatever oracle/_ref already holds is used.

include Makefile

.DEFAULT_GOAL := quantize

ifneq ($(wildcard $(REF)/src/quantize.cpp),)
quantize: $(OUT)/quantize_ref
else
quantize:
	@:
endif

$(OUT)/quantize_ref.o: $(REF)/src/quantize.cpp | $(OUT)
	$(CXX) $(REFFLAGS) -std=gnu++17 -fno-rtti -fopenmp -I$(REF)/include -c $< -o $@

$(OUT)/quantize_ref: $(OUT)/quantize_ref.o $(OUT)/llama_ref.o $(OUT)/ggml_ref.o
	$(CXX) -o $@ $^ -fopenmp -lpthread -lm

.PHONY: quantize
