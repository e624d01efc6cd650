# oracle/ref32.mk -- builds _ref/libk4ref32.so, a CHECKER (test infrastructure), never the product:
# the reference's upstream C engine (orig/lib/lz4.c) as its 32-bit engine LL32 behaves, the one
# LZ4Codec.Enforce32 selects.  LL32 differs from LL64 only in the hash of the u32 table: 4 bytes (hash4)
# instead of 8 (hash5), LL32.tools.cs:143-150.  Upstream picks hash5 in LZ4_hashPosition by the test
# `(sizeof(reg_t)==8) && (tableType != byU16)`; sed turns that test into 0 while the source is piped into
# the compiler, so no reference source is written to disk and only the .so lands in _ref/.  The recipe
# fails unless the test occurs exactly once.  Nothing is done where $(REF) is absent.
#   make -C oracle -f ref32.mk
REF ?= /root/reference
CC ?= gcc
CFLAGS ?= -O2 -fPIC -Wall -Wextra -Wno-unused-parameter
HASH5_TEST := (sizeof(reg_t)==8) && (tableType != byU16)

ref32:
	@if [ -f $(REF)/orig/lib/lz4.c ]; then \
	  n=$$(grep -cF '$(HASH5_TEST)' $(REF)/orig/lib/lz4.c); \
	  if [ "$$n" != 1 ]; then echo "ref32.mk: '$(HASH5_TEST)' occurs $$n times in lz4.c, expected once" >&2; exit 1; fi; \
	  mkdir -p _ref && \
	  sed 's/(sizeof(reg_t)==8) && (tableType != byU16)/0/' $(REF)/orig/lib/lz4.c | \
	    $(CC) $(CFLAGS) -I$(REF)/orig/lib -shared -Wl,-Bsymbolic -o _ref/libk4ref32.so -x c - && \
	  echo "built _ref/libk4ref32.so"; \
	else echo "reference not present: keeping prebuilt _ref/libk4ref32.so (if any)"; fi

.PHONY: ref32
