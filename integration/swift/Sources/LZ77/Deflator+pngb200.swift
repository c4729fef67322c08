//  Replaces Sources/LZ77/Deflator/LZ77.Deflator.swift:8-44 (and Gzip.Deflator / Gzip.archive,
//  Sources/LZ77/Gzip/Gzip.swift:34-46, with format 2).  Call sites: PNG.Encoder.pull,
//  Sources/PNG/Encoding/PNG.Encoder.swift:68,85,101,117,121,128.
import CPNGB200

extension LZ77
{
    @frozen public
    struct Deflator
    {
        private final
        class Handle
        {
            let z:OpaquePointer
            init(format:Int32, level:Int, exponent:Int, hint:Int)
            {
                // a complete block is 2 * capacity bytes, capacity = what malloc grants for `hint` UInt16 atoms
                // (LZ77.DeflatorOut.swift:15-27): 65544 for the encoder's hint of 1 << 15; 0 selects that value
                let chunk:Int = hint == 1 << 15 ? 0 : 2 * hint
                // the online handle compresses as the pushes arrive, so pop() hands PNG.Encoder.pull each IDAT chunk
                // when the reference would
                self.z = pngb200_deflator_create_online(LZ77.GPU.shared.ctx, format, Int32.init(level), Int32.init(exponent), chunk)!
            }
            /// A copy of `other` on the device that goes on independently (pngb200_deflator_clone).
            init(cloning other:Handle)
            {
                self.z = pngb200_deflator_clone(other.z)!
            }
            deinit
            {
                pngb200_deflator_destroy(self.z)
            }
        }
        private
        var handle:Handle

        /// What `exclude()` does (LZ77.DeflatorIn.swift, LZ77.DeflatorOut.swift): a shared handle is cloned before it
        /// is written.
        fileprivate mutating
        func exclude()
        {
            if !isKnownUniquelyReferenced(&self.handle)
            {
                self.handle = .init(cloning: self.handle)
            }
        }

        public
        init(format:LZ77.Format = .zlib, level:Int, exponent:Int = 15, hint:Int = 1 << 12)
        {
            self.handle = .init(format: format.code, level: level, exponent: exponent, hint: hint)
        }
    }
}
extension LZ77.Deflator
{
    public mutating
    func push(_ data:ArraySlice<UInt8>, last:Bool = false)
    {
        self.exclude()
        let status:Int32 = data.withUnsafeBufferPointer
        {
            pngb200_deflator_push(self.handle.z, $0.baseAddress, $0.count, last ? 1 : 0)
        }
        precondition(status == 0, String.init(cString: pngb200_last_error(LZ77.GPU.shared.ctx)))
    }
    /// A block of compressed data, if available; flushes the incomplete block otherwise.
    public mutating
    func pull() -> [UInt8]?
    {
        self.exclude()
        var block:UnsafePointer<UInt8>? = nil, count:Int = 0
        return pngb200_deflator_pull(self.handle.z, &block, &count) == 1
            ? .init(UnsafeBufferPointer.init(start: block, count: count)) : nil
    }
    /// A complete block of compressed data, if available.
    public mutating
    func pop() -> [UInt8]?
    {
        self.exclude()
        var block:UnsafePointer<UInt8>? = nil, count:Int = 0
        return pngb200_deflator_pop(self.handle.z, &block, &count) == 1
            ? .init(UnsafeBufferPointer.init(start: block, count: count)) : nil
    }
}
