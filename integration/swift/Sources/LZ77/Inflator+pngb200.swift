//  Replaces Sources/LZ77/Inflator/LZ77.Inflator.swift:8-62 (and, with format 2, Gzip.Inflator,
//  Sources/LZ77/Gzip/Gzip.Inflator.swift:26-57).
import CPNGB200

extension LZ77
{
    @frozen public
    struct Inflator
    {
        private final
        class Handle
        {
            let z:OpaquePointer
            init(format:Int32)
            {
                self.z = pngb200_inflator_create(LZ77.GPU.shared.ctx, format)!
            }
            /// A copy of `other` on the device that goes on independently (pngb200_inflator_clone).
            init(cloning other:Handle)
            {
                self.z = pngb200_inflator_clone(other.z)!
            }
            deinit
            {
                pngb200_inflator_destroy(self.z)
            }
        }
        private
        var handle:Handle

        /// What `exclude()` does (LZ77.InflatorBuffers.swift): a shared handle is cloned before it is written.
        fileprivate mutating
        func exclude()
        {
            if !isKnownUniquelyReferenced(&self.handle)
            {
                self.handle = .init(cloning: self.handle)
            }
        }

        public
        init(format:LZ77.Format = .zlib)
        {
            self.handle = .init(format: format.code)
        }
    }
}
extension LZ77.Inflator
{
    /// Returns nil once a complete stream has been received (LZ77.Inflator.swift:30-50).
    public mutating
    func push(_ data:ArraySlice<UInt8>) throws -> Void?
    {
        self.exclude()
        let status:Int32 = data.withUnsafeBufferPointer
        {
            pngb200_inflator_push(self.handle.z, $0.baseAddress, $0.count)
        }
        switch status
        {
        case 0: return nil          // PNGB200_OK: the stream is complete
        case 1: return ()           // PNGB200_NEED_MORE_INPUT
        default:
            var s:Int32 = 0, a:UInt32 = 0, b:UInt32 = 0
            pngb200_inflator_error(self.handle.z, &s, &a, &b)
            throw pngb200Error(status: status, a, b)
        }
    }
    /// Exactly `count` bytes, or nil (LZ77.Inflator.swift:52-56).
    public mutating
    func pull(_ count:Int) -> [UInt8]?
    {
        self.exclude()
        var out:[UInt8] = .init(repeating: 0, count: count)
        return pngb200_inflator_pull(self.handle.z, &out, count) == 0 ? out : nil
    }
    public mutating
    func pull() -> [UInt8]
    {
        self.exclude()
        var out:[UInt8] = .init(repeating: 0, count: pngb200_inflator_available(self.handle.z))
        let n:Int = pngb200_inflator_pull_all(self.handle.z, &out, out.count)
        out.removeLast(out.count - n)
        return out
    }
}
